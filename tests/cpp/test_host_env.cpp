// C++ host-API test of ResidentEnvironment (hfb_env) and the manager's update(obj) / update(objs): the environment's
// colliding pairs and per-object flags against the batched cross form collide(robot, env, ...), before and after some
// environment objects move.  Runs on the GPU box.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <set>
#include <tuple>
#include <vector>

#include "../../hpp-fcl_b200/host/hppfcl_b200.hpp"

using namespace hppfcl_b200;

static int failures = 0;
#define CHECK(c)                                                          \
  do {                                                                    \
    if (!(c)) { std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #c); ++failures; } \
  } while (0)

typedef std::set<std::pair<uint32_t, uint32_t>> Pairs;

// the colliding pairs and the flags the cross form gives: what the environment must return
static void expected(DynamicAABBTreeCollisionManager& mr, DynamicAABBTreeCollisionManager& me, Pairs& pairs,
                     std::vector<uint8_t>& flags) {
  std::vector<uint32_t> f, s;
  const std::vector<hfb_contact> rec = collide(mr, me, CollisionRequest(), f, s);
  pairs.clear();
  flags.assign(mr.size(), 0);
  for (size_t k = 0; k < f.size(); ++k)
    if (rec[k].num_contacts) {
      pairs.insert(std::make_pair(f[k], s[k]));
      flags[f[k]] = 1;
    }
}

static bool same_box(const AABB& a, const AABB& b) {
  for (int k = 0; k < 3; ++k)
    if (a.min_[k] != b.min_[k] || a.max_[k] != b.max_[k]) return false;
  return true;
}

int main() {
  std::srand(11);
  auto rnd = [] { return std::rand() / (double)RAND_MAX; };
  std::vector<CollisionGeometryPtr_t> geoms = {CollisionGeometryPtr_t(new Box(0.6, 0.4, 0.8)),
                                               CollisionGeometryPtr_t(new Sphere(0.3)),
                                               CollisionGeometryPtr_t(new Capsule(0.2, 0.6))};
  auto pose = [&] {
    const double a = 6.2832 * rnd(), b = 6.2832 * rnd();
    const Quatf q = makeQuat(std::cos(a / 2), std::sin(a / 2) * std::cos(b), std::sin(a / 2) * std::sin(b), 0);
    return Transform3f(q.toRotationMatrix(), Vec3f(6 * rnd(), 6 * rnd(), 6 * rnd()));
  };
  std::vector<std::unique_ptr<CollisionObject>> own;
  std::vector<CollisionObject*> robot, env;
  for (int i = 0; i < 600; ++i) {
    own.emplace_back(new CollisionObject(geoms[i % 3], pose()));
    (i < 150 ? robot : env).push_back(own.back().get());
  }
  DynamicAABBTreeCollisionManager mr, me;
  mr.registerObjects(robot);
  me.registerObjects(env);
  mr.setup();
  me.setup();
  ResidentEnvironment re(me);
  Pairs want;
  std::vector<uint8_t> want_flags;
  for (int round = 0; round < 2; ++round) {
    expected(mr, me, want, want_flags);
    CHECK(want.size() > 20);
    std::vector<uint32_t> first, second;
    const std::vector<hfb_contact> rec = re.collide(mr, CollisionRequest(), first, second);
    Pairs got;
    for (size_t k = 0; k < first.size(); ++k) {
      got.insert(std::make_pair(first[k], second[k]));
      CHECK(rec[k].num_contacts > 0);
    }
    CHECK(got == want && got.size() == first.size());
    CHECK(re.collide_flags(mr, CollisionRequest()) == want_flags);
    // some environment objects move: the manager's update(objs) / update(obj) and the environment's update(objs)
    std::vector<CollisionObject*> moved(env.begin() + 10, env.begin() + 60);
    for (CollisionObject* o : moved) o->setTransform(pose());
    me.update(std::vector<CollisionObject*>(moved.begin(), moved.end() - 1));
    me.update(moved.back());
    std::vector<AABB> boxes;
    for (CollisionObject* o : env) boxes.push_back(o->getAABB());
    DynamicAABBTreeCollisionManager fresh;  // setup() over the same objects gives the same boxes
    fresh.registerObjects(env);
    fresh.setup();
    for (size_t i = 0; i < env.size(); ++i) CHECK(same_box(boxes[i], env[i]->getAABB()));
    re.update(moved);
  }
  {  // an object the manager does not hold: skipped by update(obj) / update(objs), refused by the environment
    const AABB before = robot[0]->getAABB();
    robot[0]->setTransform(pose());
    me.update(robot[0]);
    me.update(std::vector<CollisionObject*>{robot[0], env[5]});
    CHECK(same_box(before, robot[0]->getAABB()));
    bool refused = false;
    try {
      re.update(std::vector<CollisionObject*>{robot[0]});
    } catch (const std::invalid_argument&) {
      refused = true;
    }
    CHECK(refused);
  }
  std::printf(failures ? "HOST-ENV-FAILED %d\n" : "HOST-ENV-OK\n", failures);
  return failures ? 1 : 0;
}
