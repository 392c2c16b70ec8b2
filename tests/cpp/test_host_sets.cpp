// C++ host-API test of the two-set collide queries of DynamicAABBTreeCollisionManager
// (broadphase_collision_manager.h:94-118): collide(other_manager, callback), collide(obj, callback), collide(this,
// callback) and the batched form, against the brute-force overlap of the objects' boxes.  Runs on the GPU box.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <set>
#include <vector>

#include "../../hpp-fcl_b200/host/hppfcl_b200.hpp"

using namespace hppfcl_b200;

static int failures = 0;
#define CHECK(c)                                                          \
  do {                                                                    \
    if (!(c)) { std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #c); ++failures; } \
  } while (0)

int main() {
  std::srand(7);
  auto rnd = [] { return std::rand() / (double)RAND_MAX; };
  std::vector<CollisionGeometryPtr_t> geoms = {CollisionGeometryPtr_t(new Box(0.6, 0.4, 0.8)),
                                               CollisionGeometryPtr_t(new Sphere(0.3)),
                                               CollisionGeometryPtr_t(new Capsule(0.2, 0.6))};
  std::vector<std::unique_ptr<CollisionObject>> own;
  std::vector<CollisionObject*> robot, env;
  for (int i = 0; i < 450; ++i) {
    const double a = 6.2832 * rnd(), b = 6.2832 * rnd();
    const Quatf q = makeQuat(std::cos(a / 2), std::sin(a / 2) * std::cos(b), std::sin(a / 2) * std::sin(b), 0);
    own.emplace_back(new CollisionObject(geoms[i % 3], Transform3f(q.toRotationMatrix(), Vec3f(6 * rnd(), 6 * rnd(), 6 * rnd()))));
    (i < 150 ? robot : env).push_back(own.back().get());
  }
  DynamicAABBTreeCollisionManager mr, me;
  mr.registerObjects(robot);
  me.registerObjects(env);
  mr.setup();
  me.setup();
  std::set<std::pair<CollisionObject*, CollisionObject*>> want;
  for (CollisionObject* a : robot)
    for (CollisionObject* b : env)
      if (a->getAABB().overlap(b->getAABB())) want.insert(std::make_pair(a, b));
  CHECK(want.size() > 50);
  {  // collide(other, callback): o1 from the manager called, o2 from `other`
    CollisionCallBackCollect cb(0);
    mr.collide(&me, &cb);
    std::set<std::pair<CollisionObject*, CollisionObject*>> got(cb.getCollisionPairs().begin(), cb.getCollisionPairs().end());
    CHECK(got == want && cb.numCollisionPairs() == want.size());
  }
  {  // collide(obj, callback): the manager's object first, then obj
    CollisionObject q(CollisionGeometryPtr_t(new Box(2, 2, 2)), Transform3f(Vec3f(3, 3, 3)));
    CollisionCallBackCollect cb(0);
    me.collide(&q, &cb);
    size_t n = 0;
    for (CollisionObject* b : env)
      if (b->getAABB().overlap(q.getAABB())) ++n;
    CHECK(n > 5 && cb.numCollisionPairs() == n);
    for (const auto& p : cb.getCollisionPairs()) CHECK(p.second == &q && p.first != &q);
  }
  {  // collide(this, callback) is the self form
    CollisionCallBackCollect c1(0), c2(0);
    me.collide(&me, &c1);
    me.collide(&c2);
    CHECK(c1.numCollisionPairs() > 0 && c1.getCollisionPairs() == c2.getCollisionPairs());
    std::vector<uint32_t> f1, s1, f2, s2;  // and so are pairs(*this, ...) and collide(m, m, ...)
    me.pairs(me, f1, s1);
    me.pairs(f2, s2);
    CHECK(f1 == f2 && s1 == s2 && f1.size() == c1.numCollisionPairs());
    const std::vector<hfb_contact> r1 = collide(me, me, CollisionRequest(), f1, s1);
    CHECK(r1.size() == f2.size() && f1 == f2);
  }
  {  // the batched form: one record per cross candidate, as collide() of that pair
    std::vector<uint32_t> first, second;
    const std::vector<hfb_contact> rec = collide(mr, me, CollisionRequest(), first, second);
    CHECK(rec.size() == want.size() && first.size() == want.size());
    size_t hits = 0;
    for (size_t k = 0; k < first.size(); k += 7) {
      CollisionResult res;
      const size_t nc = collide(robot[first[k]], env[second[k]], CollisionRequest(), res);
      CHECK(nc == rec[k].num_contacts);
      hits += nc;
    }
    CHECK(hits > 0);
  }
  std::printf(failures ? "HOST-SETS-FAILED %d\n" : "HOST-SETS-OK\n", failures);
  return failures ? 1 : 0;
}
