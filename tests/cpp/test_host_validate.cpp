// C++ host-API test of ResidentEnvironment::validate_motions: builds the robot and the environment of
// tests/test_cpp_host_validate.py (two revolute joints, a box and a capsule on them and a sphere fixed to the world,
// one box in the way), validates its motions and prints every output with every digit (hexadecimal floating point) so
// that the Python mirror's can be compared with them field by field.  Also checks that the refusals throw
// std::invalid_argument.  Runs on the GPU box.
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "../../hpp-fcl_b200/host/hppfcl_b200.hpp"

using namespace hppfcl_b200;

static int failures = 0;
#define CHECK(c)                                                          \
  do {                                                                    \
    if (!(c)) { std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #c); ++failures; } \
  } while (0)

template <class F>
static bool throws_invalid(F f) {
  try {
    f();
  } catch (const std::invalid_argument&) {
    return true;
  }
  return false;
}

int main() {
  Context::instance();  // (no GPU: throws, there is no CPU fallback)
  const Transform3f up(Vec3f(0, 0, 0.1));
  std::vector<RobotModel::Joint> joints = {{-1, HFB_JOINT_REVOLUTE, Vec3f(0, 0, 1), Transform3f()},
                                           {0, HFB_JOINT_REVOLUTE, Vec3f(0, 1, 0), Transform3f(Vec3f(0, 0, 0.2))}};
  std::vector<RobotModel::Link> links = {{0, up, CollisionGeometryPtr_t(new Box(0.05, 0.05, 0.2))},
                                         {1, up, CollisionGeometryPtr_t(new Capsule(0.03, 0.1))},
                                         {-1, Transform3f(Vec3f(0.5, 0, 0)), CollisionGeometryPtr_t(new Sphere(0.05))}};
  RobotModel robot(joints, links);
  DynamicAABBTreeCollisionManager env_mgr;
  CollisionObject obstacle(CollisionGeometryPtr_t(new Box(0.1, 0.1, 0.1)), Transform3f(Vec3f(0.2, 0.1, 0.25)));
  env_mgr.registerObject(&obstacle);
  env_mgr.setup();
  ResidentEnvironment re(env_mgr);
  const std::vector<std::pair<uint32_t, uint32_t>> tpl = {{0, 2}};
  const std::vector<double> q_from = {0.0, 0.0, 1.0, -0.5, -2.0, 0.3, 0.4, 0.4},
                            q_to = {1.5, 1.0, -1.0, 0.5, 2.0, 0.3, 0.4, 0.4};
  for (int pass = 0; pass < 2; ++pass) {  // the whole range, then motions [1, 3) under a binding cap
    const MotionValidation v = pass == 0 ? re.validate_motions(robot, q_from, q_to, tpl, 1, 7, 1u << 20)
                                         : re.validate_motions(robot, q_from, q_to, tpl, 2, 6, 9, CollisionRequest(), 1, 2);
    CHECK(v.status.size() == 4);
    for (size_t m = 0; m < v.status.size(); ++m) {
      std::printf("val %d %zu %d %a %a %d %u %u", pass, m, (int)v.status[m], v.t_valid[m], v.t_collide[m], (int)v.kind[m],
                  v.first[m], v.second[m]);
      const unsigned char* b = reinterpret_cast<const unsigned char*>(&v.contacts[m]);
      std::printf(" ");
      for (size_t k = 0; k < sizeof(hfb_contact); ++k) std::printf("%02x", b[k]);
      std::printf("\n");
    }
    std::printf("cnt %d %u %llu %llu %llu %llu\n", pass, v.n_rounds, (unsigned long long)v.n_samples,
                (unsigned long long)v.n_env_candidates, (unsigned long long)v.n_self_candidates,
                (unsigned long long)v.n_unsupported);
  }
  CHECK(re.validate_motions(robot, {}, {}, tpl, 1, 4, 100).status.empty());
  // the refusals throw std::invalid_argument, as the Python mirror raises ValueError
  CHECK(throws_invalid([&] { re.validate_motions(robot, q_from, std::vector<double>(2), tpl, 1, 4, 100); }));
  CHECK(throws_invalid([&] { re.validate_motions(robot, std::vector<double>(3), std::vector<double>(3), tpl, 1, 4, 100); }));
  CHECK(throws_invalid([&] { re.validate_motions(robot, q_from, q_to, tpl, 5, 4, 100); }));
  CHECK(throws_invalid([&] { re.validate_motions(robot, q_from, q_to, tpl, 1, 31, 100); }));
  CHECK(throws_invalid([&] { re.validate_motions(robot, q_from, q_to, tpl, 1, 4, 1); }));
  CHECK(throws_invalid([&] { re.validate_motions(robot, q_from, q_to, {{0, 3}}, 1, 4, 100); }));
  CHECK(throws_invalid([&] { re.validate_motions(robot, q_from, q_to, tpl, 1, 4, 100, CollisionRequest(), 3, 2); }));
  if (failures) return 1;
  std::printf("HOST-VALIDATE-OK\n");
  return 0;
}
