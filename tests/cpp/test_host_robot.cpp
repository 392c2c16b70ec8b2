// C++ host-API test of RobotModel: builds the model of tests/test_cpp_host_robot.py (two revolute joints, a box and a
// capsule on them and a sphere fixed to the world), samples its motions, feeds the samples to ResidentEnvironment's
// certify_motions and configuration_flags against one box, and prints every pose, sweep bound and output with every
// digit (hexadecimal floating point) so that the Python mirror's can be compared with them.  Also checks that q of the
// wrong size and malformed offsets throw std::invalid_argument.  Runs on the GPU box.
#include <cstdio>
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
  CHECK(robot.nq() == 2 && robot.num_links() == 3);
  const std::vector<double> q_from = {0.0, 0.0, 1.0, -0.5}, q_to = {1.5, 1.0, -1.0, 0.5};
  const std::vector<uint32_t> offsets = {0, 20, 45};
  RobotSamples s = robot.sample_motions(q_from, q_to, offsets);
  CHECK(s.size() == 45 * 3 && s.q().size() == 45 * 2 && s.sweep().size() == 45 * 3 && s.offsets() == offsets);
  for (size_t k = 0; k < s.size(); ++k) {
    const hfb_transform& t = s.transforms()[k];
    std::printf("tf %zu %u", k, s.handles()[k]);
    for (double v : t.R) std::printf(" %a", v);
    for (double v : t.T) std::printf(" %a", v);
    std::printf(" %a\n", s.sweep()[k]);
  }
  // poses(q) of the samples' q are the samples' poses
  RobotSamples p = robot.poses(s.q());
  CHECK(p.size() == s.size() && p.sweep().empty() && p.offsets().empty());
  for (size_t k = 0; k < p.size(); ++k)
    for (int i = 0; i < 12; ++i)
      CHECK((i < 9 ? p.transforms()[k].R[i] : p.transforms()[k].T[i - 9]) ==
            (i < 9 ? s.transforms()[k].R[i] : s.transforms()[k].T[i - 9]));
  DynamicAABBTreeCollisionManager env_mgr;
  CollisionObject obstacle(CollisionGeometryPtr_t(new Box(0.1, 0.1, 0.1)), Transform3f(Vec3f(0.2, 0.1, 0.25)));
  env_mgr.registerObject(&obstacle);
  env_mgr.setup();
  ResidentEnvironment re(env_mgr);
  const std::vector<std::pair<uint32_t, uint32_t>> tpl = {{0, 2}};
  std::vector<int32_t> fi, fu;
  const std::vector<uint8_t> cert =
      re.certify_motions(s, 3, tpl, s.offsets(), s.sweep(), CollisionRequest(), fi, fu);
  for (size_t m = 0; m < fi.size(); ++m) std::printf("mot %zu %d %d\n", m, fi[m], fu[m]);
  for (size_t g = 0; g < cert.size(); ++g) std::printf("cfg %zu %d\n", g, (int)cert[g]);
  const std::vector<uint8_t> flags = re.configuration_flags(p, 3, tpl, CollisionRequest());
  for (size_t g = 0; g < flags.size(); ++g) std::printf("flag %zu %d\n", g, (int)flags[g]);
  // malformed input throws std::invalid_argument, as the Python mirror raises ValueError
  CHECK(throws_invalid([&] { robot.poses(std::vector<double>(3)); }));
  CHECK(throws_invalid([&] { robot.sample_motions(q_from, q_to, {1, 20, 45}); }));
  CHECK(throws_invalid([&] { robot.sample_motions(q_from, q_to, {0, 20, 10}); }));
  CHECK(throws_invalid([&] { robot.sample_motions(q_from, q_to, {}); }));
  CHECK(throws_invalid([&] { robot.sample_motions(q_from, std::vector<double>(2), offsets); }));
  CHECK(throws_invalid([&] { RobotModel bad({{0, HFB_JOINT_REVOLUTE, Vec3f(0, 0, 1), Transform3f()}}, links); }));
  CHECK(throws_invalid([&] { RobotModel bad({{-1, HFB_JOINT_REVOLUTE, Vec3f(0, 0, 0), Transform3f()}}, {links[0]}); }));
  if (failures) return 1;
  std::printf("HOST-ROBOT-OK\n");
  return 0;
}
