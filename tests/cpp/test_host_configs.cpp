// C++ host-API test of ResidentEnvironment::collide_configurations / configuration_flags: reads a scene (argv[1],
// written by tests/test_cpp_host_configs.py with every digit of every pose), runs the configurations query and prints
// the verdicts and the colliding pairs so that the Python mirror's can be compared with them.  Runs on the GPU box.
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <utility>
#include <vector>

#include "../../hpp-fcl_b200/host/hppfcl_b200.hpp"

using namespace hppfcl_b200;

static int failures = 0;
#define CHECK(c)                                                          \
  do {                                                                    \
    if (!(c)) { std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #c); ++failures; } \
  } while (0)

static bool read_pose(std::FILE* f, int& type, Transform3f& tf) {
  double v[12];
  if (std::fscanf(f, "%d", &type) != 1) return false;
  for (double& x : v)
    if (std::fscanf(f, "%lf", &x) != 1) return false;  // (hexadecimal floating point: every digit)
  Matrix3f R;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R(r, c) = v[3 * r + c];
  tf = Transform3f(R, Vec3f(v[9], v[10], v[11]));
  return true;
}

int main(int argc, char** argv) {
  Context::instance();  // (no GPU: throws, there is no CPU fallback)
  if (argc < 2) return 2;
  std::FILE* f = std::fopen(argv[1], "r");
  if (!f) return 2;
  size_t links, n_configs, n_tpl, n_env;
  if (std::fscanf(f, "%zu %zu %zu %zu", &links, &n_configs, &n_tpl, &n_env) != 4) return 2;
  std::vector<std::pair<uint32_t, uint32_t>> tpl(n_tpl);
  for (auto& p : tpl)
    if (std::fscanf(f, "%u %u", &p.first, &p.second) != 2) return 2;
  // the geometry of tests/test_cpp_host_configs.py: two link kinds, three environment kinds and the floor
  std::vector<CollisionGeometryPtr_t> link_geom = {CollisionGeometryPtr_t(new Capsule(0.05, 0.14)),
                                                   CollisionGeometryPtr_t(new Box(0.08, 0.08, 0.22))};
  std::vector<CollisionGeometryPtr_t> env_geom = {
      CollisionGeometryPtr_t(new Box(0.3, 0.2, 0.25)), CollisionGeometryPtr_t(new Sphere(0.15)),
      CollisionGeometryPtr_t(new Capsule(0.1, 0.3)), CollisionGeometryPtr_t(new Halfspace(Vec3f(0, 0, 1), 0.02))};
  std::vector<std::unique_ptr<CollisionObject>> own;
  std::vector<CollisionObject*> robot, env;
  for (size_t k = 0; k < links * n_configs + n_env; ++k) {
    int type;
    Transform3f tf;
    if (!read_pose(f, type, tf)) return 2;
    const bool is_robot = k < links * n_configs;
    own.emplace_back(new CollisionObject(is_robot ? link_geom[type] : env_geom[type], tf));
    (is_robot ? robot : env).push_back(own.back().get());
  }
  std::fclose(f);
  DynamicAABBTreeCollisionManager mr, me;
  mr.registerObjects(robot);
  me.registerObjects(env);
  mr.setup();
  me.setup();
  ResidentEnvironment re(me);
  ResidentEnvironment::Pairs env_pairs, self_pairs;
  const std::vector<uint8_t> v = re.collide_configurations(mr, links, tpl, CollisionRequest(), env_pairs, self_pairs);
  CHECK(v.size() == n_configs);
  CHECK(re.configuration_flags(mr, links, tpl, CollisionRequest()) == v);
  for (const std::vector<std::pair<uint32_t, uint32_t>>& bad :
       {std::vector<std::pair<uint32_t, uint32_t>>{{0, 2}, {2, 0}}, {{1, 1}}, {{0, (uint32_t)links}}}) {
    bool refused = false;
    try {
      re.configuration_flags(mr, links, bad, CollisionRequest());
    } catch (const std::invalid_argument&) {
      refused = true;
    }
    CHECK(refused);
  }
  std::printf("verdicts ");
  for (uint8_t x : v) std::printf("%d", (int)x);
  std::printf("\n");
  const char* names[2] = {"env", "self"};
  const ResidentEnvironment::Pairs* kinds[2] = {&env_pairs, &self_pairs};
  for (int k = 0; k < 2; ++k)
    for (size_t i = 0; i < kinds[k]->first.size(); ++i) {
      const hfb_contact& c = kinds[k]->contacts[i];
      CHECK(c.num_contacts > 0);
      std::printf("%s %u %u %u %a\n", names[k], kinds[k]->first[i], kinds[k]->second[i], c.num_contacts, c.distance);
    }
  std::printf(failures ? "HOST-CONFIGS-FAILED %d\n" : "HOST-CONFIGS-OK\n", failures);
  return failures ? 1 : 0;
}
