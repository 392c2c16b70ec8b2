// C++ host-API test of ResidentEnvironment::distance_configurations / configuration_clearance: reads a scene (argv[1],
// written by tests/test_cpp_host_distance_configs.py with every digit of every pose), runs the configurations distance
// query with argv[3] links per configuration and the chain template (j >= i + 2) at the cutoff argv[2], and prints each
// configuration's winner, so that the Python mirror's can be compared with it.  Runs on the GPU box.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <limits>
#include <memory>
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
  if (argc < 4) return 2;
  const double max_distance = std::strtod(argv[2], nullptr);
  const size_t links = std::strtoul(argv[3], nullptr, 10);
  std::FILE* f = std::fopen(argv[1], "r");
  if (!f) return 2;
  size_t n_robot, n_env;
  if (std::fscanf(f, "%zu %zu", &n_robot, &n_env) != 2) return 2;
  // the geometry of tests/test_cpp_host_distance_configs.py: two link kinds, three environment kinds and the floor
  std::vector<CollisionGeometryPtr_t> link_geom = {CollisionGeometryPtr_t(new Capsule(0.05, 0.14)),
                                                   CollisionGeometryPtr_t(new Box(0.08, 0.08, 0.22))};
  std::vector<CollisionGeometryPtr_t> env_geom = {
      CollisionGeometryPtr_t(new Box(0.3, 0.2, 0.25)), CollisionGeometryPtr_t(new Sphere(0.15)),
      CollisionGeometryPtr_t(new Capsule(0.1, 0.3)), CollisionGeometryPtr_t(new Halfspace(Vec3f(0, 0, 1), 0.02))};
  std::vector<std::unique_ptr<CollisionObject>> own;
  std::vector<CollisionObject*> robot, env;
  for (size_t k = 0; k < n_robot + n_env; ++k) {
    int type;
    Transform3f tf;
    if (!read_pose(f, type, tf)) return 2;
    const bool is_robot = k < n_robot;
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
  std::vector<std::pair<uint32_t, uint32_t>> tpl;
  for (uint32_t i = 0; i < links; ++i)
    for (uint32_t j = i + 2; j < links; ++j) tpl.emplace_back(i, j);
  std::vector<int8_t> kind;
  std::vector<uint32_t> first, second;
  std::vector<FCL_REAL> dist;
  const std::vector<hfb_distance_result> rec =
      re.distance_configurations(mr, links, tpl, DistanceRequest(), kind, first, second, dist, max_distance);
  const size_t n_configs = n_robot / links;
  CHECK(rec.size() == n_configs && kind.size() == n_configs && first.size() == n_configs && dist.size() == n_configs);
  const std::vector<FCL_REAL> clear = re.configuration_clearance(mr, links, tpl, max_distance);
  CHECK(clear.size() == n_configs);
  for (size_t g = 0; g < n_configs && g < clear.size(); ++g) {
    CHECK(clear[g] == dist[g]);
    CHECK(rec[g].min_distance == dist[g]);
  }
  for (double bad : {std::nan(""), -1.0}) {
    bool refused = false;
    try {
      re.configuration_clearance(mr, links, tpl, bad);
    } catch (const std::invalid_argument&) {
      refused = true;
    }
    CHECK(refused);
  }
  for (const std::vector<std::pair<uint32_t, uint32_t>>& bad :
       {std::vector<std::pair<uint32_t, uint32_t>>{{0, (uint32_t)links}}, {{1, 1}}, {{0, 2}, {2, 0}}}) {
    bool refused = false;
    try {
      re.configuration_clearance(mr, links, bad, max_distance);
    } catch (const std::invalid_argument&) {
      refused = true;
    }
    CHECK(refused);
  }
  for (size_t g = 0; g < n_configs; ++g)
    std::printf("cfg %zu %d %u %u %a\n", g, (int)kind[g], first[g], second[g], dist[g]);
  std::printf(failures ? "HOST-DISTANCE-CONFIGS-FAILED %d\n" : "HOST-DISTANCE-CONFIGS-OK\n", failures);
  return failures ? 1 : 0;
}
