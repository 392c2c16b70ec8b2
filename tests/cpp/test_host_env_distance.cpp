// C++ host-API test of ResidentEnvironment::distance / clearance: reads a scene (argv[1], written by
// tests/test_cpp_host_env_distance.py with every digit of every pose), runs the distance query at the cutoff argv[2]
// and prints each robot object's nearest environment object and distance, so that the Python mirror's can be compared
// with them.  Runs on the GPU box.
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
  if (argc < 3) return 2;
  const double max_distance = std::strtod(argv[2], nullptr);
  std::FILE* f = std::fopen(argv[1], "r");
  if (!f) return 2;
  size_t n_robot, n_env;
  if (std::fscanf(f, "%zu %zu", &n_robot, &n_env) != 2) return 2;
  // the geometry of tests/test_cpp_host_env_distance.py: two link kinds, three environment kinds and the floor
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
  std::vector<int32_t> nearest;
  std::vector<FCL_REAL> dist;
  const std::vector<hfb_distance_result> rec = re.distance(mr, DistanceRequest(), nearest, dist, max_distance);
  CHECK(rec.size() == n_robot && nearest.size() == n_robot && dist.size() == n_robot);
  const std::vector<FCL_REAL> clear = re.clearance(mr, max_distance);
  CHECK(clear.size() == n_robot);
  for (size_t i = 0; i < n_robot && i < clear.size(); ++i) {
    CHECK(clear[i] == dist[i]);
    CHECK(rec[i].min_distance == dist[i]);
  }
  for (double bad : {std::nan(""), -1.0}) {
    bool refused = false;
    try {
      re.clearance(mr, bad);
    } catch (const std::invalid_argument&) {
      refused = true;
    }
    CHECK(refused);
  }
  for (size_t i = 0; i < n_robot; ++i) std::printf("near %zu %d %a\n", i, nearest[i], dist[i]);
  std::printf(failures ? "HOST-ENV-DISTANCE-FAILED %d\n" : "HOST-ENV-DISTANCE-OK\n", failures);
  return failures ? 1 : 0;
}
