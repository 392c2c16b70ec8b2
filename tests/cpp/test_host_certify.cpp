// C++ host-API test of ResidentEnvironment::certify_motions: reads a scene (argv[1], written by
// tests/test_cpp_host_certify.py with every digit of every pose), the motion offsets (argv[2], one per line) and the
// sweep bounds (argv[4], one per robot object, hexadecimal floating point), runs the certification with argv[3] links
// per configuration and the chain template (j >= i + 2), and prints each motion's first colliding and first
// uncertified sample and each configuration's certified flag, so that the Python mirror's can be compared with them.
// Runs on the GPU box.
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
  if (argc < 5) return 2;
  const size_t links = std::strtoul(argv[3], nullptr, 10);
  std::FILE* f = std::fopen(argv[1], "r");
  if (!f) return 2;
  size_t n_robot, n_env;
  if (std::fscanf(f, "%zu %zu", &n_robot, &n_env) != 2) return 2;
  // the geometry of tests/test_cpp_host_certify.py: two link kinds, three environment kinds and the floor
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
  std::vector<uint32_t> offsets;
  std::FILE* fo = std::fopen(argv[2], "r");
  if (!fo) return 2;
  for (unsigned v; std::fscanf(fo, "%u", &v) == 1;) offsets.push_back(v);
  std::fclose(fo);
  std::vector<double> sweep;
  std::FILE* fs = std::fopen(argv[4], "r");
  if (!fs) return 2;
  for (double v; std::fscanf(fs, "%lf", &v) == 1;) sweep.push_back(v);
  std::fclose(fs);
  DynamicAABBTreeCollisionManager mr, me;
  mr.registerObjects(robot);
  me.registerObjects(env);
  mr.setup();
  me.setup();
  ResidentEnvironment re(me);
  std::vector<std::pair<uint32_t, uint32_t>> tpl;
  for (uint32_t i = 0; i < links; ++i)
    for (uint32_t j = i + 2; j < links; ++j) tpl.emplace_back(i, j);
  std::vector<int32_t> first_invalid, first_uncertified;
  const std::vector<uint8_t> certified =
      re.certify_motions(mr, links, tpl, offsets, sweep, CollisionRequest(), first_invalid, first_uncertified);
  const size_t n_motions = offsets.size() - 1;
  CHECK(first_invalid.size() == n_motions && first_uncertified.size() == n_motions);
  CHECK(certified.size() == n_robot / links);
  // first_invalid is collide_motions'
  CHECK(re.first_invalid_samples(mr, links, tpl, offsets) == first_invalid);
  std::vector<int32_t> fi, fu;
  std::vector<std::vector<uint32_t>> bad_offsets = {{1, (uint32_t)(n_robot / links)}, {0, 2, 1, (uint32_t)(n_robot / links)},
                                                    {0, (uint32_t)(n_robot / links) + 1}, {}};
  for (const std::vector<uint32_t>& bad : bad_offsets) {
    bool refused = false;
    try {
      re.certify_motions(mr, links, tpl, bad, sweep, CollisionRequest(), fi, fu);
    } catch (const std::invalid_argument&) {
      refused = true;
    }
    CHECK(refused);
  }
  for (const std::vector<double>& bad : {std::vector<double>(sweep.begin(), sweep.end() - 1), std::vector<double>()}) {
    bool refused = false;
    try {
      re.certify_motions(mr, links, tpl, offsets, bad, CollisionRequest(), fi, fu);
    } catch (const std::invalid_argument&) {
      refused = true;
    }
    CHECK(refused);
  }
  {
    bool refused = false;
    try {
      re.certify_motions(mr, links, {{1, 1}}, offsets, sweep, CollisionRequest(), fi, fu);
    } catch (const std::invalid_argument&) {
      refused = true;
    }
    CHECK(refused);
  }
  {  // no motions over an empty robot: nothing comes back
    DynamicAABBTreeCollisionManager none;
    none.setup();
    CHECK(re.certify_motions(none, links, tpl, {0}, {}, CollisionRequest(), fi, fu).empty() && fi.empty() && fu.empty());
  }
  for (size_t m = 0; m < n_motions; ++m) std::printf("mot %zu %d %d\n", m, first_invalid[m], first_uncertified[m]);
  for (size_t g = 0; g < certified.size(); ++g) std::printf("cfg %zu %u\n", g, (unsigned)certified[g]);
  std::printf(failures ? "HOST-CERTIFY-FAILED %d\n" : "HOST-CERTIFY-OK\n", failures);
  return failures ? 1 : 0;
}
