// TEST HARNESS ONLY -- not part of the product and never loaded by it.
//
// The round bookkeeping of hfb_env_validate_motions (hpp-fcl_b200/csrc/hfb_validate.cuh) compiled with g++ and driven
// as the k_val_* kernels of hfb_scene.cu drive it -- round 0 without its list, the cost and run scans, admission, the
// samples and run offsets, the per-motion minima, the rules, the frontier and the compaction -- one pass after another
// on the host.  The certification's outcomes are not computed: a seeded hash decides, per sample, whether it collides
// and, per segment, whether it is certified and whether its sweeps are finite, so that tests/test_env_validate_reference.py
// can drive validate_reference (tests/validate_common.py) with the same outcomes and compare the bookkeeping.
#include <cstdint>
#include <vector>

#include "../../hpp-fcl_b200/csrc/hfb_validate.cuh"

using namespace hfb;

namespace {

uint64_t mix(uint64_t x) {  // splitmix64's finaliser
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}
// outcome `kind` (0: the sample collides, 1: the segment is certified, 2: its sweeps are not finite) of motion m at
// position a (and depth d for segments): true with probability per_mille / 1000
bool outcome(uint64_t seed, uint32_t kind, uint32_t m, uint32_t a, uint32_t d, uint32_t per_mille) {
  const uint64_t h = mix(mix(mix(mix(seed ^ kind) ^ m) ^ a) ^ (kind ? d : 0));
  return h % 1000 < per_mille;
}

}  // namespace

extern "C" int val_emu(uint64_t seed, uint32_t n_motions, uint32_t m0, uint32_t n_range, uint32_t d0, uint32_t D,
                       uint32_t cap, const uint32_t* per_mille, int8_t* status, double* t_valid, double* t_collide,
                       uint32_t* n_rounds, uint64_t* n_samples) {
  const uint32_t per = 1u << d0;
  std::vector<uint32_t> c(n_range, kValNone), f(n_range), u(n_range), sw, sa;
  uint64_t n_full = 0;
  uint32_t partial = 0;
  val_round0(n_range, per, cap, &n_full, &partial);
  const uint64_t n0 = n_full * per + partial;
  for (uint64_t t = 0; t < n0; ++t) {
    sw.push_back((uint32_t)(t / per));
    sa.push_back((uint32_t)(t % per) * (1u << (D - d0)));
  }
  for (uint32_t w = 0; w < n_range; ++w) {
    const uint32_t adm = val_round0_admitted(w, n_full, partial, per);
    f[w] = u[w] = adm < per ? adm * (1u << (D - d0)) : kValNone;
  }
  *n_rounds = 0;
  *n_samples = 0;
  for (uint32_t depth = d0; !sw.empty() && depth <= D; ++depth) {
    const uint32_t len = 1u << (D - depth), n = (uint32_t)sw.size();
    std::vector<uint32_t> cscan(n), nr(n), rscan(n);
    for (uint32_t i = 0; i < n; ++i) {  // k_val_cost and the two inclusive scans
      nr[i] = val_new_run(i == 0, i ? sw[i - 1] : 0, i ? sa[i - 1] : 0, sw[i], sa[i], len);
      cscan[i] = (i ? cscan[i - 1] : 0) + val_cost(nr[i]);
      rscan[i] = (i ? rscan[i - 1] : 0) + nr[i];
    }
    uint32_t n_adm = 0;  // k_val_admit
    while (n_adm < n && val_admitted(cscan[n_adm], cap)) ++n_adm;
    if (n_adm == 0) break;
    const uint32_t smp = cscan[n_adm - 1], runs = rscan[n_adm - 1];
    ++*n_rounds;
    *n_samples += smp;
    std::vector<uint32_t> pw(smp), pk(smp), off(runs + 1);  // k_val_samples
    std::vector<uint8_t> seg(smp);
    for (uint32_t i = 0; i < n_adm; ++i) {
      const uint32_t g = val_start_sample(cscan[i]);
      pw[g] = sw[i], pk[g] = sa[i], seg[g] = 1;
      if (nr[i]) off[rscan[i] - 1] = g;
      if (i + 1 == n_adm || nr[i + 1]) pw[g + 1] = sw[i], pk[g + 1] = sa[i] + len, seg[g + 1] = 0;
      if (i + 1 == n_adm) off[rscan[i]] = cscan[i];
    }
    // the certification's outcomes: per run its first colliding sample, per sample the certified and finite flags
    std::vector<uint8_t> cert(smp), fin(smp);
    for (uint32_t g = 0; g < smp; ++g) {
      cert[g] = seg[g] && outcome(seed, 1, m0 + pw[g], pk[g], depth, per_mille[1]);
      fin[g] = !(seg[g] && outcome(seed, 2, m0 + pw[g], pk[g], depth, per_mille[2]));
    }
    for (uint32_t r = 0; r < runs; ++r)  // k_val_collide
      for (uint32_t g = off[r]; g < off[r + 1]; ++g)
        if (outcome(seed, 0, m0 + pw[g], pk[g], 0, per_mille[0])) {
          if (pk[g] < c[pw[g]]) c[pw[g]] = pk[g];
          break;
        }
    std::vector<uint32_t> kids(n);
    for (uint32_t i = 0; i < n; ++i) {  // k_val_rules
      const bool admitted = i < n_adm;
      const uint32_t g = admitted ? val_start_sample(cscan[i]) : 0;
      const ValRule rule = val_rule(admitted, admitted && cert[g], sa[i], c[sw[i]], depth == D, !admitted || fin[g]);
      if (rule == VAL_DROPPED || rule == VAL_STUCK) u[sw[i]] = sa[i] < u[sw[i]] ? sa[i] : u[sw[i]];
      if (rule == VAL_STUCK) f[sw[i]] = sa[i] < f[sw[i]] ? sa[i] : f[sw[i]];
      kids[i] = rule == VAL_SPLIT ? 2u : 0u;
    }
    std::vector<uint32_t> nw, na;  // k_val_keep and k_val_compact
    for (uint32_t i = 0; i < n; ++i) {
      if (!kids[i]) continue;
      for (uint32_t b : {sa[i], sa[i] + len / 2})
        if (val_keep(b, f[sw[i]])) nw.push_back(sw[i]), na.push_back(b);
    }
    sw.swap(nw);
    sa.swap(na);
  }
  for (uint32_t m = 0; m < n_motions; ++m) {  // k_val_final
    if (m < m0 || m - m0 >= n_range) {
      status[m] = -1, t_valid[m] = 0.0, t_collide[m] = -1.0;
      continue;
    }
    val_result(c[m - m0], u[m - m0], D, status + m, t_valid + m, t_collide + m);
  }
  return 0;
}
