// EPA for one shape pair on an index-based polytope that lives in a per-pair
// workspace (shared memory for the lane-group kernels).
//
// Replaces GJK::encloseOrigin (src/narrowphase/gjk.cpp:437-492) and
// EPA::{reset,newFace,findClosestFace,evaluate,expand,getWitnessPointsAndNormal}
// (:1012-1466).
//
// Design differences from the reference (same arithmetic and same outcomes):
//  * faces are slots addressed by u8 ids, not a std::vector of pointer-linked
//    nodes (gjk.h:261-308).  The reference's `hull` list is newest-first and
//    findClosestFace keeps the first strict minimum, so "list order" is carried
//    by a per-face append sequence number: the closest face is the argmin of d^2
//    with ties broken towards the LARGEST sequence number.  That makes the scan a
//    lane-parallel reduction.
//  * `stock` is a LIFO of free slots (slot identity has no numerical meaning;
//    only the count matters for OutOfFaces).
//  * the recursive expand (:1361-1449) and encloseOrigin run on explicit stacks.
//  * newFace is split into its two halves: the slot/topology part runs inside the
//    horizon walk (every lane of the group executes it redundantly), the geometry
//    part (normal, offset, ignore flag, convexity verdict) is deferred to the end of
//    the round and spread over the group's lanes, one new face per lane.  The walk
//    never reads the geometry of a face created in the same round unless it steps on
//    a re-used slot; in that case the pending faces are completed on the spot, in
//    creation order, which is the order the reference meets their verdicts in.
//  * the closest-face scan stops at the highest slot ever handed out.
#pragma once
#include "hfb_gjk.cuh"

namespace hfb {

#define HFB_EPA_CAP_IT 64
#define HFB_EPA_MAXV (HFB_EPA_CAP_IT + 4)
#define HFB_EPA_MAXF (2 * HFB_EPA_CAP_IT + 4)
#define HFB_EPA_NONE 0xff

// internal verdict of a run in a workspace smaller than the request's caps: the polytope outgrew it
// before the reference would have stopped; the pair is run again in the full-size workspace
#define HFB_EPA_WS_OVERFLOW 0x7f
// free face slots a reduced-size workspace wants at the top of an iteration (a round makes one face per horizon edge)
#ifndef HFB_EPA_ROUND_FACES
#define HFB_EPA_ROUND_FACES 6
#endif

// the polytope: the vertices' w (w0 - w1), the faces, the walk's scratch
template <int MAXV_, int MAXF_>
struct EpaPolyT {
  static constexpr int MAXV = MAXV_;
  static constexpr int MAXF = MAXF_;
  double vw[MAXV_ * 3];  // w0 - w1
  double fn[MAXF_ * 3];
  double fd[MAXF_];
  uint16_t fseq[MAXF_];
  uint8_t fvid[MAXF_ * 3];
  uint8_t fadj[MAXF_ * 3];
  uint8_t fedge[MAXF_ * 3];
  uint8_t fpass[MAXF_];
  uint8_t fflag[MAXF_];  // bit0: in hull, bit1: ignore
  uint8_t stock[MAXF_];
  uint8_t stk_f[MAXF_ + 4];
  uint8_t stk_s[MAXF_ + 4];  // e | stage << 2
  uint8_t newf[MAXF_ + 4];   // faces whose geometry is pending, in creation order
};
// the polytope and the vertices' support points w0 / w1, which the loop writes and never reads (a run's side, below)
template <int MAXV_, int MAXF_>
struct EpaWsT : EpaPolyT<MAXV_, MAXF_> {
  double vw0[MAXV_ * 3];
  double vw1[MAXV_ * 3];
};
// full size: any request up to epa_max_iterations = HFB_EPA_CAP_IT fits
typedef EpaWsT<HFB_EPA_MAXV, HFB_EPA_MAXF> EpaWs;
// first-try size of the EPA kernel: room for 24 iterations (99% of the penetrating pairs of the benchmark workloads stop
// within 20).  k_epa's first tier holds the polytope alone (EpaPolySmall) and keeps the support points of its vertices
// in a store of their own (EpaSupArray, 6 doubles per vertex, in global memory); EpaWsSmall is the same size with the
// support points in the workspace, for host callers
#define HFB_EPA_SMALL_IT 24
typedef EpaPolyT<HFB_EPA_SMALL_IT + 4, 2 * HFB_EPA_SMALL_IT + 4> EpaPolySmall;
typedef EpaWsT<HFB_EPA_SMALL_IT + 4, 2 * HFB_EPA_SMALL_IT + 4> EpaWsSmall;

// A run's side: where it keeps what its loop writes and never reads back, the support points w0 / w1 of the polytope's
// vertices (the witness points read those of the result face's three vertices, the hand-over copies them all).  Every
// side has:
//   put<G>(i, sv)             stores w0 / w1 of vertex i
//   get(i, c), set(i, c, v)   component c of vertex i: w0.x w0.y w0.z w1.x w1.y w1.z
// EpaSideWs: w0 / w1 in the workspace's own arrays (EpaWsT).
template <class WS>
struct EpaSideWs {
  WS* ws;
  template <int G>
  HFB_HD void put(int i, const SV& s) const {
    ws->vw0[3 * i] = s.w0.x;
    ws->vw0[3 * i + 1] = s.w0.y;
    ws->vw0[3 * i + 2] = s.w0.z;
    ws->vw1[3 * i] = s.w1.x;
    ws->vw1[3 * i + 1] = s.w1.y;
    ws->vw1[3 * i + 2] = s.w1.z;
  }
  HFB_HD double get(int i, int c) const { return c < 3 ? ws->vw0[3 * i + c] : ws->vw1[3 * i + c - 3]; }
  HFB_HD void set(int i, int c, double v) const {
    if (c < 3) ws->vw0[3 * i + c] = v;
    else ws->vw1[3 * i + c - 3] = v;
  }
};
// EpaSupArray: w0 / w1 in an array of their own, [vertex][w0.x w0.y w0.z w1.x w1.y w1.z].  On the device the G lanes of
// a group share the six stores of a vertex; on the host (where every lane thread of the lane simulation owns a private
// copy) one thread makes all six.
struct EpaSupArray {
  double* p;
  template <int G>
  HFB_HD void put(int i, const SV& s) const {
#if defined(__CUDA_ARCH__)
    for (int c = Coop<G>::lane(); c < 6; c += G)
      p[6 * i + c] = c == 0 ? s.w0.x : c == 1 ? s.w0.y : c == 2 ? s.w0.z : c == 3 ? s.w1.x : c == 4 ? s.w1.y : s.w1.z;
#else
    p[6 * i] = s.w0.x;
    p[6 * i + 1] = s.w0.y;
    p[6 * i + 2] = s.w0.z;
    p[6 * i + 3] = s.w1.x;
    p[6 * i + 4] = s.w1.y;
    p[6 * i + 5] = s.w1.z;
#endif
  }
  HFB_HD double get(int i, int c) const { return p[6 * i + c]; }
  HFB_HD void set(int i, int c, double v) const { p[6 * i + c] = v; }
};

struct EpaParams {
  double tolerance;
  unsigned max_iterations;
};

// The counters and the status of a run.  The result (normal, depth, the three vertices of the closest face, the
// iteration count) is not kept here: it is read from EpaLoop and the workspace once the run is over (pair_epa_result).
struct EpaState {
  int status;       // EPA::Status value
  int hint0, hint1;
  // bookkeeping
  int num_vertices, hull_count, stock_top, seq;  // stock_top: freed slots waiting in EpaWs::stock
  int hwm;        // slots [0, hwm) have been handed out at least once
  int n_pending;  // entries of EpaWs::newf
  unsigned nfaces_cap, nverts_cap;
};

template <class WS>
HFB_HD v3 ws_vw(const WS* ws, int i) { return mk(ws->vw[3 * i], ws->vw[3 * i + 1], ws->vw[3 * i + 2]); }
template <int G, class WS, class Side>
HFB_HD void ws_put_v(WS* ws, const Side& sd, int i, const SV& s) {
  sd.template put<G>(i, s);
  ws->vw[3 * i] = s.w.x;
  ws->vw[3 * i + 1] = s.w.y;
  ws->vw[3 * i + 2] = s.w.z;
}
template <class WS>
HFB_HD v3 ws_fn(const WS* ws, int f) { return mk(ws->fn[3 * f], ws->fn[3 * f + 1], ws->fn[3 * f + 2]); }

template <class WS>
HFB_HD int ws_fedge(const WS* ws, int f, int e) { return ws->fedge[3 * f + e]; }
// plain stores only: every lane of a group writes the same topology redundantly, which is race-free
// as long as no write is a read-modify-write of a word that another lane also updates
template <class WS>
HFB_HD void ws_set_fedge(WS* ws, int f, int e, int v) { ws->fedge[3 * f + e] = (uint8_t)v; }
template <class WS>
HFB_HD void epa_bind(WS* ws, int fa, int ea, int fb, int eb) {  // gjk.h:312-320
  ws_set_fedge(ws, fa, ea, eb);
  ws->fadj[3 * fa + ea] = (uint8_t)fb;
  ws_set_fedge(ws, fb, eb, ea);
  ws->fadj[3 * fb + eb] = (uint8_t)fa;
}
template <class WS>
HFB_HD void epa_hull_remove(WS* ws, EpaState& E, int f) {  // hull.remove + stock.append
  ws->fflag[f] = 0;
  E.hull_count -= 1;
  ws->stock[E.stock_top++] = (uint8_t)f;
}

// EPA::newFace (:1068-1138), first half: take a slot from the stock, link it into the hull and
// record its vertices.  Returns the slot id, or HFB_EPA_NONE with status OutOfFaces (:1131-1137).
template <class WS>
HFB_HD int epa_alloc_face(WS* ws, EpaState& E, int ia, int ib, int ic) {
  // the reference's stock hands out fc_store[0], [1], ... and re-uses freed faces last-in first-out
  // (:1034-1035, gjk.h:292-298): a LIFO of freed slots on top of a counter of untouched ones
  if (E.stock_top > 0 || E.hwm < (int)E.nfaces_cap) {
    if (E.stock_top == 0 && E.hwm >= WS::MAXF) {  // the request allows more faces than this workspace holds
      E.status = HFB_EPA_WS_OVERFLOW;
      return HFB_EPA_NONE;
    }
    const int f = E.stock_top > 0 ? ws->stock[--E.stock_top] : E.hwm++;
    E.hull_count += 1;
    ws->fflag[f] = 1;
    ws->fseq[f] = (uint16_t)(E.seq++);
    ws->fpass[f] = 0;
    ws->fvid[3 * f] = (uint8_t)ia;
    ws->fvid[3 * f + 1] = (uint8_t)ib;
    ws->fvid[3 * f + 2] = (uint8_t)ic;
    ws->newf[E.n_pending++] = (uint8_t)f;
    return f;
  }
  E.status = HFB_EPA_OUT_OF_FACES;
  return HFB_EPA_NONE;
}

// EPA::newFace, second half (:1081-1128): normal, signed offset, ignore flag.  Returns 0 when the
// face is kept, else the status the reference sets (Degenerated / NonConvex).
template <class WS>
HFB_HD int epa_face_geometry(WS* ws, int f, double tol, bool force) {
  const v3 a = ws_vw(ws, ws->fvid[3 * f]), b = ws_vw(ws, ws->fvid[3 * f + 1]), c = ws_vw(ws, ws->fvid[3 * f + 2]);
  v3 n = cross(b - a, c - a);
  if (nrm(n) > DBL_EPSILON) {
    n = unit(n);
    ws->fn[3 * f] = n.x;
    ws->fn[3 * f + 1] = n.y;
    ws->fn[3 * f + 2] = n.z;
    const double a_dot_nab = dot(a, cross(b - a, n));
    const double b_dot_nbc = dot(b, cross(c - b, n));
    const double c_dot_nca = dot(c, cross(a - c, n));
    double d;
    if (a_dot_nab >= -tol && b_dot_nbc >= -tol && c_dot_nca >= -tol) {
      d = dot(a, n);
    } else {
      d = DBL_MAX;
      ws->fflag[f] = 3;  // in hull + ignore
    }
    ws->fd[f] = d;
    if (d >= -tol || force) return 0;
    return HFB_EPA_NON_CONVEX;
  }
  return HFB_EPA_DEGENERATED;
}

// Completes the pending faces in creation order, every lane doing all of them (the rare path: the
// horizon walk is about to read a face created in this round).  Returns false, with the status of the
// first face the reference would have rejected, if one fails.
template <class WS>
HFB_HD bool epa_flush_pending_serial(WS* ws, EpaState& E, double tol, bool force) {
  const int n = E.n_pending;
  E.n_pending = 0;
  for (int k = 0; k < n; ++k) {
    const int st = epa_face_geometry(ws, ws->newf[k], tol, force);
    if (st) {
      E.status = st;
      return false;
    }
  }
  return true;
}

// Completes the pending faces, one per lane.  Same verdict as the serial form: the first rejected
// face in creation order decides the status.
template <int G, class WS>
HFB_HD bool epa_flush_pending(WS* ws, EpaState& E, double tol, bool force) {
  const int n = E.n_pending;
  E.n_pending = 0;
  Coop<G>::sync();  // every lane is done reading the slots' previous occupants
  int first_bad = 0x7fffffff;  // creation index << 8 | status
  for (int k = Coop<G>::lane(); k < n; k += G) {
    const int st = epa_face_geometry(ws, ws->newf[k], tol, force);
    if (st && first_bad == 0x7fffffff) first_bad = (k << 8) | st;
  }
  if (G > 1) {
#pragma unroll
    for (int off = G / 2; off > 0; off >>= 1) {
      const int o = Coop<G>::shfl_xor(first_bad, off);
      if (o < first_bad) first_bad = o;
    }
    Coop<G>::sync();  // the other lanes' faces are read by the scan that follows
#if !defined(__CUDACC__) && defined(HFB_LANE_SIM)
    // host lane simulation only (tests/emu): every lane thread owns a private copy of the workspace (the
    // redundant serial parts of an iteration are sound for converged lanes of a warp, not for free-running
    // threads), so what the owner lanes computed above is fetched from their copies
    for (int k = 0; k < n; ++k) {
      const int owner = k % G;
      if (owner == Coop<G>::lane()) continue;
      const WS* peer = static_cast<const WS*>(lanesim::peer_workspace(owner));
      const int f = ws->newf[k];
      ws->fn[3 * f] = peer->fn[3 * f];
      ws->fn[3 * f + 1] = peer->fn[3 * f + 1];
      ws->fn[3 * f + 2] = peer->fn[3 * f + 2];
      ws->fd[f] = peer->fd[f];
      ws->fflag[f] = peer->fflag[f];
    }
    Coop<G>::sync();  // peers may move on only after everybody has read
#endif
  }
  if (first_bad != 0x7fffffff) {
    E.status = first_bad & 0xff;
    return false;
  }
  return true;
}

// EPA::findClosestFace (:1141-1154): argmin d^2 over non-ignored hull faces,
// ties -> newest (largest seq); all ignored -> hull.root (newest face).
template <int G, class WS>
HFB_HD int epa_find_closest(const WS* ws, const EpaState& E) {
  double best = DBL_MAX;
  int bseq = -1, bidx = HFB_EPA_NONE;
  int rseq = -1, ridx = HFB_EPA_NONE;  // newest face in the hull
  for (int f = Coop<G>::lane(); f < E.hwm; f += G) {
    const int fl = ws->fflag[f];
    if (!(fl & 1)) continue;
    const int sq = ws->fseq[f];
    if (sq > rseq) {
      rseq = sq;
      ridx = f;
    }
    if (fl & 2) continue;
    const double sqd = ws->fd[f] * ws->fd[f];
    if (sqd < best || (sqd == best && sq > bseq && bidx != HFB_EPA_NONE)) {
      best = sqd;
      bseq = sq;
      bidx = f;
    }
  }
  if (G > 1) {
#pragma unroll
    for (int off = G / 2; off > 0; off >>= 1) {
      const double ob = Coop<G>::shfl_xor(best, off);
      const int os = Coop<G>::shfl_xor(bseq, off);
      const int oi = Coop<G>::shfl_xor(bidx, off);
      const int ors = Coop<G>::shfl_xor(rseq, off);
      const int ori = Coop<G>::shfl_xor(ridx, off);
      // candidate validity first (a lane with no candidate has bidx == NONE)
      const bool mine = bidx != HFB_EPA_NONE, theirs = oi != HFB_EPA_NONE;
      if (theirs && (!mine || ob < best || (ob == best && os > bseq))) {
        best = ob;
        bseq = os;
        bidx = oi;
      }
      if (ors > rseq) {
        rseq = ors;
        ridx = ori;
      }
    }
  }
  return bidx != HFB_EPA_NONE ? bidx : ridx;
}

// EPA::expand (:1361-1449), iterative.  Returns `valid`.
template <class WS>
HFB_HD bool epa_expand(WS* ws, EpaState& E, double tol, int pass, int round_seq0, v3 ww, int id_w, int f0,
                       int e0, int& hz_first, int& hz_cur, int& hz_num) {
  const double dummy_precision = 3 * sqrt(DBL_EPSILON);
  int sp = 0;
  ws->stk_f[0] = (uint8_t)f0;
  ws->stk_s[0] = (uint8_t)e0;
  bool ret = false;
  while (sp >= 0) {
    const int f = ws->stk_f[sp];
    const int e = ws->stk_s[sp] & 3;
    const int stage = ws->stk_s[sp] >> 2;
    const int e1 = e == 2 ? 0 : e + 1;
    const int e2 = e == 0 ? 2 : e - 1;
    if (stage == 0) {
      if (ws->fpass[f] == pass) {
        E.status = HFB_EPA_INVALID_HULL;
        return false;
      }
      if (E.n_pending > 0 && ws->fseq[f] >= round_seq0) {
        // stepping on a face created in this round (a slot freed and handed out again): its geometry,
        // and every verdict the reference reached before this point, must exist now
        if (!epa_flush_pending_serial(ws, E, tol, false)) return false;
      }
      const v3 vf = ws_vw(ws, ws->fvid[3 * f + e]);
      if (dot(ws_fn(ws, f), ww - vf) < dummy_precision) {
        // case 1: support point "below" f -> new face on edge e of f
        const int nf = epa_alloc_face(ws, E, ws->fvid[3 * f + e1], ws->fvid[3 * f + e], id_w);
        if (nf == HFB_EPA_NONE) return false;
        epa_bind(ws, nf, 0, f, e);
        if (hz_cur != HFB_EPA_NONE) epa_bind(ws, nf, 2, hz_cur, 1);
        else hz_first = nf;
        hz_cur = nf;
        ++hz_num;
        ret = true;
        --sp;
        continue;
      }
      // case 2: "above" f -> recurse on the two other edges
      ws->fpass[f] = (uint8_t)pass;
      ws->stk_s[sp] = (uint8_t)(e | (1 << 2));
      ++sp;
      ws->stk_f[sp] = ws->fadj[3 * f + e1];
      ws->stk_s[sp] = (uint8_t)ws_fedge(ws, f, e1);
      continue;
    }
    if (!ret) return false;  // a failed sub-expand fails every caller (&& short-circuit)
    if (stage == 1) {
      ws->stk_s[sp] = (uint8_t)(e | (2 << 2));
      ++sp;
      ws->stk_f[sp] = ws->fadj[3 * f + e2];
      ws->stk_s[sp] = (uint8_t)ws_fedge(ws, f, e2);
      continue;
    }
    // stage 2: both sub-expands succeeded
    epa_hull_remove(ws, E, f);
    ret = true;
    --sp;
  }
  return ret;
}

// GJK::encloseOrigin (:437-492), iterative depth-first search.
template <int G, int CAPS>
HFB_HD bool gjk_enclose_origin(const ShapeD& sa, const ShapeD& sb, const MinkD& md, GjkState& g) {
  const int base = g.rank;
  int cnt1 = 0, cnt2 = 0, cnt3 = 0;
  int h0 = 0, h1 = 0;  // fresh zero hint per call in the reference; unused by the exhaustive argmax
  for (;;) {
    const int r = g.rank;
    if (r == 4) {
      if (fabs(triple(g.s0.w - g.s3.w, g.s1.w - g.s3.w, g.s2.w - g.s3.w)) > 0) return true;
      if (base == 4) return false;
      g.rank = 3;  // removeVertex, back in the rank-3 frame
      continue;
    }
    const int c = r == 1 ? cnt1 : (r == 2 ? cnt2 : cnt3);
    const int ncand = r == 3 ? 2 : 6;
    if (c >= ncand) {
      if (r == base) return false;
      if (r == 2) cnt2 = 0; else if (r == 3) cnt3 = 0;
      g.rank = r - 1;  // removeVertex in the parent frame
      continue;
    }
    if (r == 1) cnt1 = c + 1; else if (r == 2) cnt2 = c + 1; else cnt3 = c + 1;
    v3 dir;
    if (r == 1) {
      // both tries of axis i query +e_i (axis[i] = -1; appendVertex(-axis), :447-448)
      const int i = c >> 1;
      if (c & 1) dir = -mk(i == 0 ? -1.0 : 0.0, i == 1 ? -1.0 : 0.0, i == 2 ? -1.0 : 0.0);
      else dir = mk(i == 0 ? 1.0 : 0.0, i == 1 ? 1.0 : 0.0, i == 2 ? 1.0 : 0.0);
    } else if (r == 2) {
      const int i = c >> 1;
      const v3 d = g.s1.w - g.s0.w;
      const v3 axis = mk(i == 0 ? 1.0 : 0.0, i == 1 ? 1.0 : 0.0, i == 2 ? 1.0 : 0.0);
      const v3 p = cross(d, axis);
      if (is_zero(p, HFB_DUMMY_PRECISION)) continue;
      dir = (c & 1) ? -p : p;
    } else {
      const v3 axis = cross(g.s1.w - g.s0.w, g.s2.w - g.s0.w);
      if (is_zero(axis, HFB_DUMMY_PRECISION)) continue;
      dir = (c & 1) ? -axis : axis;
    }
    const SV nv = gjk_support<G, CAPS>(sa, sb, md, dir, h0, h1);
    put(g, r, nv);
    g.rank = r + 1;
  }
}

// EPA::evaluate (:1156-1316)
// what the expansion loop of EPA::evaluate carries from one iteration to the next, besides EpaState and the workspace
struct EpaLoop {
  unsigned it;
  int pass;
  int closest;
  v3 outer_n;  // `outer` is a COPY of the last good closest face (:1208,1284)
  double outer_d;
  int ov0, ov1, ov2;
  int resumable;  // the loop stopped at the top of an iteration because the workspace is full: it can go on, from
                  // exactly this state, in a larger one (epa_ws_grow)
};

// EPA::evaluate (:1156-1316) in three parts, so that a run which outgrows a reduced-size workspace can continue in the
// full-size one instead of starting over (k_epa, tier 0 -> tier 1).
// part 1: encloseOrigin, the initial tetrahedron and its four faces.  False: FallBack (E is final).
template <int G, int CAPS, class WS, class Side>
HFB_HD bool epa_begin(const ShapeD& sa, const ShapeD& sb, const MinkD& md, const EpaParams& P, GjkState& g, WS* ws,
                      const Side& sd, EpaState& E, EpaLoop& L) {
  const double tol = P.tolerance;
  E.hint0 = g.hint0;
  E.hint1 = g.hint1;
  E.nverts_cap = P.max_iterations + 4;
  E.nfaces_cap = 2 * P.max_iterations + 4;
  L.it = 0;
  L.pass = 0;
  L.resumable = 0;

  const bool enclosed = gjk_enclose_origin<G, CAPS>(sa, sb, md, g);
  if (g.rank > 1 && enclosed) {
    // reset (:1014-1037): all faces in stock, first allocation = slot 0
    E.hull_count = 0;
    E.seq = 0;
    E.hwm = 0;
    E.n_pending = 0;
    E.stock_top = 0;
    E.status = HFB_EPA_VALID;
    E.num_vertices = 0;
    // outward orientation (:1178-1184)
    if (dot(g.s0.w - g.s3.w, cross(g.s1.w - g.s3.w, g.s2.w - g.s3.w)) < 0) {
      const SV tmp = g.s0;
      g.s0 = g.s1;
      g.s1 = tmp;
    }
    ws_put_v<G>(ws, sd, 0, g.s0);
    ws_put_v<G>(ws, sd, 1, g.s1);
    ws_put_v<G>(ws, sd, 2, g.s2);
    ws_put_v<G>(ws, sd, 3, g.s3);
    E.num_vertices = 4;
    Coop<G>::sync();  // vertices written above are read by other lanes below
    const int t0 = epa_alloc_face(ws, E, 0, 1, 2);
    const int t1 = epa_alloc_face(ws, E, 1, 0, 3);
    const int t2 = epa_alloc_face(ws, E, 2, 1, 3);
    const int t3 = epa_alloc_face(ws, E, 0, 2, 3);
    // a forced face can only be rejected as Degenerated; the reference then has fewer than 4 faces in
    // the hull and falls through to FallBack (:1196)
    if (epa_flush_pending<G>(ws, E, tol, true)) {
      epa_bind(ws, t0, 0, t1, 0);
      epa_bind(ws, t0, 1, t2, 0);
      epa_bind(ws, t0, 2, t3, 0);
      epa_bind(ws, t1, 1, t3, 2);
      epa_bind(ws, t1, 2, t2, 1);
      epa_bind(ws, t2, 2, t3, 1);
      L.closest = epa_find_closest<G>(ws, E);
      L.outer_n = ws_fn(ws, L.closest);
      L.outer_d = ws->fd[L.closest];
      L.ov0 = ws->fvid[3 * L.closest];
      L.ov1 = ws->fvid[3 * L.closest + 1];
      L.ov2 = ws->fvid[3 * L.closest + 2];
      E.status = HFB_EPA_VALID;
      return true;
    }
  }
  // FallBack (:1299-1315); the solver maps it to EPAFailedExtract... (narrowphase.h:574-582), which reads neither the
  // depth nor the result vertex (g.s0) the reference sets here
  E.status = HFB_EPA_FALLBACK;
  return false;
}

// part 2: the expansion loop (:1209-1290), from the state (E, L, *ws) -- that of epa_begin, or of an earlier epa_run
// that stopped with L.resumable set
template <int G, int CAPS, class WS, class Side>
HFB_HD void epa_run(const ShapeD& sa, const ShapeD& sb, const MinkD& md, const EpaParams& P, WS* ws, const Side& sd,
                    EpaState& E, EpaLoop& L) {
  const double tol = P.tolerance;
  unsigned it = L.it;
  int pass = L.pass;
  int closest = L.closest;
  L.resumable = 0;
  E.status = HFB_EPA_VALID;
  for (; it < P.max_iterations; ++it) {
    if (E.num_vertices >= (int)E.nverts_cap) {
      E.status = HFB_EPA_OUT_OF_VERTICES;
      break;
    }
    // a reduced-size workspace (the request allows more than it holds) stops HERE, where the run can be handed over
    // to the full-size one, when it is out of vertices -- or so short of face slots that this iteration might not
    // fit: a round that runs out half-way (epa_alloc_face) cannot be continued, only started over
    if (E.num_vertices >= WS::MAXV ||
        (WS::MAXF < (int)E.nfaces_cap && (WS::MAXF - E.hwm) + E.stock_top < HFB_EPA_ROUND_FACES)) {
      E.status = HFB_EPA_WS_OVERFLOW;
      L.resumable = 1;  // nothing of this iteration has happened yet
      break;
    }
    int hz_first = HFB_EPA_NONE, hz_cur = HFB_EPA_NONE, hz_num = 0;
    const int id_w = E.num_vertices++;
    ws->fpass[closest] = (uint8_t)(++pass);
    const v3 cn = ws_fn(ws, closest);
    const SV w = gjk_support<G, CAPS>(sa, sb, md, cn, E.hint0, E.hint1);
    ws_put_v<G>(ws, sd, id_w, w);

    const v3 vf1 = ws_vw(ws, ws->fvid[3 * closest]);
    const v3 vf2 = ws_vw(ws, ws->fvid[3 * closest + 1]);
    const v3 vf3 = ws_vw(ws, ws->fvid[3 * closest + 2]);
    const double fdist = dot(cn, w.w - vf1);
    const double wnorm = nrm(w.w);
    if (fdist <= tol + tol * wnorm) {
      E.status = HFB_EPA_ACCURACY_REACHED;
      break;
    }
    if (nrm(w.w - vf1) <= tol + tol * wnorm || nrm(w.w - vf2) <= tol + tol * wnorm ||
        nrm(w.w - vf3) <= tol + tol * wnorm) {
      E.status = HFB_EPA_ACCURACY_REACHED;
      break;
    }
    bool valid = true;
    const int round_seq0 = E.seq;
    for (int j = 0; (j < 3) && valid; ++j)
      valid = valid && epa_expand(ws, E, tol, pass, round_seq0, w.w, id_w, ws->fadj[3 * closest + j],
                                  ws_fedge(ws, closest, j), hz_first, hz_cur, hz_num);
    // verdicts of the faces created in this round come before whatever stopped the walk after them
    if (!epa_flush_pending<G>(ws, E, tol, false)) valid = false;
    if (!valid || hz_num < 3) break;
    epa_bind(ws, hz_first, 2, hz_cur, 1);
    epa_hull_remove(ws, E, closest);
    closest = epa_find_closest<G>(ws, E);
    L.outer_n = ws_fn(ws, closest);
    L.outer_d = ws->fd[closest];
    L.ov0 = ws->fvid[3 * closest];
    L.ov1 = ws->fvid[3 * closest + 1];
    L.ov2 = ws->fvid[3 * closest + 2];
  }
  L.it = it;
  L.pass = pass;
  L.closest = closest;
}

// part 3: the final status (:1291-1298).  The rest of the result is that of the last good closest face: its normal
// and offset in L (outer_n, outer_d), its vertices (result.vertex[0..2]) at L.ov0..2 in the workspace, the iteration
// count in L.it; the depth is outer_d plus the two radii (epa_depth).
HFB_HD void epa_finish(const EpaParams& P, EpaState& E, const EpaLoop& L) {
  if (!(L.it < P.max_iterations)) E.status = HFB_EPA_FAILED;
}
HFB_HD double epa_depth(const MinkD& md, const EpaLoop& L) { return L.outer_d + (md.ssr0 + md.ssr1); }

template <int G, int CAPS, class WS, class Side>
HFB_HD void epa_evaluate(const ShapeD& sa, const ShapeD& sb, const MinkD& md, const EpaParams& P, GjkState& g, WS* ws,
                         const Side& sd, EpaState& E, EpaLoop& L) {
  if (epa_begin<G, CAPS>(sa, sb, md, P, g, ws, sd, E, L)) {
    epa_run<G, CAPS>(sa, sb, md, P, ws, sd, E, L);
    if (!(E.status == HFB_EPA_WS_OVERFLOW && L.resumable)) epa_finish(P, E, L);
  }
}

// the live part of a workspace (a) and its side (sa) copied into a larger workspace (b) and its side (sb), same slot and
// vertex numbers, by the G lanes of the group: vertices [0, num_vertices) and their support points, face slots
// [0, hwm), the stock of freed slots.  The per-iteration scratch (walk stack, pending faces) is empty at the top of an
// iteration, which is the only place a run is resumed from.
template <int G, class WSA, class SideA, class WSB, class SideB>
HFB_HD void epa_ws_grow(const WSA* a, const SideA& sa, WSB* b, const SideB& sb, const EpaState& E) {
#if !defined(__CUDACC__) && defined(HFB_LANE_SIM)
  const int l = 0, G_ = 1;  // host lane simulation: every lane thread owns private copies of both workspaces
#else
  const int l = Coop<G>::lane(), G_ = G;
#endif
  for (int i = l; i < 3 * E.num_vertices; i += G_) b->vw[i] = a->vw[i];
  for (int i = l; i < 6 * E.num_vertices; i += G_) sb.set(i / 6, i % 6, sa.get(i / 6, i % 6));
  for (int i = l; i < 3 * E.hwm; i += G_) {
    b->fn[i] = a->fn[i];
    b->fvid[i] = a->fvid[i];
    b->fadj[i] = a->fadj[i];
    b->fedge[i] = a->fedge[i];
  }
  for (int i = l; i < E.hwm; i += G_) {
    b->fd[i] = a->fd[i];
    b->fseq[i] = a->fseq[i];
    b->fpass[i] = a->fpass[i];
    b->fflag[i] = a->fflag[i];
  }
  for (int i = l; i < E.stock_top; i += G_) b->stock[i] = a->stock[i];
  Coop<G>::sync();
}
// the same between two workspaces that keep the support points themselves (EpaWsT)
template <int G, int VA, int FA, int VB, int FB>
HFB_HD void epa_ws_grow(const EpaWsT<VA, FA>* a, EpaWsT<VB, FB>* b, const EpaState& E) {
  epa_ws_grow<G>(a, EpaSideWs<const EpaWsT<VA, FA>>{a}, b, EpaSideWs<EpaWsT<VB, FB>>{b}, E);
}

// the support points of a result vertex, read from the run's side (the store closest_points_inl sums them from; the
// vertex is its w and its id in the workspace)
template <class Side>
struct WsStore {
  using V = SVSlot;
  static constexpr bool inline_projections = false;
  const Side& sd;
  HFB_HD void support_points(const SVSlot& v, v3& w0, v3& w1) const {
    w0 = mk(sd.get(v.slot, 0), sd.get(v.slot, 1), sd.get(v.slot, 2));
    w1 = mk(sd.get(v.slot, 3), sd.get(v.slot, 4), sd.get(v.slot, 5));
  }
};

// EPA::getWitnessPointsAndNormal (:1451-1466) of a finished run (not FallBack): the result simplex is the closest
// face's three vertices, read from the workspace and the side where the run left them.  Inlined, with the vertices
// passed by value: handed by reference to the out-of-line closest_points, they would go through local memory.
template <class WS, class Side>
HFB_HD void epa_witness(const WS* ws, const Side& sd, const EpaLoop& L, double depth, const MinkD& md, v3& w0, v3& w1,
                        v3& normal) {
  SVSlot r0, r1, r2;
  r0.w = ws_vw(ws, L.ov0);
  r0.slot = L.ov0;
  r1.w = ws_vw(ws, L.ov1);
  r1.slot = L.ov1;
  r2.w = ws_vw(ws, L.ov2);
  r2.slot = L.ov2;
  const WsStore<Side> st = {sd};
  closest_points_inl(r0, r1, r2, r0, 3, w0, w1, st);
  if (nrm(w0 - w1) > HFB_DUMMY_PRECISION) {
    if (depth >= 0) normal = unit(w0 - w1);
    else normal = unit(w1 - w0);
  } else {
    normal = L.outer_n;
  }
  inflate(md, normal, w0, w1);
}

}  // namespace hfb
