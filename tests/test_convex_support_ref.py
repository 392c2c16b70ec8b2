"""A plain numpy statement of the ConvexBase support argmax (`support_ref`), pinned here against the oracle's linear
scan (oracle_batch_convex_support, the restatement of the reference's getShapeSupportLinear,
support_functions.cpp:401-421) on hulls at the edges of the kernel's scan: odd vertex counts lying behind a plane (where a scan over
the zero padding of a vertex block would win), duplicated vertices (ties), NaN, +-0, infinite and axis-aligned
directions.  tests/test_gpu_full_size.py holds k_convex_support to it at bench.py's roofline size."""
import numpy as np

from tests.common import P
from oracle import oracle_lib


def support_ref(verts, nv, ids, dirs):
    """verts: (H, V, 3) vertex rows of H hulls (rows at and past nv[h] are ignored); nv: (H,) vertex counts;
    ids: (n,) hull of each query; dirs: (n, 3).  -> (index (n,) int32, support point (n, 3)).
    The dot is (x*dx + y*dy) + z*dz, elementwise in that order; the first index of the maximum wins; a NaN dot at
    index 0 wins, a NaN elsewhere never does (DESIGN.md section 4: the reference's linear scan starts from vertex 0
    and nothing compares greater than NaN)."""
    verts = np.asarray(verts, dtype=np.float64)
    ids = np.asarray(ids, dtype=np.int64)
    d = np.asarray(dirs, dtype=np.float64).reshape(-1, 3)
    v = verts[ids]
    with np.errstate(invalid="ignore"):  # 0 * inf, inf - inf: NaN dots are part of the rule
        dots = (v[..., 0] * d[:, None, 0] + v[..., 1] * d[:, None, 1]) + v[..., 2] * d[:, None, 2]
    nan = np.isnan(dots)
    live = np.arange(verts.shape[1])[None, :] < np.asarray(nv)[ids][:, None]
    idx = np.argmax(np.where(nan | ~live, -np.inf, dots), axis=1)
    idx[nan[:, 0]] = 0
    return idx.astype(np.int32), v[np.arange(len(ids)), idx]


def pad_hulls(hulls):
    """list of (nv_k, 3) point sets -> (verts (H, max nv, 3) zero-padded, nv (H,))"""
    nv = np.array([len(h) for h in hulls])
    verts = np.zeros((len(hulls), nv.max(), 3))
    for k, h in enumerate(hulls):
        verts[k, :len(h)] = h
    return verts, nv


SPECIAL_DIRS = np.array([
    [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1],        # axis-aligned: tie-prone
    [0.0, -0.0, 1], [-0.0, -0.0, -0.0], [0, 0, 0], [-0.0, 1, -0.0],              # signed zeros
    [np.nan, 0, 0], [np.nan] * 3, [1, np.nan, 0], [0, 0, np.nan],                # NaN: every dot NaN
    [np.inf, 0, 0], [-np.inf, 1, 0], [0, np.inf, -np.inf], [np.inf] * 3,        # 0 * inf: NaN at some indices
], dtype=np.float64)


def edge_hulls(seed=2024):
    """-> (hulls, ids, dirs, far): the edge point sets, queries on them, and a mask of the queries whose every dot is
    negative (odd vertex counts behind the plane z = -1, asked along directions close to +z)"""
    rng = np.random.default_rng(seed)
    hulls, ids, dirs, far = [], [], [], []

    def ask(k, d, is_far=False):
        ids.extend([k] * len(d))
        dirs.extend(d)
        far.extend([is_far] * len(d))

    for nv in (1, 3, 33, 63):
        pts = np.concatenate([rng.uniform(-0.5, 0.5, (nv, 2)), rng.uniform(-2, -1, (nv, 1))], axis=1)
        hulls.append(pts)
        up = np.concatenate([rng.uniform(-0.5, 0.5, (64, 2)), np.ones((64, 1))], axis=1)
        ask(len(hulls) - 1, np.concatenate([up, [[0, 0, 1], [0.0, -0.0, 1]]]), True)
        ask(len(hulls) - 1, SPECIAL_DIRS)
    # duplicated vertices: 8 distinct points, each repeated at several indices; a cube's corners, twice; one point, 5x
    base = rng.normal(size=(8, 3))
    hulls.append(base[rng.permutation(np.repeat(np.arange(8), 5))])
    cube = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], dtype=np.float64)
    hulls.append(np.concatenate([cube, cube[::-1]]))
    hulls.append(np.repeat(rng.normal(size=(1, 3)), 5, axis=0))
    # coordinates that are exactly zero at index 0 and elsewhere (0 * inf = NaN there), and a -0.0
    z = rng.normal(size=(37, 3))
    z[[0, 4, 9], 0] = 0.0
    z[[2, 30], 1] = -0.0
    z[[0, 17], 2] = 0.0
    hulls.append(z)
    for k in range(4, len(hulls)):
        ask(k, np.concatenate([SPECIAL_DIRS, rng.normal(size=(64, 3)), np.eye(3)[rng.integers(0, 3, 32)]]))
    return hulls, np.array(ids, dtype=np.uint32), np.array(dirs, dtype=np.float64), np.array(far)


def test_support_ref_equals_the_oracle():
    hulls, ids, dirs, far = edge_hulls()
    verts, nv = pad_hulls(hulls)
    want_i, want_s = support_ref(verts, nv, ids, dirs)
    orc = oracle_lib.OracleScene(P)
    for k, h in enumerate(hulls):
        assert orc.register_convex(h) == k
    gi, gs = orc.batch_convex_support(ids, dirs)
    bad = np.nonzero(gi != want_i)[0]
    assert not len(bad), "support index differs at queries %s" % bad[:10]
    assert gs.view(np.uint64).tobytes() == want_s.view(np.uint64).tobytes()
    # the inputs reach every rule: all dots negative, NaN at index 0, NaN elsewhere only, ties that the first index wins
    v = verts[ids.astype(np.int64)]
    with np.errstate(invalid="ignore"):
        dots = (v[..., 0] * dirs[:, None, 0] + v[..., 1] * dirs[:, None, 1]) + v[..., 2] * dirs[:, None, 2]
    live = np.arange(verts.shape[1])[None, :] < nv[ids][:, None]
    assert far.sum() >= 4 * 66 and np.all(np.where(live[far], dots[far], -1) < 0)
    assert np.all(want_s[far, 2] <= -1)  # never a zero row of the padding
    nan0 = np.isnan(dots[:, 0])
    nan_else = ~nan0 & (np.isnan(dots) & live).any(axis=1)
    assert nan0.sum() > 20 and nan_else.sum() >= 4
    best = np.where(np.isnan(dots) | ~live, -np.inf, dots)
    ties = ((best == best.max(axis=1, keepdims=True)) & live).sum(axis=1) > 1
    assert (ties & ~nan0).sum() > 50
