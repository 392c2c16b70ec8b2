"""Self pairs within robot configurations (hfb_broadphase_config_pairs) and the argument checks of the configurations
query (hfb_env_collide_configs*): no GPU needed.  The definition the finder must meet: for every configuration g of the
range and every template pair (i, j), the pair (g * L + i, g * L + j) when both objects have a box and the boxes overlap
(AABB::overlap, closed intervals: a NaN coordinate never separates two boxes), configuration by configuration in the
template's order."""
import ctypes as C
import gzip
import hashlib
import json
import os

import numpy as np
import pytest

from tests import common
from tests.common import P, compare_distance, hf, make_scenes, ref_agrees
from oracle import oracle_lib
from hppfcl_b200 import workloads as W

BIG = np.finfo(np.float64).max
INVALID = 1
NONE = [BIG, BIG, BIG, -BIG, -BIG, -BIG]  # the boxless marker

# the reference's recorded outputs for reference_sample's call (HFB_RECORD_REFERENCE=<this file> records them), looked
# up with those of tests/golden/reference_outputs.json.gz where oracle/_ref is not built
REF_OUTPUTS = os.path.join(common.ROOT, "tests", "golden", "reference_outputs_configs.json.gz")


def load_recorded():
    if os.path.exists(REF_OUTPUTS):
        common._load_recorded().update(json.load(gzip.open(REF_OUTPUTS, "rt")))


def reference_sample(sc):
    """128 configurations of the robot workload (bending joints in +-2.8 rad) registered in every backend of sc, which
    holds the host build of the device code ("emu") -> (w, ha, tfa, first, second): the self candidates of the chain
    template from the host build's boxes, the same wherever this runs"""
    w = W.robot_vs_environment(n_configs=128, n_env=16, room=1.6, seed=41, joint_range=2.8)
    hs = w["register"](sc, oracle=True)
    sc.commit()
    ha, tfa = hs[w["geom_a"]].astype(np.uint32), w["tf_a"]
    f, s = hf.broadphase_config_pairs(sc.b["emu"].scene_aabbs(ha, tfa), 16, W.chain_self_pairs(16))
    return w, ha, tfa, f, s


def brute_config(bb, links, tpl, g0=0, ng=None):
    """the self candidates, in the finder's order, by definition"""
    tpl = np.asarray(tpl, dtype=np.int64).reshape(-1, 2)
    ng = len(bb) // links - g0 if ng is None else ng
    boxless = (bb[:, 0] == BIG) & (bb[:, 3] == -BIG)
    out = []
    for g in range(g0, g0 + ng):
        for i, j in tpl:
            a, b = g * links + i, g * links + j
            apart = np.any(bb[a, :3] > bb[b, 3:]) or np.any(bb[a, 3:] < bb[b, :3])
            if not apart and not boxless[a] and not boxless[b]:
                out.append((int(a), int(b)))
    return out


def found(bb, links, tpl, g0=0, ng=None):
    f, s = hf.broadphase_config_pairs(bb, links, tpl, first_config=g0, num_configs=ng)
    return list(zip(f.tolist(), s.tolist()))


def chain_boxes(rng, n_configs, links, spread=0.25):
    """a chain per configuration: link boxes along a random walk, so near links overlap and far ones sometimes"""
    c = np.cumsum(rng.normal(scale=spread, size=(n_configs, links, 3)), axis=1).reshape(-1, 3)
    e = 0.05 + 0.15 * rng.random((n_configs * links, 3))
    return np.concatenate([c - e, c + e], axis=1)


def test_random_boxes_match_the_definition():
    rng = np.random.default_rng(1)
    for links, skip in ((16, 2), (7, 1), (3, 2)):
        bb = chain_boxes(rng, 200, links)
        tpl = W.chain_self_pairs(links, skip)
        want = brute_config(bb, links, tpl)
        assert found(bb, links, tpl) == want and len(want) > 20
        # the template's order is the order of o1 and o2, and of the output within a configuration
        rev = tpl[::-1, ::-1]
        assert found(bb, links, rev) == brute_config(bb, links, rev)
        assert {(b, a) for a, b in found(bb, links, rev)} == set(want)


def test_touching_boxes_overlap():
    links = 4
    bb = np.array([[0, 0, 0, 1, 1, 1.0], [1, 0, 0, 2, 1, 1], [1 + 1e-12, 0, 0, 3, 1, 1], [1, 1, 1, 2, 2, 2]] * 2)
    bb[4:] += 10.0
    tpl = [(0, 1), (0, 2), (0, 3), (1, 2)]
    want = [(0, 1), (0, 3), (1, 2), (4, 5), (4, 7), (5, 6)]
    assert found(bb, links, tpl) == brute_config(bb, links, tpl) == want


def test_unbounded_nonfinite_and_boxless_links():
    rng = np.random.default_rng(3)
    links = 6
    bb = chain_boxes(rng, 40, links)
    floor = [-BIG, -BIG, -BIG, BIG, BIG, 0.0]  # a halfspace link
    tilted = [-np.inf, -np.inf, -np.inf, np.inf, np.inf, np.inf]
    bb[[2, 9, 20]] = [floor, tilted, floor]
    bb[[3, 31]] = NONE
    bb[13, 1] = np.nan  # a NaN coordinate: never apart along that axis
    bb[14, 4] = np.nan
    bb[15, 0] = np.inf
    bb[16, 5] = -np.inf
    bb[17] = np.nan
    tpl = W.chain_self_pairs(links, 1)
    want = brute_config(bb, links, tpl)
    assert found(bb, links, tpl) == want
    got = set(want)
    assert (2, 4) in got and (8, 9) in got and (12, 17) in got and (13, 17) in got
    assert not any(3 in p or 31 in p for p in got)  # a boxless link takes no part, not even against the floor


def test_partial_ranges_and_capacity():
    rng = np.random.default_rng(4)
    links = 16
    bb = chain_boxes(rng, 100, links)
    tpl = W.chain_self_pairs(links)
    whole = found(bb, links, tpl)
    parts = []
    for g0, ng in ((0, 1), (1, 33), (34, 0), (34, 66)):
        part = found(bb, links, tpl, g0, ng)
        assert part == brute_config(bb, links, tpl, g0, ng)
        assert all(g0 * links <= a < (g0 + ng) * links for a, _ in part)
        parts += part
    assert parts == whole
    # at most `capacity` stored, all counted
    L = hf.load_library()
    tp = np.ascontiguousarray(tpl)
    f, s = np.zeros(5, np.uint32), np.zeros(5, np.uint32)
    cnt = C.c_size_t(0)
    assert L.hfb_broadphase_config_pairs(len(bb), bb.ctypes.data, links, len(tp), tp.ctypes.data, 0, 100, f.ctypes.data,
                                         s.ctypes.data, 5, C.byref(cnt)) == 0
    assert cnt.value == len(whole) and list(zip(f.tolist(), s.tolist())) == whole[:5]
    assert L.hfb_broadphase_config_pairs(len(bb), bb.ctypes.data, links, len(tp), tp.ctypes.data, 0, 100, None, None, 0,
                                         C.byref(cnt)) == 0 and cnt.value == len(whole)


def test_empty_template_and_empty_sets():
    rng = np.random.default_rng(5)
    bb = chain_boxes(rng, 10, 4)
    assert found(bb, 4, np.zeros((0, 2), np.uint32)) == []
    assert found(bb[:0], 4, [(0, 2)]) == []
    assert found(bb[:4], 4, [(0, 1), (1, 3)]) == brute_config(bb[:4], 4, [(0, 1), (1, 3)])


@pytest.mark.parametrize("tpl,why", [([(0, 4)], "j >= L"), ([(4, 0)], "i >= L"), ([(1, 1)], "i == j"),
                                     ([(0, 2), (1, 3), (0, 2)], "listed twice"), ([(0, 2), (2, 0)], "listed twice, reversed"),
                                     ([(0, 0xffffffff)], "j far out of range")])
def test_malformed_templates_are_refused(tpl, why):
    L = hf.load_library()
    bb = chain_boxes(np.random.default_rng(6), 3, 4)
    tp = np.ascontiguousarray(np.array(tpl, dtype=np.uint32))
    f, s = np.zeros(8, np.uint32), np.zeros(8, np.uint32)
    cnt = C.c_size_t(12345)
    assert L.hfb_broadphase_config_pairs(12, bb.ctypes.data, 4, len(tp), tp.ctypes.data, 0, 3, f.ctypes.data,
                                         s.ctypes.data, 8, C.byref(cnt)) == INVALID, why
    assert cnt.value == 12345  # nothing written
    with pytest.raises(hf.EngineError):
        hf.broadphase_config_pairs(bb, 4, tpl)


def test_layout_range_and_null_arguments_are_refused():
    L = hf.load_library()
    bb = chain_boxes(np.random.default_rng(7), 3, 4, spread=0.05)
    tp = np.ascontiguousarray(np.array([(0, 2), (1, 3)], dtype=np.uint32))
    f, s = np.zeros(8, np.uint32), np.zeros(8, np.uint32)
    cnt = C.c_size_t(0)
    fn = L.hfb_broadphase_config_pairs
    B, T, F, S = bb.ctypes.data, tp.ctypes.data, f.ctypes.data, s.ctypes.data

    def call(n=12, links=4, g0=0, ng=3, aabbs=B, n_tpl=2, tpl=T, first=F, second=S, cap=8, out=C.byref(cnt)):
        return fn(n, aabbs, links, n_tpl, tpl, g0, ng, first, second, cap, out)

    assert call() == 0 and cnt.value == len(brute_config(bb, 4, tp)) > 0
    for bad in (dict(links=0), dict(n=11), dict(links=5), dict(g0=4, ng=0), dict(g0=1, ng=3), dict(g0=0, ng=4),
                dict(ng=2 ** 64 - 1), dict(aabbs=None), dict(tpl=None), dict(first=None), dict(second=None), dict(out=None)):
        assert call(**bad) == INVALID, bad
    assert call(g0=3, ng=0) == 0 and cnt.value == 0  # an empty range at the end
    assert call(n_tpl=0, tpl=None) == 0 and cnt.value == 0
    assert call(first=None, second=None, cap=0) == 0 and cnt.value > 0  # counted, none stored
    assert call(n=0, aabbs=None, ng=0) == 0 and cnt.value == 0


def test_configs_abi_argument_checks():
    """the configurations query refuses null and malformed arguments before it touches the context or the env"""
    L = hf.load_library()
    ctx = C.create_string_buffer(4096)  # stand-ins: the calls must refuse before reading them
    env = C.create_string_buffer(4096)
    h = np.zeros(8, dtype=np.uint32)
    t = np.zeros(8, dtype=P.transform_dtype)
    tp = np.ascontiguousarray(np.array([(0, 2), (1, 3)], dtype=np.uint32))
    hp, tfp, tpp = h.ctypes.data, t.ctypes.data, tp.ctypes.data
    req = P.CollisionRequestPOD()
    f, s = np.zeros(8, dtype=np.uint32), np.zeros(8, dtype=np.uint32)
    rec = np.zeros(8, dtype=P.contact_dtype)
    cnt = np.zeros(4, dtype=np.uint32)
    v = np.zeros(2, dtype=np.uint8)

    def kind(k):
        return P.SceneContacts(f.ctypes.data, s.ctypes.data, rec.ctypes.data, 8, cnt[2 * k:].ctypes.data,
                               cnt[2 * k + 1:].ctypes.data)

    ok = P.ConfigsOut(v.ctypes.data, kind(0), kind(1))
    for fn in (L.hfb_env_collide_configs, L.hfb_env_collide_configs_device):
        extra = [None] if fn is L.hfb_env_collide_configs_device else []

        def call(c=ctx, e=env, a_h=hp, a_t=tfp, tpl=tpp, r=C.byref(req), o=C.byref(ok)):
            return fn(c, e, 8, a_h, a_t, 4, 2, tpl, 0, 2, r, o, *extra)

        for bad in (dict(c=None), dict(e=None), dict(a_h=None), dict(a_t=None), dict(tpl=None), dict(r=None), dict(o=None)):
            assert call(**bad) == INVALID, bad
        for which in ("env", "self"):
            for k in range(3):  # a capacity without one of the three pair buffers of either kind
                good = getattr(ok, which)
                broken = P.SceneContacts(*[None if j == k else getattr(good, n) for j, (n, _) in enumerate(P.SceneContacts._fields_)])
                bad = P.ConfigsOut(ok.verdicts, broken if which == "env" else ok.env, broken if which == "self" else ok.self)
                assert call(o=C.byref(bad)) == INVALID, (which, k)


def test_robot_workload_default_is_unchanged():
    """joint_range=1.2 is the default: the same random draws and the same arrays as before the parameter existed
    (fingerprints taken from the generator as it was; trigonometry may differ in the last bit between numpy builds)"""
    w = W.robot_vs_environment()
    digest = lambda a: hashlib.sha256(np.ascontiguousarray(a, dtype=np.int64).tobytes()).hexdigest()[:16]  # noqa: E731
    assert digest(w["geom_a"]) == "11c90487808eea87" and digest(w["geom_b"]) == "19cb8561284f6e75"
    assert w["room"] == 3.6203867196751234
    want = {
        "tf_a": (16384, 76053.37379736634, 6157.369080324325, 188827.989386869, 2340,
                 [[3.16702788583671, 2.6558277436418645, 0.11], [1.867925225940639, 3.547876289760399, 0.963886472698416],
                  [-0.05665505984056449, 0.5076937524994785, 0.03284833378744917],
                  [5.427121995716777, 4.255087660191926, 0.5123019004095944], [3.583486763713546, 2.6248349649504634, 0.11],
                  [0.4244206079424373, 0.5513356250944509, 0.8892761891520893],
                  [2.353072570664305, 2.6755152617498665, 0.9435461984966971]],
                 [-0.50139351809215, 0.7582322840385183, -0.41675933517668073, -0.004168519742940748, 0.47955800856814756,
                  0.8775002791232064, 0.8652093177135403, 0.44171022159316703, -0.23728657079949925]),
        "tf_b": (100000, 446603.1237191329, 3488.8632487453083, 969340.4149366615, 14285,
                 [[0.0, 0.0, 0.0], [2.4693843643605105, 0.8089084095146029, 0.6323264647969961],
                  [2.3240194670119334, 1.5195672919763505, 1.2147096549630534],
                  [0.9708081544544628, 1.6519920037287728, 1.006626455850322],
                  [0.5396983667841555, 3.327536219911803, 0.946362627772705],
                  [0.2947670955382099, 1.8714390605816418, 1.1898825185234898],
                  [1.7590213139592379, 3.5180943835325653, 0.7353836980181581]],
                 [0.24716267894887545, -0.8624307184257449, 0.44172827173554174, 0.02728836484215047, 0.46188662086672294,
                  0.886519088688203, -0.9685896733287305, -0.20706039065927995, 0.13769545867954247]),
    }
    for k, (n, sum_t, sum_r, sum_t2, step, rows_t, row_r) in want.items():
        t = w[k]
        rows = np.arange(0, n, step)[:7]
        assert len(t) == n
        np.testing.assert_allclose([t["T"].sum(), t["R"].sum(), (t["T"] ** 2).sum()], [sum_t, sum_r, sum_t2], rtol=1e-12)
        np.testing.assert_allclose(t["T"][rows], rows_t, rtol=1e-13, atol=1e-15)
        np.testing.assert_allclose(t["R"][rows[3]], row_r, rtol=1e-13, atol=1e-15)
    assert len(W.chain_self_pairs(16)) == 105
    assert all(j >= i + 2 for i, j in W.chain_self_pairs(16))


def test_self_pairs_reference_sample():
    """the sample the GPU test compares the device's self records on: oracle, host build of the device code and reference
    build agree on every record, and the template's pairs include colliding ones"""
    oracle_lib.build_ref()
    load_recorded()
    sc = make_scenes(ref=True)
    w, ha, tfa, f, s = reference_sample(sc)
    args = (ha[f], tfa[f], ha[s], tfa[s])
    ro = sc.b["oracle"].batch_collide(*args, nthreads=0)
    compare_distance(ro, sc.b["emu"].batch_collide(*args), what="self pairs, host build")
    ref_agrees(sc, "batch_collide", ro, args, "self pairs")
    assert len(f) > 200 and (ro["num_contacts"] > 0).sum() > 20
