"""Shared test helpers: the same geometry registered in the oracle (CPU
restatement of the reference), the CPU emulation of the device code (tests/emu)
and -- on a GPU box -- the CUDA engine; plus the parity comparison."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import hppfcl_b200 as hf  # noqa: E402
from hppfcl_b200 import _pod as P  # noqa: E402
from oracle import oracle_lib  # noqa: E402

EMU_DIR = os.path.join(ROOT, "tests", "emu")
_EMU = None


def emu_lib():
    global _EMU
    if _EMU is None:
        so = os.environ.get("HFB_EMU_SO") or os.path.join(EMU_DIR, "libemu.so")  # another build under test
        src = os.path.join(EMU_DIR, "emu.cpp")
        csrc = os.path.join(ROOT, "hpp-fcl_b200", "csrc")
        deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
        if "HFB_EMU_SO" not in os.environ and (
                not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps)):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off",
                                   "-march=x86-64-v2", "-Wno-unknown-pragmas", "-pthread", "-shared", "-o", so, src])
        L = C.CDLL(so)
        L.emu_create.restype = C.c_void_p
        L.emu_destroy.argtypes = [C.c_void_p]
        L.emu_register_convex.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        L.emu_register_shapes.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.emu_register_shapes.restype = C.c_int64
        L.emu_register_halfspaces.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t]
        L.emu_register_halfspaces.restype = C.c_int64
        for name in ("emu_batch_distance", "emu_batch_collide"):
            getattr(L, name).argtypes = [C.c_void_p, C.c_size_t] + [C.c_void_p] * 7
        L.emu_batch_convex_support.argtypes = [C.c_void_p, C.c_size_t] + [C.c_void_p] * 4
        L.emu_register_bvh.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                       C.c_uint32]
        L.emu_register_bvh_obb.argtypes = L.emu_register_bvh.argtypes
        L.emu_update_shapes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        L.emu_update_convex.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
        _EMU = L
    return _EMU


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class EmuScene:
    def __init__(self):
        self.L = emu_lib()
        self.h = C.c_void_p(self.L.emu_create())

    def __del__(self):
        try:
            self.L.emu_destroy(self.h)
        except Exception:
            pass

    def register_convex(self, points):
        pts = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        return self.L.emu_register_convex(self.h, _ptr(pts), pts.shape[0])

    def register_bvh_obbrss(self, nodes, vertices, triangles):
        nodes = np.ascontiguousarray(nodes, dtype=P.bvh_node_dtype)
        v = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
        t = np.ascontiguousarray(triangles, dtype=np.uint32).reshape(-1, 3)
        bid = self.L.emu_register_bvh(self.h, _ptr(nodes), nodes.shape[0], _ptr(v), v.shape[0], _ptr(t), t.shape[0])
        assert bid >= 0
        return bid

    def register_bvh_obb(self, nodes, vertices, triangles):
        nodes = np.ascontiguousarray(nodes, dtype=P.bvh_node_dtype)
        v = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
        t = np.ascontiguousarray(triangles, dtype=np.uint32).reshape(-1, 3)
        bid = self.L.emu_register_bvh_obb(self.h, _ptr(nodes), nodes.shape[0], _ptr(v), v.shape[0], _ptr(t), t.shape[0])
        assert bid >= 0
        return bid

    def register_shapes(self, shapes):
        shapes = np.ascontiguousarray(shapes, dtype=P.shape_dtype)
        first = self.L.emu_register_shapes(self.h, _ptr(shapes), shapes.shape[0])
        assert first >= 0
        return np.arange(first, first + shapes.shape[0], dtype=np.uint32)

    def register_halfspaces(self, kind, n_d, ssr=None):
        nd = np.ascontiguousarray(n_d, dtype=np.float64).reshape(-1, 4)
        r = None if ssr is None else np.ascontiguousarray(ssr, dtype=np.float64).reshape(-1)
        first = self.L.emu_register_halfspaces(self.h, int(kind), _ptr(nd), None if r is None else _ptr(r), nd.shape[0])
        assert first >= 0
        return np.arange(first, first + nd.shape[0], dtype=np.uint32)

    def scene_aabbs(self, handles, tfs):
        h = np.ascontiguousarray(handles, dtype=np.uint32)
        tf = np.ascontiguousarray(tfs, dtype=P.transform_dtype)
        out = np.zeros((len(h), 6))
        self.L.emu_scene_aabbs.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
        assert self.L.emu_scene_aabbs(self.h, len(h), _ptr(h), _ptr(tf), _ptr(out)) == 0
        return out

    def commit(self):
        pass

    def update_shapes(self, handles, shapes):
        handles = np.ascontiguousarray(handles, dtype=np.uint32)
        shapes = np.ascontiguousarray(shapes, dtype=P.shape_dtype)
        rc = self.L.emu_update_shapes(self.h, _ptr(handles), _ptr(shapes), C.c_size_t(handles.shape[0]))
        if rc != 0:
            raise ValueError("emu error %d" % rc)

    def update_convex(self, convex_id, points):
        pts = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        rc = self.L.emu_update_convex(self.h, C.c_uint32(int(convex_id)), _ptr(pts), C.c_uint32(pts.shape[0]))
        if rc != 0:
            raise ValueError("emu error %d" % rc)

    lanes = 1  # > 1: shape pairs run through lane groups of that many threads (tests/emu lanesim)

    def _run(self, fn, dtype, h1, tf1, h2, tf2, req, want_guess):
        h1 = np.ascontiguousarray(h1, dtype=np.uint32)
        h2 = np.ascontiguousarray(h2, dtype=np.uint32)
        tf1 = np.ascontiguousarray(tf1, dtype=P.transform_dtype)
        tf2 = np.ascontiguousarray(tf2, dtype=P.transform_dtype)
        n = h1.shape[0]
        out = np.zeros(n, dtype=dtype)
        g = gg = gh = None
        if want_guess:
            gg = np.zeros((n, 3))
            gh = np.zeros((n, 2), dtype=np.int32)
            g = P.GuessOut(_ptr(gg), _ptr(gh))
        if self.lanes > 1:
            lfn = self.L.emu_batch_distance_lanes if fn is self.L.emu_batch_distance else self.L.emu_batch_collide_lanes
            lfn.restype = C.c_long
            lfn.argtypes = [C.c_void_p, C.c_int, C.c_size_t] + [C.c_void_p] * 7
            rc = lfn(self.h, self.lanes, n, _ptr(h1), _ptr(tf1), _ptr(h2), _ptr(tf2), C.byref(req), _ptr(out),
                     C.byref(g) if g is not None else None)
            if rc == -1:
                raise RuntimeError("a lane of a group never reached a barrier (divergent control flow)")
            if rc > 0:
                raise RuntimeError("the lanes of a group disagreed on %d pairs" % rc)
            if rc == -2:  # meshes in the batch (one lane per query on the device as well) or a special request
                rc = fn(self.h, n, _ptr(h1), _ptr(tf1), _ptr(h2), _ptr(tf2), C.byref(req), _ptr(out),
                        C.byref(g) if g is not None else None)
        else:
            rc = fn(self.h, n, _ptr(h1), _ptr(tf1), _ptr(h2), _ptr(tf2), C.byref(req), _ptr(out),
                    C.byref(g) if g is not None else None)
        if rc != 0:
            raise ValueError("emu error %d" % rc)
        return (out, gg, gh) if want_guess else out

    def batch_distance(self, h1, tf1, h2, tf2, req=None, want_guess=False):
        return self._run(self.L.emu_batch_distance, P.distance_result_dtype, h1, tf1, h2, tf2,
                         req or P.DistanceRequestPOD(), want_guess)

    def batch_collide(self, h1, tf1, h2, tf2, req=None, want_guess=False):
        return self._run(self.L.emu_batch_collide, P.contact_dtype, h1, tf1, h2, tf2,
                         req or P.CollisionRequestPOD(), want_guess)

    def batch_collide_contacts(self, h1, tf1, h2, tf2, req=None, max_extra=3):
        req = req or P.CollisionRequestPOD()
        h1 = np.ascontiguousarray(h1, dtype=np.uint32)
        h2 = np.ascontiguousarray(h2, dtype=np.uint32)
        tf1 = np.ascontiguousarray(tf1, dtype=P.transform_dtype)
        tf2 = np.ascontiguousarray(tf2, dtype=P.transform_dtype)
        n = h1.shape[0]
        out = np.zeros(n, dtype=P.contact_dtype)
        extra = np.zeros((n, max(max_extra, 1)), dtype=P.contact_dtype)
        counts = np.zeros(n, dtype=np.uint32)
        fn = self.L.emu_batch_collide_contacts
        fn.argtypes = [C.c_void_p, C.c_size_t] + [C.c_void_p] * 6 + [C.c_uint32, C.c_void_p, C.c_void_p]
        rc = fn(self.h, n, _ptr(h1), _ptr(tf1), _ptr(h2), _ptr(tf2), C.byref(req), _ptr(out), max_extra, _ptr(extra),
                _ptr(counts))
        if rc != 0:
            raise ValueError("emu error %d" % rc)
        return out, extra[:, :max_extra], counts

    def batch_convex_support(self, ids, dirs):
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        d = np.ascontiguousarray(dirs, dtype=np.float64).reshape(-1, 3)
        idx = np.zeros(ids.shape[0], dtype=np.int32)
        sup = np.zeros((ids.shape[0], 3))
        rc = self.L.emu_batch_convex_support(self.h, ids.shape[0], _ptr(ids), _ptr(d), _ptr(idx), _ptr(sup))
        assert rc == 0
        return idx, sup


class MultiScene:
    """Registers identical geometry in every backend given."""

    def __init__(self, backends):
        self.b = backends  # dict name -> scene object

    def register_convex(self, points, tris=None):
        ids = set()
        for name, s in self.b.items():
            if name == "oracle":
                ids.add(int(s.register_convex(points, tris)))
            elif name == "ref":  # Convex<Triangle> needs its faces; a TriangleP's vertex set is a bare point set
                ids.add(int(s.register_points(points) if tris is None else s.register_convex(points, tris)))
            else:
                ids.add(int(s.register_convex(points)))
        assert len(ids) == 1
        return ids.pop()

    def register_bvh(self, vertices, triangles):
        """The oracle builds the tree with the reference's builder; the other backends get the exported
        node array through the product ABI (what a binding copies out of BVHModel<OBBRSS>::bvs)."""
        bid, nodes = self.b["oracle"].register_bvh(vertices, triangles)
        for name, s in self.b.items():
            if name == "ref":  # (builds its own tree: the reference's builder, which the oracle's restates)
                assert s.register_bvh(vertices, triangles)[0] == bid
            elif name != "oracle":
                assert s.register_bvh_obbrss(nodes, vertices, triangles) == bid
        return bid, nodes

    def register_bvh_obb(self, vertices, triangles):
        """a plain BVHModel<OBB> of the mesh: in the oracle and the reference build a model serves both kinds (its id
        is shared), the product registers the node array a second time as an OBB model"""
        bid, nodes = self.b["oracle"].register_bvh(vertices, triangles)
        for name, s in self.b.items():
            if name == "ref":
                assert s.register_bvh(vertices, triangles)[0] == bid
            elif name != "oracle":
                assert s.register_bvh_obb(nodes, vertices, triangles) == bid
        return bid, nodes

    def register_shapes(self, shapes):
        hs = [s.register_shapes(shapes) for s in self.b.values()]
        for h in hs[1:]:
            assert np.array_equal(h, hs[0])
        return hs[0]

    def register_halfspaces(self, kind, n_d, ssr=None):
        hs = [s.register_halfspaces(kind, n_d, ssr) for s in self.b.values()]
        for h in hs[1:]:
            assert np.array_equal(h, hs[0])
        return hs[0]

    def commit(self):
        for name, s in self.b.items():
            if hasattr(s, "commit"):
                s.commit()


def make_scenes(gpu=False, emu=True, ref=False):
    """ref=True adds the reference build (oracle/_ref) where it exists: the known-answer tests then check their
    literal numbers on records the reference's own code agrees with bit for bit"""
    b = {"oracle": oracle_lib.OracleScene(P)}
    if ref:
        b["ref"] = reference_scene()
    if emu:
        b["emu"] = EmuScene()
    if gpu:
        b["gpu"] = hf.Engine(0)
    return MultiScene(b)


# ---------------------------------------------------------------------------------------------------
# The reference build (oracle/_ref) is compiled from the reference's sources, which a checkout of this project does
# not carry.  Its outputs for the tests that compare against it are kept, as per-field digests, in
# tests/golden/reference_outputs.json.gz: where the reference build is absent, reference_scene() answers every call with
# the oracle's (box queries: the host build of the device code's) output, after checking that each field the reference
# defines has the digest the reference's own output had.  HFB_RECORD_REFERENCE=<file> (with oracle/_ref built)
# records the digests of a run into <file>.
REF_OUTPUTS = os.path.join(ROOT, "tests", "golden", "reference_outputs.json.gz")
import base64  # noqa: E402
import zlib  # noqa: E402

_RECORDED = {}


def _canon(a):
    """bytes of an array with every NaN and every zero in one bit pattern (the comparisons treat them as equal)"""
    a = np.array(a)
    if a.dtype.kind == "f":
        a = a.astype(np.float64)
        a[np.isnan(a)] = np.nan
        a[a == 0] = 0.0
    return np.ascontiguousarray(a).tobytes()


def _digest(x):
    import hashlib
    if isinstance(x, tuple):
        return [_digest(v) for v in x]
    if not isinstance(x, np.ndarray):
        return repr(x)
    h = lambda a: hashlib.sha256(_canon(a)).hexdigest()[:10]  # noqa: E731
    if x.dtype.names is None:
        return {"": h(x)}
    x = x.copy()
    if "num_contacts" in x.dtype.names:  # the reference leaves `distance` unset without a contact
        x["distance"][x["num_contacts"] == 0] = 0
    return {f: h(x[f]) for f in x.dtype.names if not f.startswith("_")}


class _StandIn:
    """the oracle (box queries: the host build of the device code, with the same geometry registered in it on first
    use) answers for the reference"""

    def __init__(self):
        self.orc, self.emu, self.log = oracle_lib.OracleScene(P), None, []

    def register_convex(self, points, tris=None):
        self.log.append(("register_convex", (points,)))
        return self.orc.register_convex(points, tris)

    def register_points(self, points):
        return self.register_convex(points)

    def register_shapes(self, shapes):
        self.log.append(("register_shapes", (shapes,)))
        return self.orc.register_shapes(shapes)

    def register_halfspaces(self, kind, n_d, ssr=None):
        self.log.append(("register_halfspaces", (kind, n_d, ssr)))
        return self.orc.register_halfspaces(kind, n_d, ssr)

    def object_aabbs(self, handles, tfs):
        if self.emu is None:
            self.emu = EmuScene()
            for name, args in self.log:
                getattr(self.emu, name)(*args)
        return self.emu.scene_aabbs(handles, tfs)

    def obb_is_obbrss_half(self, bvh_id):
        return None  # a property of the reference's own builder: the recorded value answers

    def __getattr__(self, name):  # register_bvh, batch_distance, batch_collide, batch_collide_contacts
        return getattr(self.orc, name)


_NUMBERING = ("register_convex", "register_points", "register_shapes", "register_halfspaces")


class ReferenceScene:
    """RefScene's interface.  Live (oracle/_ref built): the reference build answers, and with HFB_RECORD_REFERENCE the
    digests of its outputs are recorded.  Replay: the stand-in answers, checked against the recorded digests."""

    def __init__(self):
        self.live = oracle_lib.RefScene(P) if oracle_lib.ref_available() else None
        self.record = bool(os.environ.get("HFB_RECORD_REFERENCE")) and self.live is not None
        self.stand_in = _StandIn() if self.live is None or self.record else None
        self.pod = P
        import hashlib
        self._h = hashlib.sha256()

    def _key(self, name, args, kw):
        """a call's key: the geometry registered so far and the call's own inputs.  Registrations extend the scene's
        state; queries do not, so adding a query to a test leaves the keys of the other calls as they were."""
        h = self._h if name.startswith("register_") else self._h.copy()
        h.update(name.encode())
        for v in list(args) + sorted(kw.items()):
            if isinstance(v, tuple) and len(v) == 2 and isinstance(v[0], str):  # keyword argument
                if v[0] == "nthreads":
                    continue
                h.update(v[0].encode())
                v = v[1]
            if isinstance(v, C.Structure):  # request: pointer fields (cached guesses) vary from run to run
                v = type(v).from_buffer_copy(bytes(v))
                v.q.cached_gjk_guess = v.q.cached_support_func_guess = None
                h.update(bytes(v))
            else:
                h.update(_canon(v) if isinstance(v, np.ndarray) else repr(v).encode())
        return h.copy().hexdigest()[:16]

    def _call(self, name, *args, **kw):
        key = self._key(name, args, kw)
        if self.live is not None and not self.record:
            return getattr(self.live, name)(*args, **kw)
        std_kw = {k: v for k, v in kw.items() if k != "nthreads" or name.startswith("batch_")}
        got = getattr(self.stand_in, name)(*args, **std_kw)
        if name in _NUMBERING:
            # handle numbering only: every caller asserts it equal across backends, so nothing is recorded for it
            return getattr(self.live, name)(*args, **kw) if self.record else got
        if self.record:
            out = getattr(self.live, name)(*args, **kw)
            want, have = _digest(out), _digest(got)
            diff = _differing(want, have)
            _RECORDED[key] = {"call": name, "out": want if name != "obb_is_obbrss_half" else out,
                              "not_reproduced": diff, "patch": _patches(out, got, diff)}
            return out
        rec = _load_recorded().get(key)
        assert rec is not None and rec["call"] == name, (
            "%s: no recorded output of the reference for this call (tests/golden/reference_outputs.json.gz)" % name)
        if name == "obb_is_obbrss_half":
            return rec["out"]
        patch = rec.get("patch", {})
        for p, (rows, vals) in patch.items():
            leaf = _leaf(got, p)
            rows = np.cumsum(_unpack(rows, np.uint32))
            leaf[rows] = _unpack(vals, leaf.dtype).reshape((len(rows),) + leaf.shape[1:])
        have = _digest(got)
        bad = [p for p in _differing(rec["out"], have) if p not in rec["not_reproduced"] or p in patch]
        assert not bad, "%s: %s differ from the reference's recorded output" % (name, bad)
        return _blank(got, [p for p in rec["not_reproduced"] if p not in patch])

    def __getattr__(self, name):
        if name.startswith(("register_", "batch_")) or name in ("object_aabbs", "obb_is_obbrss_half"):
            return lambda *a, **k: self._call(name, *a, **k)
        raise AttributeError(name)


def _differing(want, have, path=""):
    if isinstance(want, list):
        return [p for k, (w, h) in enumerate(zip(want, have)) for p in _differing(w, h, "%s%d." % (path, k))]
    if isinstance(want, dict):
        return [path + f for f in want if want[f] != have.get(f)]
    return [] if want == have else [path]


def _prepared(x):
    if isinstance(x, tuple):
        return tuple(_prepared(v) for v in x)
    if isinstance(x, np.ndarray) and x.dtype.names and "num_contacts" in x.dtype.names:
        x = x.copy()
        x["distance"][x["num_contacts"] == 0] = 0  # as in _digest
    return x


def _leaf(x, path):
    """the array a digest path ("field", "k.field", "k.") names in an output"""
    if isinstance(x, tuple):
        k, rest = path.split(".", 1)
        return _leaf(x[int(k)], rest)
    return x if path == "" else x[path]


def _pack(a):
    return base64.b64encode(zlib.compress(np.ascontiguousarray(a).tobytes(), 9)).decode()


def _unpack(s, dtype):
    return np.frombuffer(zlib.decompress(base64.b64decode(s)), dtype=dtype)


def _patches(out, got, paths, limit=4096):
    """where the stand-in differs from the reference in a few rows of a field only (TriangleP pairs the reference does
    not serve, say), the reference's rows are kept: path -> [row numbers (as steps), its canonical values there]"""
    res = {}
    ro, go = _prepared(out), _prepared(got)
    for p in paths:
        a, b = _leaf(ro, p), _leaf(go, p)
        if not isinstance(a, np.ndarray) or not isinstance(b, np.ndarray) or a.shape != b.shape or a.ndim == 0:
            continue
        ca = np.frombuffer(_canon(a), np.uint8).reshape(len(a), -1)
        cb = np.frombuffer(_canon(b), np.uint8).reshape(len(b), -1)
        rows = np.nonzero((ca != cb).any(axis=1))[0]
        if len(rows) <= limit:
            res[p] = [_pack(np.diff(rows, prepend=0).astype(np.uint32)), _pack(ca[rows])]
    return res


def _blank(x, paths, path=""):
    """the fields the stand-in does not reproduce (the reference defines them differently or not at all) are
    returned as NaN / all-ones, so that no comparison can pass on them by accident"""
    if isinstance(x, tuple):
        return tuple(_blank(v, paths, "%s%d." % (path, k)) for k, v in enumerate(x))
    if not isinstance(x, np.ndarray):
        return x
    for p in paths:
        if not p.startswith(path):
            continue
        f = p[len(path):]
        tgt = x if f == "" else x[f]
        tgt[...] = np.nan if tgt.dtype.kind == "f" else np.iinfo(tgt.dtype).max
    return x


_LOADED = None


def _load_recorded():
    global _LOADED
    if _LOADED is None:
        import gzip
        import json
        _LOADED = json.load(gzip.open(REF_OUTPUTS, "rt")) if os.path.exists(REF_OUTPUTS) else {}
    return _LOADED


def _write_recorded():
    import gzip
    import json
    path = os.environ.get("HFB_RECORD_REFERENCE")
    if not path or not _RECORDED:
        return
    old = json.load(gzip.open(path, "rt")) if os.path.exists(path) else {}
    old.update(_RECORDED)
    with gzip.GzipFile(path, "wb", mtime=0) as f:  # (mtime 0: the same records give the same bytes)
        f.write((json.dumps(old, sort_keys=True, separators=(",", ":")) + "\n").encode())


import atexit  # noqa: E402

atexit.register(_write_recorded)


def reference_scene():
    return ReferenceScene()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def compare_distance(ref, got, rtol=1e-6, exact=True, what=""):
    """north_star bar: status/flags/indices bit-exact; distances, points, normals within
    1e-6 relative.  With exact=True additionally require bitwise-identical doubles
    (oracle and device code execute the same IEEE operation sequence)."""
    assert ref.shape == got.shape
    assert np.array_equal(ref["status"], got["status"]), "%s: status words differ at %s" % (
        what, np.nonzero(ref["status"] != got["status"])[0][:10])
    if exact:
        assert np.array_equal(ref["iterations"], got["iterations"]), "%s: iteration counts differ" % what
    assert np.array_equal(ref["b1"], got["b1"]) and np.array_equal(ref["b2"], got["b2"])
    dname = "min_distance" if "min_distance" in ref.dtype.names else "distance"
    for f in (dname, "p1", "p2", "normal") + (("pos", "distance_lower_bound") if "pos" in ref.dtype.names else ()):
        a, b = ref[f], got[f]
        assert np.array_equal(np.isnan(a), np.isnan(b)), "%s: NaN pattern differs in %s" % (what, f)
        if exact:
            bad = _bits(a) != _bits(b)
            bad &= ~(np.isnan(a) & np.isnan(b))
            bad &= ~((a == 0) & (b == 0))
            assert not bad.any(), "%s: %s not bit-identical at rows %s (max abs diff %g)" % (
                what, f, np.unique(np.nonzero(bad)[0])[:10], np.nanmax(np.abs(a - b)))
        else:
            m = ~np.isnan(a)
            scale = np.maximum(1.0, np.abs(a[m]))
            assert np.all(np.abs(a[m] - b[m]) <= rtol * scale), "%s: %s exceeds rtol" % (what, f)
    if "num_contacts" in ref.dtype.names:
        assert np.array_equal(ref["num_contacts"], got["num_contacts"]), "%s: collide flags differ" % what


def ref_agrees(sc, fn, ro, args, what, fields=None):
    """where oracle/_ref exists: the reference build returns the same bits (it leaves `distance` of a collide()
    without a contact unset).  `fields`: compare only these (mesh queries: the BV / leaf test counters and the path
    byte of the record are the oracle's own, and the reference writes no normal on the mesh-mesh distance path)"""
    if "ref" not in sc.b:
        return
    rr = getattr(sc.b["ref"], fn)(*args)
    if fields is not None:
        for f in fields:
            x, y = rr[f], ro[f]
            ok = (x == y) | (np.isnan(x) & np.isnan(y)) if x.dtype.kind == "f" else x == y
            assert np.all(ok), "%s (reference build): field %s differs at rows %s" % (what, f, np.unique(np.nonzero(~ok)[0])[:8])
        return
    a, b = rr.copy(), ro.copy()
    if "num_contacts" in a.dtype.names:
        nc = a["num_contacts"] == 0
        a["distance"][nc] = 0
        b["distance"][nc] = 0
    compare_distance(a, b, what=what + " (reference build)")


def compare_hill_climb(ref, got):
    """Exhaustive-argmax device code vs the reference's hill-climbing support (hulls > 32
    vertices).  The chosen vertex can differ only on maxima tied to rounding, i.e. at GJK/EPA
    convergence; the solver may then stop one iteration earlier or later.  Bar: status words and
    collide flags bit-exact; distances within 1e-6 (north_star); witness points / normals equal
    to 1e-9 on all but a vanishing fraction of pairs (tolerance-limited early stops), and within
    the solver's own accuracy (1e-3) everywhere."""
    assert np.array_equal(ref["status"], got["status"])
    assert np.array_equal(ref["num_contacts"], got["num_contacts"])
    m = ~np.isnan(ref["p1"][:, 0])
    assert np.array_equal(m, ~np.isnan(got["p1"][:, 0]))
    assert np.all(np.abs(ref["distance"][m] - got["distance"][m]) <= 1e-6 * np.maximum(1, np.abs(ref["distance"][m])))
    for f in ("p1", "p2", "normal"):
        d = np.abs(ref[f][m] - got[f][m]).max(axis=1)
        assert (d > 1e-9).mean() < 1e-3, f
        assert d.max() < 1e-3, f
