"""Seeded synthetic workloads for the BASELINE.json configs (SURVEY.md section 8d).

Pure numpy/scipy generators; they produce POD arrays (see _pod.py) that are fed
identically to the CUDA engine, to the oracle and to the CPU emulation harness.
Generators mirror the reference's test helpers:
  generateRandomTransforms  test/utility.cpp:198-247
  constructPolytopeFromEllipsoid / random hulls  test/utility.cpp:501-557
"""
import numpy as np

from . import _pod as P


def random_rotations(rng, n):
    """Uniform unit quaternions -> rotation matrices (n,3,3) (math/transform.h:228-250)."""
    u1, u2, u3 = rng.random(n), rng.random(n), rng.random(n)
    m1, m2 = np.sqrt(1.0 - u1), np.sqrt(u1)
    w, x = m1 * np.sin(2 * np.pi * u2), m1 * np.cos(2 * np.pi * u2)
    y, z = m2 * np.sin(2 * np.pi * u3), m2 * np.cos(2 * np.pi * u3)
    return quat_to_rot(w, x, y, z)


def quat_to_rot(w, x, y, z):
    w, x, y, z = [np.asarray(a, dtype=np.float64) for a in (w, x, y, z)]
    R = np.empty(w.shape + (3, 3))
    R[..., 0, 0] = 1 - 2 * (y * y + z * z)
    R[..., 0, 1] = 2 * (x * y - z * w)
    R[..., 0, 2] = 2 * (x * z + y * w)
    R[..., 1, 0] = 2 * (x * y + z * w)
    R[..., 1, 1] = 1 - 2 * (x * x + z * z)
    R[..., 1, 2] = 2 * (y * z - x * w)
    R[..., 2, 0] = 2 * (x * z - y * w)
    R[..., 2, 1] = 2 * (y * z + x * w)
    R[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def random_transforms(rng, n, lo, hi):
    lo = np.asarray(lo, dtype=np.float64)
    hi = np.asarray(hi, dtype=np.float64)
    T = lo + (hi - lo) * rng.random((n, 3))
    return P.make_transforms(random_rotations(rng, n), T)


def identity_transforms(n, T=None):
    R = np.broadcast_to(np.eye(3), (n, 3, 3))
    return P.make_transforms(R, np.zeros((n, 3)) if T is None else T)


def random_primitive_shapes(rng, n, types):
    """n shape records with type drawn uniformly from `types`; sizes as in
    test/normal_and_nearest_points.cpp:283-… (U[0.05,1] radii / half sides)."""
    types = np.asarray(types, dtype=np.uint32)
    t = types[rng.integers(0, len(types), n)]
    p = 0.05 + 0.95 * rng.random((n, 3))
    out = P.make_shapes(t, p)
    # capsule/cylinder/cone: p[0] = radius, p[1] = halfLength in [0.075, 0.5]
    lz = 0.15 + 0.85 * rng.random(n)
    m = (t == P.GEOM_CAPSULE) | (t == P.GEOM_CYLINDER) | (t == P.GEOM_CONE)
    out["p"][m, 1] = lz[m] / 2
    out["p"][m, 2] = 0.0
    ms = t == P.GEOM_SPHERE
    out["p"][ms, 1:] = 0.0
    return out


def config2_mixed_primitives(n_pairs, seed=0xFC1 + 2, pool=65536,
                             types=(P.GEOM_SPHERE, P.GEOM_CAPSULE, P.GEOM_BOX, P.GEOM_CYLINDER)):
    """BASELINE config 2: mixed primitive pairs (sphere/capsule/box/cylinder), random poses;
    relative translation U[-3,3]^2 x U[0,3] as test/accelerated_gjk.cpp:122."""
    rng = np.random.default_rng(seed)
    shapes = random_primitive_shapes(rng, pool, types)
    h1 = rng.integers(0, pool, n_pairs).astype(np.uint32)
    h2 = rng.integers(0, pool, n_pairs).astype(np.uint32)
    tf1 = random_transforms(rng, n_pairs, (0, 0, 0), (0, 0, 0))
    tf2 = random_transforms(rng, n_pairs, (-3, -3, 0), (3, 3, 3))
    # move the whole scene so poses are not origin-centred
    off = -5 + 10 * rng.random((n_pairs, 3))
    tf1["T"] += off
    tf2["T"] += off
    return dict(shapes=shapes, h1=h1, tf1=tf1, h2=h2, tf2=tf2)


def config2_scene(n_objects=100_000, n_pairs=1_000_000, seed=0xFC1 + 2, pool=65536,
                  types=(P.GEOM_SPHERE, P.GEOM_CAPSULE, P.GEOM_BOX, P.GEOM_CYLINDER)):
    """BASELINE config 2 as a SCENE: n_objects mixed primitives (sphere/capsule/box/cylinder, sizes as in
    config2_mixed_primitives) with random poses in a cube, and the n_pairs object pairs a broadphase would hand to the
    narrow phase -- every ordered pair (i, j) whose relative translation lies in [-3,3]^2 x [0,3], the box
    test/accelerated_gjk.cpp:122 draws relative translations from, so the pairs have config 2's statistics (uniform
    relative translation in that box, independent uniform rotations) while 1 M pairs share 100 k objects, as pairs do
    in a real scene.  -> shapes (the pool), obj_h (pool index per object), obj_tf, first, second."""
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(seed)
    shapes = random_primitive_shapes(rng, pool, types)
    obj_h = rng.integers(0, pool, n_objects).astype(np.uint32)
    # expected pairs = N^2 / 2 * 6^3 / side^3; aim 8 % above n_pairs, then cut
    side = (0.5 * n_objects * n_objects * 216.0 / (1.08 * n_pairs)) ** (1.0 / 3.0)
    for _ in range(6):
        tf = random_transforms(rng, n_objects, (0, 0, 0), (side, side, side))
        pr = cKDTree(tf["T"]).query_pairs(3.0, p=np.inf, output_type="ndarray")
        if len(pr) >= n_pairs:
            break
        side *= 0.96
    assert len(pr) >= n_pairs, "scene too sparse"
    pr = pr[rng.permutation(len(pr))[:n_pairs]]
    dz = tf["T"][pr[:, 1], 2] - tf["T"][pr[:, 0], 2]
    first = np.where(dz >= 0, pr[:, 0], pr[:, 1]).astype(np.uint32)
    second = np.where(dz >= 0, pr[:, 1], pr[:, 0]).astype(np.uint32)
    return dict(shapes=shapes, obj_h=obj_h, obj_tf=tf, first=first, second=second)


def ellipsoid_hull(rng, nv=64, radii=None):
    """nv points on a random ellipsoid (all are hull vertices) + triangulated hull faces."""
    from scipy.spatial import ConvexHull
    if radii is None:
        radii = 0.05 + 0.95 * rng.random(3)
    while True:
        v = rng.normal(size=(nv, 3))
        v /= np.linalg.norm(v, axis=1, keepdims=True)
        pts = v * radii
        hull = ConvexHull(pts)
        if len(hull.vertices) == nv:
            break
    tris = hull.simplices.astype(np.uint32)
    # orient faces outward (fillNeighbors only needs adjacency, convex.hxx:231-280)
    c = pts.mean(axis=0)
    a, b, cc = pts[tris[:, 0]], pts[tris[:, 1]], pts[tris[:, 2]]
    flip = np.einsum("ij,ij->i", np.cross(b - a, cc - a), a - c) < 0
    tris[flip] = tris[flip][:, [0, 2, 1]]
    return pts, tris


def config3_convex_pairs(n_pairs, seed=0xFC1 + 3, pool=1024, nv=64):
    """BASELINE config 3: ConvexBase(nv) x ConvexBase(nv); ~half of the pairs overlap."""
    rng = np.random.default_rng(seed)
    hulls = [ellipsoid_hull(rng, nv) for _ in range(pool)]
    h1 = rng.integers(0, pool, n_pairs).astype(np.uint32)
    h2 = rng.integers(0, pool, n_pairs).astype(np.uint32)
    tf1 = random_transforms(rng, n_pairs, (0, 0, 0), (0, 0, 0))
    tf2 = random_transforms(rng, n_pairs, (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
    off = -5 + 10 * rng.random((n_pairs, 3))
    tf1["T"] += off
    tf2["T"] += off
    return dict(hulls=hulls, h1=h1, tf1=tf1, h2=h2, tf2=tf2)


def icosahedron_from_ellipsoid(radii):
    """constructPolytopeFromEllipsoid (test/utility.cpp:486-557): 12 vertices, 20 faces.
    toEllipsoid: point /= ||point||, then scaled per axis by the radii."""
    phi = (1 + np.sqrt(5)) / 2
    pts = np.array([
        [-1, phi, 0], [1, phi, 0], [-1, -phi, 0], [1, -phi, 0],
        [0, -1, phi], [0, 1, phi], [0, -1, -phi], [0, 1, -phi],
        [phi, 0, -1], [phi, 0, 1], [-phi, 0, -1], [-phi, 0, 1]], dtype=np.float64)
    pts /= np.linalg.norm(pts, axis=1, keepdims=True)
    pts *= np.asarray(radii, dtype=np.float64)
    tris = np.array([
        [0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4],
        [11, 10, 2], [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8],
        [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]], dtype=np.uint32)
    return pts, tris


def sphere_mesh(radius=1.0, seg=100, ring=50, noise=0.0, rng=None):
    """generateBVHModel(Sphere, seg, ring) (shape/geometric_shape_to_BVH_model.h:100-150):
    2*seg*ring triangles (seg=100, ring=50 -> 10 000); optional radial noise breaks symmetric ties."""
    pts, tris = [], []
    phid, thetad = 2 * np.pi / seg, np.pi / (ring + 1)
    for i in range(ring):
        theta = thetad * (i + 1)
        for j in range(seg):
            phi = phid * j
            pts.append([radius * np.sin(theta) * np.cos(phi), radius * np.sin(theta) * np.sin(phi),
                        radius * np.cos(theta)])
    pts.append([0, 0, radius])
    pts.append([0, 0, -radius])
    for i in range(ring - 1):
        for j in range(seg):
            a = i * seg + j
            b = i * seg if j == seg - 1 else i * seg + j + 1
            c = (i + 1) * seg + j
            d = (i + 1) * seg if j == seg - 1 else (i + 1) * seg + j + 1
            tris.append([a, c, b])
            tris.append([b, c, d])
    for j in range(seg):
        a, b, c = j, (0 if j == seg - 1 else j + 1), ring * seg
        tris.append([c, a, b])
        a = (ring - 1) * seg + j
        b = (ring - 1) * seg if j == seg - 1 else (ring - 1) * seg + j + 1
        c = ring * seg + 1
        tris.append([a, c, b])
    pts = np.array(pts, dtype=np.float64)
    if noise and rng is not None:
        pts *= 1 + noise * rng.standard_normal((len(pts), 1))
    return pts, np.array(tris, dtype=np.uint32)


def config4_mesh_vs_capsules(n_queries, seed=0xFC1 + 4, seg=100, ring=50, pool=4096):
    """BASELINE config 4: 10k-triangle OBBRSS mesh vs capsules, distance + nearest points."""
    rng = np.random.default_rng(seed)
    verts, tris = sphere_mesh(1.0, seg, ring, noise=0.01, rng=rng)
    caps = P.make_shapes([P.GEOM_CAPSULE] * pool,
                         np.stack([0.02 + 0.08 * rng.random(pool), (0.05 + 0.25 * rng.random(pool)) / 2,
                                   np.zeros(pool)], axis=1))
    hc = rng.integers(0, pool, n_queries).astype(np.uint32)
    tf_mesh = random_transforms(rng, n_queries, (-0.2, -0.2, -0.2), (0.2, 0.2, 0.2))
    tf_caps = random_transforms(rng, n_queries, (-2, -2, -2), (2, 2, 2))
    return dict(verts=verts, tris=tris, capsules=caps, hc=hc, tf_mesh=tf_mesh, tf_caps=tf_caps)


def config5_moving_boxes(n_objects=100_000, env_scale=None, seed=0xFC1 + 5, target_pairs=1_000_000):
    """BASELINE config 5: n Box(5, 10, 20) objects (generateEnvironments, test/utility.cpp:392-404) with random poses in
    [-env_scale, env_scale]^3; `step(k)` moves every object by a small random delta (generateRandomTransforms with
    delta_trans / delta_rot, utility.cpp:249-...).  env_scale defaults to the value that gives about `target_pairs`
    overlapping AABB pairs (the reference's 2000 for 1000 objects would give ~50 pairs for 100 k)."""
    rng = np.random.default_rng(seed)
    shapes = P.make_shapes([P.GEOM_BOX], [[2.5, 5.0, 10.0]])  # half sides of Box(5, 10, 20)
    if env_scale is None:
        # a rotated box's AABB has a mean side of about 16.5; two cubes of side s overlap with probability (2 s / L)^3
        s = 16.5
        env_scale = 0.5 * 2 * s / (2.0 * target_pairs / (float(n_objects) ** 2)) ** (1.0 / 3.0)
    tf = random_transforms(rng, n_objects, (-env_scale,) * 3, (env_scale,) * 3)
    obj_h = np.zeros(n_objects, dtype=np.uint32)

    def step(k, delta_trans=1.0, delta_rot=0.05):
        """poses of step k: the base poses moved by a seeded random delta"""
        r = np.random.default_rng(seed + 7919 * (k + 1))
        out = tf.copy()
        out["T"] += delta_trans * (2 * r.random((n_objects, 3)) - 1)
        # small rotation about a random axis, applied on the left: R' = dR * R
        ax = r.standard_normal((n_objects, 3))
        ax /= np.linalg.norm(ax, axis=1, keepdims=True)
        ang = delta_rot * (2 * r.random(n_objects) - 1)
        K = np.zeros((n_objects, 3, 3))
        K[:, 0, 1], K[:, 0, 2], K[:, 1, 0] = -ax[:, 2], ax[:, 1], ax[:, 2]
        K[:, 1, 2], K[:, 2, 0], K[:, 2, 1] = -ax[:, 0], -ax[:, 1], ax[:, 0]
        dR = np.eye(3)[None] + np.sin(ang)[:, None, None] * K + (1 - np.cos(ang))[:, None, None] * (K @ K)
        R = out["R"].reshape(n_objects, 3, 3).transpose(0, 2, 1)  # stored column-major
        Rn = dR @ R
        out["R"] = Rn.transpose(0, 2, 1).reshape(out["R"].shape)
        return out

    return dict(shapes=shapes, obj_h=obj_h, obj_tf=tf, env_scale=env_scale, step=step)


def _axis_rotations(axis, ang):
    """rotations by `ang` (n,) about the unit axis x (0), y (1) or z (2) -> (n, 3, 3)"""
    c, s = np.cos(ang), np.sin(ang)
    R = np.zeros(ang.shape + (3, 3))
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    R[..., axis, axis] = 1
    R[..., i, i] = c
    R[..., j, j] = c
    R[..., i, j] = -s
    R[..., j, i] = s
    return R


def robot_vs_environment(n_configs=1024, n_links=16, n_env=100_000, room=None, seed=0xFC1 + 6, target_pairs=1_000_000,
                         joint_range=1.2):
    """A planner's collision query: a seeded chain robot of n_links links (capsules, boxes and two small hulls, joint
    axes alternating z / y) at n_configs configurations (random base in the room, random joint angles, the bending
    joints within +-joint_range rad: at 2.8 the chain folds back onto itself in some configurations) -- set A,
    n_configs * n_links objects, configuration-major -- against a static environment -- set B: small primitives
    (spheres, boxes, capsules, cylinders of 2-8 cm), about 1 % large boxes (tables, shelves: 0.4-1.2 m), a few OBBRSS
    meshes and a Halfspace floor z <= 0.  `room` (side of the square room, 1.7 m high) defaults to the value that gives
    about `target_pairs` candidate pairs.
    -> dict: link_len; geometry to register (`register(scene, oracle=False)` -> one handle per geometry slot);
    geom_a / geom_b (geometry slot of every object) and tf_a / tf_b (poses)."""
    rng = np.random.default_rng(seed)
    link_len = 0.22
    # robot geometry: slot k = link k; links 5 and 11 are hulls, every third of the others a box, the rest capsules
    hull_links = (5, 11)
    link_rec = []
    for k in range(n_links):
        if k % 3 == 2 and k not in hull_links:
            link_rec.append((P.GEOM_BOX, [0.04, 0.04, 0.5 * link_len]))
        else:
            link_rec.append((P.GEOM_CAPSULE, [0.035, 0.5 * link_len - 0.035, 0.0]))
    hulls = [ellipsoid_hull(rng, 24, radii=(0.05, 0.05, 0.5 * link_len)) for _ in hull_links]
    # environment pools: 64 small primitives, 16 large boxes, one mesh
    small = random_primitive_shapes(rng, 64, (P.GEOM_SPHERE, P.GEOM_BOX, P.GEOM_CAPSULE, P.GEOM_CYLINDER))
    small["p"] *= 0.04  # radii / half sides 2 mm - 4 cm, so boxes of 2-8 cm
    big = P.make_shapes([P.GEOM_BOX] * 16, 0.2 + 0.4 * rng.random((16, 3)))
    mesh = sphere_mesh(0.15, 16, 8, noise=0.02, rng=rng)
    n_prims = n_links + len(small) + len(big)
    prim_types = np.array([t for t, _ in link_rec], dtype=np.uint32)
    prim_p = np.array([p for _, p in link_rec], dtype=np.float64)
    shapes = np.concatenate([P.make_shapes(prim_types, prim_p), small, big])
    slot_hull = [n_prims, n_prims + 1]
    slot_mesh = n_prims + 2
    slot_floor = n_prims + 3

    def register(sc, oracle=False):
        h = [np.asarray(sc.register_shapes(shapes), dtype=np.uint32)]
        for pts, tris in hulls:
            cid = sc.register_convex(pts, tris) if oracle else sc.register_convex(pts)
            h.append(np.asarray(sc.register_shapes(P.make_shapes([P.GEOM_CONVEX], [[0, 0, 0]], data=[cid])), dtype=np.uint32))
        if oracle:
            bid = sc.register_bvh(*mesh)[0]
        else:
            from .engine import build_bvh_obbrss
            bid = sc.register_bvh_obbrss(build_bvh_obbrss(*mesh), *mesh)
        h.append(np.asarray(sc.register_shapes(P.make_shapes([P.BV_OBBRSS], [[0, 0, 0]], data=[bid])), dtype=np.uint32))
        h.append(np.asarray(sc.register_halfspaces(P.GEOM_HALFSPACE, [[0, 0, 1, 0.0]]), dtype=np.uint32))
        return np.concatenate(h)

    if room is None:
        # candidates per link ~ density * (link box + object box)^3, about 0.25^3 for this robot and the small objects
        room = float(np.sqrt(n_env * n_configs * n_links * 0.0136 / (1.7 * target_pairs)))
    # ---- set B: the environment
    geom_b = np.empty(n_env, dtype=np.int64)
    kind = rng.random(n_env)
    n_mesh = 8
    geom_b[:] = n_links + rng.integers(0, len(small), n_env)
    nbig = kind < 0.01
    geom_b[nbig] = n_links + len(small) + rng.integers(0, len(big), int(nbig.sum()))
    geom_b[1:1 + n_mesh] = slot_mesh
    geom_b[0] = slot_floor
    tf_b = random_transforms(rng, n_env, (0, 0, 0), (room, room, 1.7))
    tf_b[nbig] = identity_transforms(int(nbig.sum()), T=tf_b["T"][nbig])  # axis-aligned furniture
    tf_b[0] = identity_transforms(1)[0]
    # ---- set A: the robot at n_configs configurations
    K, L = n_configs, n_links
    base = rng.random((K, 3)) * np.array([room, room, 0.0])
    R = _axis_rotations(2, 2 * np.pi * rng.random(K))
    p = base.copy()
    Rs, Ts = np.empty((K, L, 3, 3)), np.empty((K, L, 3))
    for k in range(L):
        R = R @ _axis_rotations(2 if k % 2 == 0 else 1, rng.uniform(-joint_range, joint_range, K) if k else rng.uniform(0, 2 * np.pi, K))
        axis = R[:, :, 2]
        Rs[:, k] = R
        Ts[:, k] = p + 0.5 * link_len * axis
        p = p + link_len * axis
    tf_a = P.make_transforms(Rs.reshape(-1, 3, 3), Ts.reshape(-1, 3))
    geom_a = np.tile(np.where(np.isin(np.arange(L), hull_links), 0, np.arange(L)), K)
    for s, k in zip(slot_hull, hull_links):
        geom_a[np.arange(K) * L + k] = s
    return dict(register=register, geom_a=geom_a, tf_a=tf_a, geom_b=geom_b, tf_b=tf_b, room=room, link_len=link_len,
                n_configs=K, n_links=L)


def robot_motions(n_motions, n_links=16, n_env=100_000, room=None, seed=0xFC1 + 7, target_pairs=1_000_000,
                  joint_range=1.2, max_step=1.0, resolution=0.025):
    """A planner's motion validation: n_motions straight-line joint-space motions of robot_vs_environment's chain robot,
    in its room and against its environment.  A motion's joints are the base yaw and the n_links - 1 bending joints
    (within +-joint_range rad), its base position fixed in the room.  Each motion goes from a random start towards a
    goal up to 1.25 steps away for at most `max_step` (Euclidean, joint space), as an RRT extension does, and is sampled every
    `resolution` rad along it, end points included, so sample counts vary.  The samples' poses come from forward
    kinematics, one configuration per sample, motion after motion.  `room` defaults to robot_vs_environment's for the
    total sample count.
    -> robot_vs_environment's dict with tf_a / geom_a holding the samples (n_configs of them), plus `offsets`
    (n_motions + 1: motion m is configurations [offsets[m], offsets[m+1])), `n_motions` and `q` (the joint values,
    n_configs x n_links)."""
    rng = np.random.default_rng(seed)
    K, L = n_motions, n_links
    lo = np.concatenate([[-np.pi], np.full(L - 1, -joint_range)])
    hi = np.concatenate([[np.pi], np.full(L - 1, joint_range)])
    q0 = lo + (hi - lo) * rng.random((K, L))
    d = rng.standard_normal((K, L))  # towards a goal up to 1.25 steps away, in a random direction
    d *= (1.25 * max_step * rng.random(K) / np.maximum(np.linalg.norm(d, axis=1), 1e-300))[:, None]
    d *= (max_step / np.maximum(np.linalg.norm(d, axis=1), max_step))[:, None]
    d[:, 1:] = np.clip(q0[:, 1:] + d[:, 1:], lo[1:], hi[1:]) - q0[:, 1:]  # (the bending joints stay in range)
    n_samples = 1 + np.ceil(np.linalg.norm(d, axis=1) / resolution).astype(np.int64)
    offsets = np.concatenate([[0], np.cumsum(n_samples)]).astype(np.uint32)
    total = int(offsets[-1])
    w = robot_vs_environment(total, n_links, n_env, room, seed=seed, target_pairs=target_pairs, joint_range=joint_range)
    base = np.repeat(rng.random((K, 3)) * np.array([w["room"], w["room"], 0.0]), n_samples, axis=0)
    motion = np.repeat(np.arange(K), n_samples)
    step = np.arange(total) - offsets[motion]
    frac = step / np.maximum(n_samples[motion] - 1, 1)
    q = q0[motion] + frac[:, None] * d[motion]

    def fk(base, q):  # the chain of robot_vs_environment: joint k turns about z (k even) or y (k odd)
        R = np.broadcast_to(np.eye(3), (len(q), 3, 3))
        p = base.copy()
        Rs, Ts = np.empty((len(q), L, 3, 3)), np.empty((len(q), L, 3))
        for k in range(L):
            R = R @ _axis_rotations(2 if k % 2 == 0 else 1, q[:, k])
            axis = R[:, :, 2]
            Rs[:, k] = R
            Ts[:, k] = p + 0.5 * w["link_len"] * axis
            p = p + w["link_len"] * axis
        return P.make_transforms(Rs.reshape(-1, 3, 3), Ts.reshape(-1, 3))

    w["tf_a"] = fk(base, q)
    w["geom_a"] = np.tile(w["geom_a"][:L], total)
    w.update(offsets=offsets, n_motions=K, q=q)
    return w


def chain_sweep_bounds(w):
    """Sweep bounds for robot_motions' chain, as hfb_env_certify_motions takes them: (n_configs * n_links,) float64,
    entry g * L + l bounding the path length of every point of link l from sample g to sample g + 1 of its motion, 0 at
    a motion's last sample (never read there).

    Joint k turns about an axis through p_k, the start of link k (joint 0, the base yaw, through the base).  Every point
    of link l >= k lies within rho_{k,l} = (l - k + 1) * link_len + 0.06 of p_k: l - k links of length link_len up to
    p_l, then link l itself, whose points lie within link_len along its axis and, across it, within the box corner
    0.04 * sqrt(2) < 0.06 (capsules 0.035, hulls 0.05).  A point's speed is at most the sum over the joints below it
    of |dq_k/dt| times its distance to joint k's axis, which is at most its distance to p_k.  The samples are linear
    in q, so over a segment the path length of link l's points is at most
    s_{g,l} = sum_{k <= l} |q_{g+1,k} - q_{g,k}| * rho_{k,l}; it is computed in float64 and rounded up by a relative
    margin far above the sum's rounding error."""
    q, off, L, ll = np.asarray(w["q"], dtype=np.float64), np.asarray(w["offsets"], dtype=np.int64), w["n_links"], w["link_len"]
    n = q.shape[0]
    dq = np.zeros_like(q)
    dq[:-1] = np.abs(q[1:] - q[:-1])
    dq[off[1:][off[1:] > 0] - 1] = 0.0  # a motion's last sample (the next row is another motion's)
    k, l = np.meshgrid(np.arange(L), np.arange(L), indexing="ij")
    rho = np.where(k <= l, (l - k + 1) * ll + 0.06, 0.0)
    s = dq @ rho
    s = np.nextafter(s * (1.0 + 64 * L * np.finfo(np.float64).eps), np.inf)
    s[dq.sum(axis=1) == 0] = 0.0
    return np.ascontiguousarray(s.reshape(n * L))


def resample_motions(w, configs, n_interior):
    """the poses of robot_motions' chain at n_interior evenly spaced interior points of each segment from configuration
    g to g + 1, g in `configs` (each with a successor in its motion): linear in q, through the same forward kinematics
    -> transforms, n_interior * n_links per segment, segment after segment"""
    L, ll = w["n_links"], w["link_len"]
    g = np.asarray(configs, dtype=np.int64)
    tf0 = w["tf_a"][g * L]  # link 0 of each start sample: its start is the base
    base = tf0["T"] - 0.5 * ll * tf0["R"].reshape(-1, 3, 3)[:, 2, :]
    t = np.arange(1, n_interior + 1) / (n_interior + 1.0)
    q = w["q"][g][:, None, :] + t[None, :, None] * (w["q"][g + 1] - w["q"][g])[:, None, :]
    base = np.repeat(base, n_interior, axis=0)
    q = q.reshape(-1, L)
    R = np.broadcast_to(np.eye(3), (len(q), 3, 3))
    p = base.copy()
    Rs, Ts = np.empty((len(q), L, 3, 3)), np.empty((len(q), L, 3))
    for k in range(L):
        R = R @ _axis_rotations(2 if k % 2 == 0 else 1, q[:, k])
        axis = R[:, :, 2]
        Rs[:, k] = R
        Ts[:, k] = p + 0.5 * ll * axis
        p = p + ll * axis
    return P.make_transforms(Rs.reshape(-1, 3, 3), Ts.reshape(-1, 3))


def chain_self_pairs(n_links, skip=2):
    """the self-pair template of a chain: every link pair (i, j) with j >= i + skip (neighbours touch at their joint
    and are not checked, as an SRDF disables adjacent links) -> (P, 2) uint32; 105 pairs for 16 links"""
    i, j = np.triu_indices(n_links, k=skip)
    return np.stack([i, j], axis=1).astype(np.uint32)


def chain_robot_model(w):
    """robot_motions' (or robot_vs_environment's) chain as a robot model, in the arrays hfb_robot_desc takes: prismatic
    joints x and y carry the base (joints 0 and 1, on the world), then the yaw joint (about z, at the base) and the
    bending joints, about z (link k even) or y (k odd), each placed link_len along its parent's z axis; link k hangs on
    joint k + 2 at link_len / 2 along its z axis.  The q layout is [x, y, q_0 .. q_{L-1}].
    -> dict: parent, types, axis, placement (J = L + 2 joints), link_joint, link_placement, geom (the geometry slot of
    each link, as w["geom_a"] and w["register"] number them); with w from robot_motions also q (the samples' joint
    values, n_configs x J, the base read back from link 0's pose) and q_from / q_to (each motion's first and last
    sample, n_motions x J)."""
    L, ll = w["n_links"], w["link_len"]
    J = L + 2
    parent = np.arange(-1, J - 1, dtype=np.int32)
    types = np.array([P.JOINT_PRISMATIC] * 2 + [P.JOINT_REVOLUTE] * L, dtype=np.uint32)
    axis = np.zeros((J, 3))
    axis[0, 0] = axis[1, 1] = 1.0
    axis[2 + np.arange(L), np.where(np.arange(L) % 2 == 0, 2, 1)] = 1.0
    placement = identity_transforms(J)
    placement["T"][3:, 2] = ll
    link_placement = identity_transforms(L)
    link_placement["T"][:, 2] = 0.5 * ll
    out = dict(parent=parent, types=types, axis=axis, placement=placement, link_joint=np.arange(2, J, dtype=np.int32),
               link_placement=link_placement, geom=np.asarray(w["geom_a"][:L]))
    if "q" in w:
        tf0 = w["tf_a"][::L]  # link 0 of every sample: its start is the base
        base = tf0["T"] - 0.5 * ll * tf0["R"].reshape(-1, 3, 3)[:, 2, :]  # (R is column-major: row 2 is the z axis)
        q = np.concatenate([base[:, :2], w["q"]], axis=1)
        off = np.asarray(w["offsets"], dtype=np.int64)
        first = off[:-1]
        q_from = q[np.minimum(first, len(q) - 1)]
        q_to = q[np.maximum(off[1:] - 1, 0)]
        q_to[:, :2] = q_from[:, :2]  # (the base stays put along a motion)
        out.update(q=q, q_from=np.ascontiguousarray(q_from), q_to=np.ascontiguousarray(q_to))
    return out
