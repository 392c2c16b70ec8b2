"""The contract of hfb_env_validate_motions (include/hppfcl_b200.h) in Python: validate_reference() runs the rounds --
runs, admission under the cap, one certification of the runs, the segment rules and the frontier -- over a narrow
phase passed in, so that the same bookkeeping can be driven by the host builds and the oracle (cpu_narrow) or by the
library's existing public calls.  Also a hand-made scene of spheres on a two-joint robot where each rule decides
something."""
import numpy as np

from tests.common import P
from tests.robot_common import emu_poses, emu_sample, local_boxes
from hppfcl_b200 import workloads as W


def q_at(q_from, q_to, k, D):
    """the joint values at position k of [0, 2^D]: kin_sample's formula (t = k * 2^-D is exact)"""
    if k == 0:
        return np.array(q_from, dtype=np.float64)
    if k == 1 << D:
        return np.array(q_to, dtype=np.float64)
    t = k / float(1 << D)
    return q_from + t * (q_to - q_from)


def effective_cap(max_samples, n_b, links):
    return min(int(max_samples), 1 << 29, (0xFFFFFFFF - n_b) // links)


def validate_reference(narrow, n_motions, d0, D, cap, first_motion=0, num_motions=None):
    """the rounds of hfb_env_validate_motions.  narrow(depth, runs) certifies runs = [(motion, [positions])] as
    hfb_env_certify_motions would and returns (first colliding sample per run or -1, certified flags per run (one per
    segment), finite-sweep flags per run (one per segment), counts = (env candidates, self candidates, unsupported)).
    -> dict: status, t_valid, t_collide (n_motions each), c (the colliding position per motion or None), n_rounds,
    n_samples, n_env_candidates, n_self_candidates, n_unsupported"""
    nm = n_motions - first_motion if num_motions is None else num_motions
    rng = range(first_motion, first_motion + nm)
    c = {m: None for m in rng}
    f = {m: None for m in rng}
    u = {m: None for m in rng}
    lo = lambda x, y: y if x is None or (y is not None and y < x) else x
    per, len0 = 1 << d0, 1 << (D - d0)
    seg = [(m, j * len0) for m in rng for j in range(per)]
    rounds = samples = n_env = n_self = n_unsup = 0
    depth = d0
    while seg:
        ln = 1 << (D - depth)
        # runs and admission
        total, adm, runs = 0, [], []
        for i, (m, a) in enumerate(seg):
            new = i == 0 or seg[i - 1][0] != m or seg[i - 1][1] + ln != a
            total += 2 if new else 1
            if total > cap:
                break
            adm.append(new)
            if new:
                runs.append((m, [a, a + ln], [i]))
            else:
                runs[-1][1].append(a + ln)
                runs[-1][2].append(i)
        n_adm = len(adm)
        rounds += 1
        samples += sum(len(r[1]) for r in runs)
        fi, cert, fin, cnt = narrow(depth, [(r[0], r[1]) for r in runs])
        n_env, n_self, n_unsup = n_env + cnt[0], n_self + cnt[1], n_unsup + cnt[2]
        certified, finite = {}, {}
        for r, (m, pos, idx) in enumerate(runs):
            if fi[r] >= 0:
                c[m] = lo(c[m], pos[fi[r]])
            for s, i in enumerate(idx):
                certified[i], finite[i] = bool(cert[r][s]), bool(fin[r][s])
        split = []
        for i, (m, a) in enumerate(seg):
            admitted = i < n_adm
            if admitted and certified[i]:
                continue
            if c[m] is not None and a >= c[m]:
                u[m] = lo(u[m], a)
                continue
            if not admitted or depth == D or not finite[i]:
                u[m], f[m] = lo(u[m], a), lo(f[m], a)
                continue
            split.append((m, a))
        half = ln // 2
        seg = [(m, b) for m, a in split for b in (a, a + half) if f[m] is None or b < f[m]]
        depth += 1
    status = np.full(n_motions, -1, np.int8)
    t_valid = np.zeros(n_motions)
    t_collide = np.full(n_motions, -1.0)
    for m in rng:
        status[m] = 1 if c[m] is not None else 0 if u[m] is None else 2
        t_valid[m] = 1.0 if u[m] is None else u[m] / float(1 << D)
        t_collide[m] = -1.0 if c[m] is None else c[m] / float(1 << D)
    return dict(status=status, t_valid=t_valid, t_collide=t_collide, c=c, n_rounds=rounds, n_samples=samples,
                n_env_candidates=n_env, n_self_candidates=n_self, n_unsupported=n_unsup)


def run_layout(runs, q_from, q_to, D):
    """the runs' samples as motions: joint values (n_samples, J), offsets, and the segments' end points"""
    qs, off, qa, qb = [], [0], [], []
    for m, pos in runs:
        qs += [q_at(q_from[m], q_to[m], k, D) for k in pos]
        off.append(off[-1] + len(pos))
        qa += [q_at(q_from[m], q_to[m], k, D) for k in pos[:-1]]
        qb += [q_at(q_from[m], q_to[m], k, D) for k in pos[1:]]
    return np.array(qs), np.array(off, dtype=np.uint32), np.array(qa), np.array(qb)


def sweeps_of(sample, runs, qa, qb, L):
    """the sweep bounds per run sample (0 at a run's last sample) from sample(qa, qb, off2), the robot's sweeps of the
    segments as 2-sample motions, and each segment's finite flag"""
    ns = len(qa)
    sw2 = sample(qa, qb, np.arange(0, 2 * ns + 1, 2, dtype=np.uint32)).reshape(-1, L)[::2] if ns else np.zeros((0, L))
    sweep, fin, k = [], [], 0
    for m, pos in runs:
        s = len(pos) - 1
        sweep += [sw2[k:k + s], np.zeros((1, L))]
        fin.append([bool((sw2[j] <= np.finfo(np.float64).max).all()) for j in range(k, k + s)])
        k += s
    return np.concatenate(sweep).reshape(-1), fin


def cpu_narrow(orc, emu, model, boxes, hb, tfb, tpl, q_from, q_to, D, req):
    """the narrow phase on the CPU: poses and sweeps from the host build of the kinematics, the certification by the
    brute-force contract of tests/test_env_certify_reference.py (the oracle's collide())"""
    from tests.test_env_certify_reference import contract
    L = len(model["link_joint"])

    def narrow(depth, runs):
        qs, off, qa, qb = run_layout(runs, q_from, q_to, D)
        tfa = emu_poses(model, boxes, qs)
        ha = np.tile(np.asarray(model["handles"], dtype=np.uint32), len(qs))
        sweep, fin = sweeps_of(lambda a, b, o: emu_sample(model, boxes, a, b, o)[3], runs, qa, qb, L)
        fi, _, cert, cnt, _, _ = contract(orc, emu, ha, tfa, hb, tfb, L, tpl, off, sweep, req=req)
        return fi, [cert[off[r]:off[r + 1] - 1] for r in range(len(runs))], fin, cnt[:3]
    return narrow


def hand_scene(sc):
    """a robot of two prismatic joints (x on the world, y on x) carrying a sphere link (radius 0.25), a second sphere
    link fixed to the world far away (self pair (0, 1)), and environment spheres (radius 0.25) placed so that each rule
    of the rounds decides something -> (model, hb, tfb, q_from, q_to, names)"""
    sph = int(sc.register_shapes(P.make_shapes([P.GEOM_SPHERE], [[0.25, 0, 0]]))[0])
    B, Q0, Q1, names = [], [], [], []

    def motion(name, y, x0, x1, env=()):
        names.append(name)
        Q0.append((x0, y))
        Q1.append((x1, y))
        B.extend((x, y + dy, 0.0) for x, dy in env)

    motion("free", 0.0, 0.0, 4.0)                           # certified in round 0
    motion("near", 10.0, 0.0, 4.0, [(2.0, 0.7)])            # 0.2 from the obstacle at x = 2: certified after splits
    motion("hit", 20.0, 0.0, 4.0, [(1.0, 0.0)])             # touches at x = 0.5, a sample of depth 3
    motion("graze", 30.0, 0.0, 4.0, [(4.0 / 3.0, 0.5)])     # touches at x = 4/3, never at a sample: stuck at D
    motion("nan", 40.0, np.nan, 4.0)                        # a NaN joint value: stuck at once
    motion("still", 50.0, 1.0, 1.0)                         # q_from == q_to
    motion("late", 60.0, 0.0, 4.0, [(3.6, 0.0)])            # collides near the end
    motion("free2", 70.0, 0.0, -4.0)
    model = dict(parent=np.array([-1, 0], np.int32), types=np.array([P.JOINT_PRISMATIC] * 2, np.uint32),
                 axis=np.array([[1.0, 0, 0], [0, 1.0, 0]]), placement=W.identity_transforms(2),
                 link_joint=np.array([1, -1], np.int32), link_placement=W.identity_transforms(2, T=[(0, 0, 0), (0, -100, 0)]),
                 handles=np.array([sph, sph], np.uint32))
    hb = np.full(len(B), sph, np.uint32)
    tfb = W.identity_transforms(len(B), T=B)
    return model, hb, tfb, np.array(Q0), np.array(Q1), names
