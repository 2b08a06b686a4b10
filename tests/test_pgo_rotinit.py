"""Chordal rotation initialisation (include/d2pgo.h d2pgo_rot_init; d2pgo's rotInitial, RotationInitialization<double>):
the numpy oracle (oracle/pgo_rotinit_oracle.py) against the reference's own rotation_initialization_base.hpp (live through
oracle/_ref/libd2ref_rotinit.so, and through the frozen tests/golden/ref_rotinit.npz), and on the GPU the device against both."""
import ctypes as C
import os

import numpy as np
import pytest

from d2slam_b200 import pgo, synth
from oracle import pgo_oracle as po
from oracle import pgo_rotinit_oracle as ro

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_rotinit.npz")
FIELDS = ("ids", "poses", "fixed", "id_a", "id_b", "rel", "sqrt_info", "ego_ids", "ego", "gravity")


def _qexp(th):
    return pgo._qexp(np.asarray(th, np.float64))


def graph_case(seed, n_agents=3, n=12, loops=30, tilt=0.5, gravity=False, quirk=False, self_loop=False, untouched=False, fixed_heads=1):
    """A make_pose_graph graph with tens of degrees of attitude error on the free frames (random rotations of `tilt` rad per
    axis on the drifting odometry guess), square-root informations with random upper-triangular rotation blocks (so that the
    edges' weights s = |S_rot|_F differ), the head frames of the first `fixed_heads` agents fixed, and optionally: a loop from a
    fixed frame and one into it (the b-fixed quirk), a self loop, a pose no edge names, gravity rows with make_gravity_case's
    ego poses."""
    g = pgo.make_pose_graph(seed=seed, n_agents=n_agents, poses_per_agent=n, loops=loops)
    rng = np.random.default_rng(seed + 1000)
    ids = np.array(g["ids"]); poses = np.array(g["init"]); fixed = np.zeros(len(ids), np.uint8)
    for a in range(fixed_heads):
        fixed[a * n] = 1; poses[a * n] = g["gt"][a * n]
    free = fixed == 0
    q = pgo._qmul(poses[free, 3:7], _qexp(rng.normal(0, tilt, (int(free.sum()), 3))))
    poses[free, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    id_a, id_b, rel, S = list(g["id_a"]), list(g["id_b"]), list(g["rel"]), list(g["sqrt_info"].reshape(-1, 6, 6))
    gt = g["gt"]

    def add(i, j):
        r = pgo.relative_pose(gt[i], gt[j]).copy()
        qq = pgo._qmul(r[3:7], _qexp(rng.normal(0, 0.02, 3))); r[3:7] = qq / np.linalg.norm(qq)
        id_a.append(ids[i]); id_b.append(ids[j]); rel.append(r); S.append(np.diag([20.0, 20.0, 20.0, 57.0, 57.0, 57.0]))

    for a in range(1, n_agents):             # every agent tied to agent 0 between free frames (a loop into a fixed frame gives no rows)
        add(a * n + 2, 1)
    if quirk:
        add(0, n // 2); add(n - 2, 0)        # a fixed (a prior on b) and b fixed (dropped)
    if self_loop:
        add(3, 3)
    S = np.array(S)
    for e in range(len(S)):
        U = np.triu(rng.normal(0, 1.0, (3, 3)), 1) * 5.0 + np.diag(rng.uniform(20.0, 80.0, 3))
        S[e, 3:6, 3:6] = U
    ego = pgo.make_gravity_case(g, seed=seed)["ego"]
    ego_ids = ids.copy()
    if untouched:
        ids = np.concatenate([ids, [99_000_000]]); poses = np.concatenate([poses, [[1.0, 2.0, 3.0, 0.1, 0.2, 0.3, 0.9]]])
        poses[-1, 3:7] /= np.linalg.norm(poses[-1, 3:7]); fixed = np.concatenate([fixed, [0]]).astype(np.uint8)
    return dict(ids=ids, poses=poses, fixed=fixed, id_a=np.array(id_a, np.int64), id_b=np.array(id_b, np.int64), rel=np.array(rel),
                sqrt_info=S.reshape(-1, 36), ego_ids=ego_ids, ego=ego, gravity=np.int64(1 if gravity else 0), gt=np.concatenate([gt, poses[len(gt):]]))


def reference_cases():
    return {
        "multi": graph_case(11, untouched=True),
        "quirk_self": graph_case(12, quirk=True, self_loop=True),
        "gravity": graph_case(13, quirk=True, self_loop=True, gravity=True, untouched=True),
        "gravity_two_fixed": graph_case(14, n_agents=4, n=10, loops=40, gravity=True, fixed_heads=2, tilt=0.7),
    }


def oracle_of(c):
    return ro.rot_init(c["ids"], c["poses"], c["fixed"], c["id_a"], c["id_b"], c["rel"], c["sqrt_info"], gravity=bool(c["gravity"]),
                       ego_ids=c["ego_ids"], ego_poses=c["ego"])


def reference_outputs(cases):
    """The reference's own RotationInitialization<double>::solve on each case (oracle/_ref/libd2ref_rotinit.so)."""
    from oracle import ref_rotinit
    out = {}
    for name, c in cases.items():
        r = ref_rotinit.rot_init(c["ids"], c["poses"], c["fixed"], c["id_a"], c["id_b"], c["rel"], c["sqrt_info"], bool(c["gravity"]),
                                 10.0, c["ego_ids"], c["ego"])
        for k, v in r.items():
            out[f"ref_{name}_{k}"] = v
    return out


def golden():
    z = np.load(GOLD)
    cases = {}
    for k in z.files:
        if k.startswith("case_"):
            name, field = k[5:].rsplit("__", 1)
            cases.setdefault(name, {})[field] = z[k]
    refs = {k[4:]: z[k] for k in z.files if k.startswith("ref_")}
    return cases, refs


def _ref(refs, name):
    return {k[len(name) + 1:]: v for k, v in refs.items() if k.startswith(name + "_")}


def _compare_oracle_to_reference(c, r):
    o = oracle_of(c)
    assert [int(f) for f in o["frames"]] == [int(f) for f in r["frames"]]
    assert np.abs(o["M"] - r["M"]).max() <= 1e-10, np.abs(o["M"] - r["M"]).max()
    assert np.abs(o["R"] - r["R"]).max() <= 1e-10, np.abs(o["R"] - r["R"]).max()
    assert abs(o["state_changes"] - float(r["state_changes"])) <= 1e-12
    assert o["dropped"] == int(r["dropped"])


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_matches_the_frozen_reference_outputs():
    cases, refs = golden()
    assert set(cases) == set(reference_cases())
    for name, c in cases.items():
        _compare_oracle_to_reference(c, _ref(refs, name))


def test_oracle_matches_the_reference_live():
    from oracle import ref_rotinit
    if not ref_rotinit.available():
        pytest.skip("reference tree and prebuilt oracle/_ref/libd2ref_rotinit.so both absent")
    cases = reference_cases()
    refs = reference_outputs(cases)
    for name, c in cases.items():
        _compare_oracle_to_reference(c, _ref({k[4:]: v for k, v in refs.items()}, name))


def test_golden_inputs_are_the_seeded_cases():
    cases, _ = golden()
    for name, c in reference_cases().items():
        for f in FIELDS:
            assert np.array_equal(np.asarray(cases[name][f]), np.asarray(c[f])), (name, f)


def test_dropped_edges_follow_the_reference_rules():
    c = reference_cases()["quirk_self"]
    o = oracle_of(c)
    fixed = set(int(i) for i, f in zip(c["ids"], c["fixed"]) if f)
    want = sum(1 for a, b in zip(c["id_a"], c["id_b"]) if a == b or int(b) in fixed)
    assert o["dropped"] == want and want >= 2


def test_oracle_solution_is_a_stationary_point():
    for c in reference_cases().values():
        o = oracle_of(c)
        A, b, x = o["A"], o["b"], o["x"]
        g = A.T @ (A @ x - b)
        assert np.abs(g).max() <= 1e-9 * max(1.0, np.abs(A.T @ b).max())


def test_projection_is_the_nearest_rotation():
    rng = np.random.default_rng(5)
    M = rng.normal(size=(200, 3, 3))
    R = ro.project_so3(M)
    assert np.abs(R @ np.swapaxes(R, 1, 2) - np.eye(3)).max() <= 1e-12 and np.abs(np.linalg.det(R) - 1).max() <= 1e-12
    # polar check: where det M > 0, R^T M is symmetric positive semi-definite (R is the polar factor)
    pos = np.linalg.det(M) > 0
    P = np.swapaxes(R[pos], 1, 2) @ M[pos]
    assert np.abs(P - np.swapaxes(P, 1, 2)).max() <= 1e-12 and np.linalg.eigvalsh((P + np.swapaxes(P, 1, 2)) / 2).min() >= -1e-12
    # and no sampled rotation is closer
    for k in range(20):
        d0 = np.linalg.norm(R[k] - M[k])
        for _ in range(50):
            Q = R[k] @ ro.quat_R(_qexp(rng.normal(0, 0.2, 3)))
            assert np.linalg.norm(Q - M[k]) >= d0 - 1e-12


def test_unanchored_component_is_refused_by_the_oracle():
    c = reference_cases()["multi"]
    with pytest.raises(ValueError):
        ro.rot_init(c["ids"], c["poses"], np.zeros_like(c["fixed"]), c["id_a"], c["id_b"], c["rel"], c["sqrt_info"])


# ---------------------------------------------------------------------------------------------------------------- GPU
def _solver(c, **kw):
    s = pgo.PgoSolver(**kw)
    s.set_poses(c["ids"], c["poses"], c["fixed"]); s.add_edges(c["id_a"], c["id_b"], c["rel"], c["sqrt_info"])
    return s


def _rot_init(s, c, **cfg):
    if c.get("gravity", 0):
        return s.rot_init(c["ego_ids"], c["ego"], enable_gravity_prior=1, **cfg)
    return s.rot_init(**cfg)


def _rots(poses):
    return ro.quat_R(np.asarray(poses)[:, 3:7])


@pytest.mark.gpu
def test_device_matches_the_frozen_reference_outputs():
    cases, refs = golden()
    for name, c in cases.items():
        r = _ref(refs, name)
        s = _solver(c)
        rep = _rot_init(s, c)
        out = s.get_poses(c["ids"])
        pos = {int(i): k for k, i in enumerate(c["ids"])}
        rows = [pos[int(f)] for f in r["frames"]]
        err = np.abs(_rots(out[rows]) - r["R"]).max()
        print(f"{name}: frames {rep['frames']} dropped {rep['edges_dropped']} pcg {rep['pcg_iterations']} residual {rep['residual']} "
              f"|R - R_ref| {err:.2e} state_changes {rep['state_changes']:.6e} (ref {float(r['state_changes']):.6e})")
        assert err <= 1e-9, (name, err)
        assert abs(rep["state_changes"] - float(r["state_changes"])) <= 1e-9
        assert rep["edges_dropped"] == int(r["dropped"]) and rep["frames"] == len(r["frames"])
        assert rep["edges_used"] + rep["edges_dropped"] == len(c["id_a"])
        # positions of every frame, and fixed and untouched poses entirely, keep every bit
        assert np.array_equal(out[:, :3], c["poses"][:, :3])
        keep = np.ones(len(c["ids"]), bool); keep[rows] = False
        assert keep.sum() >= 1 and np.array_equal(out[keep], c["poses"][keep])
        s.close()


@pytest.mark.gpu
def test_device_matches_the_oracle_on_a_larger_graph():
    for grav in (False, True):
        c = graph_case(21, n_agents=3, n=300, loops=900, tilt=0.4, gravity=grav, quirk=True, self_loop=True)
        o = oracle_of(c)
        s = _solver(c)
        rep = _rot_init(s, c)
        out = s.get_poses(c["ids"])
        pos = {int(i): k for k, i in enumerate(c["ids"])}
        rows = [pos[int(f)] for f in o["frames"]]
        err = np.abs(_rots(out[rows]) - o["R"]).max()
        print(f"gravity {grav}: {rep['frames']} frames, pcg {rep['pcg_iterations']}, residual {rep['residual']}, {rep['device_ms']:.1f} ms, "
              f"|R - R_oracle| {err:.2e}, state_changes {rep['state_changes']:.6e} vs {o['state_changes']:.6e}")
        assert err <= 1e-8, err
        assert abs(rep["state_changes"] - o["state_changes"]) <= 1e-8
        assert max(rep["residual"]) <= 1e-12 and rep["edges_dropped"] == o["dropped"]
        s.close()


def _refusal_cases():
    c = reference_cases()["gravity"]
    bad_ego = c["ego"].copy(); bad_ego[3, 4] = np.nan
    return c, [
        ("no ego pose for a frame", dict(ego_ids=c["ego_ids"][:-3], ego=c["ego"][:-3]), 2),
        ("unknown ego id", dict(ego_ids=np.concatenate([c["ego_ids"], [123456789]]), ego=np.concatenate([c["ego"], c["ego"][:1]])), 2),
        ("duplicate ego id", dict(ego_ids=np.concatenate([c["ego_ids"], c["ego_ids"][:1]]), ego=np.concatenate([c["ego"], c["ego"][:1]])), 2),
        ("non-finite ego pose", dict(ego_ids=c["ego_ids"], ego=bad_ego), 2),
        ("negative count", dict(ego_ids=c["ego_ids"], ego=c["ego"], n=-1), 1),
    ]


def _call(s, ego_ids, ego, n=None, grav=1):
    L = pgo._lib()
    cfg = pgo.RotInitConfig(); L.d2pgo_default_rot_init_config(C.byref(cfg)); cfg.enable_gravity_prior = grav
    ids = np.ascontiguousarray(ego_ids, np.int64); e = np.ascontiguousarray(np.asarray(ego, np.float64).reshape(-1, 7))
    rep = pgo.RotInitReport()
    return L.d2pgo_rot_init(s.h, C.byref(cfg), C.c_int32(len(ids) if n is None else n), pgo._p(ids), pgo._p(e), C.byref(rep))


@pytest.mark.gpu
def test_refusals_leave_the_handle_unchanged():
    c, calls = _refusal_cases()
    kw = dict(max_iterations=8, pcg_max_iterations=100)
    ref = _solver(c, **kw); ref_rep = ref.solve(); ref_out = ref.get_poses(c["ids"]); ref.close()

    def check(s, rc, want, what):
        assert rc == want, (what, rc)
        assert pgo._lib().d2pgo_last_error(s.h)
        assert np.array_equal(s.get_poses(c["ids"]), c["poses"]), what
        rep = s.solve()
        assert rep.final_cost == ref_rep.final_cost and np.array_equal(s.get_poses(c["ids"]), ref_out), what
        s.close()

    for what, a, want in calls:
        s = _solver(c, **kw)
        check(s, _call(s, a["ego_ids"], a["ego"], a.get("n")), want, what)
    # a component of free frames without a fixed frame: no fixed flag at all, and a free frame named only by a b-fixed edge
    g = dict(c); g["fixed"] = np.zeros_like(c["fixed"])
    s = _solver(g, **kw)
    rc = _call(s, c["ego_ids"], c["ego"])
    assert rc == 2 and np.array_equal(s.get_poses(c["ids"]), c["poses"])
    s.close()
    h = dict(c)
    h["ids"] = np.concatenate([c["ids"], [77_000_000]]); h["poses"] = np.concatenate([c["poses"], c["poses"][1:2]])
    h["fixed"] = np.concatenate([c["fixed"], [0]]).astype(np.uint8)
    h["id_a"] = np.concatenate([c["id_a"], [77_000_000]]); h["id_b"] = np.concatenate([c["id_b"], [c["ids"][0]]])
    h["rel"] = np.concatenate([c["rel"], c["rel"][:1]]); h["sqrt_info"] = np.concatenate([c["sqrt_info"], c["sqrt_info"][:1]])
    s = _solver(h, **kw)
    rc = _call(s, np.concatenate([c["ego_ids"], [77_000_000]]), np.concatenate([c["ego"], c["ego"][:1]]))
    assert rc == 2 and "77000000" in pgo._lib().d2pgo_last_error(s.h).decode() and np.array_equal(s.get_poses(h["ids"]), h["poses"])
    s.close()
    # a 4-DoF handle, and an ARock handle: 5; a null config: 1
    s4 = pgo.PgoSolver(pose_dof=4)
    s4.set_poses_4d(c["ids"], pgo.poses_to_4d(c["poses"]), c["fixed"])
    assert _call(s4, c["ego_ids"], c["ego"]) == 5
    s4.close()
    s = _solver(c, **kw)
    assert pgo._lib().d2pgo_rot_init(s.h, None, 0, None, None, None) == 1
    s.arock_enable(c["ids"], np.zeros(len(c["ids"]), np.int32), self_id=0)
    check(s, _call(s, c["ego_ids"], c["ego"]), 5, "ARock mode")


@pytest.mark.gpu
def test_bitwise_reproducible():
    c = graph_case(22, n_agents=3, n=100, loops=300, gravity=True, quirk=True)
    outs, reps = [], []
    a = _solver(c)
    for _ in range(2):
        a.set_poses(c["ids"], c["poses"], c["fixed"]); a.add_edges(c["id_a"], c["id_b"], c["rel"], c["sqrt_info"])
        reps.append(_rot_init(a, c)); outs.append(a.get_poses(c["ids"]))
    b = _solver(c)
    reps.append(_rot_init(b, c)); outs.append(b.get_poses(c["ids"]))
    for o, r in zip(outs[1:], reps[1:]):
        assert np.array_equal(o, outs[0]) and r["state_changes"] == reps[0]["state_changes"] and r["pcg_iterations"] == reps[0]["pcg_iterations"]
    a.close(); b.close()


@pytest.mark.gpu
def test_rot_init_then_solve_lands_on_the_sparse_direct_optimum():
    # seed 7 rather than test_pgo.py's 6: there agent 2's only tie to the rest is a loop into the fixed frame, which gives no
    # rows (the b-fixed quirk), and rot init refuses the graph
    g = pgo.make_pose_graph(seed=7, n_agents=4, poses_per_agent=60, loops=300)
    c = dict(ids=g["ids"], poses=g["init"], fixed=g["fixed"], id_a=g["id_a"], id_b=g["id_b"], rel=g["rel"], sqrt_info=g["sqrt_info"])
    s = _solver(c, max_iterations=40, pcg_max_iterations=400, pcg_tolerance=1e-12, lambda0=0.0, function_tolerance=1e-14)
    s.rot_init()
    start = s.get_poses(g["ids"])
    rep = s.solve()
    x_ref, costs = po.solve(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], iters=40)
    assert rep.final_cost < rep.initial_cost and abs(rep.final_cost - costs[-1]) <= 1e-8 * costs[-1], (rep.final_cost, costs[-1])
    dp, dr = synth.pose_errors(s.get_poses(g["ids"]), x_ref)
    assert dp <= 1e-6 and dr <= 1e-6, (dp, dr)
    assert np.array_equal(start[:, :3], g["init"][:, :3])
    s.close()


def _rot_rms_deg(poses, gt):
    R, G = _rots(poses), _rots(gt)
    c = (np.einsum("nij,nij->n", R, G) - 1.0) / 2.0
    return np.rad2deg(np.sqrt(np.mean(np.arccos(np.clip(c, -1.0, 1.0)) ** 2)))


@pytest.mark.gpu
def test_rot_init_removes_attitude_drift():
    g = pgo.make_pose_graph(seed=7, n_agents=4, poses_per_agent=250, loops=2000)
    c = dict(ids=g["ids"], poses=g["init"], fixed=g["fixed"], id_a=g["id_a"], id_b=g["id_b"], rel=g["rel"], sqrt_info=g["sqrt_info"])
    s = _solver(c)
    rep = s.rot_init()
    e0, e1 = _rot_rms_deg(g["init"], g["gt"]), _rot_rms_deg(s.get_poses(g["ids"]), g["gt"])
    print(f"rotation RMS error to the ground truth: {e0:.2f} deg before, {e1:.2f} deg after; pcg {rep['pcg_iterations']}")
    assert e1 < 0.6 * e0, (e0, e1)
    s.close()
