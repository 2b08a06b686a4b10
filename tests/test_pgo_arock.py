"""d2pgo's ARock distributed mode (pgo_mode 1): the oracle's restatement of the reference's ARock loop, the agents' sub-graphs,
and the device agents (include/d2pgo.h d2pgo_arock_*) against the oracle, in the two configurations the reference runs: 4-DoF
[x y z yaw] duals (d2pgo_test's default) and 6-DoF perturbation duals [p ; theta] (the node's perturb_mode)."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from d2slam_b200 import pgo, synth  # noqa: E402
from oracle import pgo4d_oracle as p4  # noqa: E402
from oracle import pgo_arock_oracle as ao  # noqa: E402
from oracle import pgo_gravity_oracle as go  # noqa: E402
from oracle import pgo_oracle as po  # noqa: E402

SEED = 4            # 3 agents x 15 frames: every |yaw| < 0.4 rad, inter-agent loops, and frames of one agent in loops with both others
SHIPPED = {"default": dict(rho_frame_T=0.1, rho_frame_theta=0.1, eta_k=0.9),           # ARockSolverConfig defaults (ARock.hpp:6-19)
           "d435_multi": dict(rho_frame_T=0.7, rho_frame_theta=0.625, eta_k=0.1)}      # config/realsense_d435/d435_multi.yaml
TIGHT = dict(max_iterations=200, pcg_max_iterations=2000, pcg_tolerance=1e-12, lambda0=1e-8, function_tolerance=1e-15)


def graph(dof, seed=SEED):
    g = pgo.make_pose_graph(seed=seed, n_agents=3, poses_per_agent=15, loops=60, loop_radius=8.0)
    return g if dof == 6 else pgo.pose_graph_to_4d(g, seed=seed)


def gravity_of(g, split):
    """ego poses of a split's frames (make_gravity_case on the whole graph) and the oracle's prior tuple"""
    c = pgo.make_gravity_case(g, seed=SEED)
    pos = {int(i): k for k, i in enumerate(g["ids"])}
    ego = c["ego"][[pos[int(i)] for i in split["ids"]]]
    n = len(ego)
    return ego, (np.arange(n), go.ego_gravity(ego), np.tile(pgo.GRAVITY_SQRT_INFO * np.eye(3), (n, 1, 1)))


def oracle_agents(gg, cfg, gravity_graph=None, splits=None, **kw):
    out = []
    for s in range(3):
        sp = pgo.arock_split(gg, s) if splits is None else splits[s]
        pri = gravity_of(gravity_graph, sp)[1] if gravity_graph is not None else None
        out.append(ao.OracleAgent(sp, priors=pri, **cfg, **kw))
    return out


def third_party(agents):
    """duals (agent, neighbour, frame) whose frame belongs to neither the agent nor the neighbour"""
    return [(a.self_id, n, f) for a in agents for (n, f) in a.duals if int(a.owner[a.pos[f]]) not in (n, a.self_id)]


# ------------------------------------------------------------------------------------------------ CPU: sub-graphs
def test_arock_split_takes_own_odometry_and_the_loops_between_known_frames():
    g = graph(6)
    agent = g["agent"]; n_odo = len(g["ids"]) - 3
    for s in range(3):
        sp = pgo.arock_split(g, s)
        e = sp["edges"]
        odo = e[e < n_odo]
        assert np.all(agent[g["ea"][odo]] == s)                        # only s's own ego-motion edges
        assert len(odo) == 14
        mine = set(g["ids"][agent == s].tolist())
        known = mine | {int(v) for a, b in zip(g["id_a"][n_odo:], g["id_b"][n_odo:]) if int(a) in mine or int(b) in mine for v in (a, b)}
        want = [k for k in range(n_odo, len(g["id_a"])) if int(g["id_a"][k]) in known and int(g["id_b"][k]) in known]
        assert e[e >= n_odo].tolist() == want                          # every loop whose two frames s knows
        assert set(sp["ids"].tolist()) == known
        assert sp["fixed"].sum() == (1 if s == 0 else 0)               # only main_id's head frame is constant
        if s == 0:
            assert sp["ids"][sp["fixed"] == 1][0] == g["ids"][0]
        assert np.all(sp["owner"] == sp["ids"] // 1_000_000)


def test_arock_split_from_the_per_agent_g2o_layout(tmp_path):
    g = graph(6)
    pgo.write_g2o_agents(str(tmp_path), g["ids"], g["init"], g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    r = pgo.read_g2o_agents(str(tmp_path), 3)
    for s in range(3):
        a, b = pgo.arock_split(g, s), pgo.arock_split(r, s)
        assert a["ids"].tolist() == b["ids"].tolist() and a["fixed"].tolist() == b["fixed"].tolist() and a["owner"].tolist() == b["owner"].tolist()
        ka = sorted(zip(a["id_a"].tolist(), a["id_b"].tolist())); kb = sorted(zip(b["id_a"].tolist(), b["id_b"].tolist()))
        assert ka == kb
        assert np.abs(a["poses"] - b["poses"]).max() < 1e-12


# ------------------------------------------------------------------------------------------------ CPU: the oracle's bookkeeping
def one_frame_agent(dof, self_id=0, owner=1, **cfg):
    """agent self_id holding frame 7 (owned by `owner`) and its own frame 5, one edge between them"""
    x = np.array([[0.0, 0.0, 0.0, 0.1], [1.0, 0.0, 0.0, 0.2]]) if dof == 4 else np.array([[0.0, 0, 0, 0, 0, 0, 1], [1.0, 0, 0, 0, 0, np.sin(0.1), np.cos(0.1)]])
    D = dof
    rel = x[1:2].copy() if dof == 4 else pgo.relative_pose(x[0], x[1])[None]
    split = dict(self_id=self_id, ids=np.array([5, 7]), poses=x, fixed=np.array([1, 0], np.uint8), owner=np.array([self_id, owner], np.int32),
                 id_a=np.array([5]), id_b=np.array([7]), rel=rel, sqrt_info=np.eye(D).reshape(1, -1))
    return ao.OracleAgent(split, **cfg), split


@pytest.mark.parametrize("dof", [4, 6])
def test_scan_creates_duals_at_the_pose_or_zero(dof):
    a, _ = one_frame_agent(dof)
    a._process(); a._scan()
    assert list(a.duals) == [(1, 7)]
    c = ao.coords(a.x, a.qi)[1]
    assert np.array_equal(a.duals[(1, 7)][0], c) and np.array_equal(a.duals[(1, 7)][1], c)
    z, _ = one_frame_agent(dof, dual_state_init_to_zero=True)
    z._process(); z._scan()
    assert not z.duals[(1, 7)][0].any() and not z.duals[(1, 7)][1].any()


@pytest.mark.parametrize("dof", [4, 6])
def test_receive_honours_the_target_and_the_existing_dual_rule(dof):
    a, _ = one_frame_agent(dof)
    v1, v2, v3 = (np.full(dof, k * 0.01) for k in (1, 2, 3))
    a.receive((2, 9, [7], [v1]))          # no dual (2, 7) yet: created, y_l = y_r = v1 although the target is another agent
    a.receive((2, 9, [7], [v2]))          # exists, target is not self: ignored
    a.receive((1, 9, [99], [v2]))         # a frame outside the problem: ignored
    a._process()
    assert list(a.duals) == [(2, 7)] and np.array_equal(a.duals[(2, 7)][0], v1) and np.array_equal(a.duals[(2, 7)][1], v1)
    a.receive((2, 0, [7], [v3]))          # target = self: y_r only
    a._process()
    assert np.array_equal(a.duals[(2, 7)][0], v1) and np.array_equal(a.duals[(2, 7)][1], v3)


def test_dual_update_keeps_the_unwrapped_mean_and_normalises_late():
    # y_l, y_r on both sides of +-pi: the reference averages the raw numbers ((3.1 - 3.1) / 2 = 0) and wraps y_l's yaw only once
    # it leaves [-pi, pi] (ARock.cpp:51-62)
    yl = np.array([0.0, 0.0, 0.0, 3.1]); yr = np.array([0.0, 0.0, 0.0, -3.1]); x = np.array([0.0, 0.0, 0.0, 3.12])
    out = ao.update_duals(yl, yr, x, 0.9)
    assert out[3] == 3.1 - (0.0 - 3.12) * 0.9 - 2 * np.pi            # 5.908 wrapped once
    out = ao.update_duals(yl, yr, x, 0.01)
    assert out[3] == 3.1 - (0.0 - 3.12) * 0.01                        # 3.1312 > pi? no: pi = 3.14159, left as it is
    out = ao.update_duals(np.array([0, 0, 0, 3.14]), np.array([0, 0, 0, 3.14]), np.array([0, 0, 0, 3.10]), 0.9)
    assert out[3] == 3.14 - (3.14 - 3.10) * 0.9
    six = ao.update_duals(np.full(6, 4.0), np.full(6, 4.0), np.zeros(6), 0.9)   # 6-DoF: Euclidean, never wrapped
    assert np.all(six == 4.0 - 4.0 * 0.9)


@pytest.mark.parametrize("dof", [4, 6])
def test_proximal_jacobians_match_finite_differences(dof):
    rng = np.random.default_rng(1)
    for _ in range(20):
        if dof == 4:
            x = np.concatenate([rng.normal(size=3), [rng.uniform(-3, 3)]]); qi = None; y = np.concatenate([rng.normal(size=3), [rng.uniform(-3, 3)]])
        else:
            qi = pgo._qexp(rng.normal(size=3))
            x = np.concatenate([rng.normal(size=3), pgo._qmul(qi, pgo._qexp(rng.normal(0, 0.8, 3)))]); y = rng.normal(size=6)
        r, J = ao.prox_eval(x[None], None if qi is None else qi[None], y[None], 0.7, 0.625)
        h = 1e-6
        for k in range(dof):
            d = np.zeros(dof); d[k] = h
            if dof == 4:
                xp, xm = x + d, x - d
            else:
                xp, xm = synth.pose_plus(x, d), synth.pose_plus(x, -d)
            rp = ao.prox_eval(xp[None], None if qi is None else qi[None], y[None], 0.7, 0.625)[0][0]
            rm = ao.prox_eval(xm[None], None if qi is None else qi[None], y[None], 0.7, 0.625)[0][0]
            assert np.abs((rp - rm) / (2 * h) - J[0][:, k]).max() < 1e-6


def test_theta_is_the_principal_log_and_small_angles_use_the_series():
    rng = np.random.default_rng(2)
    qi = pgo._qexp(rng.normal(size=(50, 3)))
    for scale in (1e-9, 1e-3, 0.3, 2.5):
        th = rng.normal(size=(50, 3)); th *= scale / np.linalg.norm(th, axis=1, keepdims=True)
        q = pgo._qmul(qi, pgo._qexp(th))
        got, Jinv = ao.theta_of(-q if scale > 1 else q, qi)                 # either sign of q
        assert np.abs(got - th).max() < 1e-12
        # J_r^-1 is the inverse of J_r(theta) = I - (1 - cos a)/a^2 [th]x + (a - sin a)/a^3 [th]x^2
        a = np.linalg.norm(th, axis=1)[:, None, None]; K = po._vskew(th)
        Jr = np.eye(3) - (1 - np.cos(a)) / a ** 2 * K + (a - np.sin(a)) / a ** 3 * np.einsum("kij,kjl->kil", K, K)
        if scale > 1e-6:
            assert np.abs(np.einsum("kij,kjl->kil", Jinv, Jr) - np.eye(3)).max() < 1e-9


@pytest.mark.parametrize("dof", [4, 6])
def test_third_party_discovery_happens_on_the_test_graph(dof):
    agents = oracle_agents(graph(dof), SHIPPED["default"])
    ao.arock_run(agents, 2)
    tp = third_party(agents)
    assert tp, "the graph must exercise the path where an agent latches onto another pair's dual"
    for s, n, f in tp:                                                  # the latched pair is symmetric
        assert (n, s, f) in tp


def centralised(dof, gg):
    if dof == 4:
        return p4.solve_4d(gg["init"], gg["fixed"], gg["ea"], gg["eb"], gg["rel"], gg["sqrt_info"])[0]
    return po.solve(gg["init"], gg["fixed"], gg["ea"], gg["eb"], gg["rel"], gg["sqrt_info"])[0]


@pytest.mark.parametrize("dof", [4, 6])
@pytest.mark.parametrize("params", list(SHIPPED))
def test_oracle_arock_with_the_shipped_parameters(dof, params, capsys):
    """What the synchronous ARock loop does on a small connected graph (3 agents x 15 frames, 41 loops): copies of a shared
    frame and the agents' own poses against the centralised sparse-direct optimum, per round.  With the ARockSolverConfig
    defaults (0.1 / 0.1 / 0.9) the copies come within 1 cm of each other after ~30 (4-DoF) / ~44 (6-DoF) rounds and the own poses
    within 1 cm of the optimum after ~38 / ~46; with d435_multi's 0.7 / 0.625 / 0.1 neither happens in 100 rounds (copies still
    4-7 cm apart, own poses ~0.12 m from the optimum)."""
    gg = graph(dof)
    xc = centralised(dof, gg)
    pos = {int(i): k for k, i in enumerate(gg["ids"])}
    hist = []

    def cb(r, agents):
        dp, dr = ao.copy_disagreement(agents)
        own = max(float(np.linalg.norm(a.x[i, :3] - xc[pos[int(f)], :3])) for a in agents for i, f in enumerate(a.ids) if a.owner[i] == a.self_id)
        hist.append((dp, dr, own))
    agents = oracle_agents(gg, SHIPPED[params])
    rounds = 100
    ao.arock_run(agents, rounds, cb)
    h = np.array(hist)
    first = lambda col, tol: next((r + 1 for r in range(rounds) if h[r, col] < tol), None)
    with capsys.disabled():
        print(f"\n[arock {dof}-DoF {params}] copies apart (m): round 1 {h[0, 0]:.3f}, 10 {h[9, 0]:.3f}, 100 {h[-1, 0]:.3f}; "
              f"own poses vs centralised (m): round 1 {h[0, 2]:.3f}, 100 {h[-1, 2]:.3f}; rounds to copies < 1 cm: {first(0, 1e-2)}, "
              f"to own poses within 1 cm of the centralised optimum: {first(2, 1e-2)}")
    assert h[-1, 0] < h[0, 0] / 10 and h[-1, 2] < h[0, 2] / 5           # it pulls the copies together and towards the optimum
    want = {(4, "default"): (30, 38), (6, "default"): (44, 46), (4, "d435_multi"): (None, None), (6, "d435_multi"): (None, None)}[(dof, params)]
    for got, w in zip((first(0, 1e-2), first(2, 1e-2)), want):
        assert (got is None) if w is None else (got is not None and abs(got - w) <= 3), (got, w)


def test_new_kernels_do_not_spill():
    from d2slam_b200 import build
    build.build()
    log = open(os.path.join(ROOT, "d2slam_b200", "build", "ptxas.log")).read()
    blocks = re.findall(r"Compiling entry function '(\w*k_pgo_arock\w*)'.*?\n(.*?)\n(.*?)\n", log)
    assert len(blocks) == 10
    for name, _, props in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props, (name, props)


# ------------------------------------------------------------------------------------------------ GPU
def device_agents(gg, cfg, gravity_graph=None, solver_kw=TIGHT, splits=None, **kw):
    out = []
    for s in range(3):
        sp = pgo.arock_split(gg, s) if splits is None else splits[s]
        ego = gravity_of(gravity_graph, sp)[0] if gravity_graph is not None else None
        out.append(pgo.ArockAgent(sp, ego_poses=ego, solver_kw=solver_kw, **cfg, **kw))
    return out


def pose_diff(dof, a, b):
    if dof == 4:
        return float(np.abs(a[:, :3] - b[:, :3]).max()), float(np.abs(pgo.normalize_angle(a[:, 3] - b[:, 3])).max())
    dp, dr = synth.pose_errors(a, b)
    return float(dp), float(dr)


def compare_rounds(dof, gg, cfg, rounds=10, gravity=False, fix_heads=False, **kw):
    splits = [pgo.arock_split(gg, s) for s in range(3)]
    if fix_heads:   # every agent holds its own head frame (a well-posed local problem even when the duals start at zero)
        for sp in splits:
            sp["fixed"][sp["ids"] == sp["ids"][sp["owner"] == sp["self_id"]].min()] = 1
    dev = device_agents(gg, cfg, graph(6) if gravity else None, splits=splits, **kw)
    orc = oracle_agents(gg, cfg, graph(6) if gravity else None, splits=splits, **kw)
    worst = [0.0, 0.0, 0.0]
    for r in range(rounds):
        pgo.arock_run(dev, 1); ao.arock_run(orc, 1)
        for d, o in zip(dev, orc):
            dp, dr = pose_diff(dof, d.poses(), o.x)
            assert dp < 1e-6 and dr < 1e-6, (r, d.self_id, dp, dr)
            dd = d.duals()
            assert sorted(dd) == sorted(o.duals), (r, d.self_id)
            dy = max(max(np.abs(dd[k][0] - o.duals[k][0]).max(), np.abs(dd[k][1] - o.duals[k][1]).max()) for k in dd)
            assert dy < 1e-6, (r, d.self_id, dy)
            worst = [max(worst[0], dp), max(worst[1], dr), max(worst[2], dy)]
    for a in dev:
        a.close()
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("dof", [4, 6])
@pytest.mark.parametrize("params", list(SHIPPED))
def test_device_arock_matches_the_oracle_every_round(dof, params):
    w = compare_rounds(dof, graph(dof), SHIPPED[params])
    print(f"arock {dof}-DoF {params}: worst pose diff {w[0]:.2e} m {w[1]:.2e} rad, dual diff {w[2]:.2e}")


@pytest.mark.gpu
def test_device_arock_with_gravity_priors_and_zero_initialised_duals():
    compare_rounds(6, graph(6), SHIPPED["d435_multi"], gravity=True)
    # zero-initialised duals pull every shared frame towards the origin; with the gauge held by those pulls alone (agents 1
    # and 2) the local problem is too ill-conditioned for a 1e-6 comparison, so here every agent fixes its own head frame
    compare_rounds(4, graph(4), SHIPPED["default"], rounds=5, fix_heads=True, dual_state_init_to_zero=1)
    compare_rounds(6, graph(6), SHIPPED["default"], rounds=5, fix_heads=True, dual_state_init_to_zero=1)


@pytest.mark.gpu
@pytest.mark.parametrize("dof", [4, 6])
def test_device_proximal_terms_match_the_oracle(dof):
    gg = graph(dof)
    dev = device_agents(gg, SHIPPED["d435_multi"])
    pgo.arock_run(dev, 2)
    for d in dev:
        o = ao.OracleAgent(d.split, **SHIPPED["d435_multi"])
        o.x = d.poses()
        for k, (yl, yr) in d.duals().items():
            o.duals[k] = [yl, yr]
        want = o.terms()
        got = d.s.debug_arock_terms(len(want))
        assert len(want) > 0
        assert np.abs(got - want).max() <= 1e-11 * max(1.0, np.abs(want).max())
        d.close()


@pytest.mark.gpu
def test_device_dual_update_across_pi_matches_the_reference_arithmetic():
    """A 4-DoF dual whose y_l and y_r lie on both sides of +-pi: the device keeps the unwrapped mean and wraps y_l's yaw only
    once it leaves [-pi, pi], bit for bit the oracle's update at the device's solved pose."""
    _, split = one_frame_agent(4)
    split["poses"] = np.array([[0.0, 0.0, 0.0, 0.0], [1.0, 0.0, 0.0, 3.05]]); split["rel"] = np.array([[1.0, 0.0, 0.0, 3.05]])
    a = pgo.ArockAgent(split, solver_kw=TIGHT, eta_k=0.9)
    a.receive((1, 0, [7], [np.array([1.0, 0.0, 0.0, 3.1])]))             # creates (1, 7): y_l = y_r = yaw 3.1
    a.step()
    _, yl1, _ = a.s.arock_duals(1)
    a.receive((1, 0, [7], [np.array([1.0, 0.0, 0.0, -3.1])]))            # y_r across pi
    a.step()
    f, yl2, yr2 = a.s.arock_duals(1)
    x = a.poses()[1]
    assert f.tolist() == [7] and yr2[0, 3] == -3.1
    raw = yl1[0, 3] - ((yl1[0, 3] + yr2[0, 3]) / 2 - x[3]) * 0.9
    assert raw > np.pi                                                   # the case the late normalisation is for
    assert np.array_equal(yl2[0], ao.update_duals(yl1[0], yr2[0], x, 0.9))
    assert -np.pi <= yl2[0, 3] < np.pi
    a.close()


@pytest.mark.gpu
def test_arock_steps_are_bitwise_reproducible():
    def run():
        dev = device_agents(graph(6), SHIPPED["default"], gravity_graph=graph(6))
        pgo.arock_run(dev, 4)
        out = [(d.poses(), d.duals()) for d in dev]
        for d in dev:
            d.close()
        return out
    a, b = run(), run()
    for (pa, da), (pb, db) in zip(a, b):
        assert np.array_equal(pa, pb)
        assert sorted(da) == sorted(db) and all(np.array_equal(da[k][0], db[k][0]) and np.array_equal(da[k][1], db[k][1]) for k in da)


@pytest.mark.gpu
def test_the_dual_table_survives_set_poses():
    gg = graph(4)
    dev = device_agents(gg, SHIPPED["default"])
    pgo.arock_run(dev, 2)
    a = dev[1]
    before = a.duals()
    sp = a.split
    keep = np.ones(len(sp["ids"]), bool)
    gone = [f for (_, f) in before][0]
    keep[list(sp["ids"]).index(gone)] = False
    a.s.set_poses_4d(sp["ids"][keep], a.poses()[keep], sp["fixed"][keep])
    after = a.duals()
    assert sorted(after) == sorted(k for k in before if k[1] != gone)
    for k in after:
        assert np.array_equal(after[k][0], before[k][0]) and np.array_equal(after[k][1], before[k][1])
    for d in dev:
        d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dof", [4, 6])
def test_receive_rules_on_the_device(dof):
    _, split = one_frame_agent(dof)
    a = pgo.ArockAgent(split, solver_kw=TIGHT)
    v1, v2, v3 = (np.full(dof, k * 0.01) for k in (1, 2, 3))
    a.receive((2, 9, [7], [v1])); a.receive((2, 9, [7], [v2])); a.receive((1, 9, [99], [v2]))
    a.step()
    d = a.duals()
    assert sorted(d) == [(1, 7), (2, 7)]                                 # (1, 7) by scanning, (2, 7) by the first message
    assert np.array_equal(d[(2, 7)][1], v1)                              # the second message (target 9, dual exists) was ignored
    a.receive((2, 0, [7], [v3]))
    a.step()
    assert np.array_equal(a.duals()[(2, 7)][1], v3)                     # target = self: y_r set
    a.close()


@pytest.mark.gpu
def test_bad_arock_calls_are_refused_and_keep_nothing():
    from d2slam_b200.solver import lib
    L = lib()
    _, split = one_frame_agent(4)
    a = pgo.ArockAgent(split, solver_kw=TIGHT)
    h = a.s.h
    f = np.array([7], np.int64)
    good = np.array([1.0, 0, 0, 0.2])
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    assert L.d2pgo_arock_receive(h, 1, 0, 1, p(f), 6, p(good)) == 2                      # wrong D
    assert L.d2pgo_arock_receive(h, 1, 0, 1, p(f), 4, p(np.array([1.0, np.nan, 0, 0]))) == 2
    assert L.d2pgo_arock_receive(h, 0, 1, 1, p(f), 4, p(good)) == 2                      # from itself
    assert L.d2pgo_arock_receive(h, 1, 0, 2, p(np.array([7, 7], np.int64)), 4, p(np.tile(good, 2))) == 2
    assert L.d2pgo_arock_receive(h, 1, 0, 1, None, 4, p(good)) == 1
    assert L.d2pgo_arock_receive(h, 1, 0, -1, p(f), 4, p(good)) == 1
    cfg = pgo.ArockConfig(); L.d2pgo_default_arock_config(C.byref(cfg))
    assert (cfg.rho_frame_T, cfg.rho_frame_theta, cfg.eta_k, cfg.dual_state_init_to_zero) == (0.1, 0.1, 0.9, 0)
    ids = np.array([5, 1234], np.int64); own = np.array([0, 1], np.int32)
    assert L.d2pgo_arock_enable(h, C.byref(cfg), 2, p(ids), p(own), None) == 2           # unknown id
    bad = pgo.ArockConfig(); L.d2pgo_default_arock_config(C.byref(bad)); bad.rho_frame_T = float("inf")
    assert L.d2pgo_arock_enable(h, C.byref(bad), 0, None, None, None) == 2
    a.step()
    assert sorted(a.duals()) == [(1, 7)]                                 # nothing of the refused calls was kept
    assert L.d2pgo_comm_init(h, (C.c_uint8 * 128)(), 0, 1) == 5          # ARock and edge sharding exclude each other
    assert "ARock" in L.d2pgo_last_error(h).decode()
    a.close()
    # 6-DoF: zero q_init; a pose without an owner stops the step
    _, split6 = one_frame_agent(6)
    s = pgo.PgoSolver(pose_dof=6)
    s.set_poses(split6["ids"], split6["poses"], split6["fixed"]); s.add_edges(split6["id_a"], split6["id_b"], split6["rel"], split6["sqrt_info"])
    ids = np.array([5, 7], np.int64); own = np.array([0, 1], np.int32)
    assert L.d2pgo_arock_enable(s.h, C.byref(cfg), 2, p(ids), p(own), p(np.zeros(8))) == 2
    assert L.d2pgo_arock_step(s.h, None) == 5                           # not in ARock mode
    assert L.d2pgo_arock_enable(s.h, C.byref(cfg), 1, p(ids), p(own), None) == 0
    assert L.d2pgo_arock_step(s.h, None) == 2                           # pose 7 has no owner
    s.close()


@pytest.mark.gpu
def test_solves_without_arock_on_the_bench_graph_keep_their_counts_at_the_exact_pcg_cap():
    """The bench's pose graph (seed 7) solved with bench.py's settings: the LM / PCG counts of the solver without ARock, pinned
    since CG stops at exactly pcg_max_iterations (it used to round the cap up to a multiple of 16, 208 instead of 200 here,
    which gave 60 LM / 10 289 PCG iterations on 6-DoF and 59 / 11 167 on 4-DoF; with the shorter steps the 6-DoF LM meets its
    function tolerance at 23 iterations instead of running all 60).  No LM iteration runs more than 200 CG iterations."""
    settings = dict(max_iterations=60, pcg_max_iterations=200, pcg_tolerance=1e-1, lambda0=1e-4, function_tolerance=1e-5)
    g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)
    s = pgo.PgoSolver(**settings)
    s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    r = s.solve(); s.close()
    assert (r.iterations, r.pcg_iterations, r.converged) == (23, 2302, 1)
    assert r.pcg_iterations <= 200 * r.iterations
    h = pgo.pose_graph_to_4d(g, seed=7)
    s = pgo.PgoSolver(pose_dof=4, **settings)
    s.set_poses_4d(h["ids"], h["init"], h["fixed"]); s.add_edges_4d(h["id_a"], h["id_b"], h["rel"], h["sqrt_info"])
    r = s.solve(); s.close()
    assert (r.iterations, r.pcg_iterations) == (59, 10749)
    assert r.pcg_iterations <= 200 * r.iterations


PARENT = "9392526"   # the last commit before ARock: its d2pgo.cu kernels are the ones a graph without ARock must still run


def test_kernels_without_arock_compile_to_the_same_sass_as_before():
    """Every kernel of d2pgo.cu as it was before ARock compiles to the same instructions now, in d2pgo.cu or d2pgo_pcm.cu (the
    proximal terms live in kernels of their own).  Needs the git history and the CUDA toolkit; skipped without them."""
    import shutil
    import subprocess
    import tempfile
    from d2slam_b200 import build
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (shutil.which("git") and shutil.which("cuobjdump") and os.path.exists(nvcc)):
        pytest.skip("git, nvcc or cuobjdump unavailable")
    objs = [os.path.join(ROOT, "d2slam_b200", "build", o) for o in ("d2pgo.o", "d2pgo_pcm.o")]   # PCM's kernels have their own file
    build.build(force=not all(os.path.exists(o) for o in objs))
    with tempfile.TemporaryDirectory() as td:
        files = {"d2slam_b200/csrc/d2pgo.cu": "x/csrc/d2pgo.cu", "d2slam_b200/csrc/d2ba_math.cuh": "x/csrc/d2ba_math.cuh", "include/d2pgo.h": "include/d2pgo.h"}
        for src, dst in files.items():
            r = subprocess.run(["git", "-C", ROOT, "show", f"{PARENT}:{src}"], capture_output=True)
            if r.returncode:
                pytest.skip(f"commit {PARENT} not in this checkout")
            os.makedirs(os.path.dirname(os.path.join(td, dst)), exist_ok=True)
            open(os.path.join(td, dst), "wb").write(r.stdout)
        flags = [f for f in build.NVCC_FLAGS if f not in ("-Xptxas", "-v")]
        obj = os.path.join(td, "parent.o")
        subprocess.check_call([nvcc] + flags + ["-c", os.path.join(td, "x", "csrc", "d2pgo.cu"), "-o", obj])
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        import sass_diff
        old = sass_diff.kernels(obj)
        new = {}
        for o in objs:
            new.update(sass_diff.kernels(o))
    assert len(old) == 31
    assert [k for k in old if new.get(k) != old[k]] == []
    assert sum("k_pgo_arock" in k for k in new) == 10


# ------------------------------------------------------------------------------------------------ CPU: the reference's ARock loop
# The reference's own ARock.cpp (oracle/_ref/libd2ref_arock.so) replays the oracle's local solutions: after every round, every
# agent's dual table and the proximal factors it created must be the oracle's.  Live where the pin library is built, and
# through tests/golden/ref_arock.npz (made by tests/golden/make_ref_arock_golden.py) everywhere.
from oracle import ref_arock  # noqa: E402

LIVE = pytest.mark.skipif(not ref_arock.available(), reason="reference ARock library not built")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_arock.npz")
PIN_ROUNDS = 6
PIN_CASES = {   # name: (dof, parameter set, dual_state_init_to_zero, global yaw offset of the 4-DoF graph)
    "dof4": (4, "default", False, 0.0),
    "dof4_across_pi": (4, "d435_multi", False, np.pi - 0.1),     # every yaw near +-pi: unwrapped means, late normalisation
    "dof4_zero": (4, "default", True, 0.0),
    "dof6": (6, "d435_multi", False, 0.0),
    "dof6_zero": (6, "default", True, 0.0),
}


def rotate4(h, a):
    """the 4-DoF graph turned by yaw a about the origin (relative measurements unchanged)"""
    out = dict(h)
    for k in ("init", "gt"):
        x = np.array(h[k]); c, s = np.cos(a), np.sin(a)
        x[:, :2] = np.stack([c * x[:, 0] - s * x[:, 1], s * x[:, 0] + c * x[:, 1]], 1); x[:, 3] = pgo.normalize_angle(x[:, 3] + a)
        out[k] = x
    return out


def pin_case(name):
    """The oracle's run of a case: its agents' sub-graphs, config and local solutions per round."""
    dof, params, zero, yaw = PIN_CASES[name]
    gg = graph(dof) if not yaw else rotate4(graph(4), yaw)
    cfg = dict(SHIPPED[params], dual_state_init_to_zero=zero)
    agents = oracle_agents(gg, cfg)
    solved = []
    ao.arock_run(agents, PIN_ROUNDS, lambda r, ags: solved.append([a.x.copy() for a in ags]))
    return dict(splits=[a.split for a in agents], cfg=cfg, solved=solved)


def replay_oracle(splits, cfg, solved):
    """the oracle's bookkeeping with the given local solutions; per round and agent: (keys, y_l, y_r, r | J) after the step"""
    agents = [ao.OracleAgent(sp, **cfg) for sp in splits]
    for k, a in enumerate(agents):
        a.replay = iter([solved[r][k] for r in range(len(solved))])
    out = []
    for r in range(len(solved)):
        row = []
        for a in agents:
            a.step()
            keys, _, yl, yr = a.table()
            row.append((keys, yl, yr, a.terms()))
        out.append(row)
        msgs = [m for a in agents for m in a.messages()]
        for a in agents:
            for m in msgs:
                if m[0] != a.self_id:
                    a.receive(m)
    return out


def to_ref_inputs(splits, solved, dof):
    """dual-coordinate states for the reference: initial and per-round solutions"""
    qi = [None if dof == 4 else sp["poses"][:, 3:7] / np.linalg.norm(sp["poses"][:, 3:7], axis=1, keepdims=True) for sp in splits]
    init = [ao.coords(sp["poses"], q) for sp, q in zip(splits, qi)]
    sol = [[ao.coords(x, q) for x, q in zip(row, qi)] for row in solved]
    return init, sol, qi


def tangent_jacobian(fac, coords_of, dof):
    """the reference's factor Jacobians are w.r.t. the state [p ; theta]; in the right-multiplicative tangent they are
    J blockdiag(I, J_r^-1(theta))"""
    D = dof
    out = np.array(fac)
    if dof == 6 and len(out):
        J = out[:, D:].reshape(-1, 6, 6)
        th = coords_of[:, 3:]
        q = pgo._qexp(th)
        Jinv = ao.theta_of(q, np.tile([0.0, 0.0, 0.0, 1.0], (len(q), 1)))[1]
        J[:, :, 3:] = np.einsum("kij,kjl->kil", J[:, :, 3:], Jinv)
        out[:, D:] = J.reshape(len(out), -1)
    return out


def compare_to_reference(splits, cfg, solved, ref, dof):
    orc = replay_oracle(splits, cfg, solved)
    init, sol, _ = to_ref_inputs(splits, solved, dof)
    worst = 0.0
    for r in range(len(solved)):
        for a, sp in enumerate(splits):
            keys, yl, yr, terms = orc[r][a]
            got = ref[r][a]
            assert list(got["keys"]) == keys, (r, a)
            if not keys:
                continue
            pos = {int(f): i for i, f in enumerate(sp["ids"])}
            c = np.array([sol[r][a][pos[f]] for _, f in keys])
            fac = tangent_jacobian(got["fac"], c, dof)
            for u, v in ((got["yl"], yl), (got["yr"], yr), (fac, terms)):
                d = float(np.abs(np.asarray(u) - v).max())
                assert d <= 1e-12 * max(1.0, float(np.abs(v).max())), (r, a, d)
                worst = max(worst, d)
    return worst


@LIVE
@pytest.mark.parametrize("name", list(PIN_CASES))
def test_oracle_matches_the_reference_arock_loop_live(name):
    c = pin_case(name)
    dof = PIN_CASES[name][0]
    init, sol, _ = to_ref_inputs(c["splits"], c["solved"], dof)
    ref = ref_arock.run([sp["self_id"] for sp in c["splits"]], [sp["ids"] for sp in c["splits"]], [sp["owner"] for sp in c["splits"]], init, sol,
                        c["cfg"]["rho_frame_T"], c["cfg"]["rho_frame_theta"], c["cfg"]["eta_k"], c["cfg"]["dual_state_init_to_zero"])
    compare_to_reference(c["splits"], c["cfg"], c["solved"], ref, dof)


def load_golden():
    z = np.load(GOLDEN)
    cases = {}
    for name in PIN_CASES:
        dof = int(z[f"{name}/dof"]); A = int(z[f"{name}/agents"]); R = int(z[f"{name}/rounds"])
        cfg = dict(rho_frame_T=float(z[f"{name}/rho_T"]), rho_frame_theta=float(z[f"{name}/rho_theta"]), eta_k=float(z[f"{name}/eta"]),
                   dual_state_init_to_zero=bool(z[f"{name}/init_zero"]))
        splits = [{k: z[f"{name}/a{a}/{k}"] for k in ("ids", "poses", "fixed", "owner", "id_a", "id_b", "rel", "sqrt_info")} for a in range(A)]
        for a, sp in enumerate(splits):
            sp["self_id"] = int(z[f"{name}/a{a}/self_id"])
        solved = [[z[f"{name}/r{r}/a{a}/solved"] for a in range(A)] for r in range(R)]
        ref = [[dict(keys=[(int(u), int(v)) for u, v in z[f"{name}/r{r}/a{a}/keys"]], yl=z[f"{name}/r{r}/a{a}/yl"], yr=z[f"{name}/r{r}/a{a}/yr"],
                     fac=z[f"{name}/r{r}/a{a}/fac"]) for a in range(A)] for r in range(R)]
        cases[name] = (dof, splits, cfg, solved, ref)
    return cases


@pytest.mark.parametrize("name", list(PIN_CASES))
def test_oracle_matches_the_frozen_reference_arock_loop(name):
    dof, splits, cfg, solved, ref = load_golden()[name]
    compare_to_reference(splits, cfg, solved, ref, dof)


def test_frozen_cases_cover_the_wrap_the_third_party_path_and_zero_duals():
    cases = load_golden()
    _, splits, _, solved, ref = cases["dof4_across_pi"]
    yl = np.concatenate([t["yl"][:, 3] for row in ref for t in row if len(t["keys"])])
    assert (np.abs(yl) > 2.5).any() and (yl > 0).any() and (yl < 0).any()      # duals on both sides of +-pi
    for name, (dof, splits, cfg, solved, ref) in cases.items():
        owner = [{int(f): int(o) for f, o in zip(sp["ids"], sp["owner"])} for sp in splits]
        tp = [(a, n, f) for row in ref for a, t in enumerate(row) for n, f in t["keys"] if owner[a][f] not in (n, splits[a]["self_id"])]
        assert tp, name                                                          # an agent latched onto another pair's dual
    _, _, _, _, ref = cases["dof6_zero"]
    assert any(len(t["keys"]) and not t["yr"].any(axis=1).all() for t in ref[0])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dof4", "dof4_across_pi", "dof6"])
def test_device_proximal_terms_match_the_frozen_reference(name):
    """Each agent of a frozen case at its round-3 solution, its dual table loaded as messages that create every dual with the
    reference's y_r; a step without LM iterations processes them, and the device's terms must be the reference's factors."""
    dof, splits, cfg, solved, ref = load_golden()[name]
    r = 3
    _, sol, _ = to_ref_inputs(splits, solved, dof)
    for a, sp in enumerate(splits):
        got = ref[r][a]
        if not got["keys"]:
            continue
        ag = pgo.ArockAgent(sp, solver_kw=dict(max_iterations=0), **cfg)
        x = solved[r][a]
        if dof == 4:
            ag.s.set_poses_4d(sp["ids"], x, sp["fixed"]); ag.s.add_edges_4d(sp["id_a"], sp["id_b"], sp["rel"], sp["sqrt_info"])
        else:
            ag.s.set_poses(sp["ids"], x, sp["fixed"]); ag.s.add_edges(sp["id_a"], sp["id_b"], sp["rel"], sp["sqrt_info"])
        for n in sorted({k[0] for k in got["keys"]}):
            rows = [i for i, k in enumerate(got["keys"]) if k[0] == n]
            ag.receive((n, sp["self_id"], [got["keys"][i][1] for i in rows], got["yr"][rows]))
        ag.step()
        assert sorted(ag.duals()) == got["keys"]
        pos = {int(f): i for i, f in enumerate(sp["ids"])}
        want = tangent_jacobian(got["fac"], np.array([sol[r][a][pos[f]] for _, f in got["keys"]]), dof)
        dev = ag.s.debug_arock_terms(len(want))
        assert np.abs(dev - want).max() <= 1e-11 * max(1.0, np.abs(want).max()), (a, np.abs(dev - want).max())
        ag.close()
