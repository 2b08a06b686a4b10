"""Distributed chordal rotation initialisation (include/d2pgo.h d2pgo_arock_rot_*; d2pgo's RotationInitARock<double> in
pgo_mode 1): the numpy oracle (oracle/pgo_rotinit_arock_oracle.py) against the reference's own RotationInitARock loop (live
through oracle/_ref/libd2ref_rotinit_arock.so, and through the frozen tests/golden/ref_rotinit_arock.npz) after every round, and
on the GPU the device against both -- one step from a common state, free-running rounds -- plus the receive rules, the
hand-off to d2pgo_arock_step, the refusals and reproducibility."""
import os
import re
import sys

import numpy as np
import pytest

from d2slam_b200 import pgo
from oracle import pgo_rotinit_arock_oracle as ra
from oracle.pgo_rotinit_oracle import quat_R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PARENT = "0061495"   # the last commit before the distributed rotation initialisation
TOL = 1e-12          # pcg_tolerance of the device runs
PARAMS = {           # name: (rho_rot_mat, eta_k, gravity rows)
    "multi_launch": (0.16, 0.9, False),   # d2pgo_test_multi.launch:13-16
    "multi_launch_gravity": (0.16, 0.9, True),
    "default_gravity_slow": (0.1, 0.1, True),
    "default_slow": (0.1, 0.1, False),
}


def graph(seed, n_agents=3, n=40, loops=60, tilt=0.3):
    """A make_pose_graph graph with `tilt` rad per axis of attitude error on the initial guess of every frame but agent 0's head,
    plus a loop from agent 1 into agent 0's head frame (fixed in agent 0's sub-graph: the b-fixed quirk there), a loop from
    that head frame to a frame of agent 0, and a self loop."""
    g = pgo.make_pose_graph(seed=seed, n_agents=n_agents, poses_per_agent=n, loops=loops)
    rng = np.random.default_rng(seed + 77)
    init = np.array(g["init"])
    q = pgo._qmul(init[1:, 3:7], pgo._qexp(rng.normal(0, tilt, (len(init) - 1, 3))))
    init[1:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    ea, eb, rel, S = list(g["ea"]), list(g["eb"]), list(g["rel"]), list(g["sqrt_info"])
    for i, j in ((n + 3, 0), (0, n // 2), (5, 5)):
        r = pgo.relative_pose(g["gt"][i], g["gt"][j]).copy()
        ea.append(i); eb.append(j); rel.append(r); S.append(np.diag([20.0, 20.0, 20.0, 57.0, 57.0, 57.0]).ravel())
    ea = np.array(ea); eb = np.array(eb)
    out = dict(g, init=init, ea=ea, eb=eb, id_a=g["ids"][ea], id_b=g["ids"][eb], rel=np.array(rel), sqrt_info=np.array(S))
    out["ego"] = pgo.make_gravity_case(out, seed=seed)["ego"]
    return out


def ego_of(g, split):
    pos = {int(i): k for k, i in enumerate(g["ids"])}
    return g["ego"][[pos[int(i)] for i in split["ids"]]]


def oracle_agents(g, rho, eta, grav):
    return [ra.RotAgent(sp, eta_k=eta, rho_rot_mat=rho, enable_gravity_prior=grav, ego_poses=ego_of(g, sp))
            for sp in (pgo.arock_split(g, s) for s in range(int(g["agent"].max()) + 1))]


def qdist(a, b):
    a = np.asarray(a).reshape(-1, 4); b = np.asarray(b).reshape(-1, 4)
    return np.minimum(np.abs(a - b).max(1), np.abs(a + b).max(1))


def sv_ratio(M):
    """sigma_2 / sigma_1 per 3x3 (0 for the zero matrix)"""
    s = np.linalg.svd(np.asarray(M).reshape(-1, 3, 3), compute_uv=False)
    return np.where(s[:, 0] > 0, s[:, 1] / np.where(s[:, 0] > 0, s[:, 0], 1.0), 0.0)


def owner_ratio(states, splits):
    """per split, sigma_2 / sigma_1 of each frame's M as its owner solved it (0 where the owner has none): a frame's attitude
    anywhere is its owner's projection of that M"""
    own = {}
    for (M, *_), sp in zip(states, splits):
        for i, f in enumerate(sp["ids"]):
            if int(sp["owner"][i]) == int(sp["self_id"]):
                own[int(f)] = M[i]
    return [sv_ratio([own.get(int(f), np.zeros((3, 3))) for f in sp["ids"]]) for sp in splits]


# ---------------------------------------------------------------------------------------------------------------- the pin
# The reference's own RotationInitARock rounds on seeded cases, frozen in tests/golden/ref_rotinit_arock.npz (made by
# tests/golden/make_ref_rotinit_arock_golden.py).  Cases: 3 and 4 agents; gravity rows on and off; rho_rot_mat 0.1 / 0.16 and
# eta_k 0.9 / 0.1; a loop from a free frame into the fixed frame, a loop from it, a self loop (graph()); third-party duals (every
# message reaches every agent); without gravity rows the non-main agents' first M is zero.
from oracle import ref_rotinit_arock  # noqa: E402

LIVE = pytest.mark.skipif(not ref_rotinit_arock.available(), reason="reference RotationInitARock library not built")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_rotinit_arock.npz")
PIN_ROUNDS = 6
PIN_CASES = {   # name: (seed, agents, rho_rot_mat, eta_k, gravity rows)
    "three_multi_launch": (31, 3, 0.16, 0.9, False),
    "three_gravity_slow": (32, 3, 0.1, 0.1, True),
    "four_gravity": (33, 4, 0.16, 0.9, True),
    "four_default_slow": (34, 4, 0.1, 0.1, False),
}
SPLIT_FIELDS = ("self_id", "ids", "poses", "fixed", "owner", "id_a", "id_b", "rel", "sqrt_info", "ego")


def pin_case(name):
    """(splits with their ego poses, rho, eta, gravity) of a pin case"""
    seed, A, rho, eta, grav = PIN_CASES[name]
    g = graph(seed, n_agents=A, n=10, loops=24)
    splits = []
    for s in range(A):
        sp = pgo.arock_split(g, s)
        splits.append({k: np.asarray(ego_of(g, sp) if k == "ego" else sp[k]) for k in SPLIT_FIELDS})
    return splits, rho, eta, grav


def reference_outputs(name, splits, rho, eta, grav):
    out = {}
    for r, R in enumerate(ref_rotinit_arock.run(splits, [s["ego"] for s in splits], PIN_ROUNDS, rho, eta, grav)):
        out[f"ref_{name}__r{r}_chg"] = R["state_changes"]
        for a in range(len(splits)):
            out[f"ref_{name}__r{r}_a{a}_state"] = R["state"][a]; out[f"ref_{name}__r{r}_a{a}_poses"] = R["poses"][a]
            out[f"ref_{name}__r{r}_a{a}_keys"] = np.array(R["keys"][a], np.int64).reshape(-1, 2)
            out[f"ref_{name}__r{r}_a{a}_yl"] = R["yl"][a]; out[f"ref_{name}__r{r}_a{a}_yr"] = R["yr"][a]
    return out


def golden():
    """{name: (splits, rho, eta, grav)}, {key: array} of the frozen file"""
    z = np.load(GOLDEN)
    cases = {}
    for name in PIN_CASES:
        rho, eta, grav = z[f"case_{name}__params"]
        A = int(z[f"case_{name}__agents"])
        splits = [{k: z[f"case_{name}__a{a}_{k}"] for k in SPLIT_FIELDS} for a in range(A)]
        cases[name] = (splits, float(rho), float(eta), bool(grav))
    return cases, {k: z[k] for k in z.files if k.startswith("ref_")}


def check_against_reference(name, splits, rho, eta, grav, refs, agents=None, step=None, tol=1e-10, tol_chg=1e-12):
    """Every round of the agents (the oracle's by default; `step(agents)` runs one round) against the reference's outputs:
    M (every frame's R_state) and both duals within tol, the dual keys exactly, state_changes within tol_chg (or the same
    non-finite value), positions bit-identical, attitudes within tol / (sigma_2 / sigma_1) of the owner's M where that ratio is
    above 1e-8 (the projection of a nearly rank-1 M is decided by its last digits; the shim's SVD stand-in differs from
    Eigen's on rank-deficient input).  Returns the worst differences."""
    A = len(splits)
    if agents is None:
        agents = [ra.RotAgent(dict(sp), eta_k=eta, rho_rot_mat=rho, enable_gravity_prior=grav, ego_poses=sp["ego"]) for sp in splits]
        step = lambda ags: ra.run(ags, 1)[0]
    worst = dict(M=0.0, dual=0.0, chg=0.0, att=0.0)
    for r in range(PIN_ROUNDS):
        reps = step(agents)
        st = [agent_state(a) for a in agents]
        ratios = owner_ratio(st, splits)
        chg = np.array([q["state_changes"] for q in reps])
        rc = refs[f"ref_{name}__r{r}_chg"]
        fin = np.isfinite(rc)
        assert np.array_equal(rc[~fin], chg[~fin], equal_nan=True) and np.array_equal(fin, np.isfinite(chg)), (r, rc, chg)
        worst["chg"] = max(worst["chg"], float(np.abs(rc[fin] - chg[fin]).max(initial=0.0)))
        for a, ((M, x, keys, yl, yr), sp) in enumerate(zip(st, splits)):
            k = f"ref_{name}__r{r}_a{a}_"
            assert [tuple(q) for q in refs[k + "keys"].tolist()] == keys, (r, a)
            worst["M"] = max(worst["M"], float(np.abs(refs[k + "state"] - M).max()))
            if len(keys):
                worst["dual"] = max(worst["dual"], float(np.abs(refs[k + "yl"] - yl).max()), float(np.abs(refs[k + "yr"] - yr).max()))
            assert np.array_equal(refs[k + "poses"][:, :3], x[:, :3]), (r, a)
            ratio = ratios[a]
            sel = ratio > 1e-8
            d = qdist(refs[k + "poses"][sel, 3:7], x[sel, 3:7])
            assert np.all(d <= tol / ratio[sel]), (r, a, d.max(initial=0.0))
            worst["att"] = max(worst["att"], float((d * ratio[sel]).max(initial=0.0)))
    assert worst["M"] <= tol and worst["dual"] <= tol and worst["chg"] <= tol_chg, worst
    return worst


def agent_state(a):
    """(R_state [n, 3, 3], poses [n, 7], dual keys, y_l [K, 9], y_r [K, 9]) of an oracle or device agent"""
    if isinstance(a, ra.RotAgent):
        keys, yl, yr = a.table()
        return a.M(), a.x.copy(), keys, yl, yr
    st = a.s.debug_arock_rot_state()
    return st["state"], a.poses(), [(int(n), int(f)) for n, f in zip(st["neighbour"], st["frame"])], st["yl"], st["yr"]


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_matches_the_frozen_reference_outputs():
    cases, refs = golden()
    assert set(cases) == set(PIN_CASES)
    for name, (splits, rho, eta, grav) in cases.items():
        print(name, check_against_reference(name, splits, rho, eta, grav, refs))


@LIVE
def test_oracle_matches_the_reference_live():
    for name in PIN_CASES:
        splits, rho, eta, grav = pin_case(name)
        check_against_reference(name, splits, rho, eta, grav, reference_outputs(name, splits, rho, eta, grav))


def test_golden_inputs_are_the_seeded_cases():
    cases, _ = golden()
    for name, (splits, rho, eta, grav) in cases.items():
        fresh, *params = pin_case(name)
        assert params == [rho, eta, grav]
        for a, b in zip(fresh, splits):
            assert all(np.array_equal(a[k], b[k]) for k in SPLIT_FIELDS), name


def test_pin_cases_cover_the_issue_cases():
    """zero first M on the non-main agents without gravity rows, third-party duals (a dual (n, f) with f owned by neither n nor
    the agent), the fixed frame's loops and a self loop"""
    cases, refs = golden()
    third = set()
    for name, (splits, rho, eta, grav) in cases.items():
        if not grav:
            for a in range(1, len(splits)):
                M = refs[f"ref_{name}__r0_a{a}_state"]
                own = splits[a]["owner"] == splits[a]["self_id"]
                assert not M[own].any()
        for a, sp in enumerate(splits):
            keys = [tuple(k) for k in refs[f"ref_{name}__r{PIN_ROUNDS - 1}_a{a}_keys"].tolist()]
            owner = dict(zip(sp["ids"].tolist(), sp["owner"].tolist()))
            if any(owner[f] != n and owner[f] != sp["self_id"] for n, f in keys):
                third.add(name)
        s0 = splits[0]
        head = int(s0["ids"][s0["fixed"].astype(bool)][0])
        assert head in s0["id_b"].tolist() and head in s0["id_a"].tolist()
        assert any(a == b for a, b in zip(s0["id_a"], s0["id_b"]))
    assert len(third) >= 2, third


def test_non_main_agents_start_from_zero_and_take_identity():
    """Without gravity rows a non-main agent's first system has b = 0: M = 0 exactly, its own frames get the identity attitude
    (JacobiSVD of 0), the remote frames keep theirs, and the next state change is not finite (R_state = 0: |M| / 0, or 0 / 0 where
    M stays 0 because no information has reached the agent yet), as in the reference."""
    g = graph(1)
    ags = oracle_agents(g, 0.16, 0.9, False)
    x0 = [a.x.copy() for a in ags]
    reps = ra.run(ags, 2)
    assert reps[0][0]["state_changes"] > 0 and np.isfinite(reps[0][0]["state_changes"])
    assert not np.isfinite(reps[1][1]["state_changes"]) and not np.isfinite(reps[1][2]["state_changes"])
    for a, x in zip(ags[1:], x0[1:]):
        a2 = ra.RotAgent(a.split, eta_k=0.9, rho_rot_mat=0.16)
        a2.rot_init_step()
        assert not a2.M()[[a2.pos[f] for f in a2.named if not a2.fixed[a2.pos[f]]]].any()
        own = a2.owner == a2.self_id
        assert np.array_equal(a2.x[own, 3:7], np.tile([0.0, 0.0, 0.0, 1.0], (int(own.sum()), 1)))
        assert np.array_equal(a2.x[~own], x[~own])
    # with gravity rows the first system is not homogeneous
    b = oracle_agents(g, 0.16, 0.9, True)[1]
    b.rot_init_step()
    assert np.abs(b.M()).max() > 0.5


def test_receipt_and_processing_rules():
    """inputDPGOData overwrites the sender's own frames (position and attitude) at once and nothing else; processPGOData creates
    a dual (y_l = y_r = value) when missing, else sets y_r only when the message targets this agent; frames no edge names are
    ignored."""
    g = graph(2)
    a = oracle_agents(g, 0.1, 0.9, False)[1]
    a.rot_init_step()
    other = int(min(o for o in a.owner if o != a.self_id))
    fr = [int(f) for f, o in zip(a.ids, a.owner) if o == other][:2]
    mine = int(a.ids[a.owner == a.self_id][0])
    pose = np.array([[1.0, 2.0, 3.0, 0.0, 0.0, 0.6, 0.8]] * 3)
    before = a.x.copy()
    a.rot_receive((other, 99, np.array(fr + [mine]), np.arange(27.0).reshape(3, 9), pose))
    for f in fr:
        assert np.array_equal(a.x[a.pos[f]], pose[0])
    assert np.array_equal(a.x[a.pos[mine]], before[a.pos[mine]])           # not the sender's frame
    key = (other, fr[0])
    yl, yr = a.duals[key][0].copy(), a.duals[key][1].copy()
    a._process()
    assert np.array_equal(a.duals[key][0], yl) and np.array_equal(a.duals[key][1], yr)   # third-party message, dual existed
    assert np.array_equal(a.duals[(other, mine)][0], np.arange(18.0, 27.0))              # missing: created from the value
    assert np.array_equal(a.duals[(other, mine)][1], np.arange(18.0, 27.0))
    a.rot_receive((other, a.self_id, np.array([fr[0], 123456789]), np.ones((2, 9)), pose[:2]))
    a._process()
    assert np.array_equal(a.duals[key][0], yl) and np.array_equal(a.duals[key][1], np.ones(9))
    assert all(k[1] != 123456789 for k in a.duals)


def test_new_duals_from_a_message_take_the_value_on_both_sides():
    g = graph(2)
    a = oracle_agents(g, 0.1, 0.9, False)[1]
    mine = int(a.ids[a.owner == a.self_id][0])
    a.rot_receive((7, 3, np.array([mine]), np.arange(9.0)[None], np.array([[0, 0, 0, 0, 0, 0, 1.0]])))
    a._process()
    assert np.array_equal(a.duals[(7, mine)][0], np.arange(9.0)) and np.array_equal(a.duals[(7, mine)][1], np.arange(9.0))


def test_fixed_frame_dual_uses_its_entry_rotation():
    """A dual on the fixed frame gets no prior, and its update reads R(attitude at entry), not a solved M."""
    g = graph(3)
    ags = oracle_agents(g, 0.16, 0.9, False)
    ra.run(ags, 3)
    a0 = ags[0]
    head = int(a0.ids[a0.fixed][0])
    keys = [k for k in a0.duals if k[1] == head]
    assert keys                                           # other agents send duals on agent 0's head frame
    assert np.array_equal(a0.rstate[head], quat_R(np.asarray(g["gt"])[0, 3:7]))
    yl, yr = a0.duals[keys[0]][0].copy(), a0.duals[keys[0]][1].copy()
    a0.inbox = []
    a0.rot_init_step()
    want = yl - ((yl + yr) / 2 - a0.rstate[head].ravel()) * 0.9
    assert np.array_equal(a0.duals[keys[0]][0], want)


def test_oracle_solution_is_a_stationary_point_with_dual_priors():
    """The step's M solves the normal equations of the edges, fixed-frame rows, dual priors w = sqrt(3 rho) and gravity rows."""
    g = graph(4)
    ags = oracle_agents(g, 0.16, 0.9, True)
    ra.run(ags, 3)
    for a in ags:
        A, b, H, x = a.last["A"], a.last["b"], a.last["H"], a.last["x"]
        assert np.abs(H @ x - A.T @ b).max() <= 1e-10 * abs(H).max() * max(1.0, np.abs(x).max())
        n_dual = sum(1 for (_, f) in a.duals if f in a.last["col"])
        tail = A[A.shape[0] - 9 * n_dual:]                     # the dual priors: one entry w = sqrt(3 rho) per row
        assert n_dual > 0 and tail.nnz == 9 * n_dual and np.all(tail.data == np.sqrt(3 * 0.16))


def test_oracle_refuses_an_unanchored_component():
    g = graph(5)
    sp = pgo.arock_split(g, 1)
    # two extra frames of agent 1 joined to each other only: no fixed-frame row and no dual prior
    sp = dict(sp, ids=np.concatenate([sp["ids"], [1_900_000, 1_900_001]]), poses=np.concatenate([sp["poses"], sp["poses"][:2]]),
              fixed=np.concatenate([sp["fixed"], [0, 0]]).astype(np.uint8), owner=np.concatenate([sp["owner"], [1, 1]]).astype(np.int32),
              id_a=np.concatenate([sp["id_a"], [1_900_000]]), id_b=np.concatenate([sp["id_b"], [1_900_001]]),
              rel=np.concatenate([sp["rel"], sp["rel"][:1]]), sqrt_info=np.concatenate([sp["sqrt_info"], sp["sqrt_info"][:1]]))
    with pytest.raises(ValueError, match="1900000"):
        ra.RotAgent(sp).rot_init_step()


class _Scripted:
    """an agent whose step reports the given state changes, counting its steps and the messages it receives"""

    def __init__(self, self_id, changes):
        self.self_id, self.changes, self.steps, self.got = self_id, list(changes), 0, 0

    def rot_init_step(self, **cfg):
        self.steps += 1
        return dict(state_changes=self.changes[self.steps - 1])

    def rot_messages(self):
        return [(self.self_id, 1 - self.self_id, np.zeros(0, np.int64), np.zeros((0, 9)), np.zeros((0, 7)))]

    def rot_receive(self, msg):
        self.got += 1


def test_convergence_gate_of_the_run():
    """rotInitial converges once state_changes < eps after more than min_rounds earlier solves (d2pgo.cpp:351-353); a
    converged agent stops stepping and keeps receiving; None where it never converges."""
    a = _Scripted(0, [1e-3] * 30)                       # below eps from the start: held back by the round count
    b = _Scripted(1, [0.5] * 13 + [5e-3] * 17)          # falls below eps at round 14
    assert pgo.arock_rot_init_run([a, b], 30) == [12, 14]
    assert a.steps == 12 and b.steps == 14 and a.got == 14 and b.got == 12
    c, d = _Scripted(0, [0.5] * 30), _Scripted(1, [1e-3] * 30)
    assert pgo.arock_rot_init_run([c, d], 20, eps=1e-2, min_rounds=3) == [None, 5]
    assert c.steps == 20
    assert pgo.rot_init_converged(0.0099, 12) and not pgo.rot_init_converged(0.0099, 11) and not pgo.rot_init_converged(0.01, 40)


def test_oracle_agents_run_to_convergence_with_gravity_rows():
    g = graph(6)
    rounds = pgo.arock_rot_init_run(oracle_agents(g, 0.16, 0.9, True), 40)
    assert all(r is not None and 12 <= r <= 40 for r in rounds), rounds


def test_new_kernels_do_not_spill():
    from d2slam_b200 import build
    build.build()
    log = open(os.path.join(ROOT, "d2slam_b200", "build", "ptxas.log")).read()
    blocks = re.findall(r"Compiling entry function '(\w*k_rotinit_arock\w*)'.*?\n(.*?)\n(.*?)\n", log)
    assert len(blocks) == 3
    for name, _, props in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props, (name, props)


def test_existing_kernels_compile_to_the_same_sass():
    """Every kernel of d2pgo.cu as it was before this feature compiles to the same instructions now.  Needs the git history and
    the CUDA toolkit; skipped without them."""
    import shutil
    import subprocess
    import tempfile
    from d2slam_b200 import build
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (shutil.which("git") and shutil.which("cuobjdump") and os.path.exists(nvcc)):
        pytest.skip("git, nvcc or cuobjdump unavailable")
    obj_new = os.path.join(ROOT, "d2slam_b200", "build", "d2pgo.o")
    build.build(force=not os.path.exists(obj_new))
    with tempfile.TemporaryDirectory() as td:
        files = ["d2pgo.cu", "d2pgo_handle.cuh", "d2pgo_chol.cuh", "d2ba_math.cuh"]
        for f in files + ["../../include/d2pgo.h"]:
            src = os.path.normpath(os.path.join("d2slam_b200/csrc", f))
            r = subprocess.run(["git", "-C", ROOT, "show", f"{PARENT}:{src}"], capture_output=True)
            if r.returncode:
                pytest.skip(f"commit {PARENT} not in this checkout")
            dst = os.path.normpath(os.path.join(td, "x", "csrc", f))
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            open(dst, "wb").write(r.stdout)
        flags = [f for f in build.NVCC_FLAGS if f not in ("-Xptxas", "-v")]
        obj = os.path.join(td, "parent.o")
        subprocess.check_call([nvcc] + flags + ["-c", os.path.join(td, "x", "csrc", "d2pgo.cu"), "-o", obj])
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        import sass_diff
        old, new = sass_diff.kernels(obj), sass_diff.kernels(obj_new)
    assert len(old) == 45
    assert [k for k in old if new.get(k) != old[k]] == []
    assert sorted(k for k in new if k not in old) == sorted(k for k in new if "k_rotinit_arock" in k) and len(new) == 48


# ---------------------------------------------------------------------------------------------------------------- GPU
def device_agents(g, rho, eta, grav):
    return [pgo.ArockAgent(sp, ego_poses=ego_of(g, sp), eta_k=eta) for sp in (pgo.arock_split(g, s) for s in range(int(g["agent"].max()) + 1))]


def dev_cfg(rho, grav):
    return dict(rho_rot_mat=rho, enable_gravity_prior=int(grav), pcg_tolerance=TOL)


def dev_run(ags, rounds, rho, grav):
    """all agents step every round (no convergence gate), then the synchronous delivery; returns the reports"""
    out = []
    for r in range(rounds):
        reps = [a.rot_init_step(**dev_cfg(rho, grav)) for a in ags]
        msgs = [m for a in ags for m in a.rot_messages()]
        for a in ags:
            for m in msgs:
                if m[0] != a.self_id:
                    a.rot_receive(m)
        out.append(reps)
    return out


def snapshot(a):
    st = a.s.debug_arock_rot_state()
    return dict(poses=a.poses(), **st)


def oracle_from_device(dev, rho, eta, grav, g, msgs, stepped):
    """An oracle agent in the device agent's state (poses, R_state once the device has stepped, rotation duals) with the same
    messages queued."""
    st = snapshot(dev)
    o = ra.RotAgent(dev.split, eta_k=eta, rho_rot_mat=rho, enable_gravity_prior=grav, ego_poses=ego_of(g, dev.split))
    o.x = st["poses"].copy()
    o.rstate = {int(f): st["state"][i].copy() for i, f in enumerate(o.ids) if st["flag"][i] and stepped}
    o.duals = {(int(n), int(f)): [yl.copy(), yr.copy()] for n, f, yl, yr in zip(st["neighbour"], st["frame"], st["yl"], st["yr"])}
    o.inbox = [(m[0], m[1], np.asarray(m[2]), np.asarray(m[3]).reshape(-1, 9)) for m in msgs if m[0] != dev.self_id]
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("params", list(PARAMS))
def test_one_step_from_a_common_state(params):
    """From the device's state after r rounds (r = 0, 1, 4), the device's next step and the oracle's sparse-direct step agree:
    M, duals and state_changes within 100 kappa pcg_tolerance, kappa the condition number of the oracle's normal matrix."""
    rho, eta, grav = PARAMS[params]
    g = graph(11)
    ags = device_agents(g, rho, eta, grav)
    worst = 0.0
    try:
        msgs = []
        for r in range(6):
            if r in (0, 1, 4):
                orcs = [oracle_from_device(a, rho, eta, grav, g, msgs, r > 0) for a in ags]
                for a, o in zip(ags, orcs):
                    rd = a.rot_init_step(**dev_cfg(rho, grav)); ro_ = o.rot_init_step()
                    st = snapshot(a)
                    bound = 100 * ra.kappa(o) * TOL
                    dM = np.abs(st["state"] - o.M()).max()
                    _, yl, yr = o.table()
                    dY = np.abs(st["yl"] - yl).max() if len(yl) else 0.0
                    assert np.array_equal(st["yr"], yr)
                    assert dM <= bound and dY <= bound, (r, a.self_id, dM, dY, bound)
                    if np.isfinite(ro_["state_changes"]):
                        assert abs(rd["state_changes"] - ro_["state_changes"]) <= bound, (rd["state_changes"], ro_["state_changes"])
                    else:
                        assert np.array_equal(rd["state_changes"], ro_["state_changes"], equal_nan=True)
                    worst = max(worst, dM / bound, dY / bound)
            else:
                for a in ags:
                    a.rot_init_step(**dev_cfg(rho, grav))
            msgs = [m for a in ags for m in a.rot_messages()]
            for a in ags:
                for m in msgs:
                    if m[0] != a.self_id:
                        a.rot_receive(m)
        print(f"{params}: worst difference / (100 kappa tol) = {worst:.3g}")
    finally:
        for a in ags:
            a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("params", list(PARAMS))
def test_ten_free_running_rounds_follow_the_oracle(params):
    """3 agents x 40 frames, ten rounds each on the device and in the oracle from the same start: M, duals and the attitudes
    where the owner's M is not degenerate (sigma_2 > 1e-8 sigma_1) within 1e-6, positions and fixed poses bit-identical, the zero-M agents on identity in round 1."""
    rho, eta, grav = PARAMS[params]
    g = graph(12)
    dev = device_agents(g, rho, eta, grav)
    orc = oracle_agents(g, rho, eta, grav)
    worst = dict(M=0.0, dual=0.0, att=0.0)
    try:
        for r in range(10):
            dr = [a.rot_init_step(**dev_cfg(rho, grav)) for a in dev]
            orr = [a.rot_init_step() for a in orc]
            ratios = owner_ratio([agent_state(o) for o in orc], [o.split for o in orc])
            for a, o, x, y, ratio in zip(dev, orc, dr, orr, ratios):
                st = snapshot(a)
                worst["M"] = max(worst["M"], float(np.abs(st["state"] - o.M()).max()))
                _, yl, _ = o.table()
                if len(yl):
                    worst["dual"] = max(worst["dual"], float(np.abs(st["yl"] - yl).max()))
                nd = ratio > 1e-8
                worst["att"] = max(worst["att"], float(qdist(st["poses"][nd, 3:7], o.x[nd, 3:7]).max(initial=0.0)))
                assert np.array_equal(st["poses"][:, :3], o.x[:, :3])
                assert np.array_equal(st["poses"][o.fixed], o.x[o.fixed])
                if r == 0 and not grav and a.self_id != 0:
                    own = o.owner == o.self_id
                    assert not st["state"][st["flag"] == 1].any()
                    assert np.array_equal(st["poses"][own, 3:7], np.tile([0.0, 0.0, 0.0, 1.0], (int(own.sum()), 1)))
                if np.isfinite(y["state_changes"]):
                    assert abs(x["state_changes"] - y["state_changes"]) <= 1e-6
                else:
                    assert np.array_equal(x["state_changes"], y["state_changes"], equal_nan=True)
            dm = [m for a in dev for m in a.rot_messages()]; om = [m for a in orc for m in a.rot_messages()]
            for ags, ms in ((dev, dm), (orc, om)):
                for a in ags:
                    for m in ms:
                        if m[0] != a.self_id:
                            a.rot_receive(m)
        print(f"{params}: worst over 10 rounds: M {worst['M']:.3g}, y_l {worst['dual']:.3g}, attitude {worst['att']:.3g}")
        assert max(worst.values()) <= 1e-6, worst
    finally:
        for a in dev:
            a.close()


@pytest.mark.gpu
def test_device_matches_the_frozen_reference_outputs():
    """The device agents, free-running on the pin cases, against the reference's rounds: M, duals and state_changes within
    1e-6, positions bit-identical, attitudes within 1e-6 / (sigma_2 / sigma_1) of the owner's M."""
    cases, refs = golden()
    for name, (splits, rho, eta, grav) in cases.items():
        ags = [pgo.ArockAgent(dict(sp), ego_poses=sp["ego"], eta_k=eta) for sp in splits]
        try:
            w = check_against_reference(name, splits, rho, eta, grav, refs, ags, lambda xs: dev_run(xs, 1, rho, grav)[0], tol=1e-6, tol_chg=1e-6)
            print(name, {k: f"{v:.3g}" for k, v in w.items()})
        finally:
            for a in ags:
                a.close()


@pytest.mark.gpu
def test_device_receive_rules():
    g = graph(13)
    ags = device_agents(g, 0.1, 0.9, False)
    try:
        a = ags[1]
        a.rot_init_step()
        ids, owner = a.split["ids"], a.split["owner"]
        other = int(min(o for o in owner if o != a.self_id))
        fr = [int(f) for f, o in zip(ids, owner) if o == other][:2]
        mine = int(ids[owner == a.self_id][0])
        frames = fr + [mine, 987654321]
        pose = np.array([[1.0, 2.0, 3.0, 0.0, 0.0, 0.6, 0.8]] * len(frames))
        duals = np.arange(9.0 * len(frames)).reshape(-1, 9)
        before = a.poses()
        pos = {int(f): i for i, f in enumerate(ids)}
        st0 = a.s.debug_arock_rot_state()
        a.s.arock_rot_receive(other, 0, np.array(frames), duals, pose)
        after = a.poses()
        for f in fr:                                                     # the sender's frames: overwritten at receipt
            assert np.array_equal(after[pos[f]], pose[0])
        assert np.array_equal(after[pos[mine]], before[pos[mine]])
        st1 = a.s.debug_arock_rot_state()
        assert np.array_equal(st0["yl"], st1["yl"]) and np.array_equal(st0["yr"], st1["yr"])   # duals wait for the step
        a.rot_init_step()
        st2 = a.s.debug_arock_rot_state()
        tab = {(int(n), int(f)): (yl, yr) for n, f, yl, yr in zip(st2["neighbour"], st2["frame"], st2["yl"], st2["yr"])}
        assert not any(f == 987654321 for _, f in tab)                  # unknown frame ignored
        assert np.array_equal(tab[(other, mine)][1], duals[len(fr)])    # created from the message (then y_l updated)
        old = {(int(n), int(f)): yr for n, f, yr in zip(st1["neighbour"], st1["frame"], st1["yr"])}
        assert np.array_equal(tab[(other, fr[0])][1], old[(other, fr[0])])      # existed, target is not self: unchanged
        a.s.arock_rot_receive(other, a.self_id, np.array([fr[0]]), np.ones((1, 9)), pose[:1])
        a.rot_init_step()
        st3 = a.s.debug_arock_rot_state()
        tab3 = {(int(n), int(f)): yr for n, f, yr in zip(st3["neighbour"], st3["frame"], st3["yr"])}
        assert np.array_equal(tab3[(other, fr[0])], np.ones(9))         # targeted at self: y_r set
    finally:
        for a in ags:
            a.close()


@pytest.mark.gpu
def test_first_arock_step_starts_at_the_rot_init_attitudes():
    """Rot-init steps set q_init with the attitudes they write, so the perturbation duals the first d2pgo_arock_step creates
    are [p ; theta = 0] at those attitudes."""
    g = graph(14)
    ags = device_agents(g, 0.16, 0.9, True)
    try:
        dev_run(ags, 4, 0.16, True)
        poses = [a.poses() for a in ags]
        for a in ags:
            a.step()
        for a, p in zip(ags, poses):
            pos = {int(f): i for i, f in enumerate(a.split["ids"])}
            d = a.duals()
            assert d
            for (n, f), (yl, yr) in d.items():
                assert np.abs(yr[3:]).max() <= 1e-14, (f, yr)
                assert np.array_equal(yr[:3], p[pos[f], :3])
    finally:
        for a in ags:
            a.close()


@pytest.mark.gpu
def test_refusals_keep_nothing():
    g = graph(15)
    ags = device_agents(g, 0.16, 0.9, True)
    try:
        dev_run(ags, 2, 0.16, True)
        a = ags[1]

        def state():
            st = a.s.debug_arock_rot_state()
            return [a.poses(), st["state"], st["yl"], st["yr"], st["frame"], a.duals()]

        def same(x, y):
            assert all(np.array_equal(u, v) for u, v in zip(x[:5], y[:5])) and x[5].keys() == y[5].keys()

        s0 = state()
        f0 = int(a.split["ids"][a.split["owner"] != 1][0])
        with pytest.raises(RuntimeError, match="rc=2"):
            a.s.arock_rot_receive(2, 1, [f0], np.zeros((1, 6)), [[0, 0, 0, 0, 0, 0, 1.0]], dim=6)
        with pytest.raises(RuntimeError, match="rc=2"):
            a.s.arock_rot_receive(2, 1, [f0], np.full((1, 9), np.nan), [[0, 0, 0, 0, 0, 0, 1.0]])
        with pytest.raises(RuntimeError, match="rc=2"):
            a.s.arock_rot_receive(2, 1, [f0], np.zeros((1, 9)), [[5.0, 0, 0, 0, 0, 0, 0]])
        with pytest.raises(RuntimeError, match="rc=2"):
            a.s.arock_rot_receive(1, 1, [f0], np.zeros((1, 9)), [[0, 0, 0, 0, 0, 0, 1.0]])
        with pytest.raises(RuntimeError, match="rc=2"):                                 # gravity rows, no ego poses
            a.s.arock_rot_init_step(None, None, enable_gravity_prior=1)
        same(s0, state())
        # an unanchored component: two extra frames of agent 1 joined only to each other
        sp = a.split
        b = pgo.PgoSolver()
        ids = np.concatenate([sp["ids"], [1_900_000, 1_900_001]])
        b.set_poses(ids, np.concatenate([sp["poses"], sp["poses"][:2]]), np.concatenate([sp["fixed"], [0, 0]]))
        b.add_edges(np.concatenate([sp["id_a"], [1_900_000]]), np.concatenate([sp["id_b"], [1_900_001]]),
                    np.concatenate([sp["rel"], sp["rel"][:1]]), np.concatenate([sp["sqrt_info"], sp["sqrt_info"][:1]]))
        b.arock_enable(ids, np.concatenate([sp["owner"], [1, 1]]), self_id=1)
        p0 = b.get_poses(ids)
        with pytest.raises(RuntimeError, match="rc=2.*1900000"):
            b.arock_rot_init_step()
        assert np.array_equal(b.get_poses(ids), p0) and len(b.debug_arock_rot_state()["frame"]) == 0
        b.close()
        # a 4-DoF handle, a handle not in ARock mode, d2pgo_rot_init on an ARock handle
        c = pgo.PgoSolver(pose_dof=4)
        with pytest.raises(RuntimeError, match="rc=5"):
            c.arock_rot_init_step()
        c.close()
        d = pgo.PgoSolver()
        d.set_poses(sp["ids"], sp["poses"], sp["fixed"]); d.add_edges(sp["id_a"], sp["id_b"], sp["rel"], sp["sqrt_info"])
        with pytest.raises(RuntimeError, match="rc=5"):
            d.arock_rot_init_step()
        d.close()
        with pytest.raises(RuntimeError, match="rc=5"):
            a.s.rot_init()
        same(s0, state())
        # once the pose dual table is non-empty
        a.step()
        s1 = state()
        with pytest.raises(RuntimeError, match="rc=5"):
            a.rot_init_step(**dev_cfg(0.16, True))
        with pytest.raises(RuntimeError, match="rc=5"):
            a.s.arock_rot_receive(2, 1, [f0], np.zeros((1, 9)), [[0, 0, 0, 0, 0, 0, 1.0]])
        same(s1, state())
    finally:
        for x in ags:
            x.close()


@pytest.mark.gpu
def test_two_runs_are_bitwise_equal():
    g = graph(16)
    outs = []
    for _ in range(2):
        ags = device_agents(g, 0.16, 0.9, True)
        reps = dev_run(ags, 5, 0.16, True)
        outs.append([(snapshot(a), [r[i]["state_changes"] for r in reps]) for i, a in enumerate(ags)])
        for a in ags:
            a.close()
    for (s, c), (t, d) in zip(*outs):
        assert np.array_equal(c, d, equal_nan=True)
        for k in s:
            assert np.array_equal(s[k], t[k]), k
