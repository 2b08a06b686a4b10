"""Writes tests/golden/ref_arock.npz: per case of tests/test_pgo_arock.py (PIN_CASES), the agents' sub-graphs, the oracle's
local solutions of every round, and what the reference's own ARock loop (oracle/_ref/libd2ref_arock.so) makes of them: every
agent's dual table after every round and the proximal factors it created.  Needs the reference tree.
`python tests/golden/make_ref_arock_golden.py`"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_pgo_arock as t  # noqa: E402
from oracle import ref_arock  # noqa: E402


def main():
    ref_arock.build()
    out = {}
    for name in t.PIN_CASES:
        c = t.pin_case(name)
        dof = t.PIN_CASES[name][0]
        splits, cfg = c["splits"], c["cfg"]
        init, sol, _ = t.to_ref_inputs(splits, c["solved"], dof)
        ref = ref_arock.run([sp["self_id"] for sp in splits], [sp["ids"] for sp in splits], [sp["owner"] for sp in splits], init, sol,
                            cfg["rho_frame_T"], cfg["rho_frame_theta"], cfg["eta_k"], cfg["dual_state_init_to_zero"])
        out.update({f"{name}/dof": dof, f"{name}/agents": len(splits), f"{name}/rounds": len(c["solved"]), f"{name}/rho_T": cfg["rho_frame_T"],
                    f"{name}/rho_theta": cfg["rho_frame_theta"], f"{name}/eta": cfg["eta_k"], f"{name}/init_zero": int(cfg["dual_state_init_to_zero"])})
        for a, sp in enumerate(splits):
            for k in ("ids", "poses", "fixed", "owner", "id_a", "id_b", "rel", "sqrt_info", "self_id"):
                out[f"{name}/a{a}/{k}"] = np.asarray(sp[k])
        for r, row in enumerate(ref):
            for a, g in enumerate(row):
                out[f"{name}/r{r}/a{a}/solved"] = np.asarray(c["solved"][r][a])
                out[f"{name}/r{r}/a{a}/keys"] = np.array(g["keys"], np.int64).reshape(-1, 2)
                for k in ("yl", "yr", "fac"):
                    out[f"{name}/r{r}/a{a}/{k}"] = g[k]
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "ref_arock.npz"), **out)


if __name__ == "__main__":
    main()
