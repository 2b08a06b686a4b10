"""Writes tests/golden/ref_rotinit_arock.npz: the reference's own RotationInitARock<double> rounds (rotation states, pose states,
state_changes and dual tables after every round) through oracle/_ref/libd2ref_rotinit_arock.so, on the seeded cases of
tests/test_pgo_rotinit_arock.py, with those cases' inputs.  Needs the reference tree.
`python tests/golden/make_ref_rotinit_arock_golden.py`"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_pgo_rotinit_arock as t  # noqa: E402


def arrays():
    out = {}
    for name in t.PIN_CASES:
        splits, rho, eta, grav = t.pin_case(name)
        out[f"case_{name}__params"] = np.array([rho, eta, 1.0 if grav else 0.0])
        out[f"case_{name}__agents"] = np.int64(len(splits))
        for a, sp in enumerate(splits):
            out.update({f"case_{name}__a{a}_{k}": np.asarray(sp[k]) for k in t.SPLIT_FIELDS})
        out.update(t.reference_outputs(name, splits, rho, eta, grav))
    return out


def main():
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "ref_rotinit_arock.npz"), **arrays())


if __name__ == "__main__":
    main()
