"""Writes tests/golden/ref_rotinit.npz: the reference's own RotationInitialization<double>::solve outputs (rotation states,
new attitudes, pose states, state_changes, dropped loops) through oracle/_ref/libd2ref_rotinit.so, on the seeded cases of
tests/test_pgo_rotinit.py.  Needs the reference tree.  `python tests/golden/make_ref_rotinit_golden.py`"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_pgo_rotinit as t  # noqa: E402


def arrays():
    cases = t.reference_cases()
    out = {f"case_{name}__{f}": np.asarray(c[f]) for name, c in cases.items() for f in t.FIELDS}
    out.update(t.reference_outputs(cases))
    return out


def main():
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "ref_rotinit.npz"), **arrays())


if __name__ == "__main__":
    main()
