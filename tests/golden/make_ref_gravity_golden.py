"""Writes tests/golden/ref_gravity.npz: the reference's own GravityPriorPerturbAD and RelPoseFactorPerturbAD outputs (doubles for
the residuals, dual numbers for the Jacobians), through oracle/_ref/libd2ref_gravity.so, on the cases of
tests/test_pgo_gravity.py.  Needs the reference tree.  `python tests/golden/make_ref_gravity_golden.py`"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_pgo_gravity as t  # noqa: E402


def arrays():
    cases = t.reference_cases()
    out = {f"case_{k}": v for k, v in cases.items()}
    out.update(t.reference_outputs(cases))
    return out


def main():
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "ref_gravity.npz"), **arrays())


if __name__ == "__main__":
    main()
