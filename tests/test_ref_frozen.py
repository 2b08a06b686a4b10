"""Every reference pin library still computes its frozen golden file, bit for bit.

All five libraries of oracle/Makefile.ref are built against the one stand-in tree oracle/_shim, so an edit made there for one
pin can change what another computes.  This test reruns each tests/golden/make_ref_*_golden.py generator through the live
library and compares every array with the committed tests/golden/ref_*.npz: same keys, dtype, shape and bytes.  The one
exception is the reference Marginalizer's output in ref_factors.npz (marg*_refs / _x0 / _J / _e0): it orders the kept blocks
by heap address, which differs from run to run, so those arrays are checked with test_ref_pin's permutation-invariant
check_marginalization instead.  A pin whose library is neither built nor buildable here is skipped.
"""
import importlib
import os
import re
import sys

import numpy as np
import pytest

from oracle import ref, ref_arock, ref_gravity, ref_pcm, ref_rotinit

import test_ref_pin as trp

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
sys.path.insert(0, GOLDEN)

# golden file -> (its generator in tests/golden, the front-end of the library it comes from)
PINS = {
    "ref_factors": ("make_ref_golden", ref),
    "ref_cases": ("make_ref_cases_golden", ref),
    "ref_pcm": ("make_ref_pcm_golden", ref_pcm),
    "ref_gravity": ("make_ref_gravity_golden", ref_gravity),
    "ref_arock": ("make_ref_arock_golden", ref_arock),
    "ref_rotinit": ("make_ref_rotinit_golden", ref_rotinit),
}
MARG = re.compile(r"marg(\d+)_(refs|x0|J|e0)")


@pytest.mark.parametrize("name", sorted(PINS))
def test_reference_pin_reproduces_its_golden_file(name):
    generator, pin = PINS[name]
    if not pin.available():
        pytest.skip(f"{os.path.basename(pin.so_path())} not built and no reference tree to build it")
    live = {k: np.asarray(v) for k, v in importlib.import_module(generator).arrays().items()}
    with np.load(os.path.join(GOLDEN, name + ".npz")) as g:
        frozen = {k: g[k] for k in g.files}
    assert sorted(live) == sorted(frozen)
    marg = [k for k in live if name == "ref_factors" and MARG.fullmatch(k)]
    differ = [k for k in live if k not in marg and not (live[k].dtype == frozen[k].dtype and live[k].shape == frozen[k].shape
                                                        and live[k].tobytes() == frozen[k].tobytes())]
    assert not differ, differ
    for i in sorted({int(MARG.fullmatch(k).group(1)) for k in marg}):
        trp.check_marginalization(trp.MARG_CASES[i], *(live[f"marg{i}_{f}"] for f in ("refs", "x0", "J", "e0")))
