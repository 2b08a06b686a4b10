"""CPU: the C-ABI library loads, exports every symbol include/d2ba.h declares, and struct layouts agree
between C and the ctypes/numpy mirrors.  No compute is called (no GPU here)."""
import ctypes as C
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions(header="d2ba.h", prefix="d2ba_"):
    src = open(os.path.join(ROOT, "include", header)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(" + prefix + r"[a-z_0-9]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from d2slam_b200 import build, solver
    build.build()
    lib = solver.lib()
    names = declared_functions()
    assert len(names) >= 20
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    assert set(solver.EXPORTED) <= set(names)
    from d2slam_b200 import pgo
    pnames = declared_functions("d2pgo.h", "d2pgo_")
    assert sorted(pnames) == sorted(pgo.PGO_EXPORTED) and not [n for n in pnames if not hasattr(lib, n)]


def test_pgo_refuses_without_a_device():
    import torch
    from d2slam_b200 import pgo
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        pgo.PgoSolver()


def test_struct_layouts_match_c():
    from d2slam_b200 import abi
    code = r'''
#include <stdio.h>
#include <stddef.h>
#include "d2ba.h"
int main(void){
 printf("%zu %zu %zu %zu %zu %zu\n", sizeof(d2ba_config), sizeof(d2ba_proj_obs), sizeof(d2ba_track_obs), sizeof(d2ba_imu), sizeof(d2ba_blockref), sizeof(d2ba_report));
 printf("%zu %zu %zu %zu\n", offsetof(d2ba_proj_obs, pts_i), offsetof(d2ba_proj_obs, depth), offsetof(d2ba_imu, jacobian), offsetof(d2ba_config, focal_length));
 return 0; }
'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(code)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = subprocess.check_output([exe]).decode().split()
    sizes = list(map(int, out))
    assert sizes[0] == C.sizeof(abi.Config)
    assert sizes[1] == abi.proj_obs_dtype.itemsize
    assert sizes[2] == abi.track_obs_dtype.itemsize
    assert sizes[3] == abi.imu_dtype.itemsize
    assert sizes[4] == abi.blockref_dtype.itemsize
    assert sizes[5] == C.sizeof(abi.Report)
    assert sizes[6] == abi.proj_obs_dtype.fields["pts_i"][1]
    assert sizes[7] == abi.proj_obs_dtype.fields["depth"][1]
    assert sizes[8] == abi.imu_dtype.fields["jacobian"][1]
    assert sizes[9] == abi.Config.focal_length.offset


def test_no_cpu_fallback():
    """Without a CUDA device the product refuses to construct a solver (and nothing under d2slam_b200/
    references the oracle)."""
    import torch
    from d2slam_b200 import solver
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(solver.D2BAError):
        solver.Solver()
    pkg = os.path.join(ROOT, "d2slam_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", ".hpp")):
                txt = open(os.path.join(dp, f), errors="ignore").read()
                assert "orc_" not in txt and "from oracle" not in txt and "import oracle" not in txt, os.path.join(dp, f)


def test_sass_has_fp64_tensor_mma():
    """The built library must contain fp64 tensor-core MMAs (DMMA) for the J^T J accumulation / Schur SYRK."""
    from d2slam_b200 import build
    so = build.build()
    try:
        sass = subprocess.check_output(["cuobjdump", "-sass", so], stderr=subprocess.DEVNULL).decode()
    except (OSError, subprocess.CalledProcessError):
        pytest.skip("cuobjdump unavailable")
    assert "DMMA" in sass
    assert "arch = sm_90a" in sass


def test_pgo_struct_layouts_match_c():
    from d2slam_b200 import pgo
    code = '#include <stdio.h>\n#include <stddef.h>\n#include "d2pgo.h"\nint main(void){printf("%zu %zu %zu %zu\\n", sizeof(d2pgo_config), sizeof(d2pgo_report), offsetof(d2pgo_config, lambda0), offsetof(d2pgo_report, device_ms));return 0;}\n'
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(code)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = list(map(int, subprocess.check_output([exe]).decode().split()))
    assert out == [C.sizeof(pgo.PgoConfig), C.sizeof(pgo.PgoReport), pgo.PgoConfig.lambda0.offset, pgo.PgoReport.device_ms.offset]
