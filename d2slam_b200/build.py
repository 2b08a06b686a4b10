"""Builds libd2ba.so (sm_90a) in-tree with nvcc.  `python -m d2slam_b200.build`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.environ.get("D2BA_OUT") or os.path.join(HERE, "libd2ba.so")
SOURCES = ["d2ba_kernels.cu", "d2ba_host.cu", "d2ba_margin.cu", "d2pgo.cu"]
EXTRA_DEPS = ["d2ba_harness.cpp"]
HEADERS = ["d2ba_types.cuh", "d2ba_math.cuh", "d2ba_proj.cuh", os.path.join("..", "..", "include", "d2ba.h"), os.path.join("..", "..", "include", "d2pgo.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS + EXTRA_DEPS] + [os.path.abspath(__file__)]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    objdir = "build_side" if os.environ.get("D2BA_OUT") else "build"
    os.makedirs(os.path.join(HERE, objdir), exist_ok=True)
    for s in SOURCES:
        o = os.path.join(HERE, objdir, s.replace(".cu", ".o"))
        objs.append(o)
        cmd = [nvcc] + NVCC_FLAGS + os.environ.get("D2BA_NVCC_EXTRA", "").split() + ["-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for s, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {s}\n{out}")
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {s}")
    link = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", OUT] + objs + ["-lcudart", "-ldl"]
    subprocess.check_call(link)
    # host-side harness (C++ stand-in for the D2Estimator call sequence), links against libd2ba.so
    harness = os.path.join(HERE, "libd2ba_harness.so")
    if os.environ.get("D2BA_OUT"):
        return OUT   # instrumented side build: library only
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", os.path.join(CSRC, "d2ba_harness.cpp"), "-o", harness,
                           "-L" + HERE, "-ld2ba", "-Wl,-rpath,$ORIGIN"])
    with open(os.path.join(HERE, "build", "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
