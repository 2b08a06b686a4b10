"""SASS evidence per hot kernel: instruction histogram (fp64 tensor MMA, TMA bulk copies, LDGSTS, reductions) + the
first lines of the fp64-MMA inner loop, from the in-tree libd2ba.so.   python tools/sass_excerpts.py r02"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
so = os.path.join(ROOT, "d2slam_b200", "libd2ba.so")
KERNELS = ["k_proj_lin_pp", "k_lm_gather16", "k_schur_small", "k_schur", "k_chol_smem", "k_sb_elim", "k_leaf_elim", "k_leaf_back", "k_imu_lin", "k_step"]
sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
funcs = re.split(r"\n\s*Function : ", sass)
out = [f"# cuobjdump -sass {os.path.relpath(so, ROOT)} (sm_90a), per-kernel instruction histogram of the mnemonics that matter\n",
       "# DMMA = fp64 tensor-core mma.sync m8n8k4; UBLKCP = cp.async.bulk (TMA bulk copy); SYNCS = mbarrier; LDGSTS = cp.async;\n",
       "# RED/ATOMG = L2 reductions; DFMA/DADD/DMUL = fp64 pipe.  wgmma (HGMMA) has no f64 kind: none expected.\n\n"]
for fn in funcs[1:]:
    name = fn.split("\n", 1)[0].strip()
    short = next((k for k in KERNELS if re.search(rf"\d+{k}(E|I)", name)), None)
    if not short:
        continue
    ops = collections.Counter()
    lines = [l for l in fn.split("\n") if re.search(r"/\*[0-9a-f]{4}\*/", l)]
    for l in lines:
        m = re.search(r"\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", l)
        if m:
            ops[m.group(1).split(".")[0]] += 1
    keys = ["DMMA", "UBLKCP", "SYNCS", "LDGSTS", "RED", "ATOMG", "ATOMS", "DFMA", "DADD", "DMUL", "MUFU", "SHFL", "LDS", "STS", "LDG", "STG", "BAR", "HMMA", "UTCHMMA", "UTCQMMA"]
    out.append(f"{name}\n  instructions {len(lines)}: " + ", ".join(f"{k} {ops[k]}" for k in keys if ops[k]) + "\n")
    first = next((i for i, l in enumerate(lines) if "DMMA" in l), None)
    if first is not None:
        out.append("  first fp64 tensor MMA and its neighbourhood:\n")
        for l in lines[max(0, first - 4): first + 8]:
            out.append("    " + re.sub(r"\s+/\* 0x[0-9a-f]+ \*/\s*$", "", l.strip()) + "\n")
    out.append("\n")
path = os.path.join(ROOT, "profiles", f"{tag}_sass_excerpts.txt")
open(path, "w").writelines(out)
print("wrote", path, len(out))
