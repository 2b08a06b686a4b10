"""Compare the SASS of every kernel of one object (or library) with the same kernel in another:
`python tools/sass_diff.py OLD NEW` lists the kernels of OLD that NEW lacks or compiles to different instructions, and exits
non-zero if there is any.  Kernel names are compared with the anonymous namespace's per-file name and its length taken out
(the name changes whenever the source file does, and it names the file, so a kernel moved to another file keeps its name).
Build OLD from the earlier source with the flags of d2slam_b200/build.py, e.g.
`nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr -c d2pgo.cu`."""
import re
import subprocess
import sys

_ANON = re.compile(r"\d+_GLOBAL__N__[0-9a-f]+_\d+_[A-Za-z0-9_]+?_[0-9a-f]{8}")


def kernels(path):
    """{kernel name: [instruction lines]} of cuobjdump -sass (addresses, encodings and the anonymous-namespace hash dropped)."""
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    out, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = _ANON.sub("_GLOBAL__N_", m.group(1)); out[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if name and m:
            out[name].append(_ANON.sub("_GLOBAL__N_", m.group(1)))
    return out


def main(old, new):
    a, b = kernels(old), kernels(new)
    bad = [k for k in a if k not in b or a[k] != b[k]]
    for k in bad:
        print(("missing   " if k not in b else "different ") + k)
    print(f"{len(a) - len(bad)} of {len(a)} kernels of {old} identical in {new}; {len(set(b) - set(a))} new kernels")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1], sys.argv[2]))
