"""Writes tests/golden/ref_pcm.npz: the reference's own PCM (SwarmLocalOutlierRejection::OutlierRejectionLoopEdges) and FMC
(maxCliqueHeu) outputs, through oracle/_ref/libd2ref_pcm.so, on the cases of tests/test_pgo_pcm.py.  Needs the reference tree.
`python tests/golden/make_ref_pcm_golden.py`"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_pcm as ref  # noqa: E402
import test_pgo_pcm as t  # noqa: E402


def main():
    out = {}
    case = t.small_case()
    for k, v in case.items():
        if isinstance(v, np.ndarray):
            out[f"case_{k}"] = v
    for name, (is4, thr, pc, yc) in t.PCM_CONFIGS.items():
        good, smd = ref.pcm(case, is4, thr, pc, yc, rel_key="rel_bad")
        out[f"{name}_good"] = good
        out[f"{name}_smd"] = t.ref_order_to_group_major(case, smd)
    graphs = t.fmc_graphs()
    out["fmc_n"] = np.array([len(a) for a in graphs], np.int32)
    out["fmc_adj"] = np.concatenate([a.ravel() for a in graphs])
    cl = [sorted(ref.fmc_heu(a)) for a in graphs]
    out["fmc_size"] = np.array([len(c) for c in cl], np.int32)
    out["fmc_clique"] = np.array(sum(cl, []), np.int32)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "ref_pcm.npz"), **out)


if __name__ == "__main__":
    main()
