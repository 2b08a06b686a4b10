"""Writes tests/golden/ref_pcm_stream.npz: the reference's own SwarmLocalOutlierRejection kept across calls (good mask and smd
of every call) on the batchings of tests/test_pgo_pcm_stream.py, and FMC::maxCliqueHeuIncremental's return value on seeded
graphs, through oracle/_ref/libd2ref_pcm_stream.so.  Needs the reference tree.  `python tests/golden/make_ref_pcm_stream_golden.py`"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from d2slam_b200 import pgo  # noqa: E402
from oracle import ref_pcm_stream as ref  # noqa: E402
import test_pgo_pcm as t  # noqa: E402
import test_pgo_pcm_stream as ts  # noqa: E402


def arrays():
    out = {}
    case = t.small_case()
    for b, calls in ts.batchings(case).items():
        out[f"{b}_frames"] = np.concatenate([f for f, _ in calls]); out[f"{b}_n_frames"] = np.array([len(f) for f, _ in calls], np.int32)
        out[f"{b}_loops"] = np.concatenate([l for _, l in calls]); out[f"{b}_n_loops"] = np.array([len(l) for _, l in calls], np.int32)
        for name, (is4, thr, pc, yc) in t.PCM_CONFIGS.items():
            s = ref.PcmStream(is4, thr, pc, yc)
            goods, smds, n_smd = [], [], []
            for f, l in ts.cumulative(calls):
                good, smd = s.call(*pgo.pcm_stream_args(case, f, l))
                goods.append(good); smds.append(smd); n_smd.append(len(smd))
            out[f"{b}_{name}_good"] = np.concatenate(goods)
            out[f"{b}_{name}_smd"] = np.concatenate(smds); out[f"{b}_{name}_n_smd"] = np.array(n_smd, np.int64)
    graphs, new, prev = ts.fmc_inc_graphs()
    out["inc_n"] = np.array([len(a) for a in graphs], np.int32)
    out["inc_adj"] = np.concatenate([a.ravel() for a in graphs])
    out["inc_new"] = np.array(new, np.int32); out["inc_prev"] = np.array(prev, np.int32)
    out["inc_ret"] = np.array([ref.fmc_heu_inc(a, k, p) for a, k, p in zip(graphs, new, prev)], np.int32)
    return out


def main():
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "ref_pcm_stream.npz"), **arrays())


if __name__ == "__main__":
    main()
