"""Python binding of libd2ba.so through its C ABI (include/d2ba.h).

This is plumbing only: every numeric step of the solve runs in the CUDA library.  The import
fails loudly when the library is missing; ``Solver()`` fails when no CUDA device is present
(d2ba_create returns an error -- there is no CPU fallback).
"""
import ctypes as C
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib_path():
    # D2BA_LIB: developer override (instrumented builds); the product always loads the in-tree library
    return os.environ.get("D2BA_LIB") or os.path.join(_HERE, "libd2ba.so")


def lib():
    global _LIB
    if _LIB is None:
        p = lib_path()
        if not os.path.exists(p):
            raise RuntimeError(f"{p} not built: run `python -m d2slam_b200.build` (nvcc, sm_90a). No CPU fallback exists.")
        # torch bundles the NCCL the library dlopens lazily; make it discoverable without importing torch
        if "D2BA_NCCL_LIB" not in os.environ:
            try:
                import importlib.util
                spec = importlib.util.find_spec("nvidia.nccl")
                if spec and spec.submodule_search_locations:
                    cand = os.path.join(list(spec.submodule_search_locations)[0], "lib", "libnccl.so.2")
                    if os.path.exists(cand):
                        os.environ["D2BA_NCCL_LIB"] = cand
            except Exception:
                pass
        _LIB = C.CDLL(p)
        _LIB.d2ba_last_error.restype = C.c_char_p
        _LIB.d2ba_last_error.argtypes = [C.c_void_p]
        _LIB.d2ba_create.argtypes = [C.POINTER(abi.Config), C.POINTER(C.c_void_p)]
    return _LIB


EXPORTED = [
    "d2ba_default_config", "d2ba_create", "d2ba_destroy", "d2ba_reset", "d2ba_last_error", "d2ba_set_blocks",
    "d2ba_add_proj", "d2ba_add_landmark_tracks", "d2ba_add_imu", "d2ba_set_prior", "d2ba_set_prior_info",
    "d2ba_set_consensus", "d2ba_comm_unique_id", "d2ba_comm_init", "d2ba_consensus_buffer", "d2ba_finalize",
    "d2ba_solve", "d2ba_solve_fixed", "d2ba_get_blocks", "d2ba_num_windows", "d2ba_marginalize",
    "d2ba_debug_linearize", "d2ba_debug_get", "d2ba_debug_kernel_times", "d2ba_debug_host_times",
]


class D2BAError(RuntimeError):
    pass


class Solver:
    """A handle holding up to ``max_windows`` windows (reference: one SolverWrapper per D2Estimator;
    several windows = throughput batch or several agents on one GPU)."""

    def __init__(self, cfg=None, **kw):
        self.cfg = cfg if cfg is not None else abi.default_config(**kw)
        self.h = C.c_void_p()
        rc = lib().d2ba_create(C.byref(self.cfg), C.byref(self.h))
        if rc != 0:
            raise D2BAError(f"d2ba_create failed rc={rc} (CUDA device required; no CPU fallback)")

    def _chk(self, rc, what):
        if rc != 0:
            msg = lib().d2ba_last_error(self.h)
            raise D2BAError(f"{what} failed rc={rc}: {msg.decode() if msg else ''}")

    def close(self):
        if self.h:
            lib().d2ba_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        self._chk(lib().d2ba_reset(self.h), "reset")

    def set_blocks(self, window, kind, ids, values, is_const=None):
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        values = np.ascontiguousarray(values, dtype=np.float64)
        c = None if is_const is None else np.ascontiguousarray(is_const, dtype=np.uint8)
        self._chk(lib().d2ba_set_blocks(self.h, C.c_int32(window), C.c_int32(kind), C.c_int32(len(ids)), abi.ptr(ids),
                                        abi.ptr(values), abi.ptr(c)), "set_blocks")

    def add_proj(self, window, obs):
        obs = np.ascontiguousarray(obs, dtype=abi.proj_obs_dtype)
        self._chk(lib().d2ba_add_proj(self.h, C.c_int32(window), C.c_int32(len(obs)), abi.ptr(obs)), "add_proj")

    def add_landmark_tracks(self, window, landmark_ids, track_ptr, tobs, fuse_dep=0, min_d=0.3, max_d=5.0, ignore_frames=()):
        landmark_ids = np.ascontiguousarray(landmark_ids, dtype=np.int64)
        track_ptr = np.ascontiguousarray(track_ptr, dtype=np.int32)
        tobs = np.ascontiguousarray(tobs, dtype=abi.track_obs_dtype)
        ign = np.ascontiguousarray(ignore_frames, dtype=np.int64)
        self._chk(lib().d2ba_add_landmark_tracks(self.h, C.c_int32(window), C.c_int32(len(landmark_ids)), abi.ptr(landmark_ids),
                                                 abi.ptr(track_ptr), abi.ptr(tobs), C.c_int32(fuse_dep), C.c_double(min_d),
                                                 C.c_double(max_d), C.c_int32(len(ign)), abi.ptr(ign) if len(ign) else None),
                  "add_landmark_tracks")

    def add_imu(self, window, imu):
        imu = np.ascontiguousarray(imu, dtype=abi.imu_dtype)
        self._chk(lib().d2ba_add_imu(self.h, C.c_int32(window), C.c_int32(len(imu)), abi.ptr(imu)), "add_imu")

    def set_prior(self, window, J, e0, refs, x0):
        J = np.ascontiguousarray(J, dtype=np.float64); e0 = np.ascontiguousarray(e0, dtype=np.float64)
        refs = np.ascontiguousarray(refs, dtype=abi.blockref_dtype); x0 = np.ascontiguousarray(x0, dtype=np.float64)
        self._chk(lib().d2ba_set_prior(self.h, C.c_int32(window), C.c_int32(len(e0)), abi.ptr(J), abi.ptr(e0), C.c_int32(len(refs)),
                                       abi.ptr(refs), abi.ptr(x0)), "set_prior")

    def set_prior_info(self, window, A, b, refs, x0):
        A = np.ascontiguousarray(A, dtype=np.float64); b = np.ascontiguousarray(b, dtype=np.float64)
        refs = np.ascontiguousarray(refs, dtype=abi.blockref_dtype); x0 = np.ascontiguousarray(x0, dtype=np.float64)
        self._chk(lib().d2ba_set_prior_info(self.h, C.c_int32(window), C.c_int32(len(b)), abi.ptr(A), abi.ptr(b), C.c_int32(len(refs)),
                                            abi.ptr(refs), abi.ptr(x0)), "set_prior_info")

    def set_consensus(self, window, refs, slots, n_slots_global):
        refs = np.ascontiguousarray(refs, dtype=abi.blockref_dtype)
        slots = np.ascontiguousarray(slots, dtype=np.int32)
        self._chk(lib().d2ba_set_consensus(self.h, C.c_int32(window), C.c_int32(len(refs)), abi.ptr(refs), abi.ptr(slots),
                                           C.c_int32(n_slots_global)), "set_consensus")

    def comm_init(self, unique_id, rank, nranks):
        uid = (C.c_uint8 * 128)(*unique_id)
        self._chk(lib().d2ba_comm_init(self.h, uid, C.c_int32(rank), C.c_int32(nranks)), "comm_init")

    def finalize(self):
        self._chk(lib().d2ba_finalize(self.h), "finalize")

    def num_windows(self):
        return lib().d2ba_num_windows(self.h)

    def solve(self, n_windows=None):
        n = n_windows or max(self.num_windows(), self.cfg.max_windows)
        reps = (abi.Report * n)()
        self._chk(lib().d2ba_solve(self.h, reps), "solve")
        return list(reps)[: self.num_windows()]

    def solve_fixed(self, iters):
        n = max(self.num_windows(), self.cfg.max_windows)
        reps = (abi.Report * n)()
        self._chk(lib().d2ba_solve_fixed(self.h, C.c_int32(iters), reps), "solve_fixed")
        return list(reps)[: self.num_windows()]

    def get_blocks(self, window, kind, ids):
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        out = np.zeros((len(ids), abi.KIND_SIZE[kind]), dtype=np.float64)
        self._chk(lib().d2ba_get_blocks(self.h, C.c_int32(window), C.c_int32(kind), C.c_int32(len(ids)), abi.ptr(ids), abi.ptr(out)),
                  "get_blocks")
        return out

    def marginalize(self, window, remove_frame_ids, max_m=1024, max_blk=256):
        """-> (A [m,m], b [m], refs, x0) of the new prior (information form)."""
        rem = np.ascontiguousarray(remove_frame_ids, dtype=np.int64)
        A = np.zeros((max_m, max_m)); b = np.zeros(max_m); refs = np.zeros(max_blk, dtype=abi.blockref_dtype); x0 = np.zeros(max_blk * 9)
        m = C.c_int32(); nb = C.c_int32()
        Aflat = np.zeros(max_m * max_m)
        self._chk(lib().d2ba_marginalize(self.h, C.c_int32(window), C.c_int32(len(rem)), abi.ptr(rem), C.byref(m), C.c_int32(max_m), abi.ptr(Aflat),
                                         abi.ptr(b), C.byref(nb), C.c_int32(max_blk), abi.ptr(refs), abi.ptr(x0)), "marginalize")
        mm = m.value
        refs = refs[: nb.value].copy()
        nx = int(sum(abi.KIND_SIZE[int(k)] for k in refs["kind"]))
        return Aflat[: mm * mm].reshape(mm, mm).copy(), b[:mm].copy(), refs, x0[:nx].copy()

    def kernel_times(self, iters):
        out = np.zeros(12)
        self._chk(lib().d2ba_debug_kernel_times(self.h, C.c_int32(iters), abi.ptr(out)), "kernel_times")
        kt = {k: out[i] / max(out[7], 1) for i, k in enumerate(KERNEL_NAMES)}
        # the speed-bias elimination is timed inside the gather bucket, its back substitution inside the chol bucket
        se, sbk = out[8] / max(out[7], 1), out[9] / max(out[7], 1)
        le, lb = out[10] / max(out[7], 1), out[11] / max(out[7], 1)
        kt["lm_gather"] -= se; kt["chol"] -= sbk + lb; kt["sb_elim"] = se; kt["sb_back"] = sbk
        if le > 0 or lb > 0:
            kt["schur"] -= le; kt["leaf_elim"] = le; kt["leaf_back"] = lb
        self.chol_split = {"sb_elim": se, "sb_back": sbk}
        return kt

    def host_times(self):
        """Wall-clock ms of the phases of the last finalize()."""
        out = np.zeros(16)
        self._chk(lib().d2ba_debug_host_times(self.h, abi.ptr(out)), "host_times")
        d = dict(zip(("plan", "prefix", "fill", "enqueue", "wait", "mirror"), out[:6].round(3).tolist()))
        d.update(zip(("dev_upload", "dev_prep"), out[6:8].round(3).tolist()))
        d.update(zip(("solve_enqueue", "solve_wait", "solve_writeback"), out[12:15].round(3).tolist()))
        d["h2d_bytes"] = int(out[15])
        d.update(zip(("add_lookup", "add_stamps", "add_copy", "add_cuda"), out[8:12].round(3).tolist()))
        return d

    def debug_linearize(self):
        self._chk(lib().d2ba_debug_linearize(self.h), "debug_linearize")

    def debug_get(self, window, item, dtype=np.float64):
        need = C.c_int64()
        self._chk(lib().d2ba_debug_get(self.h, C.c_int32(window), C.c_int32(item), None, C.c_int64(0), C.byref(need)), "debug_get")
        out = np.zeros(need.value // np.dtype(dtype).itemsize + 1, dtype=dtype)
        self._chk(lib().d2ba_debug_get(self.h, C.c_int32(window), C.c_int32(item), abi.ptr(out), C.c_int64(out.nbytes), C.byref(need)),
                  "debug_get")
        return out[: need.value // np.dtype(dtype).itemsize]


KERNEL_NAMES = ["lm_gather", "schur", "chol", "step", "misc_lin", "proj_lin", "control"]


def comm_unique_id():
    uid = (C.c_uint8 * 128)()
    rc = lib().d2ba_comm_unique_id(uid)
    if rc != 0:
        raise D2BAError(f"d2ba_comm_unique_id failed rc={rc}")
    return bytes(uid)


class _WindowView:
    """Adapter so that synth.Problem.load(solver_view) can target one window of a Solver."""

    def __init__(self, solver, window):
        self.s, self.w = solver, window

    def __getattr__(self, name):
        f = getattr(self.s, name)
        return lambda *a, **k: f(self.w, *a, **k)
