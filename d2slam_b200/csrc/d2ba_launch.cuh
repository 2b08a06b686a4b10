// d2ba_launch.cuh -- the interface between the host side (d2ba_host.cu) and the kernels (d2ba_kernels.cu,
// d2ba_margin.cu): what d2ba_finalize derives for the launches, the shared-memory sizes its planner decides with, and the
// host-callable launchers.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <algorithm>

#include "d2ba_types.cuh"

namespace d2ba {

// What d2ba_finalize derives for the handle as a whole: array totals, the maxima the kernels are sized and configured for,
// and which kernels the iteration launches.  Value-initialised by every finalize.
struct LaunchSummary {
  int n_used = 0, n6_total = 0, nsb_total = 0, nl_total = 0, n_tiles = 0, n_imu_total = 0, n_slots = 0;   // windows, blocks, ...
  int n_grp = 0, n_lmptr = 0, n_pblk = 0, n_leaf_total = 0, n_hseg = 0, n_leaf_lm = 0, n_chunks = 0, n_g12 = 0;
  int n_schur = 0, n_schur0 = 0;                     // Schur tiles; the first n_schur0 are stage 0 (leaf columns)
  int n_jobs = 0, job_begin[8] = {}, job_count[8] = {};   // reprojection jobs per launch_proj_lin variant
  int tpj_target = 1;                                // observation tiles per reprojection job (D2BA_DBG_LIN_JOBS)
  int64_t totH = 0, totW = 0, totc = 0, totLE = 0, totLL = 0, tot_rec = 0, tot_pJ = 0, tot_pv = 0;   // doubles
  int max_nc = 1, max_prior_m = 0, max_row_tiles = 1, max_ldw_small = 0;
  int max_n_smem = 0, max_rows_glob = 1; bool any_chol_glob = false;   // dense Cholesky: shared-memory / global kernel
  int any_compact = 0, any_wide = 0;                 // record widths present (which gather kernels to launch)
  bool any_admm = false, any_info = false;           // consensus terms / a prior given in information form
  // dynamic shared memory of k_leaf_elim, k_leaf_back, k_sb_elim and k_sb_back (0 = no window uses the kernel)
  size_t leaf_smem = 0, leafb_smem = 0, sbe_smem = 0, sbb_smem = 0;
  // one-kernel reduced-system solve (k_solve_small) of the windows with WinDesc::fused_solve; the separate kernels are
  // launched only when some window still needs them
  int n_fused = 0; size_t fused_smem = 0;
  bool ss_unfused = false, cs_unfused = false, sbb_unfused = false;
};

// ------------------------------------------------------------------------------------------------ per-window limits
// Shared memory of the eliminations and dense factorisations: d2ba_finalize picks each window's solve path by these
// functions, and the kernels lay out their shared memory by them.
// k_chol_smem: the bordered matrix with an even leading dimension, 1/d, and the panel / fail-flag scratch
constexpr int kCsThreads = 512;
constexpr int kCsNB = 8;
__host__ __device__ inline int chol_smem_ld(int n) { return (n + 1) & ~1; }
__host__ __device__ inline size_t chol_smem_bytes(int n) {
  size_t pr = (size_t)kCsNB * ((n + 2) & ~1), need = (size_t)n + 1 + 16 * 32;
  return ((size_t)(n + 1) * chol_smem_ld(n) + (size_t)((n + 1) & ~1) + (pr > need ? pr : need)) * 8 + 32;   // invd padded to even: P stays 16 B aligned
}
// small systems (after the speed-bias elimination): 4 warps per window so that several windows share an SM
inline int chol_smem_threads(int max_n) { return max_n <= 96 ? 128 : kCsThreads; }
// k_sb_elim / k_sb_back
constexpr int kSeMaxBlocks = 32;   // speed-bias blocks per window (mbarrier table)
constexpr int kSeSlotRows = 9;
__host__ __device__ inline size_t sbe_smem_bytes(int ldw, int n_c, int nb) {
  return ((size_t)3 * kSeSlotRows * ldw + (size_t)nb * 2 * 81 + (size_t)nb * 9 + (size_t)n_c + (size_t)9 * nb + 16) * 8;
}
__host__ __device__ inline size_t sb_back_smem_bytes(int nlc, int nb) { return (size_t)(((nlc + 31) & ~31) + 9 * nb + 171 * nb) * 8; }
// k_leaf_elim / k_leaf_back
constexpr int kLeafMaxCols = 96;
constexpr int kLeafLmChunk = 16;   // landmarks whose coupling rows are staged at a time (a multiple of the MMA k = 4)
__host__ __device__ inline int leaf_lda(int n) { return n | 1; }   // odd: the one-row-per-thread TRSM walks the rows without bank conflicts (all accesses are scalar)
__host__ __device__ inline size_t leaf_elim_smem_bytes(int n, int nh) {
  const int n1 = n + nh + 1;
  return ((size_t)n1 * leaf_lda(n) + (size_t)((n + 1) & ~1) + (size_t)kCsNB * ((n1 + 1) & ~1) + 64 + (size_t)kLeafLmChunk * n1 + 8) * 8;
}
__host__ __device__ inline size_t leaf_back_smem_bytes(int n, int nh) { return ((size_t)n * n + 2 * (size_t)n + (size_t)nh + 8) * 8; }
// k_solve_small: the phases share one region, sized for the largest
constexpr int kSolveThreads = 128;
constexpr int kSolveMaxB = 12;   // 9*10/2 = 45 lower blocks (ldw <= 72) over 4 warps
__host__ __device__ inline size_t solve_small_smem_bytes(int ldw, int n_lc, int n_c, int nb) {
  size_t b = (size_t)2 * 32 * (ldw + 4) * 8;
  b = std::max(b, chol_smem_bytes(n_lc));
  b = std::max(b, sb_back_smem_bytes(n_lc, nb));
  return std::max(b, (size_t)(40 + 3 * n_c) * 8);
}
// the 8x8 blocks of the lower triangle fit the accumulators of k_solve_small's warps
inline bool solve_small_fits(int ldw) { const int nb8 = ldw / 8; return nb8 * (nb8 + 1) / 2 <= kSolveMaxB * (kSolveThreads / 32); }

// ------------------------------------------------------------------------------------------------ launchers
// d2ba_kernels.cu.  A launcher given the summary launches its kernel only when some window of the handle needs it.
// Raises every kernel's dynamic shared-memory limit to what the summary's launches ask for (once per d2ba_finalize, not
// in the launchers: those also run under stream capture).  Returns nullptr, or the message of the refused request.
const char *configure_launches(const LaunchSummary &L);
// finalize: tiles, state, IMU and prior preparation
void launch_build_tiles(const LaunchSummary &L, const long long *raw_off, const int *tile_src, const int *tile_win, const double *xtd,
                        double *obs, cudaStream_t s);
void launch_state_prep(const Dev &d, const LaunchSummary &L, cudaStream_t s);
void launch_imu_prep(const Dev &d, const LaunchSummary &L, const double *packed, double *full, cudaStream_t s);
void launch_prior_prep(const Dev &d, cudaStream_t s);
// the iteration
void launch_misc_lin(const Dev &d, const LaunchSummary &L, int eval_cur, cudaStream_t s);
void launch_imu_lin(const Dev &d, const LaunchSummary &L, int eval_cur, cudaStream_t s);
void launch_proj_lin(const Dev &d, const LaunchSummary &L, int eval_cur, cudaStream_t s);   // all eight variants, in order
void launch_lm_gather(const Dev &d, const LaunchSummary &L, const int *lm_win, cudaStream_t s);
void launch_sb_elim(const Dev &d, const LaunchSummary &L, cudaStream_t s);
void launch_zero_sb_rows(const Dev &d, const LaunchSummary &L, cudaStream_t s);
void launch_leaf_elim(const Dev &d, const LaunchSummary &L, cudaStream_t s);
void launch_zero_leaf_rows(const Dev &d, const LaunchSummary &L, cudaStream_t s);
// with_fused = 0: the windows the separate kernels solve; 1: every window k_schur_small serves (the full Schur complement)
void launch_schur_small(const Dev &d, const LaunchSummary &L, int with_fused, cudaStream_t s);
void launch_schur(const Dev &d, const SchurTile *tiles, int n_tiles, cudaStream_t s);
void launch_chol_smem(const Dev &d, const LaunchSummary &L, cudaStream_t s);
void launch_chol(const Dev &d, const LaunchSummary &L, cudaStream_t s);
void launch_sb_back(const Dev &d, const LaunchSummary &L, cudaStream_t s);
void launch_leaf_back(const Dev &d, const LaunchSummary &L, cudaStream_t s);
// phase_ts: nullptr, or 5 timestamps per window (d2ba_debug_solve_phases: the timestamped instantiation)
void launch_solve_small(const Dev &d, const LaunchSummary &L, unsigned long long *phase_ts, cudaStream_t s);
int solve_small_occupancy(size_t smem);   // CTAs per SM, -1 if the query fails
void launch_step(const Dev &d, const LaunchSummary &L, cudaStream_t s);
void launch_control(const Dev &d, int init, cudaStream_t s);
void launch_tr_reset(const Dev &d, int first, cudaStream_t s);
// ADMM consensus (only a handle with consensus windows runs them)
void launch_cons_init(const Dev &d, const LaunchSummary &L, cudaStream_t s);
void launch_cons_pack(const Dev &d, const LaunchSummary &L, const int *blk_win, cudaStream_t s);
void launch_cons_apply(const Dev &d, const LaunchSummary &L, const int *blk_win, cudaStream_t s);
void launch_cons_refs(const Dev &d, const LaunchSummary &L, const int *sb_win, const int *lm_win, cudaStream_t s);
// debug views
void launch_proj_debug(const Dev &d, const LaunchSummary &L, double *out, const int *tile_win, cudaStream_t s);
void launch_imu_debug(const Dev &d, double *out, const int *imu_win, int n, cudaStream_t s);
void launch_cons_debug(const Dev &d, const LaunchSummary &L, double *out, const int *blk_win, cudaStream_t s);
// marginalization: S (landmarks eliminated) -> the kept columns' A, b.  Returns non-zero when the shared memory is refused.
int launch_marg_reduce(const double *S, int ld, int n, const int *keep_idx, int nk, const int *rem_idx, int nr, double *A, double *b, int *fail_flag,
                       cudaStream_t s);
// d2ba_margin.cu: priors given in information form -> Jacobian form (L.any_info)
void launch_prior_from_info(const LaunchSummary &L, const int *m_of, const long long *offJ, const long long *offv, const int *is_info,
                            double *A, double *V, double *b, cudaStream_t s);

}  // namespace d2ba
