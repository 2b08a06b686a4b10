// d2ba_types.cuh -- device-visible data layout of libd2ba (sm_90a).
//
// HBM layout (DESIGN.md section 3).  One handle holds B windows; every array below is a single
// allocation shared by all windows, indexed through the per-window WinDesc offsets so that one
// launch covers the whole batch (grid.y / flattened job lists).
#pragma once
#include <stdint.h>

namespace d2ba {

constexpr int kTile = 32;        // observations per tile == warp width
constexpr int kObsFields = 21;   // pts_i(3) pts_j(3) vel_i(3) vel_j(3) td_i td_j tangent_base(6) inv_depth_j
constexpr int kMaxImuPerWin = 64;

enum ProjType { P2F1C = 0, P2F2C = 1, P1F2C = 2, P2F1CD = 3, PDEPTH = 4 };

// A "group" = all reprojection residuals of one window that share (type, pose_i, pose_j, ext_a, ext_b):
// they share every camera-side parameter block, so their J^T J contributions reduce into the same
// blocks (pair-major ordering, DESIGN.md 4.1).
struct Group {
  int type;
  int blk[4];       // window-local six-dof block index of pose_i, pose_j, ext_a, ext_b (-1 = absent)
  int slot_src[4];  // which factor block (0..3) feeds J-slot s, -1 = slot unused
  int slot_col[4];  // reduced-system column of slot s
  int td_col;       // reduced column of td or -1
  int nct;          // column tiles of the staged J (2: [s0 s1 r], 4: [s0 s1 s2 s3 td r])
  int rows;         // residual rows (1, 2 or 3)
  int need_ext;     // any extrinsic Jacobian needed
  int need_td;
  int shift0;       // every observation has td - td_i == td - td_j == 0 (td constant): velocity terms vanish
};

struct Job {       // one warp's work: a run of tiles of one group
  int win, grp, tile_begin, ntiles;
};

// Compact upload format of the observation constants (built by d2ba_add_proj, consumed by k_build_tiles).  Geometry and
// motion (feature velocity, stamp) are separate arrays: with a constant td equal to every stamp of the window -- the
// reference's default, estimate_td: 0 -- the time shift td - td_i is exactly zero, the velocities multiply zero, and the
// motion arrays never cross PCIe.
struct ObsJ {        // per residual block: the observing half of a reprojection record (40 bytes)
  double pts_j[3];
  double depth;      // measured depth (2F1C_DEPTH, DEPTH_PRIOR), else 0
  int32_t anchor;    // index into the window's ObsAnchor table
  int32_t type;      // d2ba_proj_type
};
struct ObsJm { double vel_j[3], td_j; };          // motion half of ObsJ (32 bytes), same index
struct ObsAnchor { double pts_i[3]; };            // the anchor half, stored once per run of residual blocks that share it (24 bytes)
struct ObsAnchorM { double vel_i[3], td_i; };     // motion half of ObsAnchor (32 bytes), same index

// One run of a row of Hcc that some factor writes (the per-linearisation zero-fill touches only these; everything else
// of Hcc stays at the zero of the finalize-time memset).  Hcc is LOWER triangular storage: writers put (max, min).
struct HSeg { int row, c0, len; };

// A "leaf" = a set of pose blocks that couples (through landmarks) only to itself and to the hub (own frames, extrinsics,
// td): the remote frames of one other drone in a multi-agent window.  Leaves are eliminated from the reduced system
// before the dense Cholesky of the hub (k_leaf_elim), the way the speed-bias chain is (k_sb_elim).
struct Leaf {
  int win, col0, n;      // window, first reduced column, columns
  int row0;              // first of its n rows Y = L^-1 [S_leaf,hub | g_leaf] behind the landmark / speed-bias rows of Wt (window-local row)
  long long offL;        // offset (doubles) into Dev::leafL: L (n x n row-major) then 1/diag(L) (n)
  int lm_begin, lm_count;  // its landmarks (the rows of Wt with entries in its columns): Dev::leaf_lm[lm_begin ..), window-local indices
};

// Reduced camera system tiles: kind 0 = SYRK tile in W-space (32x32) over the listed 32-row chunks of Wt,
// kind 1 = copy tile (rows / cols of a not eliminated speed-bias part, which has no landmark coupling)
struct SchurTile { int win, kind, tm, tn, cb, cn; };

struct ImuDesc {
  int pi, si, pj, sj;  // window-local indices (six-dof table / speed-bias table)
  int win;             // window of the factor (k_imu_lin runs one warp per factor over the whole batch)
};

struct WinDesc {
  int n6, np, ne, nsb, nl, has_td, td_col;
  int n_lc, n_c, ldh;          // reduced dims, leading dim of Hcc/S (multiple of 4)
  int ldw;                     // leading dim of Wt rows (>= n_lc+1, multiple of 8)
  int nl_pad;                  // landmarks padded to a multiple of 32
  int off6, offsb, offlm;      // offsets into block tables
  int off_tile, n_tile;
  int off_grp, n_grp;
  int off_imu, n_imu;
  int rec_stride;              // doubles per landmark-side record (16 or 32)
  int64_t off_rec;             // offset of the window's records (doubles)
  int64_t offH;                // Hcc / S offset (doubles)
  int64_t offW;                // Wt offset (doubles)
  int64_t offc;                // offset into n_c sized vectors
  int off_lmptr;               // landmark CSR pointer offset (nl+1 entries)
  int64_t off_lmobs;           // landmark CSR entries
  // prior
  int prior_m, prior_nblk, off_prior_blk;
  int64_t off_prior_J, off_prior_v;
  // consensus
  int admm_on;
  int chol_smem;               // reduced system fits the shared-memory Cholesky
  int schur_small;             // landmark-coupled part <= 127 columns: one-CTA Schur kernel
  // speed-bias elimination (k_sb_elim): block-tridiagonal speed-bias part eliminated before the dense Cholesky
  int sb_elim, n_sbe;          // enabled, number of (non-constant) speed-bias blocks
  int wt_rows;                 // rows of Wt the Schur kernels sum over: nl landmark rows + 9 n_sbe eliminated speed-bias rows, padded to 32
  int64_t offLE;               // offset (doubles) into Dev::sbLE
  // leaves (multi-agent windows): columns are ordered [leaf 0 | leaf 1 | ... | hub | speed-bias]
  int hub0, n_hub;             // first hub column, hub columns (n_lc - hub0); hub0 == 0 when the window has no leaves
  int n_leaf, off_leaf;
  int off_hseg, n_hseg;        // Hcc zero-fill segments
  int hub_small;               // leaves present and n_hub + 1 <= 96: the hub x hub part of the reduced system comes from the one-CTA Schur kernel
  int gather_nosync;           // compact records: within a landmark no column block appears at both slot positions (k_lm_gather16 needs no barrier between records)
  int row_tiles;               // most 32-column tiles any landmark's coupling row touches (row buffers of the gather kernels)
};

struct PriorBlk {
  int kind, index, off, eff;   // index: window-local (six-dof index for POSE/EXTRINSIC)
  double x0[9];
};

// Trust-region state of one window (device resident; the whole solve runs without host round trips).
struct Ctl {
  int cur;            // which linearisation / state buffer holds the accepted point
  int reuse;          // previous step rejected: reuse GN / Cauchy data (dogleg_strategy reuse_)
  int done;
  int term;
  int step_valid;     // 0: this iteration produced no candidate (solver failure / model change <= 0)
  int invalid_run;
  int iter, succ;
  int chol_fail;
  int lin_count;
  double radius, mu;
  double cost, cand_cost_misc, cand_cost_proj, model_change;
  double gg, nn, gdn, alpha, step_norm;
  double x_norm2, dx_norm2;
  double gmax_c, gmax_l;
  double uHu_cam, gg_cam;   // camera-part partial sums of the Cauchy quadratic form
  double initial_cost;
  unsigned long long gmax_l_bits;
};

struct SolverParams {
  double sqrt_info_px, depth_sqrt_inf, gravity, huber;
  double rho_T, rho_theta, rho_landmark, relaxation_alpha;
  double initial_radius, max_radius, min_rel_decrease, ftol, gtol, ptol;
  int max_iter, fixed_mode;
  double mu0;   // initial LM regularisation of the dogleg GN solve (1e-8; 0 for marginalization)
};

// All device pointers of a handle (passed to kernels by value).
struct Dev {
  const WinDesc *win;
  Ctl *ctl;
  int n_win;
  // block tables
  double *x6[2];        // [N6][8]  (x y z qx qy qz qw pad)
  double *R6[2];        // [N6][12] rotation matrix row-major (9) + pad
  double *xsb[2];       // [NSB][9]
  double *xlm[2];       // [NL]
  double *xtd[2];       // [B]
  const int *col6;      // [N6] reduced column or -1
  const int *colsb;     // [NSB]
  // reprojection
  const Group *grp;
  const Job *job;
  int n_job;
  const int *tile_grp;  // [T]
  const double *obs;    // [T][kObsFields][32]
  const int *obs_lm;    // [T][32] window-local landmark index, -1 = padding
  double *rec[2];       // landmark-side per-observation records
  // landmark CSR
  const int *lm_ptr;
  const unsigned long long *lm_mask;  // [NL] bit t set: the landmark's coupling row has entries in W-space columns [32 t, 32 t + 32)
  const HSeg *hseg;
  const Leaf *leaf; int n_leaf_total;
  int n_plain_win;      // windows without leaves
  double *leafL;        // per leaf: L, 1/diag(L)
  const int *schur_chunks;
  const int *leaf_lm;
  const int *obs_slot;  // [T][32] position of the observation's record in its landmark's run (window-local), -1 = padding
  // imu
  const ImuDesc *imu;
  const double *imu_c;  // [NIMU][kImuStride]
  double *imu_U;        // [NIMU][225] sqrt_info
  double *imu_raw;      // [NIMU][465] raw Jacobian (15 x 30) + residual (15) of the current linearisation (k_imu_raw -> k_imu_lin)
  // prior
  const PriorBlk *prior_blk;
  const double *prior_J;  // m x m
  const double *prior_e0; // packed in prior_v: e0[m]
  double *prior_A;        // J^T J (m x m) computed on device
  // consensus
  const int *slot6;       // [N6] global slot or -1
  double *z6;             // [N6][8]
  double *tilde6;         // [N6][6]
  double *lm_ref, *sb_ref, *td_ref;
  double *cons_buf;       // [n_slots][14] all-reduce payload
  int n_slots;
  // linearisation (double buffered)
  double *Hcc[2];
  double *gc[2];
  // Schur / solve
  double *Wt;           // [nl_pad][ldw] scaled coupling rows (+ g~ column)
  double *dinv;         // [NL] 1/sqrt(h + mu d^2)
  double *hl, *gl;      // [NL]
  double *S;            // reduced system (lower) per window
  double *sbLE;         // speed-bias elimination: L_kk, E'_k, 1/diag(L_kk) blocks (the rows Y live behind the landmark rows of Wt)
  double *gred;         // n_c
  double *D2c;          // n_c
  double *gn_c, *gn_l;  // Gauss-Newton step
  double *step_c, *step_l;
  double *wu;           // [NL] w_l . u_c
  double *uc;           // n_c : g_c / D_c^2 of the accepted linearisation
  double *D2l;          // [NL] landmark trust-region metric
  SolverParams prm;
};

constexpr int kImuStride = 1 + 3 + 4 + 3 + 3 + 3 + 225 + 225;  // sum_dt dp dq dv ba bg jac cov = 467
// upload format of the same constants: the 17 scalars, rows 0..8 x columns 9..14 of the pre-integration Jacobian (the only
// bias blocks IMUFactor reads) and the lower triangle of the covariance (the only half its Cholesky reads) -- 191 doubles
constexpr int kImuPack = 17 + 54 + 120;

}  // namespace d2ba
