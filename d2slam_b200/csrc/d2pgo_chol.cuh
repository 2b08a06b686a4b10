// d2pgo_chol.cuh -- the pose graph's sparse Cholesky path (d2pgo_set_linear_solver(h, D2PGO_LINEAR_SPARSE_CHOLESKY)):
// host symbolic analysis and the device state of the supernodal multifrontal factorisation in d2pgo_chol.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/d2pgo.h"

namespace d2pgo_chol {

constexpr int kMaxFront = 1024;              // scalar rows of one front: a factorisation panel and the solves' vectors sit in shared memory
constexpr double kAmalgamateZeros = 0.25;    // relaxed amalgamation: largest share of explicit zeros in a merged supernode
constexpr double kArenaShare = 0.5;          // largest share of the free device memory the fronts may take
constexpr int kNdLeaf = 64;                  // nested dissection: parts of at most this many poses keep their natural order

// The symbolic analysis of one graph structure: block columns are free poses in elimination order, a supernode is a range of
// consecutive block columns sharing one row structure below them.  Everything is in blocks (D x D) unless named scalar.
struct Symbolic {
  int n_pose = 0, n_edge = 0, D = 0, n_free = 0;
  std::vector<unsigned char> fixed; std::vector<int> ea, eb;   // the structure this was computed for
  std::vector<int> perm;       // [n_free] pose index of each block column
  std::vector<int> col_of;     // [n_pose] block column of each pose, -1 for a fixed pose
  std::vector<int> pair_lo, pair_ptr, pair_edge;   // distinct free-free pose pairs (lo < hi), their edges ascending
  std::vector<int> self_ptr, self_edge;            // [n_free + 1] self-loop edges of each block column
  std::vector<int> sn_first, sn_width, sn_parent, sn_level;   // supernodes in column order; parent -1 = root
  std::vector<int> idx_ptr, idx;     // each supernode's front rows: its own columns, then the rows below them (ascending)
  std::vector<int> relmap;           // aligned with idx: the row's position in the parent's front (-1 on the own columns)
  std::vector<int> ch_ptr, ch;       // children of each supernode, ascending
  std::vector<int> po_ptr, po_pair, po_row, po_col, po_tr;   // off-diagonal H blocks each front assembles (tr: transposed)
  std::vector<int> lvl_ptr, lvl_sn;  // level sets of the supernodal tree, leaves first
  std::vector<long long> sn_off, sn_uoff;   // scalar offsets of each front (M x M) and of its update vector (M - W)
  long long arena = 0, uarena = 0;          // doubles of all fronts and of all update vectors
  int64_t nnz_L = 0, nnz_stored = 0;        // blocks of L: exact, and as stored after amalgamation
  int n_pairs = 0, sn_fundamental = 0, levels_fundamental = 0, max_front_rows = 0, max_front_cols = 0;   // front sizes scalar
};

// 0, or 2 with `err` on an out-of-range edge end or a block size other than 4 or 6
int analyse(int n_pose, const unsigned char *fixed, int n_edge, const int *ea, const int *eb, int D, Symbolic &s, std::string &err);
// the structure counts of d2pgo_cholesky_info (the run counters are left alone)
void fill_info(const Symbolic &s, d2pgo_cholesky_info *out);
// "" or why the kernels cannot take this structure (a front above kMaxFront rows, fronts beyond kArenaShare of free_bytes)
std::string check_limits(const Symbolic &s, size_t free_bytes);

// inputs of one factorisation: the linearisation buffer the LM loop is at
struct Lin {
  const double *lin, *Dg, *g;   // edge records [D + 2 D^2][E] field-major, block diagonal [N][D^2], gradient [N][D]
  const unsigned char *fixed; const int *ea, *eb;
  double *dx;                   // [N][D] output
};

// the damping of a ceres Levenberg-Marquardt step (d2pgo_set_minimizer): scale [N][D] the Jacobi scale s, par -> {radius,
// min_lm_diagonal, max_lm_diagonal}, both in device memory
struct LmDamping { const double *scale, *par; };

struct Numeric {
  Symbolic sym;
  bool dev_ready = false;
  std::vector<void *> bufs;     // device allocations of the symbolic tables and the arenas
  int *d_i = nullptr;           // all int tables, one allocation (offsets below)
  long long *d_off = nullptr;   // sn_off | sn_uoff
  double *d_pairH = nullptr, *d_diagH = nullptr, *d_front = nullptr, *d_uvec = nullptr, *d_b = nullptr, *d_y = nullptr, *d_x = nullptr, *d_lambda = nullptr;
  int *d_fail = nullptr;
  size_t o_perm, o_col_of, o_pair_lo, o_pair_ptr, o_pair_edge, o_self_ptr, o_self_edge, o_sn_first, o_sn_width, o_idx_ptr, o_idx, o_relmap,
      o_ch_ptr, o_ch, o_po_ptr, o_po_pair, o_po_row, o_po_col, o_po_tr, o_lvl_sn;
  cudaGraphExec_t gfac[2] = {nullptr, nullptr}, gsol[2] = {nullptr, nullptr};
  Lin gkey[2] = {};             // the buffers each parity's graphs were captured with
  cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
  double h_lambda = 0.0; int h_fail = 0;
  bool has_system = false;      // d_pairH / d_diagH / d_b hold the system of a step on these buffers
  // counters of the last solve
  int factorizations = 0, failed = 0; double factor_ms = 0.0, solve_ms = 0.0;
  int generation = 0;           // set by every upload, unique in the process: graphs that captured other buffers are stale

  ~Numeric() { release(); }
  void release();
  void drop_graphs();
  // device tables and arenas of `sym` (once per structure)
  int upload(cudaStream_t st, std::string &err);
  // (H + damping) dx = -g at the buffers `in` (parity `par` picks the captured graphs): *failed = a non-positive or non-finite
  // pivot.  Synchronises the stream.
  int step(cudaStream_t st, int par, const Lin &in, double lambda, bool *failed, std::string &err);
  // the same factorisation and solve with the damping of lm, enqueued on `st` (not launched, not synchronised: for capture
  // into the minimiser's graph); the pivot flag is left in d_fail
  int enqueue_lm(cudaStream_t st, const Lin &in, const LmDamping &lm, std::string &err);
  // copies of the last step's assembled system by pose index (has_system): diag[n_pose][D*D] (lower triangle as factored,
  // mirrored; 0 on fixed poses), b[n_pose][D] (0 on fixed poses), the first max_pairs pairs' pose indices pair_ab[][2] (lo, hi)
  // and blocks pair_H[][D*D] (sum J_lo^T J_hi).  Synchronises the stream.
  int system(cudaStream_t st, double *diag, double *b, int max_pairs, int32_t *pair_ab, double *pair_H, std::string &err);
};

}  // namespace d2pgo_chol
