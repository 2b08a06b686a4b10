// d2pgo_handle.cuh -- what the pose-graph solver (d2pgo.cu) and PCM (d2pgo_pcm.cu) share: the handle behind include/d2pgo.h,
// its self-freeing device buffers, and the error helpers.
#pragma once
#include <array>
#include <map>
#include <memory>
#include <unordered_map>

#include "d2pgo_chol.cuh"   // and with it cuda_runtime.h, <string>, <vector> and include/d2pgo.h

namespace d2pgo_host {

// a device array that only grows, freed with its owner
template <typename T> struct Buf {
  T *p = nullptr; size_t n = 0;
  Buf() = default;
  Buf(const Buf &) = delete;
  Buf &operator=(const Buf &) = delete;
  ~Buf() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t c) { if (c <= n && p) return cudaSuccess; if (p) cudaFree(p); p = nullptr; n = 0; cudaError_t e = cudaMalloc(&p, (c ? c : 1) * sizeof(T)); if (e == cudaSuccess) n = c; return e; }
};

struct PgoScalars {      // device-resident CG state that is not a per-block partial
  double bb;             // |b|^2 of the current linear system
  int done, iters;
};

// an ARock dual table: the duals keyed (neighbour, frame id) in ascending order, y_l and y_r of up to W doubles each (the
// exchange's width: the pose table's is the pose dof, 4 or 6; the rotation table's 9, a row-major 3x3 matrix), and the
// messages received since the last step (duals [n][width])
template <int W> struct ArockDual { double yl[W], yr[W]; };
template <int W> using ArockDuals = std::map<std::pair<int32_t, int64_t>, ArockDual<W>>;
struct ArockMsg { int32_t sender, target; std::vector<int64_t> frames; std::vector<double> duals; };
template <int W> struct ArockTable { ArockDuals<W> duals; std::vector<ArockMsg> inbox; };

// the ceres minimiser's device state (d2pgo_set_minimizer): its config and its trust region, written by the one-thread control
// kernels of d2pgo.cu only
struct LmState {
  double radius, min_diag, max_diag;   // in this order: the Cholesky's damping reads them (d2pgo_chol::LmDamping::par)
  double radius0, max_radius, min_radius, min_rel_dec, ftol, gtol, ptol, budget_s;
  int max_iter, max_invalid, jacobi, trace_cap;
  double decrease_factor, cost, cost0, x_norm, model, step_norm;
  unsigned long long t0, t_end;        // %globaltimer at the first device work and at the last decision
  int iter, ok, bad, invalid_run, pivot_fail, pending_grad, done, type, reason, cand;
};

struct PcmBufs;                                               // d2pgo_pcm.cu
struct PcmBufsFree { void operator()(PcmBufs *p) const; };    // defined beside PcmBufs
struct PcmStream;                                             // d2pgo_pcm.cu
struct PcmStreamFree { void operator()(PcmStream *p) const; };

}  // namespace d2pgo_host

struct d2pgo_handle {
  template <typename T> using Buf = d2pgo_host::Buf<T>;
  d2pgo_config cfg;
  int dof = 6;              // pose block size: 6 (RelPoseFactorAD on SE(3)) or 4 (RelPoseFactor4D on [x y z yaw])
  std::string err;
  cudaStream_t stream = nullptr;
  bool own_stream = false;  // d2pgo_create's handles; the rotation-init inner handle (rot) runs on its outer handle's stream
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::vector<int64_t> ids; std::unordered_map<int64_t, int> index;
  std::vector<double> poses; std::vector<unsigned char> fixed;   // [N][8], the device layout of PgoDev::x
  std::vector<int> ea, eb; std::vector<double> rel, sinfo;         // rel [E][8], sinfo [E][dof^2]
  std::vector<int> gp_pose; std::vector<double> gp_u, gp_S;        // gravity priors: pose index, u_ego [G][3], S [G][9]
  Buf<double> d_gp_u, d_gp_S, d_glin[2]; Buf<int> d_gp_pose, d_prior_of;
  Buf<double> d_x[2], d_rel, d_sinfo, d_lin[2], d_g[2], d_D[2], d_Minv, d_dx, d_r, d_z, d_p, d_Ap, d_cost, d_damp, d_t, d_part, d_cost_part;
  Buf<unsigned char> d_fixed; Buf<int> d_ea, d_eb, d_inc_ptr, d_inc; Buf<d2pgo_host::PgoScalars> d_s;
  // single rank, per linearisation buffer 0 / 1: [0] a chunk of kCgChunk CG iterations, [1] the shorter last chunk that stops
  // at pcg_max_iterations; cg_args: the bytes of the kernel arguments (and the chunk length) each graph was captured with
  cudaGraphExec_t cg_graph[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};
  std::string cg_args[2][2];
  bool uploaded = false;
  void *comm = nullptr; int rank = 0, nranks = 1;
  std::unique_ptr<d2pgo_host::PcmBufs, d2pgo_host::PcmBufsFree> pcm;   // d2pgo_pcm's device buffers, from its first call
  std::unique_ptr<d2pgo_host::PcmStream, d2pgo_host::PcmStreamFree> pcm_stream;   // the PCM stream, from d2pgo_pcm_stream_reset
  // ARock (d2pgo_arock_enable): owner agent and 6-DoF q_init per pose id, the pose dual table, and the device copy of the table
  // (in table order)
  bool arock = false; d2pgo_arock_config acfg = {};
  std::unordered_map<int64_t, int32_t> owner; std::unordered_map<int64_t, std::array<double, 4>> qinit;
  d2pgo_host::ArockTable<6> pose_table;
  Buf<int> d_ak_pose, d_ak_ptr, d_ak_of; Buf<double> d_ak_yr, d_ak_yl, d_ak_qinit, d_ak_lin[2], d_ak_coord;
  int ak_n = -1;                      // duals on the device, -1 = none synced
  // distributed rotation initialisation (d2pgo_arock_rot_*): its own dual table, each frame's rotation state R_state
  // (row-major; R(attitude) when the frame first enters a step, then the last unprojected M), and the device copies
  d2pgo_host::ArockTable<9> rot_table;
  std::unordered_map<int64_t, std::array<double, 9>> rot_state;
  Buf<int> d_rk_pose, d_rk_prior; Buf<double> d_rk_yl, d_rk_yr, d_rk_state;
  std::unique_ptr<d2pgo_handle> rot;  // the row systems (dof 3) of both rotation initialisations, kept between calls for their buffers
  int linear_solver = D2PGO_LINEAR_PCG;   // d2pgo_set_linear_solver
  std::unique_ptr<d2pgo_chol::Numeric> chol;   // the sparse Cholesky's analysis and device state (d2pgo_chol.cu)
  // d2pgo_set_minimizer: the kind and ceres LM's config; its device state, Jacobi scale, per-block partials and trace; the
  // graph of one whole solve and the bytes it was built from; the last solve's report (lm_ran: that solve was ceres LM)
  int minimizer = D2PGO_MINIMIZER_RESTATED; d2pgo_ceres_lm_config lm_cfg = {};
  Buf<d2pgo_host::LmState> d_lm; Buf<double> d_lm_scale, d_lm_part; Buf<d2pgo_minimizer_iteration> d_lm_trace;
  cudaGraphExec_t lm_graph = nullptr; std::string lm_key;
  bool lm_ran = false; d2pgo_minimizer_summary lm_report = {}; int lm_trace_n = 0;
  // d2pgo_set_chart: in the perturbation chart the pose records hold [p, theta, 0, 0] and chart_qinit [N][4] (unit, xyzw) the
  // attitude each theta is taken from; d_qinit is its device copy, uploaded with the poses
  int chart = D2PGO_CHART_RETRACTION; std::vector<double> chart_qinit; Buf<double> d_qinit;
  int driver_version = 0;

  ~d2pgo_handle() {   // the device buffers free themselves
    if (lm_graph) cudaGraphExecDestroy(lm_graph);
    for (auto &pair : cg_graph) for (cudaGraphExec_t g : pair) if (g) cudaGraphExecDestroy(g);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (own_stream) cudaStreamDestroy(stream);
  }
};

#define PCK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { h->err = std::string(#call) + ": " + cudaGetErrorString(e_); return 100 + (int)e_; } } while (0)

inline int pgo_fail(d2pgo_handle *h, int rc, const std::string &msg) { h->err = msg; return rc; }
