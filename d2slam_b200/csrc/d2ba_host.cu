// d2ba_host.cu -- host side of libd2ba.so: C-ABI entry points (include/d2ba.h), problem assembly
// (pair-major sorting, 32-observation tiles, landmark CSR), device arena, launch sequencing / CUDA
// graph, NCCL consensus exchange.  No numerics of the solve run on the host; there is no CPU
// fallback (d2ba_create fails without a CUDA device).
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <sched.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <map>
#include <mutex>
#include <thread>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/d2ba.h"
#include "d2ba_types.cuh"

namespace d2ba {
// launchers implemented in d2ba_kernels.cu
void launch_state_prep(const Dev &d, int n6_total, int buf, cudaStream_t s);
void launch_imu_prep(const Dev &d, const double *packed, double *full, int n_imu, cudaStream_t s);
void launch_prior_prep(const Dev &d, cudaStream_t s);
void launch_misc_lin(const Dev &d, int eval_cur, int max_prior_m, cudaStream_t s);
void launch_imu_lin(const Dev &d, int eval_cur, int n_imu_total, cudaStream_t s);
void launch_imu_raw(const Dev &d, int eval_cur, int n_imu_total, cudaStream_t s);   // the two halves of launch_imu_lin
void launch_imu_acc(const Dev &d, int eval_cur, int n_imu_total, cudaStream_t s);
int configure_kernels(int max_rows, int max_nc, int max_prior_m);
int configure_gather(int max_ldw);
void launch_proj_lin(const Dev &d, int variant, int eval_cur, int job_begin, int job_count, cudaStream_t s);
void launch_proj_debug(const Dev &d, double *out, int n_tiles, const int *tile_win, cudaStream_t s);
void launch_imu_debug(const Dev &d, double *out, const int *imu_win, int n, cudaStream_t s);
void launch_cons_debug(const Dev &d, double *out, const int *blk_win, int n, cudaStream_t s);
void launch_lm_gather(const Dev &d, const int *lm_win, int n_lm_total, int max_ldw, int any_compact, int any_wide, cudaStream_t s);
void launch_schur(const Dev &d, const void *tiles, int n_tiles, cudaStream_t s);
int configure_leaf_elim(size_t smem);
void launch_leaf_elim(const Dev &d, size_t smem, cudaStream_t s);
void launch_leaf_back(const Dev &d, size_t smem, cudaStream_t s);
size_t leaf_back_smem(int n, int n_hub);
int configure_leaf_back(size_t smem);
void launch_zero_leaf_rows(const Dev &d, cudaStream_t s);
void launch_schur_small(const Dev &d, int max_ldw, cudaStream_t s);
int configure_schur_small(int max_ldw);
void launch_chol(const Dev &d, int max_rows, cudaStream_t s);
size_t chol_smem_need(int n);
int configure_chol_smem(int max_n);
void launch_chol_smem(const Dev &d, int max_n, cudaStream_t s);
size_t sb_elim_smem(int ldw, int n_c, int nb);
size_t sb_back_smem(int nlc, int nb);
int configure_sb_back(size_t smem);
void launch_zero_sb_rows(const Dev &d, cudaStream_t s);
int configure_sb_elim(size_t smem);
void launch_sb_elim(const Dev &d, size_t smem, cudaStream_t s);
void launch_sb_back(const Dev &d, size_t smem, cudaStream_t s);
int sb_max_blocks();
void launch_step(const Dev &d, int max_nc, cudaStream_t s);
void launch_control(const Dev &d, int init, cudaStream_t s);
void launch_tr_reset(const Dev &d, int first, cudaStream_t s);
void launch_cons_init(const Dev &d, int n6_total, cudaStream_t s);
void launch_cons_pack(const Dev &d, int n6_total, const int *blk_win, cudaStream_t s);
void launch_cons_apply(const Dev &d, int n6_total, const int *blk_win, cudaStream_t s);
void launch_cons_refs(const Dev &d, int nsb_total, int nl_total, const int *sb_win, const int *lm_win, cudaStream_t s);
typedef SchurTile SchurTileH;
size_t leaf_elim_smem(int n, int n_hub);
int leaf_max_cols();
int launch_marg_reduce(const double *S, int ld, int n, const int *keep_idx, int nk, const int *rem_idx, int nr, double *A, double *b, int *fail_flag,
                       cudaStream_t s);
void launch_build_tiles(const long long *raw_off, const int *tile_src, const int *tile_win, const double *xtd, double *obs, int n_tiles, cudaStream_t s);
void launch_prior_from_info(int n_win, int max_m, const int *m_of, const long long *offJ, const long long *offv, const int *is_info,
                            double *A, double *V, double *b, cudaStream_t s);
}  // namespace d2ba

using namespace d2ba;

namespace {

// open-addressing id -> index map (no per-node allocation; capacity survives clear())
struct FlatMap {
  std::vector<int64_t> keys; std::vector<int> vals; size_t n = 0;
  static uint64_t mix(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33; return x; }
  void clear() { std::fill(vals.begin(), vals.end(), -1); n = 0; }
  int find(int64_t k) const {
    if (vals.empty()) return -1;
    size_t m = vals.size() - 1, i = mix((uint64_t)k) & m;
    while (vals[i] >= 0) { if (keys[i] == k) return vals[i]; i = (i + 1) & m; }
    return -1;
  }
  void grow() {
    std::vector<int64_t> ok; std::vector<int> ov; ok.swap(keys); ov.swap(vals);
    size_t cap = ov.empty() ? 64 : ov.size() * 2;
    keys.assign(cap, 0); vals.assign(cap, -1); n = 0;
    for (size_t i = 0; i < ov.size(); i++) if (ov[i] >= 0) put(ok[i], ov[i]);
  }
  void put(int64_t k, int v) {
    if ((n + 1) * 2 > vals.size()) grow();
    size_t m = vals.size() - 1, i = mix((uint64_t)k) & m;
    while (vals[i] >= 0) { if (keys[i] == k) { vals[i] = v; return; } i = (i + 1) & m; }
    keys[i] = k; vals[i] = v; n++;
  }
};

struct HObs { int type, pi, pj, ea, eb, lm, fa; };   // index form of one residual block (constants stay in the raw record); fa = anchor frame

// Per-window pinned staging of the observation constants in the compact upload format (d2ba_types.cuh: ObsJ /
// ObsAnchor): the anchor half of a reprojection record (pts_i, vel_i, td_i) repeats for every observation of a
// landmark, so it is stored once per run of identical anchors, and feature velocities / stamps go to separate motion
// arrays that stay on the host while td is a constant equal to every stamp -- a quarter of the caller's 160-byte records
// crosses PCIe.  The tiled layout and the tangent bases are built on the device by k_build_tiles.
// Capacity survives d2ba_reset.
template <typename T, bool WC = true>
struct PinArr {
  T *p = nullptr; size_t cap = 0, n = 0;
  bool moved = false;   // the last reserve() re-allocated (the whole array must be uploaded again)
  bool reserve(size_t extra) {
    moved = false;
    if (n + extra <= cap) return true;
    size_t want = std::max<size_t>((n + extra) * 3 / 2 + 64, 1024);
    T *q = nullptr;
    // write-combined: the feeding threads only ever append (no read-for-ownership, no cache pollution) and the DMA engine
    // does not have to snoop the CPU caches; reading it back (marginalization, growth) is slow but rare
    if (cudaHostAlloc((void **)&q, want * sizeof(T), WC ? cudaHostAllocWriteCombined : cudaHostAllocDefault) != cudaSuccess) return false;
    if (n) memcpy(q, p, n * sizeof(T));
    if (p) cudaFreeHost(p);
    p = q; cap = want; moved = true;
    return true;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = n = 0; }
};
template <typename T>
struct DevArr {   // device mirror of a PinArr, filled as the host side is appended
  T *p = nullptr; size_t cap = 0;
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
struct HImu { int pi, si, pj, sj; double c[kImuStride]; };
struct HPriorBlk { int kind, index, off, eff; double x0[9]; };

struct HostWin {
  bool used = false;
  std::vector<int64_t> pose_id, ext_id, sb_id, lm_id;
  FlatMap pose_map, ext_map, sb_map, lm_map;
  std::vector<double> pose, ext, sb, lm;
  std::vector<uint8_t> pose_c, ext_c, sb_c;
  double td = 0; bool has_td = false; uint8_t td_c = 1;
  std::vector<HObs> obs;
  PinArr<ObsJ> rawj; PinArr<ObsAnchor> anch;              // compact observation constants (pinned): geometry ...
  PinArr<ObsJm, false> rawjm; PinArr<ObsAnchorM, false> anchm;   // ... and motion (uploaded at finalize, only when the time shift can be non-zero;
                                                                  //     cacheable: normally never read by the DMA engine, and two fewer write-combining streams per feeder)
  DevArr<ObsJ> d_rawj; DevArr<ObsAnchor> d_anch;          // device copies (uploaded in batches as they are appended)
  DevArr<ObsJm> d_rawjm; DevArr<ObsAnchorM> d_anchm;
  size_t pushed_j = 0, pushed_a = 0, pushed_jm = 0, pushed_am = 0;   // records already on the copy stream
  int feed_lock = 0; bool push_pending = false;            // feeder / uploader hand-over (see flush_pending)
  double td_min = 1e300, td_max = -1e300;
  std::vector<HImu> imu;
  int prior_m = 0; std::vector<double> prior_J, prior_e0; std::vector<HPriorBlk> prior_blk; bool prior_is_info = false;
  std::vector<int> pose_slot, ext_slot; bool admm = false; int n_slots = 0;
  // derived at finalize
  std::vector<int> pose_col, ext_col, sb_col; int td_col = -1, n_lc = 0, n_c = 0;
  std::vector<int> order;            // pair-major order: sorted index -> observation index
  std::vector<int> sorted_pos;       // tile slot (window-local) of the k-th sorted observation
  std::vector<int> canon_of_dev;     // device reduced column -> canonical (insertion-order) column, for the debug views
  void clear() {   // keeps every allocation (the estimator re-adds a similar problem for the next solve)
    used = false;
    pose_id.clear(); ext_id.clear(); sb_id.clear(); lm_id.clear();
    pose_map.clear(); ext_map.clear(); sb_map.clear(); lm_map.clear();
    pose.clear(); ext.clear(); sb.clear(); lm.clear(); pose_c.clear(); ext_c.clear(); sb_c.clear();
    td = 0; has_td = false; td_c = 1;
    obs.clear(); rawj.n = 0; anch.n = 0; rawjm.n = 0; anchm.n = 0; pushed_j = pushed_a = pushed_jm = pushed_am = 0; push_pending = false; imu.clear(); td_min = 1e300; td_max = -1e300;
    prior_m = 0; prior_J.clear(); prior_e0.clear(); prior_blk.clear(); prior_is_info = false;
    pose_slot.clear(); ext_slot.clear(); admm = false; n_slots = 0;
    pose_col.clear(); ext_col.clear(); sb_col.clear(); td_col = -1; n_lc = 0; n_c = 0;
    order.clear(); sorted_pos.clear();
  }
};

// ---- minimal NCCL surface resolved with dlopen (torch ships libnccl.so.2; no link-time dependency)
typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId_t;
struct Nccl {
  void *lib = nullptr;
  int (*GetUniqueId)(ncclUniqueId_t *) = nullptr;
  int (*CommInitRank)(ncclComm_t *, int, ncclUniqueId_t, int) = nullptr;
  int (*AllReduce)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  const char *(*GetErrorString)(int) = nullptr;
  bool load(std::string &err) {
    if (lib) return true;
    const char *env = getenv("D2BA_NCCL_LIB");
    const char *names[] = {env, "libnccl.so.2", "libnccl.so"};
    for (const char *n : names) { if (!n) continue; lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
    if (!lib) { err = std::string("cannot dlopen libnccl: ") + dlerror(); return false; }
    GetUniqueId = (int (*)(ncclUniqueId_t *))dlsym(lib, "ncclGetUniqueId");
    CommInitRank = (int (*)(ncclComm_t *, int, ncclUniqueId_t, int))dlsym(lib, "ncclCommInitRank");
    AllReduce = (int (*)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t))dlsym(lib, "ncclAllReduce");
    CommDestroy = (int (*)(ncclComm_t))dlsym(lib, "ncclCommDestroy");
    GetErrorString = (const char *(*)(int))dlsym(lib, "ncclGetErrorString");
    if (!GetUniqueId || !CommInitRank || !AllReduce) { err = "libnccl lacks required symbols"; return false; }
    return true;
  }
};
Nccl g_nccl;

template <typename T>
struct DBuf {
  T *p = nullptr; size_t n = 0;
  bool view = false;   // p points into the handle's upload arena (not owned)
  void bind(void *base, size_t byte_off, size_t count) { if (p && !view) cudaFree(p); p = (T *)((char *)base + byte_off); n = count; view = true; }
  cudaError_t alloc(size_t count) {
    if (view) { p = nullptr; n = 0; view = false; }
    if (count <= n && p) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; n = 0;
    cudaError_t e = cudaMalloc(&p, std::max<size_t>(count, 1) * sizeof(T));
    if (e == cudaSuccess) n = count;
    return e;
  }
  void release() { if (p && !view) cudaFree(p); p = nullptr; n = 0; view = false; }
};

}  // namespace

namespace {
template <typename T>
struct HBuf {   // pinned host staging buffer (grows, never shrinks)
  T *p = nullptr; size_t cap = 0, n = 0;
  bool resize(size_t count) {
    n = count;
    if (count <= cap) return true;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    size_t want = count + count / 4 + 16;
    if (cudaHostAlloc((void **)&p, want * sizeof(T), cudaHostAllocDefault) != cudaSuccess) return false;
    cap = want;
    return true;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = n = 0; }
};

}  // namespace

struct d2ba_handle {
  d2ba_config cfg;
  std::string err;
  std::vector<HostWin> win;
  cudaStream_t stream = nullptr, copy_stream = nullptr;
  cudaStream_t side = nullptr;                 // second lane of the iteration: IMU chain beside the reprojection kernels, sb elimination beside the landmark gather
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_misc = nullptr;
  bool two_lanes = true;                       // D2BA_ONE_LANE=1: everything on `stream` (A/B)
  cudaEvent_t ev_copy = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaEvent_t ev_it[2] = {nullptr, nullptr};   // solver time budget: iteration k-2 complete
  cudaEvent_t evf0 = nullptr, evf1 = nullptr, evf2 = nullptr;   // device span of the last finalize: uploads | tile build + prep kernels
  bool motion_skipped = false;                 // some window's motion halves stayed on the host (debug views fetch them: ensure_motion)
  std::atomic<bool> finalized{false}, state_dirty{false};   // written by the per-window feeding calls of several threads
  std::mutex err_mu;                                        // guards err (fail() may be reached from several feeding threads)
  // device arena
  DBuf<char> d_arena;   // device image of the pinned staging arena (one H2D copy per finalize); the DBufs it backs are views
  DBuf<WinDesc> d_win; DBuf<Ctl> d_ctl;
  DBuf<double> d_x6[2], d_R6[2], d_xsb[2], d_xlm[2], d_xtd[2];
  DBuf<int> d_col6, d_colsb, d_tile_grp, d_obs_lm, d_lm_ptr, d_obs_slot, d_slot6, d_lm_win, d_blk_win, d_sb_win, d_tile_win;
  DBuf<Group> d_grp; DBuf<Job> d_job; DBuf<ImuDesc> d_imu; DBuf<PriorBlk> d_prior_blk;
  DBuf<double> d_obs, d_rec[2], d_imu_c, d_imu_pk, d_imu_U, d_imu_raw, d_prior_J, d_prior_e0, d_prior_A, d_z6, d_tilde6, d_lm_ref, d_sb_ref, d_td_ref,
      d_cons, d_H[2], d_gc[2], d_Wt, d_dinv, d_hl, d_gl, d_S, d_gred, d_D2c, d_gn_c, d_gn_l, d_step_c, d_step_l, d_wu, d_uc, d_D2l, d_dbg;
  DBuf<SchurTileH> d_schur; DBuf<int> d_schur_chunks; DBuf<Leaf> d_leaf; DBuf<HSeg> d_hseg; DBuf<unsigned long long> d_lm_mask; DBuf<double> d_leafL; DBuf<int> d_leaf_lm;
  int n_schur0 = 0, n_leaf_total = 0, max_hub = 0; size_t leaf_smem = 0, cfg_leaf_smem = 0, leafb_smem = 0, cfg_leafb_smem = 0;
  DBuf<int> d_pr_m, d_pr_info, d_tile_src; DBuf<long long> d_pr_oJ, d_pr_ov, d_raw_off;
  int cfg_max_rows = -1, cfg_max_nc = -1, cfg_max_prior = -1, cfg_max_ldw = -1;
  Dev dev;
  std::vector<WinDesc> h_win;
  HBuf<Ctl> h_ctl;   // pinned: D2H target of every solve
  std::vector<Group> h_grp;
  std::vector<int> h_tile_win;
  int n_used = 0, n6_total = 0, nsb_total = 0, nl_total = 0, n_tiles = 0, n_imu_total = 0, n_schur = 0;
  int job_begin[6] = {0, 0, 0, 0, 0, 0}, job_count[6] = {0, 0, 0, 0, 0, 0};
  int max_rows = 1, max_nc = 1, max_prior_m = 0, max_ldw = 8, n_slots = 0;
  int max_n_smem = 0, max_rows_glob = 1; bool any_chol_glob = false; int cfg_max_n_smem = -1;
  int max_ldw_small = 0, cfg_max_ldw_small = -1;
  int max_row_tiles = 1;
  int any_compact = 0, any_wide = 0;   // record widths present (which gather kernels to launch)
  size_t sbb_smem = 0, cfg_sbb_smem = 0;   // k_sb_back dynamic shared memory
  size_t sbe_smem = 0, cfg_sbe_smem = 0;   // speed-bias elimination: dynamic shared memory of k_sb_elim (0 = no window uses it)
  int64_t totLE = 0;
  DBuf<double> d_sbLE;
  int64_t totH = 0, totW = 0, totc = 0;
  bool any_admm = false;
  // host mirrors of the solved state
  HBuf<double> h_x6[2], h_xsb[2], h_xlm[2], h_xtd[2];   // pinned D2H targets
  // graph cache
  cudaGraphExec_t iter_graph = nullptr; int graph_key = -1;
  int solves_since_finalize = 0;   // the iteration graph is captured from the second solve of an unchanged structure on
  d2ba_handle *marg = nullptr;   // scratch handle of d2ba_marginalize
  double mu0 = 1e-8;
  bool force_full_S = false;     // the Schur kernels must write the complete reduced system (marginalization reads it)
  bool no_leaf = false;          // D2BA_NO_LEAF=1: keep remote-frame blocks in the dense part (A/B switch)
  bool no_sb_elim = false;       // D2BA_NO_SB_ELIM=1: keep the dense Cholesky of the whole reduced system (A/B switch for tests / profiling)
  double host_ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // wall-clock phases of the last d2ba_finalize (d2ba_debug_host_times)
  double solve_ms[4] = {0, 0, 0, 0};             // host wall-clock of the last solve: enqueue, wait for the device, write-back
  std::atomic<long long> h2d_bytes_add;          // bytes d2ba_add_proj put on the copy stream since the last reset
  std::mutex push_mu, pend_mu;                   // one uploader at a time; guards pending_win / HostWin::push_pending
  std::vector<int> pending_win;                  // windows with records not yet on the copy stream
  std::atomic<long long> pending_bytes{0};
  long long h2d_bytes_fin = 0;                   // bytes of the last finalize's arena upload
  std::atomic<long long> add_ns[4];              // thread-summed ns inside d2ba_add_proj since the last reset: index, stamps, staging copy, CUDA calls
  // comm
  ncclComm_t comm = nullptr; int rank = 0, nranks = 1;
};

namespace {

#define CK(call)                                                                                   \
  do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { h->err = std::string(#call) + ": " + cudaGetErrorString(e_); return 100 + (int)e_; } } while (0)

int fail(d2ba_handle *h, int rc, const std::string &m) { std::lock_guard<std::mutex> lk(h->err_mu); h->err = m; return rc; }

HostWin *get_win(d2ba_handle *h, int w) {
  if (!h || w < 0 || w >= (int)h->win.size()) return nullptr;
  return &h->win[w];
}

int find_in(const FlatMap &m, int64_t id) { return m.find(id); }

int kind_size(int k) { return (k == D2BA_POSE || k == D2BA_EXTRINSIC) ? 7 : (k == D2BA_SPEED_BIAS ? 9 : 1); }
int kind_eff(int k) { return (k == D2BA_POSE || k == D2BA_EXTRINSIC) ? 6 : (k == D2BA_SPEED_BIAS ? 9 : 1); }

int roundup(int v, int m) { return (v + m - 1) / m * m; }

void release_graph(d2ba_handle *h) {
  if (h->iter_graph) { cudaGraphExecDestroy(h->iter_graph); h->iter_graph = nullptr; }
  h->graph_key = -1;
}

template <typename T>
int upload(d2ba_handle *h, DBuf<T> &b, const std::vector<T> &v) {
  CK(b.alloc(v.size()));
  if (!v.empty()) CK(cudaMemcpyAsync(b.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, h->stream));
  return 0;
}
template <typename T>
int alloc_zero(d2ba_handle *h, DBuf<T> &b, size_t n) {
  CK(b.alloc(n));
  CK(cudaMemsetAsync(b.p, 0, std::max<size_t>(n, 1) * sizeof(T), h->stream));
  return 0;
}

}  // namespace

void d2ba_release_staging(d2ba_handle *h);

extern "C" {

int d2ba_default_config(d2ba_config *c) {
  if (!c) return 1;
  memset(c, 0, sizeof(*c));
  c->version = D2BA_VERSION; c->device = 0; c->max_windows = 1; c->max_num_iterations = 8; c->consensus_max_steps = 0;
  c->use_cuda_graph = 1; c->focal_length = 460.0; c->depth_sqrt_inf = 20.0; c->gravity_norm = 9.805; c->huber_delta = 1.0;
  c->rho_frame_T = 100.0; c->rho_frame_theta = 100.0; c->rho_landmark = 1.0; c->relaxation_alpha = 0.0;
  return 0;
}

int d2ba_create(const d2ba_config *cfg, d2ba_handle **out) {
  if (!cfg || !out) return 1;
  if (cfg->version != D2BA_VERSION) return 2;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { fprintf(stderr, "d2ba_create: no CUDA device (there is no CPU fallback)\n"); return 3; }
  if (cfg->device < 0 || cfg->device >= ndev) return 4;
  if (cudaSetDevice(cfg->device) != cudaSuccess) return 5;
  d2ba_handle *h = new d2ba_handle();
  { const char *e = getenv("D2BA_NO_SB_ELIM"); h->no_sb_elim = e && e[0] == '1'; }
  { const char *e = getenv("D2BA_NO_LEAF"); h->no_leaf = e && e[0] == '1'; }
  h->cfg = *cfg;
  if (h->cfg.max_windows < 1) h->cfg.max_windows = 1;
  if (h->cfg.initial_trust_region_radius <= 0) h->cfg.initial_trust_region_radius = 1e4;
  if (h->cfg.max_trust_region_radius <= 0) h->cfg.max_trust_region_radius = 1e16;
  if (h->cfg.min_relative_decrease <= 0) h->cfg.min_relative_decrease = 1e-3;
  if (h->cfg.function_tolerance <= 0) h->cfg.function_tolerance = 1e-6;
  if (h->cfg.gradient_tolerance <= 0) h->cfg.gradient_tolerance = 1e-10;
  if (h->cfg.parameter_tolerance <= 0) h->cfg.parameter_tolerance = 1e-8;
  h->win.resize(h->cfg.max_windows);
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) { delete h; return 6; }
  cudaEventCreate(&h->ev0); cudaEventCreate(&h->ev1); cudaEventCreate(&h->evf0); cudaEventCreate(&h->evf1); cudaEventCreate(&h->evf2);
  cudaEventCreateWithFlags(&h->ev_it[0], cudaEventDisableTiming); cudaEventCreateWithFlags(&h->ev_it[1], cudaEventDisableTiming);
  cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking); cudaEventCreateWithFlags(&h->ev_copy, cudaEventDisableTiming);
  cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking);
  cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming); cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming); cudaEventCreateWithFlags(&h->ev_misc, cudaEventDisableTiming);
  { const char *e = getenv("D2BA_ONE_LANE"); h->two_lanes = !(e && e[0] == '1'); }
  memset(&h->dev, 0, sizeof(h->dev));
  *out = h;
  return 0;
}

int d2ba_destroy(d2ba_handle *h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device);
  cudaStreamSynchronize(h->stream);
  release_graph(h);
  if (h->marg) { d2ba_destroy(h->marg); h->marg = nullptr; }
  if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
  // DBuf members: release explicitly
  h->d_win.release(); h->d_ctl.release(); h->h_ctl.release(); h->d_arena.release(); h->d_sbLE.release();
  for (int b = 0; b < 2; b++) { h->h_x6[b].release(); h->h_xsb[b].release(); h->h_xlm[b].release(); h->h_xtd[b].release(); }
  for (int b = 0; b < 2; b++) { h->d_x6[b].release(); h->d_R6[b].release(); h->d_xsb[b].release(); h->d_xlm[b].release(); h->d_xtd[b].release(); h->d_rec[b].release(); h->d_H[b].release(); h->d_gc[b].release(); }
  h->d_col6.release(); h->d_colsb.release(); h->d_tile_grp.release(); h->d_obs_lm.release(); h->d_lm_ptr.release(); h->d_obs_slot.release();
  h->d_slot6.release(); h->d_lm_win.release(); h->d_blk_win.release(); h->d_sb_win.release(); h->d_tile_win.release();
  h->d_grp.release(); h->d_job.release(); h->d_imu.release(); h->d_prior_blk.release(); h->d_obs.release(); h->d_imu_c.release(); h->d_imu_pk.release(); h->d_imu_U.release(); h->d_imu_raw.release();
  h->d_prior_J.release(); h->d_prior_e0.release(); h->d_prior_A.release(); h->d_z6.release(); h->d_tilde6.release(); h->d_lm_ref.release(); h->d_sb_ref.release();
  h->d_td_ref.release(); h->d_cons.release(); h->d_Wt.release(); h->d_dinv.release(); h->d_hl.release(); h->d_gl.release(); h->d_S.release(); h->d_gred.release();
  h->d_D2c.release(); h->d_gn_c.release(); h->d_gn_l.release(); h->d_step_c.release(); h->d_step_l.release(); h->d_wu.release(); h->d_uc.release(); h->d_D2l.release(); h->d_dbg.release(); h->d_schur.release(); h->d_schur_chunks.release(); h->d_leaf.release(); h->d_hseg.release(); h->d_lm_mask.release(); h->d_leafL.release(); h->d_leaf_lm.release();
  h->d_pr_m.release(); h->d_pr_info.release(); h->d_pr_oJ.release(); h->d_pr_ov.release(); h->d_tile_src.release(); h->d_raw_off.release();
  cudaStreamSynchronize(h->copy_stream);
  for (auto &w : h->win) { w.rawj.release(); w.anch.release(); w.d_rawj.release(); w.d_anch.release(); w.rawjm.release(); w.anchm.release(); w.d_rawjm.release(); w.d_anchm.release(); }
  cudaStreamDestroy(h->copy_stream); cudaEventDestroy(h->ev_copy);
  cudaStreamSynchronize(h->side); cudaStreamDestroy(h->side); cudaEventDestroy(h->ev_fork); cudaEventDestroy(h->ev_join); cudaEventDestroy(h->ev_misc);
  d2ba_release_staging(h);
  cudaEventDestroy(h->ev_it[0]); cudaEventDestroy(h->ev_it[1]);
  cudaEventDestroy(h->ev0); cudaEventDestroy(h->ev1); cudaEventDestroy(h->evf0); cudaEventDestroy(h->evf1); cudaEventDestroy(h->evf2);
  cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int d2ba_reset(d2ba_handle *h) {
  if (!h) return 1;
  for (auto &w : h->win) w.clear();
  h->finalized = false;
  for (auto &a : h->add_ns) a = 0;
  h->h2d_bytes_add = 0;
  h->pending_win.clear(); h->pending_bytes = 0;
  return 0;
}

const char *d2ba_last_error(const d2ba_handle *h) { return h ? h->err.c_str() : "null handle"; }
int d2ba_num_windows(const d2ba_handle *h) { return h ? h->n_used : 0; }

int d2ba_set_blocks(d2ba_handle *h, int32_t window, int32_t kind, int32_t n, const int64_t *ids, const double *values,
                    const uint8_t *is_const) {
  HostWin *w = get_win(h, window);
  if (!w) return 1;
  w->used = true;
  bool structural = false;
  for (int i = 0; i < n; i++) {
    uint8_t c = is_const ? is_const[i] : 0;
    switch (kind) {
      case D2BA_POSE: {
        int k = find_in(w->pose_map, ids[i]);
        if (k < 0) { k = (int)w->pose_id.size(); w->pose_id.push_back(ids[i]); w->pose_map.put(ids[i], k); w->pose.resize(7 * (k + 1)); w->pose_c.push_back(c); w->pose_slot.push_back(-1); structural = true; }
        else if (w->pose_c[k] != c) structural = true;
        memcpy(&w->pose[7 * k], values + 7 * i, 56); w->pose_c[k] = c; break;
      }
      case D2BA_EXTRINSIC: {
        int k = find_in(w->ext_map, ids[i]);
        if (k < 0) { k = (int)w->ext_id.size(); w->ext_id.push_back(ids[i]); w->ext_map.put(ids[i], k); w->ext.resize(7 * (k + 1)); w->ext_c.push_back(c); w->ext_slot.push_back(-1); structural = true; }
        else if (w->ext_c[k] != c) structural = true;
        memcpy(&w->ext[7 * k], values + 7 * i, 56); w->ext_c[k] = c; break;
      }
      case D2BA_SPEED_BIAS: {
        int k = find_in(w->sb_map, ids[i]);
        if (k < 0) { k = (int)w->sb_id.size(); w->sb_id.push_back(ids[i]); w->sb_map.put(ids[i], k); w->sb.resize(9 * (k + 1)); w->sb_c.push_back(c); structural = true; }
        else if (w->sb_c[k] != c) structural = true;
        memcpy(&w->sb[9 * k], values + 9 * i, 72); w->sb_c[k] = c; break;
      }
      case D2BA_TD:
        if (!w->has_td || w->td_c != c || w->td != values[i]) structural = true;
        w->td = values[i]; w->td_c = c; w->has_td = true; break;
      case D2BA_LANDMARK: {
        int k = find_in(w->lm_map, ids[i]);
        if (k < 0) { k = (int)w->lm_id.size(); w->lm_id.push_back(ids[i]); w->lm_map.put(ids[i], k); w->lm.push_back(0); structural = true; }
        w->lm[k] = values[i]; break;
      }
      default: return fail(h, 2, "unknown block kind");
    }
  }
  if (structural) h->finalized = false; else h->state_dirty = true;
  return 0;
}

}  // extern "C"

namespace {
// append-range upload of a pinned array into its device mirror (copy stream)
template <typename T, bool WC>
int push_range(d2ba_handle *h, PinArr<T, WC> &host, DevArr<T> &dev, size_t first_new) {
  if (host.n > dev.cap) {
    if (dev.p) { cudaStreamSynchronize(h->copy_stream); cudaFree(dev.p); }
    dev.p = nullptr; dev.cap = 0;
    if (cudaMalloc((void **)&dev.p, host.cap * sizeof(T)) != cudaSuccess) return fail(h, 12, "add_proj: device allocation failed");
    dev.cap = host.cap; first_new = 0;
  }
  if (host.moved) first_new = 0;   // the pinned array moved: everything before was re-copied on the host, upload it all again
  if (host.n > first_new &&
      cudaMemcpyAsync(dev.p + first_new, host.p + first_new, (host.n - first_new) * sizeof(T), cudaMemcpyHostToDevice, h->copy_stream) != cudaSuccess)
    return fail(h, 13, "add_proj: H2D failed");
  h->h2d_bytes_add += (long long)((host.n - first_new) * sizeof(T));
  return 0;
}

// Uploads of the compact records are issued in batches by ONE thread at a time: 32 feeding threads calling
// cudaMemcpyAsync once per window serialise on the driver's stream lock (that lock, not the copy loop, was the feed stage's
// wall time).  A feeder that finds >= kPushBatch bytes pending and the uploader role free takes it; d2ba_finalize flushes
// the rest.  A window still being appended to (feed_lock held) stays on the list.
constexpr long long kPushBatch = 4 << 20;
inline void win_lock(HostWin *w) { while (__atomic_exchange_n(&w->feed_lock, 1, __ATOMIC_ACQUIRE)) { } }
inline bool win_try_lock(HostWin *w) { return !__atomic_exchange_n(&w->feed_lock, 1, __ATOMIC_ACQUIRE); }
inline void win_unlock(HostWin *w) { __atomic_store_n(&w->feed_lock, 0, __ATOMIC_RELEASE); }
// td constant (or absent) and equal to every stamp of the window: the shift td - td_i is exactly zero for the whole solve
inline bool motion_needed(const HostWin &w) {
  if (w.td_min > w.td_max) return false;   // no reprojection factor at all
  const bool td_free = w.has_td && !w.td_c;
  return td_free || w.td_min != w.td_max || w.td_min != w.td;
}
int flush_pending(d2ba_handle *h, bool all) {   // caller holds h->push_mu
  std::vector<int> list;
  {
    std::lock_guard<std::mutex> lk(h->pend_mu);
    list.swap(h->pending_win);
    for (int wi : list) h->win[wi].push_pending = false;
    h->pending_bytes = 0;
  }
  int rc = 0;
  for (int wi : list) {
    HostWin *w = &h->win[wi];
    if (all) win_lock(w);
    else if (!win_try_lock(w)) {
      std::lock_guard<std::mutex> lk(h->pend_mu);
      if (!w->push_pending) { w->push_pending = true; h->pending_win.push_back(wi); }
      continue;
    }
    if (!rc && !(rc = push_range(h, w->rawj, w->d_rawj, w->pushed_j)) && !(rc = push_range(h, w->anch, w->d_anch, w->pushed_a))) { w->pushed_j = w->rawj.n; w->pushed_a = w->anch.n; }
    win_unlock(w);
  }
  return rc;
}
}  // namespace

extern "C" {

int d2ba_add_proj(d2ba_handle *h, int32_t window, int32_t n, const d2ba_proj_obs *in) {
  HostWin *w = get_win(h, window);
  if (!w) return 1;
  w->used = true; h->finalized = false;
  if (n <= 0) return 0;
  const size_t base = w->obs.size(), base_a = w->anch.n;
  auto tq = std::chrono::steady_clock::now();
  auto lap = [&](int k) { auto t = std::chrono::steady_clock::now(); h->add_ns[k] += std::chrono::duration_cast<std::chrono::nanoseconds>(t - tq).count(); tq = t; };
  cudaSetDevice(h->cfg.device);   // callers may feed windows from their own threads
  win_lock(w);                    // against the batch uploader (flush_pending), which reads the arrays this call may move
  struct Unlock { HostWin *w; ~Unlock() { if (w) win_unlock(w); } } unlock_at_exit{w};
  if (!w->rawj.reserve((size_t)n)) return fail(h, 11, "add_proj: pinned allocation failed");
  if (w->rawj.moved) w->pushed_j = 0;
  if (!w->anch.reserve((size_t)n)) return fail(h, 11, "add_proj: pinned allocation failed");
  if (w->anch.moved) w->pushed_a = 0;
  if (!w->rawjm.reserve((size_t)n) || !w->anchm.reserve((size_t)n)) return fail(h, 11, "add_proj: pinned allocation failed");
  if (w->rawjm.moved) w->pushed_jm = 0;
  if (w->anchm.moved) w->pushed_am = 0;
  w->obs.resize(base + n);
  lap(3);
  // one pass over the caller's records: ids -> block indices (one-entry caches: consecutive residuals of a track share
  // landmark, anchor frame and cameras), stamps, and the compact upload records written straight into pinned memory
  struct Cache { int64_t id = INT64_MIN; int idx = -1; } c_lm, c_fa, c_fb, c_ca, c_cb;
  auto cached = [](Cache &c, const FlatMap &m, int64_t id) {
    if (c.id != id) { c.id = id; c.idx = find_in(m, id); }
    return c.idx;
  };
  ObsJ *oj = w->rawj.p + w->rawj.n;
  ObsJm *ojm = w->rawjm.p + w->rawjm.n;
  ObsAnchor *an = w->anch.p;
  ObsAnchorM *anm = w->anchm.p;
  size_t na = w->anch.n;
  struct { double pts_i[3], vel_i[3], td_i; } last; memset(&last, 0, sizeof last);   // cached copy of anchor na - 1: the pinned arrays are write-only for this loop
  double tmin = w->td_min, tmax = w->td_max;
  for (int i = 0; i < n; i++) {
    const d2ba_proj_obs &p = in[i];
    HObs o;
    o.type = p.type; o.pi = o.pj = o.ea = o.eb = -1;
    o.lm = cached(c_lm, w->lm_map, p.landmark_id);
    o.fa = cached(c_fa, w->pose_map, p.frame_a);
    const char *err = nullptr;
    if (o.lm < 0) err = "add_proj: unknown landmark id";
    else if (p.type < 0 || p.type > D2BA_PROJ_DEPTH_PRIOR) err = "add_proj: unknown residual type";
    else if (p.type != D2BA_PROJ_DEPTH_PRIOR) {
      // block lists: ParamResidualInfo.hpp:34-43 (2F1C), :72-82 (2F2C), :107-115 (1F2C)
      o.ea = cached(c_ca, w->ext_map, p.cam_a);
      if (o.ea < 0) err = "add_proj: unknown camera id";
      if (!err && (p.type == D2BA_PROJ_2F2C || p.type == D2BA_PROJ_1F2C)) { o.eb = cached(c_cb, w->ext_map, p.cam_b); if (o.eb < 0) err = "add_proj: unknown camera id (b)"; }
      if (!err && p.type != D2BA_PROJ_1F2C) {
        o.pi = cached(c_fa, w->pose_map, p.frame_a); o.pj = cached(c_fb, w->pose_map, p.frame_b);
        if (o.pi < 0 || o.pj < 0) err = "add_proj: unknown frame id";
      }
    }
    if (err) { w->obs.resize(base); w->anch.n = base_a; w->anchm.n = base_a; return fail(h, 3, err); }
    w->obs[base + i] = o;
    ObsJ &r = oj[i];
    if (p.type != D2BA_PROJ_DEPTH_PRIOR) {
      tmin = std::min(tmin, std::min(p.td_i, p.td_j)); tmax = std::max(tmax, std::max(p.td_i, p.td_j));
      // anchor half: bitwise identical to the previous anchor -> share it
      if (na == base_a || memcmp(last.pts_i, p.pts_i, 24) != 0 || memcmp(last.vel_i, p.vel_i, 24) != 0 || memcmp(&last.td_i, &p.td_i, 8) != 0) {
        memcpy(last.pts_i, p.pts_i, 24); memcpy(last.vel_i, p.vel_i, 24); last.td_i = p.td_i;
        ObsAnchor ta; ObsAnchorM tm;
        memcpy(ta.pts_i, p.pts_i, 24); memcpy(tm.vel_i, p.vel_i, 24); tm.td_i = p.td_i;
        an[na] = ta; anm[na] = tm; na++;
      }
      ObsJ t; ObsJm tm;
      memcpy(t.pts_j, p.pts_j, 24); memcpy(tm.vel_j, p.vel_j, 24); tm.td_j = p.td_j;
      t.depth = p.type == D2BA_PROJ_2F1C_DEPTH ? p.depth : 0.0;
      t.anchor = (int32_t)(na - 1); t.type = p.type;
      r = t; ojm[i] = tm;   // sequential store bursts
    } else {
      ObsJ t; memset(&t, 0, sizeof t);
      ObsJm tm; memset(&tm, 0, sizeof tm);
      t.depth = p.depth; t.anchor = 0; t.type = p.type;
      r = t; ojm[i] = tm;
    }
  }
  w->td_min = tmin; w->td_max = tmax;
  w->rawj.n += (size_t)n; w->rawjm.n += (size_t)n; w->anch.n = na; w->anchm.n = na;
  lap(0);
  // the uploads overlap with the caller preparing the other blocks / windows; issued in batches (flush_pending)
  win_unlock(w); unlock_at_exit.w = nullptr;
  {
    std::lock_guard<std::mutex> lk(h->pend_mu);
    if (!w->push_pending) { w->push_pending = true; h->pending_win.push_back(window); }
  }
  int rc = 0;
  if ((h->pending_bytes += (long long)n * (long long)sizeof(ObsJ)) >= kPushBatch && h->push_mu.try_lock()) {
    rc = flush_pending(h, false);
    h->push_mu.unlock();
  }
  lap(2);
  return rc;
}

int d2ba_add_landmark_tracks(d2ba_handle *h, int32_t window, int32_t n_landmarks, const int64_t *landmark_ids,
                             const int32_t *track_ptr, const d2ba_track_obs *tobs, int32_t fuse_dep, double min_d,
                             double max_d, int32_t n_ignore, const int64_t *ignore) {
  // Anchor / factor-type dispatch of D2Estimator::setupLandmarkFactors (d2estimator.cpp:796-874).
  auto ignored = [&](int64_t f) { for (int k = 0; k < n_ignore; k++) if (ignore[k] == f) return true; return false; };
  auto depth_ok = [&](const d2ba_track_obs &t) { return t.depth_mea && fuse_dep && t.depth < max_d && t.depth > min_d; };
  std::vector<d2ba_proj_obs> out;
  for (int l = 0; l < n_landmarks; l++) {
    const int b = track_ptr[l], e = track_ptr[l + 1];
    if (e <= b) continue;
    const d2ba_track_obs &anchor = tobs[b];
    if (ignored(anchor.frame_id)) continue;
    if (depth_ok(anchor)) {
      d2ba_proj_obs p; memset(&p, 0, sizeof p);
      p.type = D2BA_PROJ_DEPTH_PRIOR; p.frame_a = anchor.frame_id; p.cam_a = anchor.camera_id; p.landmark_id = landmark_ids[l]; p.depth = anchor.depth;
      out.push_back(p);
    }
    for (int k = b + 1; k < e; k++) {
      const d2ba_track_obs &t = tobs[k];
      if (ignored(t.frame_id)) continue;
      const bool same_cam = t.camera_id == anchor.camera_id, same_frame = t.frame_id == anchor.frame_id;
      if (same_cam && same_frame) continue;
      d2ba_proj_obs p; memset(&p, 0, sizeof p);
      p.frame_a = anchor.frame_id; p.frame_b = t.frame_id; p.cam_a = anchor.camera_id; p.cam_b = t.camera_id; p.landmark_id = landmark_ids[l];
      memcpy(p.pts_i, anchor.pt3d_norm, 24); memcpy(p.pts_j, t.pt3d_norm, 24); memcpy(p.vel_i, anchor.velocity, 24); memcpy(p.vel_j, t.velocity, 24);
      p.td_i = anchor.cur_td; p.td_j = t.cur_td;
      if (same_cam) { if (depth_ok(t)) { p.type = D2BA_PROJ_2F1C_DEPTH; p.depth = t.depth; } else p.type = D2BA_PROJ_2F1C; }
      else p.type = same_frame ? D2BA_PROJ_1F2C : D2BA_PROJ_2F2C;
      out.push_back(p);
    }
  }
  return d2ba_add_proj(h, window, (int)out.size(), out.data());
}

int d2ba_add_imu(d2ba_handle *h, int32_t window, int32_t n, const d2ba_imu *in) {
  HostWin *w = get_win(h, window);
  if (!w) return 1;
  w->used = true; h->finalized = false;
  for (int i = 0; i < n; i++) {
    HImu m;
    m.pi = find_in(w->pose_map, in[i].frame_a); m.pj = find_in(w->pose_map, in[i].frame_b);
    m.si = find_in(w->sb_map, in[i].frame_a); m.sj = find_in(w->sb_map, in[i].frame_b);
    if (m.pi < 0 || m.pj < 0 || m.si < 0 || m.sj < 0) return fail(h, 6, "add_imu: unknown frame id");
    double *c = m.c;
    c[0] = in[i].sum_dt; memcpy(c + 1, in[i].delta_p, 24); memcpy(c + 4, in[i].delta_q, 32); memcpy(c + 8, in[i].delta_v, 24);
    memcpy(c + 11, in[i].linearized_ba, 24); memcpy(c + 14, in[i].linearized_bg, 24);
    memcpy(c + 17, in[i].jacobian, 225 * 8); memcpy(c + 17 + 225, in[i].covariance, 225 * 8);
    w->imu.push_back(m);
  }
  return 0;
}

static int set_prior_common(d2ba_handle *h, int32_t window, int32_t m, const double *J, const double *e0, int32_t nblk,
                            const d2ba_blockref *refs, const double *x0, bool is_info) {
  HostWin *w = get_win(h, window);
  if (!w) return 1;
  w->used = true; h->finalized = false;
  w->prior_m = m; w->prior_J.assign(J, J + (size_t)m * m); w->prior_e0.assign(e0, e0 + m); w->prior_is_info = is_info;
  w->prior_blk.clear();
  int off = 0, xo = 0;
  for (int i = 0; i < nblk; i++) {
    HPriorBlk b; memset(&b, 0, sizeof b);
    b.kind = refs[i].kind;
    switch (b.kind) {
      case D2BA_POSE: b.index = find_in(w->pose_map, refs[i].id); break;
      case D2BA_EXTRINSIC: b.index = find_in(w->ext_map, refs[i].id); break;
      case D2BA_SPEED_BIAS: b.index = find_in(w->sb_map, refs[i].id); break;
      case D2BA_TD: b.index = w->has_td ? 0 : -1; break;
      case D2BA_LANDMARK: b.index = find_in(w->lm_map, refs[i].id); break;
      default: b.index = -1;
    }
    if (b.index < 0) return fail(h, 7, "set_prior: unknown block");
    b.off = off; b.eff = kind_eff(b.kind); off += b.eff;
    memcpy(b.x0, x0 + xo, 8 * kind_size(b.kind)); xo += kind_size(b.kind);
    w->prior_blk.push_back(b);
  }
  if (off != m) return fail(h, 8, "set_prior: dimension mismatch");
  return 0;
}

int d2ba_set_prior(d2ba_handle *h, int32_t window, int32_t m, const double *J, const double *e0, int32_t nblk,
                   const d2ba_blockref *refs, const double *x0) {
  return set_prior_common(h, window, m, J, e0, nblk, refs, x0, false);
}

int d2ba_set_consensus(d2ba_handle *h, int32_t window, int32_t n, const d2ba_blockref *refs, const int32_t *slot,
                       int32_t n_slots_global) {
  HostWin *w = get_win(h, window);
  if (!w) return 1;
  if (n_slots_global <= 0) return fail(h, 9, "set_consensus: n_slots_global must be positive");
  for (int i = 0; i < n; i++)
    if (slot[i] < 0 || slot[i] >= n_slots_global) return fail(h, 9, "set_consensus: slot index outside [0, n_slots_global)");
  w->used = true; h->finalized = false; w->admm = true; w->n_slots = n_slots_global;
  for (int i = 0; i < n; i++) {
    if (refs[i].kind == D2BA_POSE) { int k = find_in(w->pose_map, refs[i].id); if (k < 0) return fail(h, 9, "set_consensus: unknown frame"); w->pose_slot[k] = slot[i]; }
    else if (refs[i].kind == D2BA_EXTRINSIC) { int k = find_in(w->ext_map, refs[i].id); if (k < 0) return fail(h, 9, "set_consensus: unknown camera"); w->ext_slot[k] = slot[i]; }
    else return fail(h, 10, "set_consensus: only POSE / EXTRINSIC blocks take part");
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------ finalize
}  // extern "C"

namespace {

struct WinPlan {
  WinDesc d;
  std::vector<Group> groups;
  std::vector<int> grp_begin, grp_cnt, grp_tile0;   // sorted-obs range and first (window-local) tile of each group
  std::vector<Job> jobs[6];                         // tile_begin window-local, grp window-local
  std::vector<SchurTileH> schur[2];                  // stage 0 (tiles with leaf columns), stage 1 (hub x hub)
  std::vector<int> schur_chunks;                     // chunk lists, window-local offsets in SchurTile::cb
  std::vector<uint64_t> hruns; std::vector<Leaf> leaves; std::vector<HSeg> hseg; std::vector<unsigned long long> lm_mask; std::vector<int> leaf_lm; int leaf_lm_off = 0;
  int n_tiles = 0, n_lmobs = 0;
  int job_off[6] = {0, 0, 0, 0, 0, 0};
  int schur_off[2] = {0, 0}, chunk_off = 0;
};

template <typename F>
void parallel_for(int n, F f) {
  int nt = (int)std::thread::hardware_concurrency();
  { cpu_set_t cs; CPU_ZERO(&cs); if (sched_getaffinity(0, sizeof cs, &cs) == 0 && CPU_COUNT(&cs) > 0) nt = CPU_COUNT(&cs); }   // the cores this process may run on
  if (nt < 1) nt = 1;
  if (nt > 32) nt = 32;
  if (nt > n) nt = n;
  if (nt <= 1) { for (int i = 0; i < n; i++) f(i); return; }
  std::atomic<int> next(0);
  std::vector<std::thread> th;
  for (int t = 0; t < nt; t++) th.emplace_back([&]() { for (;;) { int i = next.fetch_add(1); if (i >= n) break; f(i); } });
  for (auto &t : th) t.join();
}

template <typename T>
struct HView {   // typed slice of the pinned staging arena
  T *p = nullptr; size_t n = 0, off = 0;
};
struct Staging {   // every array finalize uploads lives in ONE pinned arena -> one H2D copy into one device arena
  HBuf<char> arena; size_t cursor = 0;
  HView<WinDesc> win; HView<double> x6, xsb, xlm, xtd, imu_c, prior_J, prior_e0;
  HView<int> col6, colsb, tile_grp, tile_win, obs_lm, tile_src, lm_ptr, obs_slot, slot6, lm_win, blk_win, sb_win, pr_m, pr_info;
  HView<long long> raw_off;
  HView<long long> pr_offJ, pr_offv;
  HView<Group> grp; HView<Job> job; HView<ImuDesc> imu; HView<PriorBlk> pblk; HView<SchurTileH> schur;
  HView<int> schur_chunks, leaf_lm; HView<Leaf> leaf; HView<HSeg> hseg; HView<unsigned long long> lm_mask;
  template <typename T> void reserve(HView<T> &v, size_t count) { v.n = count; v.off = cursor; cursor += (count * sizeof(T) + 255) & ~(size_t)255; }
  template <typename T> void place(HView<T> &v) { v.p = (T *)(arena.p + v.off); }
};
std::map<d2ba_handle *, Staging *> g_staging;   // owned per handle, freed in d2ba_destroy
std::mutex g_staging_mu;

Staging *staging_of(d2ba_handle *h) {
  std::lock_guard<std::mutex> lk(g_staging_mu);
  auto it = g_staging.find(h);
  if (it != g_staging.end()) return it->second;
  Staging *s = new Staging();
  g_staging[h] = s;
  return s;
}

template <typename T>
int up(d2ba_handle *h, DBuf<T> &b, const HView<T> &v) {   // the data travels with the single arena copy
  b.bind(h->d_arena.p, v.off, v.n);
  return 0;
}

}  // namespace

void d2ba_release_staging(d2ba_handle *h) {
  std::lock_guard<std::mutex> lk(g_staging_mu);
  auto it = g_staging.find(h);
  if (it == g_staging.end()) return;
  Staging *s = it->second;
  s->arena.release();
  delete s;
  g_staging.erase(it);
}

extern "C" {

int d2ba_finalize(d2ba_handle *h) {
  if (!h) return 1;
  cudaSetDevice(h->cfg.device);
  release_graph(h);
  int nw = 0;
  for (size_t i = 0; i < h->win.size(); i++) {
    if (h->win[i].used) { if ((int)i != nw) return fail(h, 20, "windows must be used contiguously from index 0"); nw++; }
  }
  if (nw == 0) return fail(h, 22, "finalize: no window in use");
  Staging &st = *staging_of(h);
  // the pinned staging buffers are rewritten below: wait for the uploads of the previous finalize of this handle
  // (normally long complete -- a solve synchronises the stream); the uploads enqueued by THIS call are not waited for
  CK(cudaStreamSynchronize(h->stream));
  { std::lock_guard<std::mutex> lk(h->push_mu); int rcp = flush_pending(h, true); if (rcp) return rcp; }   // the rest of the record uploads run beside the planning below
  for (int wi = 0; wi < nw; wi++) {   // motion halves: only where td - td_i can be non-zero (td free, or a stamp that differs from td)
    HostWin &w = h->win[wi];
    if (!motion_needed(w)) continue;
    int rcp;
    if ((rcp = push_range(h, w.rawjm, w.d_rawjm, w.pushed_jm)) || (rcp = push_range(h, w.anchm, w.d_anchm, w.pushed_am))) return rcp;
    w.pushed_jm = w.rawjm.n; w.pushed_am = w.anchm.n;
  }
  auto tp0 = std::chrono::steady_clock::now();
  auto lap = [&](int slot) { auto t = std::chrono::steady_clock::now(); h->host_ms[slot] = std::chrono::duration<double, std::milli>(t - tp0).count(); tp0 = t; };
  std::vector<WinPlan> plan(nw);
  size_t total_obs = 0;
  for (int i = 0; i < nw; i++) total_obs += h->win[i].obs.size();
  const int tiles_est = (int)(total_obs / kTile) + nw;
  int n_sm = 132;   // H100 SXM; the device's own count when it can be read
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, h->cfg.device);
  const int tpj_target = std::max(1, std::min(8, tiles_est / (n_sm * 8)));
  // ---- pass A (parallel): columns, pair-major order, groups, tiles, jobs, Schur tiles
  parallel_for(nw, [&](int wi) {
    HostWin &w = h->win[wi];
    WinPlan &pl = plan[wi];
    WinDesc &d = pl.d; memset(&d, 0, sizeof d);
    const int np = (int)w.pose_id.size(), ne = (int)w.ext_id.size(), nsb = (int)w.sb_id.size(), nl = (int)w.lm_id.size();
    d.np = np; d.ne = ne; d.n6 = np + ne; d.nsb = nsb; d.nl = nl; d.has_td = w.has_td ? 1 : 0;
    // ---- leaves: connected components (through co-observation) of the free pose blocks that no IMU factor / prior
    //      touches -- the remote frames of another drone in a multi-agent window (d2vinsstate.cpp:476-485: no speed-bias).
    //      They couple only to themselves and to the hub (own frames, extrinsics, td), so they are eliminated from the
    //      reduced system before the dense Cholesky.  Reduced columns: [leaf 0 | leaf 1 | ... | hub poses | ext | td | sb].
    std::vector<int> leaf_of(np, -1);
    std::vector<std::vector<int>> leaves;
    int nsb_free = 0, n6_free = 0;
    for (int i = 0; i < nsb; i++) if (!w.sb_c[i]) nsb_free++;
    for (int i = 0; i < np; i++) if (!w.pose_c[i]) n6_free++;
    for (int i = 0; i < ne; i++) if (!w.ext_c[i]) n6_free++;
    const bool td_free = w.has_td && !w.td_c;
    const int nlc_cnt = 6 * n6_free + (td_free ? 1 : 0), nc_cnt = nlc_cnt + 9 * nsb_free;
    bool sb_ok;
    {   // speed-bias elimination: needs a block-tridiagonal speed-bias part (IMU factors / prior blocks only between
        // neighbouring speed-bias blocks); the test does not depend on the column order
      std::vector<int> pos(nsb, -1);
      int nb = 0;
      for (int i = 0; i < nsb; i++) if (!w.sb_c[i]) pos[i] = nb++;
      sb_ok = !h->force_full_S && !h->no_sb_elim && nb >= 1 && nlc_cnt >= 1;
      for (size_t a = 0; a < w.imu.size() && sb_ok; a++) {
        const int pa = pos[w.imu[a].si], pb = pos[w.imu[a].sj];
        if (pa >= 0 && pb >= 0 && std::abs(pa - pb) > 1) sb_ok = false;
      }
      int pmin = 1 << 30, pmax = -1;
      for (const HPriorBlk &b : w.prior_blk) if (b.kind == D2BA_SPEED_BIAS && pos[b.index] >= 0) { pmin = std::min(pmin, pos[b.index]); pmax = std::max(pmax, pos[b.index]); }
      if (pmax - pmin > 1) sb_ok = false;
      if (sb_ok && nb > sb_max_blocks()) sb_ok = false;
      d.n_sbe = nb;
    }
    if (!h->force_full_S && !h->no_leaf && (sb_ok || nsb_free == 0) && nlc_cnt + 1 > 96) {   // small systems keep the one-CTA dense path (k_schur_small)
      std::vector<char> hub(np, 0);
      for (const HImu &m : w.imu) { hub[m.pi] = 1; hub[m.pj] = 1; }
      for (const HPriorBlk &b : w.prior_blk) if (b.kind == D2BA_POSE) hub[b.index] = 1;
      std::vector<int> uf(np);
      for (int i = 0; i < np; i++) uf[i] = i;
      auto find = [&](int x) { while (uf[x] != x) { uf[x] = uf[uf[x]]; x = uf[x]; } return x; };
      // two poses belong to one component when some landmark is observed from both (the landmark's elimination couples them)
      std::vector<int> first_pose(nl, -1);
      for (const HObs &o : w.obs) {
        const int ps[2] = {o.pi, o.pj};
        for (int q = 0; q < 2; q++) {
          const int pz = ps[q];
          if (pz < 0 || hub[pz] || w.pose_c[pz]) continue;
          if (first_pose[o.lm] < 0) { first_pose[o.lm] = pz; continue; }
          const int a = find(pz), b = find(first_pose[o.lm]);
          if (a != b) uf[std::max(a, b)] = std::min(a, b);
        }
      }
      std::vector<int> comp_id(np, -1);
      for (int i = 0; i < np; i++) {
        if (hub[i] || w.pose_c[i]) continue;
        const int r = find(i);
        if (comp_id[r] < 0) { comp_id[r] = (int)leaves.size(); leaves.emplace_back(); }
        leaves[comp_id[r]].push_back(i);
      }
      // a leaf must fit the elimination kernel's shared memory together with its hub coupling; otherwise it stays in the hub
      int n_hub_cols = nlc_cnt;
      for (auto &lf : leaves) n_hub_cols -= 6 * (int)lf.size();
      std::vector<std::vector<int>> kept;
      for (auto &lf : leaves) {
        const int nl6 = 6 * (int)lf.size();
        if (nl6 <= leaf_max_cols() && n_hub_cols >= 1 && leaf_elim_smem(nl6, n_hub_cols) <= (size_t)200 * 1024) kept.push_back(lf);
        else n_hub_cols += nl6;
      }
      // worthwhile only when the hub is a real reduction of the dense part
      if (kept.empty() || n_hub_cols > 3 * nlc_cnt / 4) kept.clear();
      leaves.swap(kept);
      for (size_t li = 0; li < leaves.size(); li++) for (int i : leaves[li]) leaf_of[i] = (int)li;
    }
    int c = 0;
    w.pose_col.assign(np, -1); w.ext_col.assign(ne, -1); w.sb_col.assign(nsb, -1);
    pl.leaves.clear();
    for (size_t li = 0; li < leaves.size(); li++) {
      Leaf lf; memset(&lf, 0, sizeof lf);
      lf.win = wi; lf.col0 = c; lf.n = 6 * (int)leaves[li].size();
      for (int i : leaves[li]) { w.pose_col[i] = c; c += 6; }
      pl.leaves.push_back(lf);
    }
    d.hub0 = c;
    for (int i = 0; i < np; i++) if (!w.pose_c[i] && leaf_of[i] < 0) { w.pose_col[i] = c; c += 6; }
    for (int i = 0; i < ne; i++) if (!w.ext_c[i]) { w.ext_col[i] = c; c += 6; }
    w.td_col = td_free ? c : -1;
    if (w.td_col >= 0) c += 1;
    w.n_lc = c;
    for (int i = 0; i < nsb; i++) if (!w.sb_c[i]) { w.sb_col[i] = c; c += 9; }
    w.n_c = c;
    d.n_hub = w.n_lc - d.hub0; d.n_leaf = (int)leaves.size();
    {   // canonical (insertion-order) columns for the debug views: canon_of_dev[device column] = column the oracle uses
      w.canon_of_dev.assign(w.n_c, -1);
      int cc = 0;
      for (int i = 0; i < np; i++) if (!w.pose_c[i]) { for (int q = 0; q < 6; q++) w.canon_of_dev[w.pose_col[i] + q] = cc + q; cc += 6; }
      for (int i = 0; i < ne; i++) if (!w.ext_c[i]) { for (int q = 0; q < 6; q++) w.canon_of_dev[w.ext_col[i] + q] = cc + q; cc += 6; }
      if (w.td_col >= 0) w.canon_of_dev[w.td_col] = cc++;
      for (int i = 0; i < nsb; i++) if (!w.sb_c[i]) { for (int q = 0; q < 9; q++) w.canon_of_dev[w.sb_col[i] + q] = cc + q; cc += 9; }
    }
    d.td_col = w.td_col; d.n_lc = w.n_lc; d.n_c = w.n_c; d.ldh = std::max(4, roundup(w.n_c, 4));
    d.ldw = roundup(w.n_lc + 1, 8); d.nl_pad = roundup(nl, 32);
    d.admm_on = w.admm ? 1 : 0; d.n_imu = (int)w.imu.size();
    d.chol_smem = (!h->force_full_S && w.n_c >= 1 && chol_smem_need(w.n_c) <= (size_t)232448 - 16) ? 1 : 0;   // 16 B of static shared memory (fail flag + mbarrier)
    d.prior_m = w.prior_m; d.prior_nblk = (int)w.prior_blk.size();
    // pair-major order: key = (type, pose_i, pose_j, ext_a, ext_b), ties by insertion order.  The number of distinct
    // keys is small (<= a few hundred), so this is a counting sort: key -> bucket via a flat hash, buckets ordered by key.
    const size_t M = w.obs.size();
    std::vector<std::pair<uint64_t, uint32_t>> keys(M);   // (key, bucket) then reused as (key, obs index) in sorted order
    {
      FlatMap bucket_of;                                     // key -> bucket id
      std::vector<uint64_t> bkey; std::vector<uint32_t> bcount;
      std::vector<uint32_t> ob(M);
      uint64_t last_key = ~0ull; int last_b = -1;
      for (size_t k = 0; k < M; k++) {
        const HObs &o = w.obs[k];
        const uint64_t key = ((uint64_t)(o.type & 0xF) << 60) | ((uint64_t)((o.pi + 1) & 0x7FFF) << 45) | ((uint64_t)((o.pj + 1) & 0x7FFF) << 30) |
                             ((uint64_t)((o.ea + 1) & 0x7FFF) << 15) | (uint64_t)((o.eb + 1) & 0x7FFF);
        int b;
        if (key == last_key) b = last_b;
        else {
          b = bucket_of.find((int64_t)key);
          if (b < 0) { b = (int)bkey.size(); bucket_of.put((int64_t)key, b); bkey.push_back(key); bcount.push_back(0); }
          last_key = key; last_b = b;
        }
        ob[k] = (uint32_t)b; bcount[b]++;
      }
      std::vector<uint32_t> border(bkey.size());
      for (size_t i = 0; i < border.size(); i++) border[i] = (uint32_t)i;
      std::sort(border.begin(), border.end(), [&](uint32_t a, uint32_t b) { return bkey[a] < bkey[b]; });
      std::vector<uint32_t> start(bkey.size());
      uint32_t run = 0;
      for (uint32_t bi : border) { start[bi] = run; run += bcount[bi]; }
      for (size_t k = 0; k < M; k++) { const uint32_t b = ob[k]; keys[start[b]++] = {bkey[b], (uint32_t)k}; }   // stable within a bucket
    }
    w.order.resize(M); w.sorted_pos.assign(M, -1);
    for (size_t k = 0; k < M; k++) w.order[k] = (int)keys[k].second;
    // Hcc pattern (lower triangle, block rows): rows[r] collects the [c0, c1) runs some factor writes
    // (one flat list of (row, c0, c1) runs, sorted and merged below: no per-row allocations on this per-solve path)
    std::vector<uint64_t> &hruns = pl.hruns;
    hruns.clear();
    auto hblock = [&](int ra, int rs, int ca, int cs) {
      if (ra < 0 || ca < 0) return;
      if (ra < ca) { std::swap(ra, ca); std::swap(rs, cs); }
      for (int r = 0; r < rs; r++) hruns.push_back(((uint64_t)(ra + r) << 40) | ((uint64_t)ca << 20) | (uint64_t)(ca + cs));
    };
    // landmark masks: W-space column tiles (32 columns) a landmark's coupling row touches; the rhs column n_lc always
    pl.lm_mask.assign(nl, 1ull << (w.n_lc / 32));
    auto mark = [&](int lm, int col, int width) { if (col >= 0) pl.lm_mask[lm] |= (1ull << (col / 32)) | (1ull << ((col + width - 1) / 32)); };
    bool any_wide = false;
    size_t k = 0; int tile_run = 0;
    while (k < M) {
      size_t e = k;
      while (e < M && keys[e].first == keys[k].first) e++;
      const HObs &o0 = w.obs[w.order[k]];
      Group g; memset(&g, 0, sizeof g);
      g.type = o0.type;
      g.blk[0] = o0.pi; g.blk[1] = o0.pj; g.blk[2] = o0.ea >= 0 ? np + o0.ea : -1; g.blk[3] = o0.eb >= 0 ? np + o0.eb : -1;
      int cols[4] = {o0.pi >= 0 ? w.pose_col[o0.pi] : -1, o0.pj >= 0 ? w.pose_col[o0.pj] : -1, o0.ea >= 0 ? w.ext_col[o0.ea] : -1,
                     o0.eb >= 0 ? w.ext_col[o0.eb] : -1};
      if (o0.type == D2BA_PROJ_DEPTH_PRIOR) { cols[0] = cols[1] = cols[2] = cols[3] = -1; }
      int ns = 0;
      for (int s = 0; s < 4; s++) { g.slot_src[s] = -1; g.slot_col[s] = -1; }
      for (int s = 0; s < 4; s++) if (cols[s] >= 0) { g.slot_src[ns] = s; g.slot_col[ns] = cols[s]; ns++; }
      g.td_col = (o0.type == D2BA_PROJ_DEPTH_PRIOR) ? -1 : w.td_col;
      g.need_td = g.td_col >= 0; g.need_ext = 0;
      for (int s = 0; s < ns; s++) if (g.slot_src[s] >= 2) g.need_ext = 1;
      g.nct = (ns <= 2 && !g.need_td) ? 2 : 4;
      g.rows = o0.type == D2BA_PROJ_2F1C_DEPTH ? 3 : (o0.type == D2BA_PROJ_DEPTH_PRIOR ? 1 : 2);
      if (g.nct == 4) any_wide = true;
      int variant = (g.nct == 4 ? 1 : 0) + (g.rows == 3 ? 2 : 0);
      // all shifts zero? (td constant and equal to every observation's stamp)
      g.shift0 = (!g.need_td && o0.type != D2BA_PROJ_DEPTH_PRIOR && w.td_min == w.td_max && w.td_min == w.td) ? 1 : 0;
      if (variant == 0 && !g.need_ext && (o0.type == D2BA_PROJ_2F1C || o0.type == D2BA_PROJ_2F2C) && ns == 2 && g.slot_src[0] == 0 && g.slot_src[1] == 1)
        variant = g.shift0 ? 4 : 5;
      const int cnt = (int)(e - k), ntile = (cnt + kTile - 1) / kTile;
      const int gi = (int)pl.groups.size();
      pl.groups.push_back(g); pl.grp_begin.push_back((int)k); pl.grp_cnt.push_back(cnt); pl.grp_tile0.push_back(tile_run);
      // pattern of the group's J^T J blocks and of its landmarks' coupling rows
      for (int a = 0; a < ns; a++) {
        for (int b = 0; b <= a; b++) hblock(g.slot_col[a], 6, g.slot_col[b], 6);
        if (g.td_col >= 0) hblock(g.td_col, 1, g.slot_col[a], 6);
      }
      if (g.td_col >= 0) hblock(g.td_col, 1, g.td_col, 1);
      for (size_t q = k; q < e; q++) {
        const int lm = w.obs[w.order[q]].lm;
        for (int a = 0; a < ns; a++) mark(lm, g.slot_col[a], 6);
        mark(lm, g.td_col, 1);
      }
      // balanced split of the group's tiles into jobs
      const int njob = (ntile + tpj_target - 1) / tpj_target;
      for (int j = 0; j < njob; j++) {
        int b = (int)((int64_t)ntile * j / njob), en = (int)((int64_t)ntile * (j + 1) / njob);
        Job jb; jb.win = wi; jb.grp = gi; jb.tile_begin = tile_run + b; jb.ntiles = en - b;
        pl.jobs[variant].push_back(jb);
      }
      tile_run += ntile;
      k = e;
    }
    pl.n_tiles = tile_run; d.n_tile = tile_run; d.n_grp = (int)pl.groups.size();
    {   // may k_lm_gather16 skip the barrier between records?  Only if, per landmark, no column block shows up at slot 0 of one
        // record and at slot 1 of another (then every row entry is owned by one lane).  True for the reference's graphs:
        // slot 0 is the anchor pose of the landmark, the other slot an observing frame.
      std::vector<int> s0(nl, -1);   // the landmark's slot-0 column (-2: more than one -> keep the barrier)
      bool clash = false;
      for (int gi = 0; gi < (int)pl.groups.size() && !clash; gi++) {
        const int c0g = pl.groups[gi].slot_col[0];
        if (c0g < 0) continue;
        for (int q = pl.grp_begin[gi]; q < pl.grp_begin[gi] + pl.grp_cnt[gi]; q++) {
          int &s = s0[w.obs[w.order[q]].lm];
          if (s == -1) s = c0g; else if (s != c0g) { clash = true; break; }
        }
      }
      for (int gi = 0; gi < (int)pl.groups.size() && !clash; gi++) {
        const int c1g = pl.groups[gi].slot_col[1];
        if (c1g < 0) continue;
        for (int q = pl.grp_begin[gi]; q < pl.grp_begin[gi] + pl.grp_cnt[gi]; q++) if (s0[w.obs[w.order[q]].lm] == c1g) { clash = true; break; }
      }
      d.gather_nosync = clash ? 0 : 1;
    }
    {   // landmarks of every leaf (ascending, each once) and the widest coupling row in 32-column tiles
      pl.leaf_lm.clear();
      std::vector<std::vector<int>> per_leaf(pl.leaves.size());
      if (!pl.leaves.empty()) {
        std::vector<int> last_leaf_of_lm(nl, -1);   // landmark-major obs order is not given: dedupe per (landmark, leaf) with a stamp matrix
        std::vector<char> seen((size_t)nl * pl.leaves.size(), 0);
        for (const HObs &o : w.obs) {
          const int ps[2] = {o.pi, o.pj};
          for (int q = 0; q < 2; q++) if (ps[q] >= 0 && leaf_of[ps[q]] >= 0) {
            char &sn = seen[(size_t)o.lm * pl.leaves.size() + leaf_of[ps[q]]];
            if (!sn) { sn = 1; per_leaf[leaf_of[ps[q]]].push_back(o.lm); }
          }
        }
        (void)last_leaf_of_lm;
      }
      for (size_t li = 0; li < pl.leaves.size(); li++) {
        std::sort(per_leaf[li].begin(), per_leaf[li].end());
        pl.leaves[li].lm_begin = (int)pl.leaf_lm.size(); pl.leaves[li].lm_count = (int)per_leaf[li].size();
        pl.leaf_lm.insert(pl.leaf_lm.end(), per_leaf[li].begin(), per_leaf[li].end());
      }
      int rt = 1;
      if (pl.leaves.empty()) rt = w.n_lc / 32 + 1;
      else for (int l = 0; l < nl; l++) rt = std::max(rt, __builtin_popcountll(pl.lm_mask[l]));
      d.row_tiles = rt;
    }
    d.rec_stride = any_wide ? 32 : 16;
    pl.n_lmobs = (int)M;
    d.schur_small = (d.n_lc + 1 <= 96) ? 1 : 0;
    d.hub_small = (d.n_leaf > 0 && d.n_hub + 1 <= 96) ? 1 : 0;
    {
      const int nb = d.n_sbe;
      const int hubw = roundup(d.n_hub + 1, 8);
      bool ok = sb_ok && w.n_c == w.n_lc + 9 * nb;
      if (ok && (sb_elim_smem(hubw, d.n_c, nb) > (size_t)200 * 1024 || sb_back_smem(d.n_hub, nb) > (size_t)200 * 1024)) ok = false;
      if (!ok && d.n_leaf > 0 && nb > 0) { h->err = "internal: leaves without speed-bias elimination"; }
      d.sb_elim = ok ? 1 : 0;
      // the dense Cholesky only sees the hub of the pose part then: decide its kernel with that size
      if (ok || d.n_leaf > 0) d.chol_smem = (chol_smem_need(d.n_hub) <= (size_t)232448 - 16) ? 1 : 0;
      // rows of Wt the Schur kernels sum over: landmark rows, then the eliminated speed-bias rows, then the leaves' rows
      int rows = nl + (ok ? 9 * nb : 0);
      for (Leaf &lf : pl.leaves) { lf.row0 = rows; rows += lf.n; }
      d.wt_rows = roundup(std::max(rows, 1), 32);
    }
    // other Hcc blocks: IMU factors, prior, ADMM terms
    for (const HImu &m : w.imu) {
      const int bc[4] = {w.pose_col[m.pi], w.sb_col[m.si], w.pose_col[m.pj], w.sb_col[m.sj]}, bs[4] = {6, 9, 6, 9};
      for (int a = 0; a < 4; a++) for (int b = 0; b <= a; b++) hblock(bc[a], bs[a], bc[b], bs[b]);
    }
    {
      std::vector<std::pair<int, int>> pb;
      for (const HPriorBlk &b : w.prior_blk) {
        int col = b.kind == D2BA_POSE ? w.pose_col[b.index] : b.kind == D2BA_EXTRINSIC ? w.ext_col[b.index] : b.kind == D2BA_SPEED_BIAS ? w.sb_col[b.index] : b.kind == D2BA_TD ? w.td_col : -1;
        if (col >= 0) pb.push_back({col, b.eff});
      }
      for (size_t a = 0; a < pb.size(); a++) for (size_t b = 0; b <= a; b++) hblock(pb[a].first, pb[a].second, pb[b].first, pb[b].second);
    }
    if (w.admm) {
      for (int i = 0; i < np; i++) if (w.pose_slot[i] >= 0) hblock(w.pose_col[i], 6, w.pose_col[i], 6);
      for (int i = 0; i < ne; i++) if (w.ext_slot[i] >= 0) hblock(w.ext_col[i], 6, w.ext_col[i], 6);
      for (int i = 0; i < nsb; i++) hblock(w.sb_col[i], 9, w.sb_col[i], 9);
      if (w.td_col >= 0) hblock(w.td_col, 1, w.td_col, 1);
    }
    pl.hseg.clear();
    std::sort(hruns.begin(), hruns.end());
    for (size_t q = 0; q < hruns.size();) {
      const int r = (int)(hruns[q] >> 40);
      int a = (int)((hruns[q] >> 20) & 0xFFFFF), bnd = (int)(hruns[q] & 0xFFFFF);
      size_t e2 = q + 1;
      for (; e2 < hruns.size() && (int)(hruns[e2] >> 40) == r; e2++) {
        const int c0 = (int)((hruns[e2] >> 20) & 0xFFFFF), c1 = (int)(hruns[e2] & 0xFFFFF);
        if (c0 <= bnd) { bnd = std::max(bnd, c1); continue; }
        pl.hseg.push_back(HSeg{r, a, std::min(bnd, r + 1) - a});   // lower triangle only
        a = c0; bnd = c1;
      }
      pl.hseg.push_back(HSeg{r, a, std::min(bnd, r + 1) - a});
      q = e2;
    }
    d.n_hseg = (int)pl.hseg.size();
    if (!d.schur_small) {
      // ---- Schur tiles with their 32-row chunk lists.  A chunk of Wt rows takes part in tile (tm, tn) iff some row of it
      //      has entries in both column tiles.  Stage 0 = tiles with leaf columns (computed before the leaf elimination,
      //      landmark rows only), stage 1 = tiles of the hub x hub part (after it: landmark rows + all eliminated rows).
      const int ntw = (d.n_lc + 1 + 31) / 32, nchunk = d.wt_rows / 32;
      std::vector<unsigned long long> cmask(nchunk, 0ull);
      for (int l = 0; l < nl; l++) cmask[l / 32] |= pl.lm_mask[l];
      unsigned long long hubmask = 0ull;
      for (int t = d.hub0 / 32; t <= d.n_lc / 32; t++) hubmask |= 1ull << t;
      const int first_elim_row = nl;
      for (int r = nl; r < d.wt_rows; r++) cmask[r / 32] |= hubmask;   // eliminated rows (and the zero padding): hub columns + rhs
      const int lm_chunks = (nl + 31) / 32;
      (void)first_elim_row;
      // tile pattern of Hcc (a tile without chunks still copies Hcc into S)
      std::vector<char> hpat((size_t)ntw * ntw, 0);
      for (const HSeg &sg : pl.hseg) if (sg.row < d.n_lc) for (int cidx = sg.c0; cidx < sg.c0 + sg.len; cidx += 1) { hpat[(size_t)(sg.row / 32) * ntw + cidx / 32] = 1; }
      for (int stage = 0; stage < 2; stage++)
        for (int tm = 0; tm < ntw && d.n_lc > 0; tm++)
          for (int tn = 0; tn <= tm; tn++) {
            const bool in_hub = (tm * 32 + 31 >= d.hub0) && (tn * 32 + 31 >= d.hub0);
            const bool has_leaf = tn * 32 < d.hub0;
            if (stage == 0 ? !has_leaf : (!in_hub || d.hub_small)) continue;   // hub_small: k_schur_small forms the hub x hub part
            SchurTileH t{wi, stage == 0 ? 2 : 0, tm, tn, (int)pl.schur_chunks.size(), 0};   // kind 2: only entries in leaf columns are stored
            const int kend = stage == 0 ? lm_chunks : nchunk;
            for (int kc = 0; kc < kend; kc++) if (((cmask[kc] >> tm) & 1ull) && ((cmask[kc] >> tn) & 1ull)) pl.schur_chunks.push_back(kc);
            t.cn = (int)pl.schur_chunks.size() - t.cb;
            if (t.cn == 0 && !hpat[(size_t)tm * ntw + tn] && tm != ntw - 1) continue;   // structurally zero tile: never read
            pl.schur[stage].push_back(t);
          }
      int t_lo = d.n_lc / 32, t_hi = d.n_c / 32;
      if (!d.sb_elim) for (int tm = t_lo; tm <= t_hi; tm++) for (int tn = 0; tn <= tm; tn++) pl.schur[1].push_back(SchurTileH{wi, 1, tm, tn, 0, 0});
    }
  });
  lap(0);
  // ---- serial prefix sums
  h->n_used = nw; h->max_rows = 1; h->max_nc = 1; h->max_prior_m = 0; h->max_ldw = 8; h->n_slots = 0; h->any_admm = false;
  h->max_row_tiles = 1; h->max_n_smem = 0; h->max_rows_glob = 1; h->any_chol_glob = false; h->max_ldw_small = 0; h->any_compact = h->any_wide = 0; h->sbe_smem = 0; h->sbb_smem = 0;
  int64_t offLE = 0;
  int off6 = 0, offsb = 0, offlm = 0, off_tile = 0, off_grp = 0, off_imu = 0, off_lmptr = 0, off_pblk = 0, n_schur = 0, n_sch[2] = {0, 0}, n_chunks = 0, off_leaf = 0, off_hseg = 0, n_leaf_lm = 0;
  int64_t offLL = 0; size_t leaf_smem = 0, leafb_smem = 0; int max_hub = 0;
  int64_t offH = 0, offW = 0, offc = 0, off_lmobs = 0, off_pJ = 0, off_pv = 0, off_rec = 0; long long off_raw = 0;
  int njobs[6] = {0, 0, 0, 0, 0, 0};
  bool any_info = false;
  for (int wi = 0; wi < nw; wi++) {
    HostWin &w = h->win[wi]; WinPlan &pl = plan[wi]; WinDesc &d = pl.d;
    d.off6 = off6; off6 += d.n6; d.offsb = offsb; offsb += d.nsb; d.offlm = offlm; offlm += d.nl;
    d.off_tile = off_tile; off_tile += d.n_tile; d.off_rec = off_rec; off_rec += (int64_t)std::max(pl.n_lmobs, 1) * d.rec_stride;
    d.off_grp = off_grp; off_grp += d.n_grp; d.off_imu = off_imu; off_imu += d.n_imu;
    d.off_lmptr = off_lmptr; off_lmptr += d.nl + 1; d.off_lmobs = off_lmobs; off_lmobs += pl.n_lmobs;
    d.off_prior_blk = off_pblk; off_pblk += d.prior_nblk; d.off_prior_J = off_pJ; d.off_prior_v = off_pv;
    off_pJ += (int64_t)d.prior_m * d.prior_m; off_pv += d.prior_m;
    d.offH = offH; offH += (int64_t)(d.n_c + 1) * d.ldh;
    d.offW = offW; offW += (int64_t)std::max(d.wt_rows, 32) * d.ldw;
    d.offc = offc; offc += roundup(d.n_c + 1, 4);
    for (int v = 0; v < 6; v++) { pl.job_off[v] = njobs[v]; njobs[v] += (int)pl.jobs[v].size(); }
    for (int sg = 0; sg < 2; sg++) { pl.schur_off[sg] = n_sch[sg]; n_sch[sg] += (int)pl.schur[sg].size(); }
    pl.chunk_off = n_chunks; n_chunks += (int)pl.schur_chunks.size();
    pl.leaf_lm_off = n_leaf_lm; n_leaf_lm += (int)pl.leaf_lm.size();
    h->max_row_tiles = std::max(h->max_row_tiles, d.row_tiles);
    d.off_leaf = off_leaf; off_leaf += d.n_leaf; d.off_hseg = off_hseg; off_hseg += d.n_hseg;
    for (Leaf &lf : pl.leaves) { lf.offL = offLL; offLL += (int64_t)lf.n * lf.n + lf.n; leaf_smem = std::max(leaf_smem, leaf_elim_smem(lf.n, d.n_hub)); leafb_smem = std::max(leafb_smem, leaf_back_smem(lf.n, d.n_hub)); }
    max_hub = std::max(max_hub, d.n_hub);
    h->max_rows = std::max(h->max_rows, d.n_c + 1); h->max_nc = std::max(h->max_nc, d.n_c); h->max_ldw = std::max(h->max_ldw, d.ldw);
    h->max_prior_m = std::max(h->max_prior_m, d.prior_m);
    if (d.schur_small) h->max_ldw_small = std::max(h->max_ldw_small, d.ldw);
    if (d.hub_small) h->max_ldw_small = std::max(h->max_ldw_small, roundup(d.n_hub + 1, 8));
    if (d.rec_stride == 16) h->any_compact = 1; else h->any_wide = 1;
    if (d.sb_elim) {
      d.offLE = offLE; offLE += (int64_t)d.n_sbe * 171;
      h->sbe_smem = std::max(h->sbe_smem, sb_elim_smem(roundup(d.n_hub + 1, 8), d.n_c, d.n_sbe)); h->sbb_smem = std::max(h->sbb_smem, sb_back_smem(d.n_hub, d.n_sbe));
    }
    { const int ndense = (d.sb_elim || d.n_leaf > 0) ? d.n_hub : d.n_c;
      if (d.chol_smem) h->max_n_smem = std::max(h->max_n_smem, ndense); else { h->any_chol_glob = true; h->max_rows_glob = std::max(h->max_rows_glob, ndense + 1); } }
    if (w.admm) {
      if (h->any_admm && h->n_slots != w.n_slots) return fail(h, 26, "finalize: every window of a handle must name the same n_slots_global (the all-reduce count)");
      h->any_admm = true; h->n_slots = w.n_slots;
    }
    if (w.prior_m > 0 && w.prior_is_info) any_info = true;
  }
  int jbase[6]; { int r = 0; for (int v = 0; v < 6; v++) { jbase[v] = r; h->job_begin[v] = r; h->job_count[v] = njobs[v]; r += njobs[v]; } }
  const int n_jobs = jbase[5] + njobs[5];
  h->n6_total = off6; h->nsb_total = offsb; h->nl_total = offlm; h->n_tiles = off_tile; h->n_imu_total = off_imu; n_schur = n_sch[0] + n_sch[1]; h->n_schur = n_schur; h->n_schur0 = n_sch[0];
  h->n_leaf_total = off_leaf; h->leaf_smem = leaf_smem; h->leafb_smem = leafb_smem; h->max_hub = max_hub;
  h->totH = offH; h->totW = offW; h->totc = offc; h->totLE = offLE;
  // ---- staging sizes
  st.cursor = 0;
  st.reserve(st.win, nw); st.reserve(st.x6, (size_t)off6 * 8); st.reserve(st.xsb, (size_t)offsb * 9); st.reserve(st.xlm, offlm); st.reserve(st.xtd, nw);
  st.reserve(st.col6, off6); st.reserve(st.colsb, offsb); st.reserve(st.slot6, off6); st.reserve(st.blk_win, off6); st.reserve(st.sb_win, offsb);
  st.reserve(st.lm_win, offlm); st.reserve(st.tile_grp, off_tile); st.reserve(st.tile_win, off_tile); st.reserve(st.obs_lm, (size_t)off_tile * kTile);
  st.reserve(st.tile_src, (size_t)off_tile * kTile); st.reserve(st.raw_off, 4 * (size_t)nw); st.reserve(st.lm_ptr, off_lmptr); st.reserve(st.obs_slot, (size_t)off_tile * kTile);
  st.reserve(st.grp, off_grp); st.reserve(st.job, n_jobs); st.reserve(st.imu, off_imu); st.reserve(st.imu_c, (size_t)off_imu * kImuPack);
  st.reserve(st.pblk, off_pblk); st.reserve(st.prior_J, (size_t)off_pJ); st.reserve(st.prior_e0, (size_t)off_pv); st.reserve(st.schur, n_schur); st.reserve(st.schur_chunks, n_chunks); st.reserve(st.leaf, off_leaf); st.reserve(st.hseg, off_hseg); st.reserve(st.lm_mask, offlm); st.reserve(st.leaf_lm, n_leaf_lm);
  st.reserve(st.pr_m, nw); st.reserve(st.pr_info, nw); st.reserve(st.pr_offJ, nw); st.reserve(st.pr_offv, nw);
  bool ok = st.arena.resize(st.cursor + 256);
  if (ok) {
    st.place(st.win); st.place(st.x6); st.place(st.xsb); st.place(st.xlm); st.place(st.xtd); st.place(st.col6); st.place(st.colsb); st.place(st.slot6);
    st.place(st.blk_win); st.place(st.sb_win); st.place(st.lm_win); st.place(st.tile_grp); st.place(st.tile_win); st.place(st.obs_lm); st.place(st.tile_src);
    st.place(st.raw_off); st.place(st.lm_ptr); st.place(st.obs_slot); st.place(st.grp); st.place(st.job); st.place(st.imu); st.place(st.imu_c); st.place(st.pblk);
    st.place(st.prior_J); st.place(st.prior_e0); st.place(st.schur); st.place(st.schur_chunks); st.place(st.leaf); st.place(st.hseg); st.place(st.lm_mask); st.place(st.leaf_lm); st.place(st.pr_m); st.place(st.pr_info); st.place(st.pr_offJ); st.place(st.pr_offv);
  }
  if (!ok) return fail(h, 24, "pinned staging allocation failed");
  lap(1);
  // ---- pass B (parallel): fill the staging buffers
  std::atomic<int> skipped_any{0};
  parallel_for(nw, [&](int wi) {
    HostWin &w = h->win[wi]; WinPlan &pl = plan[wi]; const WinDesc &d = pl.d;
    st.win.p[wi] = d;
    const int np = d.np, ne = d.ne;
    for (int i = 0; i < np; i++) {
      double *x = st.x6.p + (size_t)(d.off6 + i) * 8; memcpy(x, &w.pose[7 * i], 56); x[7] = 0;
      st.col6.p[d.off6 + i] = w.pose_col[i]; st.slot6.p[d.off6 + i] = w.admm ? w.pose_slot[i] : -1; st.blk_win.p[d.off6 + i] = wi;
    }
    for (int i = 0; i < ne; i++) {
      double *x = st.x6.p + (size_t)(d.off6 + np + i) * 8; memcpy(x, &w.ext[7 * i], 56); x[7] = 0;
      st.col6.p[d.off6 + np + i] = w.ext_col[i]; st.slot6.p[d.off6 + np + i] = w.admm ? w.ext_slot[i] : -1; st.blk_win.p[d.off6 + np + i] = wi;
    }
    if (d.nsb) memcpy(st.xsb.p + (size_t)d.offsb * 9, w.sb.data(), (size_t)d.nsb * 72);
    for (int i = 0; i < d.nsb; i++) { st.colsb.p[d.offsb + i] = w.sb_col[i]; st.sb_win.p[d.offsb + i] = wi; }
    if (d.nl) memcpy(st.xlm.p + d.offlm, w.lm.data(), (size_t)d.nl * 8);
    for (int i = 0; i < d.nl; i++) st.lm_win.p[d.offlm + i] = wi;
    st.xtd.p[wi] = w.td;
    // tile tables: source record of every tile slot (the device builds the AoSoA constants from the raw records)
    // + landmark CSR by counting sort
    int *lmp = st.lm_ptr.p + d.off_lmptr;
    for (int l = 0; l <= d.nl; l++) lmp[l] = 0;
    for (const HObs &o : w.obs) lmp[o.lm + 1]++;
    for (int l = 0; l < d.nl; l++) lmp[l + 1] += lmp[l];
    std::vector<int> cursor(lmp, lmp + d.nl);
    int *oslot = st.obs_slot.p + (size_t)d.off_tile * kTile;   // tile slot -> record position (landmark-major), -1 = padding
    for (int gi = 0; gi < (int)pl.groups.size(); gi++) {
      st.grp.p[d.off_grp + gi] = pl.groups[gi];
      const int cnt = pl.grp_cnt[gi], ntile = (cnt + kTile - 1) / kTile, k0 = pl.grp_begin[gi], t0 = pl.grp_tile0[gi];
      for (int t = 0; t < ntile; t++) {
        const int gt = d.off_tile + t0 + t;
        st.tile_grp.p[gt] = d.off_grp + gi; st.tile_win.p[gt] = wi;
        int *ol = st.obs_lm.p + (size_t)gt * kTile;
        int *os = st.tile_src.p + (size_t)gt * kTile;
        for (int lane = 0; lane < kTile; lane++) {
          const int idx = t * kTile + lane;
          if (idx < cnt) {
            const int oi = w.order[k0 + idx];
            ol[lane] = w.obs[oi].lm; os[lane] = oi;
            w.sorted_pos[k0 + idx] = (t0 + t) * kTile + lane;
          } else { ol[lane] = -1; os[lane] = -1; oslot[(size_t)(t0 + t) * kTile + lane] = -1; }
        }
      }
    }
    // a landmark's records in ascending tile-position order (deterministic reduction order): positions increase with sorted index
    for (size_t k = 0; k < w.order.size(); k++) { const HObs &o = w.obs[w.order[k]]; oslot[w.sorted_pos[k]] = cursor[o.lm]++; }
    for (int v = 0; v < 6; v++)
      for (size_t j = 0; j < pl.jobs[v].size(); j++) {
        Job jb = pl.jobs[v][j]; jb.grp += d.off_grp; jb.tile_begin += d.off_tile;
        st.job.p[jbase[v] + pl.job_off[v] + j] = jb;
      }
    for (int sg = 0; sg < 2; sg++)
      for (size_t t = 0; t < pl.schur[sg].size(); t++) { SchurTileH q = pl.schur[sg][t]; q.cb += pl.chunk_off; st.schur.p[(sg ? n_sch[0] : 0) + pl.schur_off[sg] + t] = q; }
    for (size_t t = 0; t < pl.schur_chunks.size(); t++) st.schur_chunks.p[pl.chunk_off + t] = pl.schur_chunks[t];
    for (size_t t = 0; t < pl.leaves.size(); t++) { Leaf lf = pl.leaves[t]; lf.lm_begin += pl.leaf_lm_off; st.leaf.p[d.off_leaf + t] = lf; }
    for (size_t t = 0; t < pl.leaf_lm.size(); t++) st.leaf_lm.p[pl.leaf_lm_off + t] = pl.leaf_lm[t];
    for (size_t t = 0; t < pl.hseg.size(); t++) st.hseg.p[d.off_hseg + t] = pl.hseg[t];
    for (int l = 0; l < d.nl; l++) st.lm_mask.p[d.offlm + l] = pl.lm_mask[l];
    for (int i = 0; i < d.n_imu; i++) {
      const HImu &m = w.imu[i];
      st.imu.p[d.off_imu + i] = ImuDesc{m.pi, m.si, m.pj, m.sj, wi};
      double *pk = st.imu_c.p + (size_t)(d.off_imu + i) * kImuPack;   // packed upload record (d2ba_types.cuh kImuPack)
      memcpy(pk, m.c, 17 * 8);
      for (int r = 0; r < 9; r++) memcpy(pk + 17 + r * 6, m.c + 17 + r * 15 + 9, 6 * 8);
      for (int r = 0, q = 0; r < 15; r++) for (int c = 0; c <= r; c++) pk[71 + q++] = m.c[17 + 225 + r * 15 + c];
    }
    st.pr_m.p[wi] = d.prior_m; st.pr_info.p[wi] = (d.prior_m > 0 && w.prior_is_info) ? 1 : 0; st.pr_offJ.p[wi] = d.off_prior_J; st.pr_offv.p[wi] = d.off_prior_v;
    if (d.prior_m > 0) {
      memcpy(st.prior_J.p + d.off_prior_J, w.prior_J.data(), (size_t)d.prior_m * d.prior_m * 8);
      memcpy(st.prior_e0.p + d.off_prior_v, w.prior_e0.data(), (size_t)d.prior_m * 8);
      for (int i = 0; i < d.prior_nblk; i++) {
        const HPriorBlk &b = w.prior_blk[i];
        PriorBlk pb; memset(&pb, 0, sizeof pb);
        pb.kind = b.kind; pb.off = b.off; pb.eff = b.eff; memcpy(pb.x0, b.x0, sizeof pb.x0);
        pb.index = (b.kind == D2BA_EXTRINSIC) ? np + b.index : b.index;
        st.pblk.p[d.off_prior_blk + i] = pb;
      }
    }
  });
  lap(2);
  h->h_win.assign(st.win.p, st.win.p + nw);
  h->h_grp.assign(st.grp.p, st.grp.p + off_grp);
  // ---- uploads (pinned -> device, async on the solver stream)
  int rc;
  CK(cudaEventRecord(h->evf0, h->stream));
  // raw observation records were uploaded as they were added (copy stream); their device addresses ride in the arena
  for (int wi = 0; wi < nw; wi++) {
    HostWin &w = h->win[wi];
    if (w.rawj.n != w.obs.size()) return fail(h, 25, "internal: raw / index record count mismatch");
    st.raw_off.p[4 * wi] = (long long)(uintptr_t)w.d_rawj.p; st.raw_off.p[4 * wi + 1] = (long long)(uintptr_t)w.d_anch.p;
    const bool mot = motion_needed(w);   // else: k_build_tiles writes zero velocities and td_i = td_j = td
    if (!mot && w.rawj.n) skipped_any = 1;
    st.raw_off.p[4 * wi + 2] = mot ? (long long)(uintptr_t)w.d_rawjm.p : 0; st.raw_off.p[4 * wi + 3] = mot ? (long long)(uintptr_t)w.d_anchm.p : 0;
  }
  if (st.cursor > h->d_arena.n) {   // growing: views of the old arena die with it
    CK(cudaStreamSynchronize(h->stream));
    CK(h->d_arena.alloc(st.cursor + st.cursor / 4 + 256));
  }
  CK(cudaMemcpyAsync(h->d_arena.p, st.arena.p, st.cursor, cudaMemcpyHostToDevice, h->stream));
  h->h2d_bytes_fin = (long long)st.cursor;
  if ((rc = up(h, h->d_win, st.win))) return rc;
  CK(h->d_ctl.alloc(nw)); CK(cudaMemsetAsync(h->d_ctl.p, 0, sizeof(Ctl) * nw, h->stream));
  if ((rc = up(h, h->d_x6[0], st.x6)) || (rc = up(h, h->d_xsb[0], st.xsb)) || (rc = up(h, h->d_xlm[0], st.xlm)) || (rc = up(h, h->d_xtd[0], st.xtd))) return rc;
  CK(h->d_x6[1].alloc(st.x6.n)); CK(h->d_xsb[1].alloc(st.xsb.n)); CK(h->d_xlm[1].alloc(st.xlm.n)); CK(h->d_xtd[1].alloc(st.xtd.n));
  const size_t rec_doubles = (size_t)off_rec;
  for (int b = 0; b < 2; b++) {
    CK(h->d_R6[b].alloc((size_t)off6 * 12)); CK(h->d_rec[b].alloc(rec_doubles));
    CK(h->d_H[b].alloc((size_t)offH)); CK(h->d_gc[b].alloc((size_t)offc));
    CK(cudaMemsetAsync(h->d_H[b].p, 0, std::max<size_t>((size_t)offH, 1) * 8, h->stream));   // entries no factor writes stay zero
  }
  if ((rc = up(h, h->d_col6, st.col6)) || (rc = up(h, h->d_colsb, st.colsb)) || (rc = up(h, h->d_tile_grp, st.tile_grp)) ||
      (rc = up(h, h->d_tile_win, st.tile_win)) || (rc = up(h, h->d_obs_lm, st.obs_lm)) || (rc = up(h, h->d_tile_src, st.tile_src)) ||
      (rc = up(h, h->d_lm_ptr, st.lm_ptr)) || (rc = up(h, h->d_obs_slot, st.obs_slot)) || (rc = up(h, h->d_slot6, st.slot6)) ||
      (rc = up(h, h->d_lm_win, st.lm_win)) || (rc = up(h, h->d_blk_win, st.blk_win)) || (rc = up(h, h->d_sb_win, st.sb_win)) ||
      (rc = up(h, h->d_grp, st.grp)) || (rc = up(h, h->d_job, st.job)) || (rc = up(h, h->d_imu, st.imu)) || (rc = up(h, h->d_imu_pk, st.imu_c)) ||
      (rc = up(h, h->d_prior_blk, st.pblk)) || (rc = up(h, h->d_prior_J, st.prior_J)) || (rc = up(h, h->d_prior_e0, st.prior_e0)) ||
      (rc = up(h, h->d_schur, st.schur)) || (rc = up(h, h->d_schur_chunks, st.schur_chunks)) || (rc = up(h, h->d_leaf, st.leaf)) || (rc = up(h, h->d_leaf_lm, st.leaf_lm)) ||
      (rc = up(h, h->d_hseg, st.hseg)) || (rc = up(h, h->d_lm_mask, st.lm_mask)))
    return rc;
  // the device builds the tiles from the raw records
  CK(h->d_obs.alloc((size_t)off_tile * kTile * kObsFields));
  if ((rc = up(h, h->d_raw_off, st.raw_off))) return rc;
  CK(cudaEventRecord(h->ev_copy, h->copy_stream));
  CK(cudaStreamWaitEvent(h->stream, h->ev_copy, 0));
  CK(cudaEventRecord(h->evf1, h->stream));
  h->motion_skipped = skipped_any.load() != 0;
  launch_build_tiles(h->d_raw_off.p, h->d_tile_src.p, h->d_tile_win.p, h->d_xtd[0].p, h->d_obs.p, off_tile, h->stream);
  CK(h->d_imu_U.alloc((size_t)off_imu * 225));
  if ((rc = alloc_zero(h, h->d_imu_c, (size_t)off_imu * kImuStride))) return rc;   // expanded from the packed upload by k_imu_unpack (launch_imu_prep)
  if ((rc = alloc_zero(h, h->d_imu_raw, (size_t)off_imu * 465))) return rc;   // structural zeros of the raw Jacobians are never rewritten
  CK(h->d_prior_A.alloc((size_t)off_pJ));
  CK(h->d_z6.alloc((size_t)off6 * 8)); CK(h->d_tilde6.alloc((size_t)off6 * 6)); CK(h->d_lm_ref.alloc(offlm)); CK(h->d_sb_ref.alloc((size_t)offsb * 9));
  CK(h->d_td_ref.alloc(nw));
  if ((rc = alloc_zero(h, h->d_cons, (size_t)std::max(h->n_slots, 1) * 14))) return rc;
  if ((rc = alloc_zero(h, h->d_Wt, (size_t)offW))) return rc;   // padding rows / columns must be zero
  CK(h->d_dinv.alloc(offlm)); CK(h->d_hl.alloc(offlm)); CK(h->d_gl.alloc(offlm));
  if ((rc = alloc_zero(h, h->d_S, (size_t)offH))) return rc;   // tiles outside the structural pattern are never written
  CK(h->d_leafL.alloc((size_t)std::max<int64_t>(offLL, 1)));
  CK(h->d_gred.alloc((size_t)offc)); CK(h->d_D2c.alloc((size_t)offc)); CK(h->d_gn_c.alloc((size_t)offc)); CK(h->d_gn_l.alloc(offlm));
  CK(h->d_sbLE.alloc((size_t)std::max<int64_t>(offLE, 1)));
  CK(h->d_step_c.alloc((size_t)offc)); CK(h->d_step_l.alloc(offlm)); CK(h->d_wu.alloc(offlm)); CK(h->d_uc.alloc((size_t)offc)); CK(h->d_D2l.alloc(offlm));
  // ---- device view
  Dev &D = h->dev;
  memset(&D, 0, sizeof D);
  D.win = h->d_win.p; D.ctl = h->d_ctl.p; D.n_win = nw;
  for (int b = 0; b < 2; b++) { D.x6[b] = h->d_x6[b].p; D.R6[b] = h->d_R6[b].p; D.xsb[b] = h->d_xsb[b].p; D.xlm[b] = h->d_xlm[b].p; D.xtd[b] = h->d_xtd[b].p; D.rec[b] = h->d_rec[b].p; D.Hcc[b] = h->d_H[b].p; D.gc[b] = h->d_gc[b].p; }
  D.col6 = h->d_col6.p; D.colsb = h->d_colsb.p; D.grp = h->d_grp.p; D.job = h->d_job.p; D.n_job = n_jobs;
  D.lm_mask = h->d_lm_mask.p; D.hseg = h->d_hseg.p; D.leaf = h->d_leaf.p; D.n_leaf_total = h->n_leaf_total; { int np_ = 0; for (int q = 0; q < nw; q++) if (plan[q].d.n_leaf == 0) np_++; D.n_plain_win = np_; } D.leafL = h->d_leafL.p; D.schur_chunks = h->d_schur_chunks.p; D.leaf_lm = h->d_leaf_lm.p;
  D.tile_grp = h->d_tile_grp.p; D.obs = h->d_obs.p; D.obs_lm = h->d_obs_lm.p; D.lm_ptr = h->d_lm_ptr.p; D.obs_slot = h->d_obs_slot.p;
  D.imu = h->d_imu.p; D.imu_c = h->d_imu_c.p; D.imu_U = h->d_imu_U.p; D.imu_raw = h->d_imu_raw.p; D.prior_blk = h->d_prior_blk.p; D.prior_J = h->d_prior_J.p;
  D.prior_e0 = h->d_prior_e0.p; D.prior_A = h->d_prior_A.p; D.slot6 = h->d_slot6.p; D.z6 = h->d_z6.p; D.tilde6 = h->d_tilde6.p;
  D.lm_ref = h->d_lm_ref.p; D.sb_ref = h->d_sb_ref.p; D.td_ref = h->d_td_ref.p; D.cons_buf = h->d_cons.p; D.n_slots = h->n_slots;
  D.Wt = h->d_Wt.p; D.dinv = h->d_dinv.p; D.hl = h->d_hl.p; D.gl = h->d_gl.p; D.S = h->d_S.p; D.gred = h->d_gred.p; D.D2c = h->d_D2c.p;
  D.sbLE = h->d_sbLE.p;
  D.gn_c = h->d_gn_c.p; D.gn_l = h->d_gn_l.p; D.step_c = h->d_step_c.p; D.step_l = h->d_step_l.p; D.wu = h->d_wu.p; D.uc = h->d_uc.p; D.D2l = h->d_D2l.p;
  SolverParams &P = D.prm;
  P.sqrt_info_px = h->cfg.focal_length / 1.5; P.depth_sqrt_inf = h->cfg.depth_sqrt_inf; P.gravity = h->cfg.gravity_norm; P.huber = h->cfg.huber_delta;
  P.rho_T = h->cfg.rho_frame_T; P.rho_theta = h->cfg.rho_frame_theta; P.rho_landmark = h->cfg.rho_landmark; P.relaxation_alpha = h->cfg.relaxation_alpha;
  P.initial_radius = h->cfg.initial_trust_region_radius; P.max_radius = h->cfg.max_trust_region_radius; P.min_rel_decrease = h->cfg.min_relative_decrease;
  P.ftol = h->cfg.function_tolerance; P.gtol = h->cfg.gradient_tolerance; P.ptol = h->cfg.parameter_tolerance;
  P.max_iter = h->cfg.max_num_iterations; P.fixed_mode = 0; P.mu0 = h->mu0;
  if (h->cfg_max_rows != h->max_rows_glob || h->cfg_max_nc != h->max_nc || h->cfg_max_prior != h->max_prior_m) {
    if (configure_kernels(std::max(h->max_rows_glob, 2), h->max_nc, h->max_prior_m)) return fail(h, 23, "cudaFuncSetAttribute failed (shared memory request too large?)");
    h->cfg_max_rows = h->max_rows_glob; h->cfg_max_nc = h->max_nc; h->cfg_max_prior = h->max_prior_m;
  }
  if (h->cfg_max_ldw < h->max_row_tiles * 32) {
    if (configure_gather(h->max_row_tiles * 32)) return fail(h, 23, "cudaFuncSetAttribute(k_lm_gather) failed (landmark-coupled part too wide for the row buffers)");
    h->cfg_max_ldw = h->max_row_tiles * 32;
  }
  if (h->max_ldw_small > 0 && h->cfg_max_ldw_small != h->max_ldw_small) {
    if (configure_schur_small(h->max_ldw_small)) return fail(h, 23, "cudaFuncSetAttribute(k_schur_small) failed");
    h->cfg_max_ldw_small = h->max_ldw_small;
  }
  if (h->sbe_smem > 0 && h->cfg_sbe_smem < h->sbe_smem) {
    if (configure_sb_elim(h->sbe_smem)) return fail(h, 23, "cudaFuncSetAttribute(k_sb_elim) failed");
    h->cfg_sbe_smem = h->sbe_smem;
  }
  if (h->sbb_smem > 0 && h->cfg_sbb_smem < h->sbb_smem) {
    if (configure_sb_back(h->sbb_smem)) return fail(h, 23, "cudaFuncSetAttribute(k_sb_back) failed");
    h->cfg_sbb_smem = h->sbb_smem;
  }
  if (h->leaf_smem > 0 && h->cfg_leaf_smem < h->leaf_smem) {
    if (configure_leaf_elim(h->leaf_smem)) return fail(h, 23, "cudaFuncSetAttribute(k_leaf_elim) failed");
    h->cfg_leaf_smem = h->leaf_smem;
  }
  if (h->leafb_smem > 0 && h->cfg_leafb_smem < h->leafb_smem) {
    if (configure_leaf_back(h->leafb_smem)) return fail(h, 23, "cudaFuncSetAttribute(k_leaf_back) failed");
    h->cfg_leafb_smem = h->leafb_smem;
  }
  if (h->max_n_smem > 0 && h->cfg_max_n_smem != h->max_n_smem) {
    if (configure_chol_smem(h->max_n_smem)) return fail(h, 23, "cudaFuncSetAttribute(k_chol_smem) failed");
    h->cfg_max_n_smem = h->max_n_smem;
  }
  launch_state_prep(D, h->n6_total, 0, h->stream);
  launch_imu_prep(D, h->d_imu_pk.p, h->d_imu_c.p, h->n_imu_total, h->stream);
  if (any_info) {
    if ((rc = up(h, h->d_pr_m, st.pr_m)) || (rc = up(h, h->d_pr_info, st.pr_info)) || (rc = up(h, h->d_pr_oJ, st.pr_offJ)) || (rc = up(h, h->d_pr_ov, st.pr_offv))) return rc;
    launch_prior_from_info(nw, h->max_prior_m, h->d_pr_m.p, h->d_pr_oJ.p, h->d_pr_ov.p, h->d_pr_info.p, h->d_prior_J.p, h->d_prior_A.p, h->d_prior_e0.p, h->stream);
  }
  launch_prior_prep(D, h->stream);
  CK(cudaEventRecord(h->evf2, h->stream));
  lap(3);
  CK(cudaGetLastError());
  lap(4);
  bool okm = h->h_ctl.resize(nw);
  for (int b = 0; b < 2; b++) okm = okm && h->h_x6[b].resize(st.x6.n) && h->h_xsb[b].resize(st.xsb.n) && h->h_xlm[b].resize(st.xlm.n) && h->h_xtd[b].resize(st.xtd.n);
  if (!okm) return fail(h, 24, "pinned read-back allocation failed");
  memset(h->h_ctl.p, 0, sizeof(Ctl) * nw);
  h->finalized = true; h->state_dirty = false; h->solves_since_finalize = 0;
  lap(5);
  return 0;
}

int d2ba_debug_host_times(d2ba_handle *h, double *ms_out) {
  if (!h || !ms_out) return 1;
  memcpy(ms_out, h->host_ms, sizeof h->host_ms);
  if (h->finalized && cudaEventSynchronize(h->evf2) == cudaSuccess) {
    float a = 0, b = 0; cudaEventElapsedTime(&a, h->evf0, h->evf1); cudaEventElapsedTime(&b, h->evf1, h->evf2);
    ms_out[6] = a; ms_out[7] = b;
  }
  for (int k = 0; k < 4; k++) ms_out[8 + k] = 1e-6 * (double)h->add_ns[k].load();
  for (int k = 0; k < 3; k++) ms_out[12 + k] = h->solve_ms[k];
  ms_out[15] = (double)(h->h2d_bytes_add.load() + h->h2d_bytes_fin);
  return 0;
}

// Prior given in information form (A, b): the reference's toJacRes (prior_factor.cpp:132-177) runs on the
// device, batched over windows, as part of d2ba_finalize (k_prior_from_info in d2ba_margin.cu).
int d2ba_set_prior_info(d2ba_handle *h, int32_t window, int32_t m, const double *A, const double *b, int32_t nblk,
                        const d2ba_blockref *refs, const double *x0) {
  if (!h) return 1;
  return set_prior_common(h, window, m, A, b, nblk, refs, x0, true);
}

// ------------------------------------------------------------------------------------------------ solve
static int upload_state(d2ba_handle *h) {
  std::vector<double> x6, xsb, xlm, xtd;
  for (auto &w : h->win) {
    if (!w.used) continue;
    for (size_t i = 0; i < w.pose_id.size(); i++) { for (int q = 0; q < 7; q++) x6.push_back(w.pose[7 * i + q]); x6.push_back(0); }
    for (size_t i = 0; i < w.ext_id.size(); i++) { for (int q = 0; q < 7; q++) x6.push_back(w.ext[7 * i + q]); x6.push_back(0); }
    xsb.insert(xsb.end(), w.sb.begin(), w.sb.end()); xlm.insert(xlm.end(), w.lm.begin(), w.lm.end()); xtd.push_back(w.td);
  }
  CK(cudaMemcpyAsync(h->d_x6[0].p, x6.data(), x6.size() * 8, cudaMemcpyHostToDevice, h->stream));
  if (!xsb.empty()) CK(cudaMemcpyAsync(h->d_xsb[0].p, xsb.data(), xsb.size() * 8, cudaMemcpyHostToDevice, h->stream));
  if (!xlm.empty()) CK(cudaMemcpyAsync(h->d_xlm[0].p, xlm.data(), xlm.size() * 8, cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->d_xtd[0].p, xtd.data(), xtd.size() * 8, cudaMemcpyHostToDevice, h->stream));
  launch_state_prep(h->dev, h->n6_total, 0, h->stream);
  CK(cudaStreamSynchronize(h->stream));   // host vectors go out of scope
  h->state_dirty = false;
  return 0;
}

static void enqueue_linearize(d2ba_handle *h, int eval_cur) {
  // two lanes: the IMU chain (latency bound, ~10 factors per window) runs beside k_misc_lin / the reprojection kernels
  // (bandwidth bound).  Order kept: k_misc_lin zero-fills the written runs of Hcc and stores cand_cost_misc before
  // k_imu_lin and k_proj_lin add to them.
  const bool fork = h->two_lanes && h->n_imu_total > 0;
  if (fork) {
    cudaEventRecord(h->ev_fork, h->stream); cudaStreamWaitEvent(h->side, h->ev_fork, 0);
    launch_imu_raw(h->dev, eval_cur, h->n_imu_total, h->side);
  }
  launch_misc_lin(h->dev, eval_cur, h->max_prior_m, h->stream);
  if (fork) {
    cudaEventRecord(h->ev_misc, h->stream); cudaStreamWaitEvent(h->side, h->ev_misc, 0);
    launch_imu_acc(h->dev, eval_cur, h->n_imu_total, h->side);
    cudaEventRecord(h->ev_join, h->side);
  } else launch_imu_lin(h->dev, eval_cur, h->n_imu_total, h->stream);
  for (int v = 0; v < 6; v++) launch_proj_lin(h->dev, v, eval_cur, h->job_begin[v], h->job_count[v], h->stream);
  if (fork) cudaStreamWaitEvent(h->stream, h->ev_join, 0);
}

// reduced camera system: tiles with leaf columns -> leaf elimination (rows Y behind the landmark rows of Wt) -> hub tiles
static void enqueue_schur(d2ba_handle *h) {
  // (the leaf kernel forms its own part of the reduced system from Hcc and its landmarks' rows: the stage-0 tiles are
  //  only launched for the debug view of S)
  if (h->n_leaf_total > 0) launch_leaf_elim(h->dev, h->leaf_smem, h->stream);
  if (h->max_ldw_small > 0) launch_schur_small(h->dev, h->max_ldw_small, h->stream);
  if (h->n_schur > h->n_schur0) launch_schur(h->dev, h->d_schur.p + h->n_schur0, h->n_schur - h->n_schur0, h->stream);
}
// dense Cholesky of the hub, then the eliminated parts' back substitutions
static void enqueue_solve_reduced(d2ba_handle *h) {
  if (h->max_n_smem > 0) launch_chol_smem(h->dev, h->max_n_smem, h->stream);
  if (h->any_chol_glob) launch_chol(h->dev, h->max_rows_glob, h->stream);
  if (h->sbe_smem > 0) launch_sb_back(h->dev, h->sbb_smem, h->stream);
  if (h->n_leaf_total > 0) launch_leaf_back(h->dev, h->leafb_smem, h->stream);
}

static void enqueue_iteration(d2ba_handle *h) {
  // the speed-bias elimination (Hcc -> its Y rows behind the landmark rows of Wt) does not touch what the landmark gather
  // reads or writes: second lane
  const bool fork = h->two_lanes && h->sbe_smem > 0;
  if (fork) { cudaEventRecord(h->ev_fork, h->stream); cudaStreamWaitEvent(h->side, h->ev_fork, 0); launch_sb_elim(h->dev, h->sbe_smem, h->side); cudaEventRecord(h->ev_join, h->side); }
  launch_lm_gather(h->dev, h->d_lm_win.p, h->nl_total, h->max_row_tiles * 32, h->any_compact, h->any_wide, h->stream);
  if (fork) cudaStreamWaitEvent(h->stream, h->ev_join, 0);
  else if (h->sbe_smem > 0) launch_sb_elim(h->dev, h->sbe_smem, h->stream);   // Y rows into Wt: the Schur kernels subtract them too
  enqueue_schur(h);
  enqueue_solve_reduced(h);
  launch_step(h->dev, h->max_nc, h->stream);
  enqueue_linearize(h, 0);
  launch_control(h->dev, 0, h->stream);
}

static int consensus_exchange(d2ba_handle *h) {
  CK(cudaMemsetAsync(h->d_cons.p, 0, (size_t)std::max(h->n_slots, 1) * 14 * 8, h->stream));
  launch_cons_pack(h->dev, h->n6_total, h->d_blk_win.p, h->stream);
  if (h->comm) {
    int r = g_nccl.AllReduce(h->d_cons.p, h->d_cons.p, (size_t)h->n_slots * 14, /*ncclFloat64*/ 8, /*ncclSum*/ 0, h->comm, h->stream);
    if (r) return fail(h, 40, std::string("ncclAllReduce: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "error"));
  }
  launch_cons_apply(h->dev, h->n6_total, h->d_blk_win.p, h->stream);
  launch_cons_refs(h->dev, h->nsb_total, h->nl_total, h->d_sb_win.p, h->d_lm_win.p, h->stream);
  return 0;
}

static int run_solve(d2ba_handle *h, int fixed_iters, d2ba_report *reports) {
  if (!h) return 1;
  cudaSetDevice(h->cfg.device);
  if (!h->finalized) { int rc = d2ba_finalize(h); if (rc) return rc; }
  if (h->state_dirty) { int rc = upload_state(h); if (rc) return rc; }
  const bool fixed = fixed_iters > 0;
  const int steps = (h->any_admm && h->cfg.consensus_max_steps > 0) ? h->cfg.consensus_max_steps : 1;
  int iters = fixed ? fixed_iters : h->cfg.max_num_iterations;
  if (steps > 1 || h->any_admm) iters = std::max(1, iters / steps);   // d2vins_params.cpp:156-158
  h->dev.prm.fixed_mode = fixed ? 1 : 0; h->dev.prm.max_iter = iters;
  const int key = (fixed ? 1 : 0) * 100000 + iters;
  if (h->graph_key != key) release_graph(h);
  auto tq = std::chrono::steady_clock::now();
  auto lap = [&](int k) { auto t = std::chrono::steady_clock::now(); h->solve_ms[k] = std::chrono::duration<double, std::milli>(t - tq).count(); tq = t; };
  CK(cudaEventRecord(h->ev0, h->stream));
  launch_tr_reset(h->dev, 1, h->stream);
  if (h->any_admm) launch_cons_init(h->dev, h->n6_total, h->stream);
  // ceres max_solver_time_in_seconds: an iteration is only started while the budget of this (sub-)step lasts.  The
  // iterations are enqueued asynchronously, so the host trails the device by at most two of them: before enqueuing
  // iteration k it waits for iteration k-2 and compares the wall clock.
  const double budget_s = (!fixed && h->cfg.max_solver_time_in_seconds > 0) ? h->cfg.max_solver_time_in_seconds / steps : 0.0;
  std::chrono::steady_clock::time_point t_step0;
  auto over_budget = [&](int it) {
    if (budget_s <= 0.0 || it < 2) return false;
    cudaEventSynchronize(h->ev_it[it & 1]);   // recorded after iteration it-2
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t_step0).count() > budget_s;
  };
  auto mark = [&](int it) { if (budget_s > 0.0) cudaEventRecord(h->ev_it[it & 1], h->stream); };
  for (int st = 0; st < steps; st++) {
    t_step0 = std::chrono::steady_clock::now();
    if (st > 0) launch_tr_reset(h->dev, 0, h->stream);
    if (h->any_admm) { int rc = consensus_exchange(h); if (rc) return rc; }
    enqueue_linearize(h, 1);
    launch_control(h->dev, st == 0 ? 1 : 2, h->stream);
    // A graph pays off when the same structure is solved repeatedly (ADMM sub-steps, re-solves, the device-resident
    // benchmark); the reference-style reset -> add -> finalize -> solve cycle launches directly and skips the instantiation.
    if (h->cfg.use_cuda_graph && (h->iter_graph || h->solves_since_finalize > 0 || st > 0)) {
      if (!h->iter_graph) {
        cudaGraph_t g;
        CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
        enqueue_iteration(h);
        CK(cudaStreamEndCapture(h->stream, &g));
        CK(cudaGraphInstantiate(&h->iter_graph, g, 0));
        cudaGraphDestroy(g);
        h->graph_key = key;
      }
      for (int it = 0; it < iters; it++) { if (over_budget(it)) break; CK(cudaGraphLaunch(h->iter_graph, h->stream)); mark(it); }
    } else {
      for (int it = 0; it < iters; it++) { if (over_budget(it)) break; enqueue_iteration(h); mark(it); }
    }
  }
  CK(cudaEventRecord(h->ev1, h->stream));
  // read back control blocks and both state buffers (the accepted buffer differs per window)
  CK(cudaMemcpyAsync(h->h_ctl.p, h->d_ctl.p, sizeof(Ctl) * h->n_used, cudaMemcpyDeviceToHost, h->stream));
  for (int b = 0; b < 2; b++) {
    CK(cudaMemcpyAsync(h->h_x6[b].p, h->d_x6[b].p, h->h_x6[b].n * 8, cudaMemcpyDeviceToHost, h->stream));
    if (h->h_xsb[b].n) CK(cudaMemcpyAsync(h->h_xsb[b].p, h->d_xsb[b].p, h->h_xsb[b].n * 8, cudaMemcpyDeviceToHost, h->stream));
    if (h->h_xlm[b].n) CK(cudaMemcpyAsync(h->h_xlm[b].p, h->d_xlm[b].p, h->h_xlm[b].n * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(h->h_xtd[b].p, h->d_xtd[b].p, h->h_xtd[b].n * 8, cudaMemcpyDeviceToHost, h->stream));
  }
  lap(0);
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  lap(1);
  float ms = 0; cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  // write the solved state back into the host windows (so a following solve starts from it)
  int wi = 0;
  for (auto &w : h->win) {
    if (!w.used) continue;
    const WinDesc &d = h->h_win[wi]; const int cur = h->h_ctl.p[wi].cur;
    double chg2 = 0.0;
    for (int i = 0; i < d.np; i++) {
      const double *xn = &h->h_x6[cur].p[(size_t)(d.off6 + i) * 8];
      for (int q = 0; q < 3; q++) { const double dq = xn[q] - w.pose[7 * i + q]; chg2 += dq * dq; }
      memcpy(&w.pose[7 * i], xn, 56);
    }
    for (int i = 0; i < d.ne; i++) memcpy(&w.ext[7 * i], &h->h_x6[cur].p[(size_t)(d.off6 + d.np + i) * 8], 56);
    if (d.nsb) memcpy(w.sb.data(), &h->h_xsb[cur].p[(size_t)d.offsb * 9], (size_t)d.nsb * 72);
    if (d.nl) memcpy(w.lm.data(), &h->h_xlm[cur].p[d.offlm], (size_t)d.nl * 8);
    w.td = h->h_xtd[cur].p[wi];
    if (reports) {
      const Ctl &c = h->h_ctl.p[wi]; d2ba_report &r = reports[wi];
      r.total_iterations = c.lin_count; r.successful_steps = c.succ; r.termination = c.term; r.succ = c.term != 4;
      r.total_time = ms * 1e-3; r.initial_cost = c.initial_cost; r.final_cost = c.cost; r.state_changes = sqrt(chg2);
      r.final_gradient_max_norm = c.gmax_c; r.final_radius = c.radius;
    }
    wi++;
  }
  h->state_dirty = true;   // device buffer 0 no longer holds the accepted state of every window
  h->solves_since_finalize++;
  lap(2);
  return 0;
}

int d2ba_solve(d2ba_handle *h, d2ba_report *reports) { return run_solve(h, 0, reports); }
int d2ba_solve_fixed(d2ba_handle *h, int32_t iters, d2ba_report *reports) { return run_solve(h, iters < 1 ? 1 : iters, reports); }

int d2ba_get_blocks(d2ba_handle *h, int32_t window, int32_t kind, int32_t n, const int64_t *ids, double *out) {
  HostWin *w = get_win(h, window);
  if (!w || !w->used) return 1;
  for (int i = 0; i < n; i++) {
    int k;
    switch (kind) {
      case D2BA_POSE: k = find_in(w->pose_map, ids[i]); if (k < 0) return fail(h, 2, "get_blocks: unknown id"); memcpy(out + 7 * i, &w->pose[7 * k], 56); break;
      case D2BA_EXTRINSIC: k = find_in(w->ext_map, ids[i]); if (k < 0) return fail(h, 2, "get_blocks: unknown id"); memcpy(out + 7 * i, &w->ext[7 * k], 56); break;
      case D2BA_SPEED_BIAS: k = find_in(w->sb_map, ids[i]); if (k < 0) return fail(h, 2, "get_blocks: unknown id"); memcpy(out + 9 * i, &w->sb[9 * k], 72); break;
      case D2BA_TD: out[i] = w->td; break;
      case D2BA_LANDMARK: k = find_in(w->lm_map, ids[i]); if (k < 0) return fail(h, 2, "get_blocks: unknown id"); out[i] = w->lm[k]; break;
      default: return 3;
    }
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------ comm
}  // extern "C"
namespace d2ba {   // the dlopen'ed NCCL entry points for the other translation units of the library (d2pgo.cu)
int nccl_comm_init(void **comm, const uint8_t *unique_id, int rank, int nranks, std::string &err) {
  if (!g_nccl.load(err)) return 2;
  ncclUniqueId_t id; memcpy(id.internal, unique_id, 128);
  ncclComm_t c = nullptr;
  const int r = g_nccl.CommInitRank(&c, nranks, id, rank);
  if (r) { err = std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "error"); return 3; }
  *comm = c;
  return 0;
}
int nccl_allreduce_f64(void *comm, double *buf, size_t n, cudaStream_t s) {
  return g_nccl.AllReduce(buf, buf, n, /*ncclFloat64*/ 8, /*ncclSum*/ 0, (ncclComm_t)comm, s);
}
void nccl_comm_destroy(void *comm) { if (comm && g_nccl.CommDestroy) g_nccl.CommDestroy((ncclComm_t)comm); }
}  // namespace d2ba
extern "C" {
int d2ba_comm_unique_id(uint8_t out[128]) {
  std::string err;
  if (!g_nccl.load(err)) { fprintf(stderr, "d2ba: %s\n", err.c_str()); return 1; }
  ncclUniqueId_t id;
  int r = g_nccl.GetUniqueId(&id);
  if (r) return 2;
  memcpy(out, id.internal, 128);
  return 0;
}
int d2ba_comm_init(d2ba_handle *h, const uint8_t unique_id[128], int32_t rank, int32_t nranks) {
  if (!h) return 1;
  if (!g_nccl.load(h->err)) return 2;
  cudaSetDevice(h->cfg.device);
  ncclUniqueId_t id; memcpy(id.internal, unique_id, 128);
  int r = g_nccl.CommInitRank(&h->comm, nranks, id, rank);
  if (r) return fail(h, 3, std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "error"));
  h->rank = rank; h->nranks = nranks;
  return 0;
}
int d2ba_consensus_buffer(d2ba_handle *h, void **dev_ptr, int64_t *n_doubles) {
  if (!h || !h->finalized) return 1;
  *dev_ptr = h->d_cons.p; *n_doubles = (int64_t)h->n_slots * 14;
  return 0;
}

// ------------------------------------------------------------------------------------------------ debug
// The debug views report the full per-factor Jacobian, whose td column holds the feature velocities even where the solve
// never needs them (td constant): fetch the motion halves that d2ba_finalize left on the host and rebuild the tiles.
static int ensure_motion(d2ba_handle *h) {
  if (!h->motion_skipped) return 0;
  std::vector<long long> off(4 * (size_t)h->n_used);
  CK(cudaMemcpy(off.data(), h->d_raw_off.p, off.size() * 8, cudaMemcpyDeviceToHost));
  for (int wi = 0; wi < h->n_used; wi++) {
    HostWin &w = h->win[wi];
    int rc;
    if ((rc = push_range(h, w.rawjm, w.d_rawjm, w.pushed_jm)) || (rc = push_range(h, w.anchm, w.d_anchm, w.pushed_am))) return rc;
    w.pushed_jm = w.rawjm.n; w.pushed_am = w.anchm.n;
    off[4 * wi + 2] = (long long)(uintptr_t)w.d_rawjm.p; off[4 * wi + 3] = (long long)(uintptr_t)w.d_anchm.p;
  }
  CK(cudaStreamSynchronize(h->copy_stream));
  CK(cudaMemcpy(h->d_raw_off.p, off.data(), off.size() * 8, cudaMemcpyHostToDevice));
  launch_build_tiles(h->d_raw_off.p, h->d_tile_src.p, h->d_tile_win.p, h->d_xtd[0].p, h->d_obs.p, h->n_tiles, h->stream);
  h->motion_skipped = false;
  return 0;
}

int d2ba_debug_linearize(d2ba_handle *h) {
  if (!h) return 1;
  cudaSetDevice(h->cfg.device);
  if (!h->finalized) { int rc = d2ba_finalize(h); if (rc) return rc; }
  { int rc = ensure_motion(h); if (rc) return rc; }
  if (h->state_dirty) { int rc = upload_state(h); if (rc) return rc; }
  h->dev.prm.fixed_mode = 1; h->dev.prm.max_iter = 1;
  launch_tr_reset(h->dev, 1, h->stream);
  enqueue_linearize(h, 1);
  launch_control(h->dev, 1, h->stream);
  launch_lm_gather(h->dev, h->d_lm_win.p, h->nl_total, h->max_row_tiles * 32, h->any_compact, h->any_wide, h->stream);
  // debug view: the landmark-only Schur complement (eliminated speed-bias rows zeroed), kept un-factored in d_dbg
  if (h->sbe_smem > 0) launch_zero_sb_rows(h->dev, h->stream);
  if (h->n_leaf_total > 0) launch_zero_leaf_rows(h->dev, h->stream);
  if (h->max_ldw_small > 0) launch_schur_small(h->dev, h->max_ldw_small, h->stream);
  launch_schur(h->dev, h->d_schur.p, h->n_schur, h->stream);   // both stages back to back: no eliminated rows in this view
  CK(h->d_dbg.alloc((size_t)h->totH));
  CK(cudaMemcpyAsync(h->d_dbg.p, h->d_S.p, (size_t)h->totH * 8, cudaMemcpyDeviceToDevice, h->stream));
  if (h->sbe_smem > 0 || h->n_leaf_total > 0) {   // now the system the solver factors: Y rows in place, Schur again
    if (h->sbe_smem > 0) launch_sb_elim(h->dev, h->sbe_smem, h->stream);
    enqueue_schur(h);
  }
  enqueue_solve_reduced(h);
  launch_step(h->dev, h->max_nc, h->stream);
  CK(cudaMemcpyAsync(h->h_ctl.p, h->d_ctl.p, sizeof(Ctl) * h->n_used, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  release_graph(h);
  return 0;
}

int d2ba_debug_get(d2ba_handle *h, int32_t window, int32_t item, void *out, int64_t out_bytes, int64_t *needed) {
  HostWin *w = get_win(h, window);
  if (!w || !w->used || !h->finalized) return 1;
  cudaSetDevice(h->cfg.device);
  const WinDesc &d = h->h_win[window];
  const int n = d.n_c, nlc = d.n_lc, nl = d.nl, ld = d.ldh;
  std::vector<uint8_t> buf;
  auto put_d = [&](const std::vector<double> &v) { buf.resize(v.size() * 8); memcpy(buf.data(), v.data(), buf.size()); };
  auto fetch = [&](const double *src, size_t cnt) { std::vector<double> v(cnt); if (cnt) cudaMemcpy(v.data(), src, cnt * 8, cudaMemcpyDeviceToHost); return v; };
  const int cur = h->h_ctl.p[window].cur;
  const std::vector<int> &cn = w->canon_of_dev;   // device column -> canonical (insertion-order) column
  auto canon_blk = [&](int c) { return c < 0 ? -1 : cn[c]; };
  switch (item) {
    case D2BA_DBG_N_CAM: { int64_t v = n; buf.resize(8); memcpy(buf.data(), &v, 8); break; }
    case D2BA_DBG_N_LC: { int64_t v = nlc; buf.resize(8); memcpy(buf.data(), &v, 8); break; }
    case D2BA_DBG_HCC: {   // Hcc is stored lower-triangular in device column order: symmetric, canonical order out
      auto H = fetch(h->d_H[cur].p + d.offH, (size_t)n * ld);
      std::vector<double> o((size_t)n * n);
      for (int i = 0; i < n; i++) for (int j = 0; j <= i; j++) { const int a = cn[i], b = cn[j]; o[(size_t)a * n + b] = H[(size_t)i * ld + j]; o[(size_t)b * n + a] = H[(size_t)i * ld + j]; }
      put_d(o); break;
    }
    case D2BA_DBG_GC: { auto g = fetch(h->d_gc[cur].p + d.offc, n); std::vector<double> o(n); for (int i = 0; i < n; i++) o[cn[i]] = g[i]; put_d(o); break; }
    case D2BA_DBG_HLL: put_d(fetch(h->d_hl.p + d.offlm, nl)); break;
    case D2BA_DBG_GL: put_d(fetch(h->d_gl.p + d.offlm, nl)); break;
    case D2BA_DBG_W: {
      auto Wt = fetch(h->d_Wt.p + d.offW, (size_t)nl * d.ldw);
      auto di = fetch(h->d_dinv.p + d.offlm, nl);
      std::vector<double> o((size_t)nl * nlc);
      for (int l = 0; l < nl; l++) for (int c = 0; c < nlc; c++) o[(size_t)l * nlc + cn[c]] = Wt[(size_t)l * d.ldw + c] / di[l];
      put_d(o); break;
    }
    case D2BA_DBG_COST: { std::vector<double> v(1, h->h_ctl.p[window].cost); put_d(v); break; }
    case D2BA_DBG_S: {
      if (h->d_dbg.n < (size_t)h->totH) return fail(h, 4, "debug_get(S): call d2ba_debug_linearize first");
      auto S = fetch(h->d_dbg.p + d.offH, (size_t)n * ld);
      if (d.sb_elim || (d.schur_small && d.chol_smem)) {
        // the speed-bias rows of such windows never pass through S (k_sb_elim / k_chol_smem read them from Hcc): rebuild them
        // for the debug view exactly as that kernel does (H + mu D^2 on the diagonal, mu = 1e-8 after tr_reset)
        auto H = fetch(h->d_H[cur].p + d.offH, (size_t)n * ld);
        for (int i = nlc; i < n; i++)
          for (int j = 0; j <= i; j++) {
            double v = H[(size_t)i * ld + j];
            if (i == j) { double dd = sqrt(v); dd = dd < 1e-6 ? 1e-6 : (dd > 1e32 ? 1e32 : dd); v += h->mu0 * dd * dd; }
            S[(size_t)i * ld + j] = v;
          }
      }
      std::vector<double> o((size_t)n * n);
      for (int i = 0; i < n; i++) for (int j = 0; j <= i; j++) { const int a = cn[i], b = cn[j]; o[(size_t)a * n + b] = S[(size_t)i * ld + j]; o[(size_t)b * n + a] = S[(size_t)i * ld + j]; }
      put_d(o); break;
    }
    case D2BA_DBG_GN_STEP: case D2BA_DBG_STEP: {
      auto a0 = fetch((item == D2BA_DBG_GN_STEP ? h->d_gn_c.p : h->d_step_c.p) + d.offc, n);
      std::vector<double> a(n);
      for (int i = 0; i < n; i++) a[cn[i]] = a0[i];
      auto b = fetch((item == D2BA_DBG_GN_STEP ? h->d_gn_l.p : h->d_step_l.p) + d.offlm, nl);
      a.insert(a.end(), b.begin(), b.end()); put_d(a); break;
    }
    case D2BA_DBG_OBS_INDEX: {
      std::vector<int32_t> v;
      for (int oi : w->order) { const HObs &o = w->obs[oi]; v.push_back(o.type); v.push_back(o.pi); v.push_back(o.pj); v.push_back(o.ea < 0 ? -1 : d.np + o.ea); v.push_back(o.eb < 0 ? -1 : d.np + o.eb); v.push_back(o.lm); }
      buf.resize(v.size() * 4); memcpy(buf.data(), v.data(), buf.size()); break;
    }
    case D2BA_DBG_COL_OF_BLOCK: {
      std::vector<int32_t> v;
      for (int c : w->pose_col) v.push_back(canon_blk(c));
      for (int c : w->ext_col) v.push_back(canon_blk(c));
      for (int c : w->sb_col) v.push_back(canon_blk(c));
      v.push_back(canon_blk(w->td_col));
      buf.resize(v.size() * 4); memcpy(buf.data(), v.data(), buf.size()); break;
    }
    case D2BA_DBG_PROJ_RESJAC: {
      DBuf<double> tmp;
      if (tmp.alloc((size_t)h->n_tiles * kTile * 81) != cudaSuccess) return fail(h, 5, "debug alloc");
      launch_proj_debug(h->dev, tmp.p, h->n_tiles, h->d_tile_win.p, h->stream);
      cudaStreamSynchronize(h->stream);
      std::vector<double> all((size_t)d.n_tile * kTile * 81);
      if (!all.empty()) cudaMemcpy(all.data(), tmp.p + (size_t)d.off_tile * kTile * 81, all.size() * 8, cudaMemcpyDeviceToHost);
      tmp.release();
      std::vector<double> o(w->obs.size() * 81, 0.0);
      for (size_t k = 0; k < w->order.size(); k++) memcpy(&o[(size_t)w->order[k] * 81], &all[(size_t)w->sorted_pos[k] * 81], 81 * 8);
      put_d(o); break;
    }
    case D2BA_DBG_IMU_RESJAC: {
      // imu -> window map built here (debug only)
      std::vector<int> iw;
      for (int wi2 = 0; wi2 < h->n_used; wi2++) iw.insert(iw.end(), h->h_win[wi2].n_imu, wi2);
      DBuf<double> tmp; DBuf<int> dw;
      if (tmp.alloc((size_t)std::max<size_t>(iw.size(), 1) * 465) != cudaSuccess || dw.alloc(std::max<size_t>(iw.size(), 1)) != cudaSuccess) return fail(h, 5, "debug alloc");
      if (!iw.empty()) cudaMemcpy(dw.p, iw.data(), iw.size() * sizeof(int), cudaMemcpyHostToDevice);
      launch_imu_debug(h->dev, tmp.p, dw.p, (int)iw.size(), h->stream);
      cudaStreamSynchronize(h->stream);
      put_d(fetch(tmp.p + (size_t)d.off_imu * 465, (size_t)d.n_imu * 465));
      tmp.release(); dw.release(); break;
    }
    case D2BA_DBG_CONS_RESJAC: {
      DBuf<double> tmp;
      if (tmp.alloc((size_t)std::max(h->n6_total, 1) * 62) != cudaSuccess) return fail(h, 5, "debug alloc");
      launch_cons_debug(h->dev, tmp.p, h->d_blk_win.p, h->n6_total, h->stream);
      cudaStreamSynchronize(h->stream);
      put_d(fetch(tmp.p + (size_t)d.off6 * 62, (size_t)d.n6 * 62));
      tmp.release(); break;
    }
    default: return fail(h, 6, "debug_get: unknown item");
  }
  if (needed) *needed = (int64_t)buf.size();
  if (out) { if (out_bytes < (int64_t)buf.size()) return 2; memcpy(out, buf.data(), buf.size()); }
  return 0;
}

// ------------------------------------------------------------------------------------------------ marginalization
// Marginalizer::marginalize (d2vins/src/estimator/marginalization/marginalization.cpp:173-254) on the device:
// the relevant residuals (filterResiduals :78-118) form a one-window sub-problem in a scratch handle; its
// linearisation (k_misc_lin / k_proj_lin, loss-corrected like ResidualInfo::Evaluate), landmark elimination
// (k_lm_gather + Schur kernel with mu = 0) and a small exact-inverse reduction of the removed pose / speed-bias
// columns (k_marg_reduce) give the information form (A, b) of the new prior.
int d2ba_marginalize(d2ba_handle *h, int32_t window, int32_t n_remove, const int64_t *remove_frame_ids, int32_t *m_out,
                     int32_t max_m, double *A_out, double *b_out, int32_t *nblk_out, int32_t max_blk, d2ba_blockref *refs_out,
                     double *x0_out) {
  HostWin *w = get_win(h, window);
  if (!w || !w->used) return 1;
  cudaSetDevice(h->cfg.device);
  const int np = (int)w->pose_id.size(), ne = (int)w->ext_id.size(), nsb = (int)w->sb_id.size(), nl = (int)w->lm_id.size();
  std::vector<char> rem_pose(np, 0), rem_sb(nsb, 0), use_pose(np, 0), use_sb(nsb, 0), use_ext(ne, 0), use_lm(nl, 0);
  bool use_td = false;
  for (int i = 0; i < np; i++) for (int k = 0; k < n_remove; k++) if (w->pose_id[i] == remove_frame_ids[k]) rem_pose[i] = 1;
  for (int i = 0; i < nsb; i++) for (int k = 0; k < n_remove; k++) if (w->sb_id[i] == remove_frame_ids[k]) rem_sb[i] = 1;
  std::vector<d2ba_proj_obs> robs;
  for (size_t k = 0; k < w->obs.size(); k++) {
    const HObs &o = w->obs[k];
    bool r;
    if (o.type == D2BA_PROJ_DEPTH_PRIOR || o.type == D2BA_PROJ_1F2C) r = o.fa >= 0 && rem_pose[o.fa];   // anchor frame only
    else r = rem_pose[o.pi] || rem_pose[o.pj];
    if (!r) continue;
    {   // back to the caller's record format from the compact constants + block indices
      d2ba_proj_obs p; memset(&p, 0, sizeof p);
      const ObsJ &r = w->rawj.p[k];
      p.type = o.type; p.landmark_id = w->lm_id[o.lm];
      p.frame_a = o.fa >= 0 ? w->pose_id[o.fa] : 0; p.frame_b = o.pj >= 0 ? w->pose_id[o.pj] : p.frame_a;
      p.cam_a = o.ea >= 0 ? (int32_t)w->ext_id[o.ea] : 0; p.cam_b = o.eb >= 0 ? (int32_t)w->ext_id[o.eb] : 0;
      if (o.type != D2BA_PROJ_DEPTH_PRIOR) {
        const ObsAnchor &a = w->anch.p[r.anchor]; const ObsAnchorM &am = w->anchm.p[r.anchor]; const ObsJm &rm = w->rawjm.p[k];
        memcpy(p.pts_i, a.pts_i, 24); memcpy(p.vel_i, am.vel_i, 24); p.td_i = am.td_i;
        memcpy(p.pts_j, r.pts_j, 24); memcpy(p.vel_j, rm.vel_j, 24); p.td_j = rm.td_j;
      }
      p.depth = r.depth;
      robs.push_back(p);
    }
    if (o.pi >= 0) { use_pose[o.pi] = 1; use_pose[o.pj] = 1; }
    if (o.type != D2BA_PROJ_DEPTH_PRIOR) { use_ext[o.ea] = 1; if (o.eb >= 0) use_ext[o.eb] = 1; use_td = true; }
    use_lm[o.lm] = 1;
  }
  std::vector<d2ba_imu> rimu;
  for (const HImu &m : w->imu) {
    if (!(rem_pose[m.pi] || rem_pose[m.pj])) continue;
    use_pose[m.pi] = use_pose[m.pj] = 1; use_sb[m.si] = use_sb[m.sj] = 1;
    d2ba_imu r; memset(&r, 0, sizeof r);
    r.frame_a = w->pose_id[m.pi]; r.frame_b = w->pose_id[m.pj];
    const double *c = m.c;
    r.sum_dt = c[0]; memcpy(r.delta_p, c + 1, 24); memcpy(r.delta_q, c + 4, 32); memcpy(r.delta_v, c + 8, 24);
    memcpy(r.linearized_ba, c + 11, 24); memcpy(r.linearized_bg, c + 14, 24); memcpy(r.jacobian, c + 17, 225 * 8); memcpy(r.covariance, c + 17 + 225, 225 * 8);
    rimu.push_back(r);
  }
  for (const HPriorBlk &b : w->prior_blk) {
    if (b.kind == D2BA_POSE) use_pose[b.index] = 1; else if (b.kind == D2BA_EXTRINSIC) use_ext[b.index] = 1;
    else if (b.kind == D2BA_SPEED_BIAS) use_sb[b.index] = 1; else if (b.kind == D2BA_TD) use_td = true; else use_lm[b.index] = 1;
  }
  // scratch handle
  if (!h->marg) {
    d2ba_config c = h->cfg; c.max_windows = 1; c.consensus_max_steps = 0; c.use_cuda_graph = 0;
    int rc = d2ba_create(&c, &h->marg);
    if (rc) return fail(h, 60, "marginalize: cannot create scratch handle");
    h->marg->mu0 = 0.0; h->marg->force_full_S = true;
  }
  d2ba_handle *t = h->marg;
  d2ba_reset(t);
  // blocks: kept poses, removed poses | extrinsics | td | kept speed-bias, removed speed-bias | landmarks (all free)
  std::vector<int> keep_cols, rem_cols;
  int nblk = 0, xo = 0, nk = 0, col = 0;
  std::vector<int64_t> ids; std::vector<double> vals; std::vector<uint8_t> cst;
  auto flush = [&](int kind, int sz) { int rc = ids.empty() ? 0 : d2ba_set_blocks(t, 0, kind, (int)ids.size(), ids.data(), vals.data(), cst.data()); ids.clear(); vals.clear(); cst.clear(); (void)sz; return rc; };
  auto emit = [&](int kind, int64_t id, const double *v, int sz) {
    if (nblk >= max_blk) return false;
    refs_out[nblk].kind = kind; refs_out[nblk].pad = 0; refs_out[nblk].id = id;
    if (x0_out) memcpy(x0_out + xo, v, 8 * sz);
    xo += sz; nblk++; return true;
  };
  int rc = 0;
  // tmp column order = [poses | ext | td | sb]; remember which reduced columns are kept / removed
  std::vector<int> pose_col(np, -1), sb_col(nsb, -1), ext_col(ne, -1);
  for (int pass = 0; pass < 2; pass++)
    for (int i = 0; i < np; i++) if (use_pose[i] && rem_pose[i] == pass) { ids.push_back(w->pose_id[i]); vals.insert(vals.end(), &w->pose[7 * i], &w->pose[7 * i] + 7); cst.push_back(0); pose_col[i] = col; col += 6; }
  if ((rc = flush(D2BA_POSE, 7))) return rc;
  for (int i = 0; i < ne; i++) if (use_ext[i]) { ids.push_back(w->ext_id[i]); vals.insert(vals.end(), &w->ext[7 * i], &w->ext[7 * i] + 7); cst.push_back(0); ext_col[i] = col; col += 6; }
  if ((rc = flush(D2BA_EXTRINSIC, 7))) return rc;
  int td_col = -1;
  { int64_t z = 0; uint8_t c0 = use_td ? 0 : 1; double tdv = w->td; if ((rc = d2ba_set_blocks(t, 0, D2BA_TD, 1, &z, &tdv, &c0))) return rc; if (use_td) { td_col = col; col += 1; } }
  for (int pass = 0; pass < 2; pass++)
    for (int i = 0; i < nsb; i++) if (use_sb[i] && rem_sb[i] == pass) { ids.push_back(w->sb_id[i]); vals.insert(vals.end(), &w->sb[9 * i], &w->sb[9 * i] + 9); cst.push_back(0); sb_col[i] = col; col += 9; }
  if ((rc = flush(D2BA_SPEED_BIAS, 9))) return rc;
  for (int i = 0; i < nl; i++) if (use_lm[i]) { ids.push_back(w->lm_id[i]); vals.push_back(w->lm[i]); cst.push_back(0); }
  if ((rc = flush(D2BA_LANDMARK, 1))) return rc;
  // kept blocks in the reference's type order (sortParams :262-270): POSE, SPEED_BIAS, EXTRINSIC, TD
  bool ok = true;
  for (int i = 0; i < np; i++) if (use_pose[i] && !rem_pose[i]) { ok = ok && emit(D2BA_POSE, w->pose_id[i], &w->pose[7 * i], 7); for (int q = 0; q < 6; q++) keep_cols.push_back(pose_col[i] + q); }
  for (int i = 0; i < nsb; i++) if (use_sb[i] && !rem_sb[i]) { ok = ok && emit(D2BA_SPEED_BIAS, w->sb_id[i], &w->sb[9 * i], 9); for (int q = 0; q < 9; q++) keep_cols.push_back(sb_col[i] + q); }
  for (int i = 0; i < ne; i++) if (use_ext[i]) { ok = ok && emit(D2BA_EXTRINSIC, w->ext_id[i], &w->ext[7 * i], 7); for (int q = 0; q < 6; q++) keep_cols.push_back(ext_col[i] + q); }
  if (use_td) { ok = ok && emit(D2BA_TD, 0, &w->td, 1); keep_cols.push_back(td_col); }
  if (!ok) return fail(h, 61, "marginalize: refs_out too small");
  for (int i = 0; i < np; i++) if (use_pose[i] && rem_pose[i]) for (int q = 0; q < 6; q++) rem_cols.push_back(pose_col[i] + q);
  for (int i = 0; i < nsb; i++) if (use_sb[i] && rem_sb[i]) for (int q = 0; q < 9; q++) rem_cols.push_back(sb_col[i] + q);
  nk = (int)keep_cols.size();
  const int nr = (int)rem_cols.size();
  if (nk > max_m) return fail(h, 62, "marginalize: A_out too small");
  if (nk == 0 || nr == 0) return fail(h, 63, "marginalize: nothing to keep or nothing to remove (reference returns nullptr)");
  if ((rc = d2ba_add_proj(t, 0, (int)robs.size(), robs.data()))) return fail(h, rc, std::string("marginalize/add_proj: ") + t->err);
  if (!rimu.empty() && (rc = d2ba_add_imu(t, 0, (int)rimu.size(), rimu.data()))) return fail(h, rc, std::string("marginalize/add_imu: ") + t->err);
  if (w->prior_m > 0) {
    std::vector<d2ba_blockref> pr; std::vector<double> px0;
    for (const HPriorBlk &b : w->prior_blk) {
      d2ba_blockref r; r.kind = b.kind; r.pad = 0;
      r.id = b.kind == D2BA_POSE ? w->pose_id[b.index] : b.kind == D2BA_EXTRINSIC ? w->ext_id[b.index] : b.kind == D2BA_SPEED_BIAS ? w->sb_id[b.index]
             : b.kind == D2BA_LANDMARK ? w->lm_id[b.index] : 0;
      pr.push_back(r); px0.insert(px0.end(), b.x0, b.x0 + kind_size(b.kind));
    }
    if ((rc = set_prior_common(t, 0, w->prior_m, w->prior_J.data(), w->prior_e0.data(), (int)pr.size(), pr.data(), px0.data(), w->prior_is_info)))
      return fail(h, rc, std::string("marginalize/prior: ") + t->err);
  }
  if ((rc = d2ba_finalize(t))) return fail(h, rc, std::string("marginalize/finalize: ") + t->err);
  if (t->h_win[0].n_c != col) return fail(h, 64, "marginalize: internal column count mismatch");
  // linearise and eliminate the landmarks (mu = 0)
  t->dev.prm.fixed_mode = 1; t->dev.prm.max_iter = 1;
  launch_tr_reset(t->dev, 1, t->stream);
  enqueue_linearize(t, 1);
  launch_control(t->dev, 1, t->stream);
  launch_lm_gather(t->dev, t->d_lm_win.p, t->nl_total, t->max_row_tiles * 32, t->any_compact, t->any_wide, t->stream);
  if (t->max_ldw_small > 0) launch_schur_small(t->dev, t->max_ldw_small, t->stream);
  launch_schur(t->dev, t->d_schur.p, t->n_schur, t->stream);
  // eliminate the removed camera columns
  DBuf<int> d_keep, d_rem, d_flag; DBuf<double> d_A, d_b;
  cudaError_t ce;
  if ((ce = d_keep.alloc(nk)) || (ce = d_rem.alloc(nr)) || (ce = d_flag.alloc(1)) || (ce = d_A.alloc((size_t)nk * nk)) || (ce = d_b.alloc(nk)))
    return fail(h, 65, "marginalize: device allocation failed");
  cudaMemcpyAsync(d_keep.p, keep_cols.data(), nk * sizeof(int), cudaMemcpyHostToDevice, t->stream);
  cudaMemcpyAsync(d_rem.p, rem_cols.data(), nr * sizeof(int), cudaMemcpyHostToDevice, t->stream);
  cudaMemsetAsync(d_flag.p, 0, sizeof(int), t->stream);
  const WinDesc &td_ = t->h_win[0];
  if (launch_marg_reduce(t->d_S.p + td_.offH, td_.ldh, td_.n_c, d_keep.p, nk, d_rem.p, nr, d_A.p, d_b.p, d_flag.p, t->stream))
    return fail(h, 66, "marginalize: reduce kernel needs more shared memory than available");
  int flag = 0;
  cudaMemcpyAsync(A_out, d_A.p, (size_t)nk * nk * 8, cudaMemcpyDeviceToHost, t->stream);
  cudaMemcpyAsync(b_out, d_b.p, (size_t)nk * 8, cudaMemcpyDeviceToHost, t->stream);
  cudaMemcpyAsync(&flag, d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, t->stream);
  ce = cudaStreamSynchronize(t->stream);
  d_keep.release(); d_rem.release(); d_flag.release(); d_A.release(); d_b.release();
  if (ce != cudaSuccess || cudaGetLastError() != cudaSuccess) return fail(h, 67, std::string("marginalize: ") + cudaGetErrorString(ce));
  if (flag) return fail(h, 68, "marginalize: removed block is not positive definite");
  *m_out = nk; *nblk_out = nblk;
  return 0;
}

// Per-kernel device time of the iteration sequence (CUDA events on the solver stream, no graph):
// ms_out[0..6] = lm_gather, schur, chol, step, misc_lin, proj_lin, control, summed over `iters` iterations;
// ms_out[7] = number of iterations timed; ms_out[8], [9] = the speed-bias elimination / back-substitution share of the
// chol bucket.  Used by bench.py for the roofline of the dominant kernel.
int d2ba_debug_kernel_times(d2ba_handle *h, int32_t iters, double *ms_out) {
  if (!h) return 1;
  cudaSetDevice(h->cfg.device);
  if (!h->finalized) { int rc = d2ba_finalize(h); if (rc) return rc; }
  if (h->state_dirty) { int rc = upload_state(h); if (rc) return rc; }
  h->dev.prm.fixed_mode = 1; h->dev.prm.max_iter = iters;
  release_graph(h);
  launch_tr_reset(h->dev, 1, h->stream);
  if (h->any_admm) { launch_cons_init(h->dev, h->n6_total, h->stream); int rc = consensus_exchange(h); if (rc) return rc; }
  enqueue_linearize(h, 1);
  launch_control(h->dev, 1, h->stream);
  cudaEvent_t ev[8], evs[2], evl[3];
  for (int i = 0; i < 3; i++) cudaEventCreate(&evl[i]);
  for (int i = 0; i < 8; i++) cudaEventCreate(&ev[i]);
  cudaEventCreate(&evs[0]); cudaEventCreate(&evs[1]);
  for (int i = 0; i < 12; i++) ms_out[i] = 0;
  for (int it = 0; it < iters; it++) {
    cudaEventRecord(ev[0], h->stream); launch_lm_gather(h->dev, h->d_lm_win.p, h->nl_total, h->max_row_tiles * 32, h->any_compact, h->any_wide, h->stream);
    cudaEventRecord(evs[0], h->stream); if (h->sbe_smem > 0) launch_sb_elim(h->dev, h->sbe_smem, h->stream);
    cudaEventRecord(ev[1], h->stream);
    cudaEventRecord(evl[0], h->stream);
    if (h->n_leaf_total > 0) launch_leaf_elim(h->dev, h->leaf_smem, h->stream);
    cudaEventRecord(evl[1], h->stream);
    if (h->max_ldw_small > 0) launch_schur_small(h->dev, h->max_ldw_small, h->stream);
    if (h->n_schur > h->n_schur0) launch_schur(h->dev, h->d_schur.p + h->n_schur0, h->n_schur - h->n_schur0, h->stream);
    cudaEventRecord(ev[2], h->stream); if (h->max_n_smem > 0) launch_chol_smem(h->dev, h->max_n_smem, h->stream); if (h->any_chol_glob) launch_chol(h->dev, h->max_rows_glob, h->stream); cudaEventRecord(evs[1], h->stream); if (h->sbe_smem > 0) launch_sb_back(h->dev, h->sbb_smem, h->stream);
    cudaEventRecord(evl[2], h->stream); if (h->n_leaf_total > 0) launch_leaf_back(h->dev, h->leafb_smem, h->stream);
    cudaEventRecord(ev[3], h->stream); launch_step(h->dev, h->max_nc, h->stream);
    cudaEventRecord(ev[4], h->stream); launch_misc_lin(h->dev, 0, h->max_prior_m, h->stream); launch_imu_lin(h->dev, 0, h->n_imu_total, h->stream);
    cudaEventRecord(ev[5], h->stream); for (int v = 0; v < 6; v++) launch_proj_lin(h->dev, v, 0, h->job_begin[v], h->job_count[v], h->stream);
    cudaEventRecord(ev[6], h->stream); launch_control(h->dev, 0, h->stream);
    cudaEventRecord(ev[7], h->stream);
    CK(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < 7; i++) { float ms = 0; cudaEventElapsedTime(&ms, ev[i], ev[i + 1]); ms_out[i] += ms; }
    { float ms = 0; cudaEventElapsedTime(&ms, evs[0], ev[1]); ms_out[8] += ms; cudaEventElapsedTime(&ms, evs[1], evl[2]); ms_out[9] += ms;
      cudaEventElapsedTime(&ms, evl[0], evl[1]); ms_out[10] += ms; cudaEventElapsedTime(&ms, evl[2], ev[3]); ms_out[11] += ms; }
  }
  ms_out[7] = iters;
  for (int i = 0; i < 8; i++) cudaEventDestroy(ev[i]);
  cudaEventDestroy(evs[0]); cudaEventDestroy(evs[1]);
  for (int i = 0; i < 3; i++) cudaEventDestroy(evl[i]);
  CK(cudaGetLastError());
  h->state_dirty = true;
  return 0;
}

}  // extern "C"
