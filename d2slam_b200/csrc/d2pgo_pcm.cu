// d2pgo_pcm.cu -- PCM loop-closure outlier rejection on the GPU (include/d2pgo.h d2pgo_pcm): the pairwise-consistency test
// of every two loops of a drone pair, then the maximum clique of each pair's consistency graph.  It shares only the handle
// (its stream, events, error string and dof) with the solver of d2pgo.cu.
#include <math.h>
#include <string.h>

#include <algorithm>

#include "d2ba_math.cuh"
#include "d2pgo_handle.cuh"

using namespace d2ba;
using d2pgo_host::PcmBufs;

namespace {

// ---- PCM: pairwise-consistency maximisation over the loop closures (SwarmLocalOutlierRejection, non-incremental, redundant;
// d2pgo/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp:46-303).  Loops are grouped by the unordered pair of drones;
// a group's loops occupy consecutive slots in input order.  Per group: a bit-packed adjacency [L][W = ceil(L/32)] words,
// bit (i, j) = smd(edge1 = max(i, j), edge2 = min(i, j)) < thres, then FMC maxCliqueHeu on it; inlier = in the clique.
constexpr int kPcmMaxGroup = 32768;   // 128 MB of adjacency bits
constexpr int kPcmWarps = 8;          // warps of a k_pcm_clique CTA = seeds examined per round

struct PcmDev {
  const int *g_loop;          // [G+1] slot offsets of the groups
  const long long *g_word;    // [G+1] adjacency word offsets (sum of L W)
  const long long *g_smd;     // [G+1] offsets of the tested pairs (sum of L (L-1) / 2)
  const int *fa, *fb;         // [n] frame index of the loop's two keyframes, by slot
  const unsigned char *flip;  // [n] drone ids in the opposite order to the other loops of the group with flip = 0
  const double *rel;          // [n][8] measured T_a^-1 T_b [t, q xyzw], by slot
  const double *cov;          // [n][21] loop covariance (S^T S)^-1, packed lower triangle, by slot
  const double *ego;          // [F][8] ego poses
  const double *path;         // [F] path length of the frame's drone from its first keyframe
  unsigned *adj; int *deg; double *smd;
  int is4; double thr, pos_cov, yaw_cov;
};

struct Pose7 { double t[3]; Q4 q; };
D2BA_DEV Q4 qnormalized(const Q4 &q) { const double s = 1.0 / sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w); return Q4{q.x * s, q.y * s, q.z * s, q.w * s}; }
D2BA_DEV Pose7 p7_load(const double *p) { return Pose7{{p[0], p[1], p[2]}, qnormalized(qload(p + 3))}; }
D2BA_DEV Pose7 p7_mul(const Pose7 &a, const Pose7 &b) {   // a * b (Swarm::Pose composition; attitude normalised as its constructor does)
  double R[9], v[3];
  q2R(a.q, R); mv3(R, b.t, v);
  return Pose7{{v[0] + a.t[0], v[1] + a.t[1], v[2] + a.t[2]}, qnormalized(qmul(a.q, b.q))};
}
D2BA_DEV Pose7 p7_inv(const Pose7 &a) {
  const Q4 qi = qinv(a.q);
  double R[9], v[3];
  q2R(qi, R); mv3(R, a.t, v);
  return Pose7{{-v[0], -v[1], -v[2]}, qnormalized(qi)};
}
D2BA_DEV double quat_yaw(const Q4 &q) { return atan2(2.0 * (q.w * q.z + q.x * q.y), 1.0 - 2.0 * (q.y * q.y + q.z * q.z)); }

// ego motion from frame f to frame g of one drone: DeltaPose(ego_f, ego_g[, yaw only]) and the diagonal of d2pgo's ego-motion
// covariance (d2pgo.cpp:482-493) at the path length between them (ASSUMED DroneTrajectory::get_relative_pose_by_frame_id)
D2BA_DEV Pose7 pcm_odom(const PcmDev &d, int f, int g, double *cp, double *cr) {
  const Pose7 a = p7_load(d.ego + (size_t)f * 8), b = p7_load(d.ego + (size_t)g * 8);
  const double len = fabs(d.path[g] - d.path[f]);
  *cp = d.pos_cov * len + 0.5 * d.yaw_cov * len * len;
  *cr = d.yaw_cov * len;
  if (!d.is4) return p7_mul(p7_inv(a), b);
  const double ya = quat_yaw(a.q), dy = quat_yaw(b.q) - ya;
  double s, c, sh, ch;
  sincos(ya, &s, &c); sincos(0.5 * dy, &sh, &ch);
  const double v[3] = {b.t[0] - a.t[0], b.t[1] - a.t[1], b.t[2] - a.t[2]};
  return Pose7{{c * v[0] + s * v[1], -s * v[0] + c * v[1], v[2]}, qnormalized(Q4{0.0, 0.0, sh, ch})};
}

// squared Mahalanobis distance of the loop pair (edge1 = slot e1, edge2 = slot e2; swarm_outlier_rejection.cpp:141-199)
D2BA_DEV double pcm_smd(const PcmDev &d, int e1, int e2) {
  const bool same = d.flip[e1] == d.flip[e2];   // same_robot_pair 1; otherwise 2
  Pose7 p2 = p7_load(d.rel + (size_t)e2 * 8);
  if (!same) p2 = p7_inv(p2);
  double ca_p, ca_r, cb_p, cb_r;
  const Pose7 oa = pcm_odom(d, d.fa[e1], same ? d.fa[e2] : d.fb[e2], &ca_p, &ca_r);
  const Pose7 ob = pcm_odom(d, d.fb[e1], same ? d.fb[e2] : d.fa[e2], &cb_p, &cb_r);
  const Pose7 err = p7_mul(p7_mul(p7_mul(oa, p2), p7_inv(ob)), p7_inv(p7_load(d.rel + (size_t)e1 * 8)));
  // log_map (ASSUMED = tangentSpace: [t ; angle-axis], angle = 2 atan2(|v|, |w|), sign of w)
  double v[6] = {err.t[0], err.t[1], err.t[2], 0.0, 0.0, 0.0};
  const double n = sqrt(err.q.x * err.q.x + err.q.y * err.q.y + err.q.z * err.q.z);
  if (n > 0.0) {
    const double k = 2.0 * atan2(n, fabs(err.q.w)) * (err.q.w < 0.0 ? -1.0 : 1.0) / n;
    v[3] = k * err.q.x; v[4] = k * err.q.y; v[5] = k * err.q.z;
  }
  // Sigma = (cov_1 + cov_2) + (cov(odom_a) + cov(odom_b)), then v^T Sigma^-1 v by Cholesky (packed lower triangle)
  double A[21];
  const double *c1 = d.cov + (size_t)e1 * 21, *c2 = d.cov + (size_t)e2 * 21;
  for (int k = 0; k < 21; k++) A[k] = c1[k] + c2[k];
  for (int k = 0; k < 6; k++) A[k * (k + 3) / 2] += k < 3 ? ca_p + cb_p : ca_r + cb_r;
  double y[6], s = 0.0;
  for (int j = 0; j < 6; j++) {
    double t = A[j * (j + 1) / 2 + j];
    for (int k = 0; k < j; k++) t -= A[j * (j + 1) / 2 + k] * A[j * (j + 1) / 2 + k];
    const double l = sqrt(t);
    A[j * (j + 1) / 2 + j] = l;
    for (int r = j + 1; r < 6; r++) {
      double u = A[r * (r + 1) / 2 + j];
      for (int k = 0; k < j; k++) u -= A[r * (r + 1) / 2 + k] * A[j * (j + 1) / 2 + k];
      A[r * (r + 1) / 2 + j] = u / l;
    }
    double w = v[j];
    for (int k = 0; k < j; k++) w -= A[j * (j + 1) / 2 + k] * y[k];
    y[j] = w / l;
    s += y[j] * y[j];
  }
  return s;
}

// per drone (one warp each): path length from its first keyframe, in trajectory order, by a fixed-order warp scan
__global__ void k_pcm_path(int n_drones, const int *traj_ptr, const int *traj, const double *ego, double *path) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n_drones) return;
  const int b = traj_ptr[w], n = traj_ptr[w + 1] - b;
  double carry = 0.0;
  for (int base = 0; base < n; base += 32) {
    const int k = base + lane;
    double x = 0.0;
    if (k > 0 && k < n) {
      const double *p = ego + (size_t)traj[b + k] * 8, *q = ego + (size_t)traj[b + k - 1] * 8;
      const double dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
      x = sqrt(dx * dx + dy * dy + dz * dz);
    }
    for (int o = 1; o < 32; o <<= 1) { const double u = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += u; }
    if (k < n) path[traj[b + k]] = carry + x;
    carry += __shfl_sync(0xffffffffu, x, 31);
  }
}

// per loop slot: measurement in slot order and covariance = (S^T S)^-1 (ASSUMED LoopEdge::getCovariance)
__global__ void k_pcm_loop(int n, const int *src, const double *rel7, const double *sqrt36, double *rel, double *cov) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const size_t s = (size_t)src[e];
  for (int k = 0; k < 7; k++) rel[(size_t)e * 8 + k] = rel7[s * 7 + k];
  rel[(size_t)e * 8 + 7] = 0.0;
  const double *S = sqrt36 + s * 36;
  double A[36], Li[36];
  for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) { double t = 0; for (int k = 0; k < 6; k++) t += S[k * 6 + i] * S[k * 6 + j]; A[i * 6 + j] = t; }
  for (int j = 0; j < 6; j++) {   // A = L L^T
    double t = A[j * 7];
    for (int k = 0; k < j; k++) t -= A[j * 6 + k] * A[j * 6 + k];
    A[j * 7] = sqrt(t);
    for (int r = j + 1; r < 6; r++) { double u = A[r * 6 + j]; for (int k = 0; k < j; k++) u -= A[r * 6 + k] * A[j * 6 + k]; A[r * 6 + j] = u / A[j * 7]; }
  }
  for (int c = 0; c < 6; c++)
    for (int r = 0; r < 6; r++) {
      double t = r == c ? 1.0 : 0.0;
      for (int k = c; k < r; k++) t -= A[r * 6 + k] * Li[k * 6 + c];
      Li[r * 6 + c] = r < c ? 0.0 : t / A[r * 7];
    }
  for (int r = 0; r < 6; r++) for (int c = 0; c <= r; c++) {   // (L L^T)^-1 = L^-T L^-1
    double t = 0;
    for (int k = r; k < 6; k++) t += Li[k * 6 + r] * Li[k * 6 + c];
    cov[(size_t)e * 21 + r * (r + 1) / 2 + c] = t;
  }
}

D2BA_DEV int pcm_group_of(const long long *off, int G, long long t) {   // the g with off[g] <= t < off[g + 1]
  int lo = 0, hi = G - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (off[mid] <= t) lo = mid; else hi = mid - 1; }
  return lo;
}

// one warp per adjacency word (row i, columns 32 w .. 32 w + 31 of a group): the word is a ballot, so no atomics.  Cell (i, j)
// is the pair with edge1 = max(i, j); the smd of j < i is kept for d2pgo_debug_pcm_smd.
__global__ void __launch_bounds__(256) k_pcm_pairs(PcmDev d, int G, long long n_words) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= n_words) return;
  const int g = pcm_group_of(d.g_word, G, t);
  const int base = d.g_loop[g], L = d.g_loop[g + 1] - base, W = (L + 31) >> 5;
  const long long local = t - d.g_word[g];
  const int i = (int)(local / W), j = (int)(local % W) * 32 + lane;
  bool ok = false;
  if (j < L && j != i) {
    const double s = pcm_smd(d, base + max(i, j), base + min(i, j));
    ok = s < d.thr;
    if (j < i) d.smd[d.g_smd[g] + (long long)i * (i - 1) / 2 + j] = s;
  }
  const unsigned word = __ballot_sync(0xffffffffu, ok);
  if (lane == 0) d.adj[t] = word;
}

__global__ void k_pcm_degree(int G, const int *g_loop, const long long *g_word, const unsigned *adj, int *deg) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= g_loop[G]) return;
  int lo = 0, hi = G - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (g_loop[mid] <= e) lo = mid; else hi = mid - 1; }
  const int L = g_loop[lo + 1] - g_loop[lo], W = (L + 31) >> 5;
  const unsigned *row = adj + g_word[lo] + (long long)(e - g_loop[lo]) * W;
  int c = 0;
  for (int k = 0; k < W; k++) c += __popc(row[k]);
  deg[e] = c;
}

// FMC's greedy from seed s under the running maximum m (findCliqueHeu.cpp:146-239): C = N(s) & {deg >= m}; repeat
// v = max C, C &= N(v).  One warp; rows `pitch` words apart; C in shared memory, word k owned by lane k % 32.  Returns the
// clique size 1 + picks, or 0 once the clique can no longer exceed m (1 + picks + |C| <= m): such a seed is never taken, so
// stopping early changes nothing.
template <typename Pitch> D2BA_DEV int pcm_greedy(int s, int m, const unsigned *rows, Pitch pitch, int W, const unsigned *degmask, unsigned *C, int lane, long long *rounds, unsigned char *member) {
  for (int k = lane; k < W; k += 32) C[k] = rows[(size_t)s * pitch + k] & degmask[k];
  if (member && lane == 0) member[s] = 1;
  int picks = 0;
  for (;;) {
    int cnt = 0, hi = -1;
    for (int k = lane; k < W; k += 32) { const unsigned c = C[k]; cnt += __popc(c); if (c) hi = k * 32 + 31 - __clz(c); }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    hi = __reduce_max_sync(0xffffffffu, hi);
    if (1 + picks + cnt <= m) return 0;
    if (cnt == 0) return 1 + picks;
    if (member && lane == 0) member[hi] = 1;
    picks++; (*rounds)++;
    for (int k = lane; k < W; k += 32) C[k] &= rows[(size_t)hi * pitch + k];
  }
}

D2BA_DEV void pcm_degmask(unsigned *degmask, const int *deg, int L, int W, int m) {   // bit u: u < L and deg(u) >= m
  for (int k = threadIdx.x; k < W; k += blockDim.x) {
    unsigned w = 0;
    for (int b = 0; b < 32; b++) { const int u = k * 32 + b; if (u < L && deg[u] >= m) w |= 1u << b; }
    degmask[k] = w;
  }
}

// one CTA per group: FMC maxCliqueHeu, exactly.  Seeds are taken kPcmWarps at a time under the current m; the first of them
// (by index) whose clique exceeds m commits, and the seeds after it are examined again under the new m.  The committed seed's
// clique is rebuilt at the end under the m it was found with.  stats[g] = {sum of degrees, greedy rounds}.
__global__ void __launch_bounds__(kPcmWarps * 32) k_pcm_clique(const int *g_loop, const long long *g_word, const unsigned *adj, const int *deg_all, unsigned char *inlier, long long *stats) {
  extern __shared__ unsigned pcm_smem[];
  __shared__ int s_size[kPcmWarps], s_m, s_best, s_best_m, s_next;
  __shared__ long long s_part[kPcmWarps * 32];
  const int g = blockIdx.x, base = g_loop[g], L = g_loop[g + 1] - base, W = (L + 31) >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned *rows = adj + g_word[g];
  const int *deg = deg_all + base;
  unsigned *degmask = pcm_smem, *C = pcm_smem + W * (1 + warp);
  long long rounds = 0, dsum = 0;
  for (int k = threadIdx.x; k < L; k += blockDim.x) { inlier[base + k] = 0; dsum += deg[k]; }
  if (threadIdx.x == 0) { s_m = -1; s_best = -1; s_best_m = -1; }
  pcm_degmask(degmask, deg, L, W, -1);
  __syncthreads();
  for (int s0 = 0; s0 < L;) {
    const int m = s_m, s = s0 + warp;
    int size = 0;
    if (s < L && !(m > deg[s])) size = pcm_greedy(s, m, rows, W, W, degmask, C, lane, &rounds, nullptr);   // Pruning 1
    if (lane == 0) s_size[warp] = size;
    __syncthreads();
    if (threadIdx.x == 0) {
      s_next = s0 + kPcmWarps;
      for (int w = 0; w < kPcmWarps; w++)
        if (s_size[w] > m) { s_best = s0 + w; s_best_m = m; s_m = s_size[w]; s_next = s0 + w + 1; break; }
    }
    __syncthreads();
    if (s_m != m) { pcm_degmask(degmask, deg, L, W, s_m); __syncthreads(); }
    s0 = s_next;
    __syncthreads();
  }
  if (s_best >= 0) {
    pcm_degmask(degmask, deg, L, W, s_best_m);
    __syncthreads();
    if (warp == 0) { long long dummy = 0; pcm_greedy(s_best, s_best_m, rows, W, W, degmask, C, lane, &dummy, inlier + base); }
  }
  s_part[threadIdx.x] = lane == 0 ? rounds : 0;   // every lane of a warp counted the same rounds
  __syncthreads();
  if (threadIdx.x == 0) { long long r = 0; for (int k = 0; k < kPcmWarps * 32; k++) r += s_part[k]; s_part[0] = r; }
  __syncthreads();
  const long long r = s_part[0];
  __syncthreads();
  s_part[threadIdx.x] = dsum;
  __syncthreads();
  if (threadIdx.x == 0) { long long t = 0; for (int k = 0; k < kPcmWarps * 32; k++) t += s_part[k]; stats[2 * g] = t; stats[2 * g + 1] = r; }
}

// one clique search of k_pcm_clique_jobs: a group's rows (row pitch `pitch` words), its degrees and its member flags.  Seeds are
// s_lo .. L-1 and the running maximum starts at m0: s_lo = 0, m0 = -1 is FMC maxCliqueHeu, as k_pcm_clique; s_lo = L0 (the first
// new vertex), m0 = the group's clique size is maxCliqueHeuIncremental's search (findCliqueHeuInc.cpp:32-96).
struct PcmCliqueJob { const unsigned *rows; int *deg; unsigned char *member; long long pitch; int L, s_lo, m0; };

// k_pcm_clique on a job table (the PCM stream, d2pgo_debug_pcm_clique_inc), one CTA per job, with the same rounds.  When a seed
// commits, the member flags [0, L) are replaced by its clique, rebuilt at the end under the m it was found with; otherwise they
// stay.  stats[j] = {sum of degrees, greedy rounds}.
__global__ void __launch_bounds__(kPcmWarps * 32) k_pcm_clique_jobs(const PcmCliqueJob *jobs, long long *stats) {
  extern __shared__ unsigned pcm_smem[];
  __shared__ int s_size[kPcmWarps], s_m, s_best, s_best_m, s_next;
  __shared__ long long s_part[kPcmWarps * 32];
  const PcmCliqueJob J = jobs[blockIdx.x];
  const int L = J.L, W = (L + 31) >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned *rows = J.rows;
  const int *deg = J.deg;
  unsigned *degmask = pcm_smem, *C = pcm_smem + W * (1 + warp);
  long long rounds = 0, dsum = 0;
  for (int k = threadIdx.x; k < L; k += blockDim.x) dsum += deg[k];
  if (threadIdx.x == 0) { s_m = J.m0; s_best = -1; s_best_m = -1; }
  pcm_degmask(degmask, deg, L, W, J.m0);
  __syncthreads();
  for (int s0 = J.s_lo; s0 < L;) {
    const int m = s_m, s = s0 + warp;
    int size = 0;
    if (s < L && !(m > deg[s])) size = pcm_greedy(s, m, rows, J.pitch, W, degmask, C, lane, &rounds, nullptr);   // Pruning 1
    if (lane == 0) s_size[warp] = size;
    __syncthreads();
    if (threadIdx.x == 0) {
      s_next = s0 + kPcmWarps;
      for (int w = 0; w < kPcmWarps; w++)
        if (s_size[w] > m) { s_best = s0 + w; s_best_m = m; s_m = s_size[w]; s_next = s0 + w + 1; break; }
    }
    __syncthreads();
    if (s_m != m) { pcm_degmask(degmask, deg, L, W, s_m); __syncthreads(); }
    s0 = s_next;
    __syncthreads();
  }
  if (s_best >= 0) {
    for (int k = threadIdx.x; k < L; k += blockDim.x) J.member[k] = 0;
    pcm_degmask(degmask, deg, L, W, s_best_m);
    __syncthreads();
    if (warp == 0) { long long dummy = 0; pcm_greedy(s_best, s_best_m, rows, J.pitch, W, degmask, C, lane, &dummy, J.member); }
  }
  s_part[threadIdx.x] = lane == 0 ? rounds : 0;   // every lane of a warp counted the same rounds
  __syncthreads();
  if (threadIdx.x == 0) { long long r = 0; for (int k = 0; k < kPcmWarps * 32; k++) r += s_part[k]; s_part[0] = r; }
  __syncthreads();
  const long long r = s_part[0];
  __syncthreads();
  s_part[threadIdx.x] = dsum;
  __syncthreads();
  if (threadIdx.x == 0) { long long t = 0; for (int k = 0; k < kPcmWarps * 32; k++) t += s_part[k]; stats[2 * blockIdx.x] = t; stats[2 * blockIdx.x + 1] = r; }
}

// ---- the PCM stream (d2pgo_pcm_stream): a group's adjacency is [cap][pitch] words with cap = 32 pitch rows; its rows 0 .. L0-1
// are the loops of earlier calls, L0 .. L-1 the loops new in this call.  slot[r] = the stream's loop index of row r.
struct PcmPairJob { unsigned *adj; const int *slot; double *smd; long long pitch; int L0, L; };

// one warp per adjacency word that a call changes: every word of the new rows, and the words of the old rows that cover columns
// >= L0.  Same cell rule and ballot as k_pcm_pairs; an old row's bits below column L0 are kept.  The smd of new row i against
// j < i is kept at smd[i (i - 1) / 2 - L0 (L0 - 1) / 2 + j] for d2pgo_debug_pcm_stream_smd.
__global__ void __launch_bounds__(256) k_pcm_stream_pairs(PcmDev d, const PcmPairJob *jobs, const long long *job_word, int n_jobs, long long n_words) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= n_words) return;
  const int g = pcm_group_of(job_word, n_jobs, t);
  const PcmPairJob &J = jobs[g];
  const int L0 = J.L0, L = J.L, W = (L + 31) >> 5;
  long long local = t - job_word[g];
  const long long n_new = (long long)(L - L0) * W;
  int i, w;
  unsigned keep = 0;
  if (local < n_new) { i = L0 + (int)(local / W); w = (int)(local % W); }
  else {
    local -= n_new;
    const int w0 = L0 >> 5, Wo = W - w0;
    i = (int)(local / Wo); w = w0 + (int)(local % Wo);
    if (w == w0) keep = (1u << (L0 & 31)) - 1u;
  }
  const int j = w * 32 + lane;
  bool ok = false;
  if (j < L && j != i && j >= (i < L0 ? L0 : 0)) {
    const double s = pcm_smd(d, J.slot[max(i, j)], J.slot[min(i, j)]);
    ok = s < d.thr;
    if (j < i) J.smd[(long long)i * (i - 1) / 2 - (long long)L0 * (L0 - 1) / 2 + j] = s;
  }
  const unsigned word = __ballot_sync(0xffffffffu, ok);
  if (lane == 0) { unsigned *p = J.adj + i * J.pitch + w; *p = (*p & keep) | word; }
}

// thread per row of the jobs' groups: degree = popcount of the row (row_off: prefix sums of the jobs' L)
__global__ void k_pcm_stream_degree(const PcmCliqueJob *jobs, const int *row_off, int n_jobs) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= row_off[n_jobs]) return;
  int lo = 0, hi = n_jobs - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (row_off[mid] <= e) lo = mid; else hi = mid - 1; }
  const PcmCliqueJob &J = jobs[lo];
  const int r = e - row_off[lo], W = (J.L + 31) >> 5;
  const unsigned *row = J.rows + r * J.pitch;
  int c = 0;
  for (int k = 0; k < W; k++) c += __popc(row[k]);
  J.deg[r] = c;
}

}  // namespace

struct d2pgo_host::PcmBufs {
  Buf<int> g_loop, fa, fb, src, traj_ptr, traj, deg; Buf<long long> g_word, g_smd, stats; Buf<unsigned char> flip, inlier;
  Buf<double> rel_in, sqrt_in, rel, cov, ego, path, smd; Buf<unsigned> adj; Buf<PcmCliqueJob> jobs;   // jobs: d2pgo_debug_pcm_clique_inc
  long long n_smd = -1;   // tested pairs of the last d2pgo_pcm call (-1: none yet)
  cudaEvent_t ev_pair = nullptr;
  ~PcmBufs() { if (ev_pair) cudaEventDestroy(ev_pair); }
};

void d2pgo_host::PcmBufsFree::operator()(PcmBufs *p) const { delete p; }

// FMC on groups already in h->pcm (g_loop, g_word, adj): degrees, one clique CTA per group; inlier flags by slot, stats per group
static int pcm_run_clique(d2pgo_handle *h, int G, int n, int max_w) {
  PcmBufs &P = *h->pcm;
  PCK(P.deg.alloc(n)); PCK(P.inlier.alloc(n)); PCK(P.stats.alloc(2 * (size_t)G));
  if (n > 0) k_pcm_degree<<<(n + 255) / 256, 256, 0, h->stream>>>(G, P.g_loop.p, P.g_word.p, P.adj.p, P.deg.p);
  if (G > 0) k_pcm_clique<<<G, kPcmWarps * 32, (size_t)(1 + kPcmWarps) * max_w * 4, h->stream>>>(P.g_loop.p, P.g_word.p, P.adj.p, P.deg.p, P.inlier.p, P.stats.p);
  PCK(cudaGetLastError());
  return 0;
}

// ---- the PCM stream's state (d2pgo_pcm_stream): frames, loops and per-group consistency graphs that stay on the device
namespace {

// grow b to hold at least `need` elements (capacity doubles), keeping the first `used`; new elements are zeroed
template <typename T> cudaError_t pcm_grow(d2pgo_host::Buf<T> &b, size_t used, size_t need, cudaStream_t st) {
  if (b.p && need <= b.n) return cudaSuccess;
  d2pgo_host::Buf<T> nb;
  cudaError_t e = nb.alloc(std::max(need, 2 * b.n));
  if (e == cudaSuccess) e = cudaMemsetAsync(nb.p, 0, nb.n * sizeof(T), st);
  if (e == cudaSuccess && used) e = cudaMemcpyAsync(nb.p, b.p, used * sizeof(T), cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);   // the old array is freed below
  if (e != cudaSuccess) return e;
  std::swap(b.p, nb.p); std::swap(b.n, nb.n);
  return cudaSuccess;
}

struct PcmStreamGroup {   // one drone pair: L loops (rows), an adjacency of cap = 32 pitch rows, the clique's member flags
  int32_t lo, hi;
  int L = 0, pitch = 0, size = 0;
  long long dsum = 0;                    // sum of the degrees after the last call that touched the group
  d2pgo_host::Buf<unsigned> adj; d2pgo_host::Buf<int> slot, deg; d2pgo_host::Buf<unsigned char> member;
  std::vector<unsigned char> member_h;   // host copy of member [L]
};

}  // namespace

struct d2pgo_host::PcmStream {
  bool ready = false; int incremental = 0, is4 = 0; double thr = 0, pos_cov = 0, yaw_cov = 0;
  std::unordered_map<int64_t, int> fidx; std::vector<int32_t> f_agent;   // keyframe id -> frame index; frame -> drone
  std::unordered_map<int32_t, int> drone_of; std::vector<std::vector<int>> trajs;
  std::unordered_map<int64_t, int> loop_of; std::vector<int> l_group, l_row;   // loop id -> loop index; loop -> group, row
  std::unordered_map<uint64_t, int> gid; std::vector<std::unique_ptr<PcmStreamGroup>> groups;
  Buf<double> ego, path, rel, cov, rel_in, sqrt_in, smd; Buf<int> fa, fb, src, traj_ptr, traj, row_off; Buf<unsigned char> flip;
  Buf<PcmPairJob> pjobs; Buf<long long> pword, stats; Buf<PcmCliqueJob> cjobs;
  long long n_smd = -1;   // pairs tested by the last stream call (-1: none yet)
  cudaEvent_t ev_pair = nullptr;
  ~PcmStream() { if (ev_pair) cudaEventDestroy(ev_pair); }
};

void d2pgo_host::PcmStreamFree::operator()(PcmStream *p) const { delete p; }

extern "C" {

int d2pgo_default_pcm_config(d2pgo_pcm_config *c) {
  if (!c) return 1;
  memset(c, 0, sizeof *c);
  c->pcm_thres = 1.635; c->pos_covariance_per_meter = 4e-3; c->yaw_covariance_per_meter = 4e-5;
  return 0;
}

int d2pgo_pcm(d2pgo_handle *h, const d2pgo_pcm_config *cfg, int32_t n_frames, const int64_t *frame_ids, const int32_t *frame_agent, const double *ego_poses7,
              int32_t n_loops, const int64_t *kf_a, const int64_t *kf_b, const double *rel7, const double *sqrt_info36, uint8_t *inlier_out, d2pgo_pcm_report *rep) {
  if (!h) return 1;
  if (!cfg || n_frames < 0 || n_loops < 0 || (n_frames && (!frame_ids || !frame_agent || !ego_poses7)) ||
      (n_loops && (!kf_a || !kf_b || !rel7 || !sqrt_info36 || !inlier_out)))
    return pgo_fail(h, 1, "pcm: null argument or negative count");
  // the reference keeps pcm_thres in a float (SwarmLocalOutlierRejectionParams, d2pgo_config.h); the test is smd < that float
  const double thr = (double)(float)cfg->pcm_thres;
  if (!(std::isfinite(thr) && thr > 0.0)) return pgo_fail(h, 2, "pcm: pcm_thres must be finite and positive");
  if (!(std::isfinite(cfg->pos_covariance_per_meter) && cfg->pos_covariance_per_meter >= 0.0 && std::isfinite(cfg->yaw_covariance_per_meter) && cfg->yaw_covariance_per_meter >= 0.0))
    return pgo_fail(h, 2, "pcm: covariance rates must be finite and non-negative");
  cudaSetDevice(h->cfg.device);
  if (!h->pcm) h->pcm.reset(new PcmBufs());
  PcmBufs &P = *h->pcm;
  P.n_smd = -1;
  // keyframes -> (drone, position in its trajectory = order of appearance)
  std::unordered_map<int64_t, int> fidx;
  std::unordered_map<int32_t, int> drone_of;
  std::vector<std::vector<int>> trajs;
  for (int f = 0; f < n_frames; f++) {
    if (!fidx.emplace(frame_ids[f], f).second) return pgo_fail(h, 3, "pcm: duplicate keyframe id " + std::to_string(frame_ids[f]));
    auto it = drone_of.emplace(frame_agent[f], (int)trajs.size());
    if (it.second) trajs.emplace_back();
    trajs[it.first->second].push_back(f);
  }
  // groups: unordered drone pairs, numbered by first appearance; a group's loops keep their input order
  std::unordered_map<uint64_t, int> gid;
  std::vector<int> lg(n_loops), la(n_loops), lb(n_loops), gsize;
  std::vector<uint64_t> gkey;
  for (int e = 0; e < n_loops; e++) {
    auto a = fidx.find(kf_a[e]), b = fidx.find(kf_b[e]);
    if (a == fidx.end() || b == fidx.end())
      return pgo_fail(h, 3, "pcm: loop " + std::to_string(e) + " names unknown keyframe id " + std::to_string(a == fidx.end() ? kf_a[e] : kf_b[e]));
    la[e] = a->second; lb[e] = b->second;
    const uint32_t x = (uint32_t)frame_agent[la[e]], y = (uint32_t)frame_agent[lb[e]];
    const uint64_t key = (uint64_t)std::min(x, y) << 32 | std::max(x, y);
    auto it = gid.emplace(key, (int)gsize.size());
    if (it.second) { gsize.push_back(0); gkey.push_back(key); }
    lg[e] = it.first->second; gsize[lg[e]]++;
  }
  const int G = (int)gsize.size();
  std::vector<int> g_loop(G + 1, 0); std::vector<long long> g_word(G + 1, 0), g_smd(G + 1, 0);
  int max_w = 1;
  for (int g = 0; g < G; g++) {
    const long long L = gsize[g], W = (L + 31) / 32;
    if (L > kPcmMaxGroup)
      return pgo_fail(h, 4, "pcm: the group of drones " + std::to_string((int32_t)(gkey[g] >> 32)) + " and " + std::to_string((int32_t)(gkey[g] & 0xffffffffu)) + " has " +
                                std::to_string(L) + " loops; at most " + std::to_string(kPcmMaxGroup) + " are supported");
    g_loop[g + 1] = g_loop[g] + (int)L; g_word[g + 1] = g_word[g] + L * W; g_smd[g + 1] = g_smd[g] + L * (L - 1) / 2;
    max_w = std::max(max_w, (int)W);
  }
  std::vector<int> src(n_loops), sfa(n_loops), sfb(n_loops), fill(g_loop.begin(), g_loop.end() - 1);
  std::vector<unsigned char> flip(n_loops);
  for (int e = 0; e < n_loops; e++) {
    const int s = fill[lg[e]]++;
    src[s] = e; sfa[s] = la[e]; sfb[s] = lb[e]; flip[s] = frame_agent[la[e]] > frame_agent[lb[e]];
  }
  std::vector<int> traj_ptr(1, 0), traj;
  for (auto &t : trajs) { traj.insert(traj.end(), t.begin(), t.end()); traj_ptr.push_back((int)traj.size()); }
  std::vector<double> ego((size_t)n_frames * 8, 0.0);
  for (int f = 0; f < n_frames; f++) memcpy(&ego[(size_t)f * 8], ego_poses7 + (size_t)f * 7, 56);
  const size_t n = n_loops, F = n_frames;
  PCK(P.g_loop.alloc(G + 1)); PCK(P.g_word.alloc(G + 1)); PCK(P.g_smd.alloc(G + 1)); PCK(P.fa.alloc(n)); PCK(P.fb.alloc(n)); PCK(P.src.alloc(n)); PCK(P.flip.alloc(n));
  PCK(P.rel_in.alloc(n * 7)); PCK(P.sqrt_in.alloc(n * 36)); PCK(P.rel.alloc(n * 8)); PCK(P.cov.alloc(n * 21)); PCK(P.ego.alloc(F * 8)); PCK(P.path.alloc(F));
  PCK(P.traj_ptr.alloc(traj_ptr.size())); PCK(P.traj.alloc(F)); PCK(P.adj.alloc(g_word[G])); PCK(P.smd.alloc(g_smd[G]));
  if (!P.ev_pair) PCK(cudaEventCreate(&P.ev_pair));
  PCK(cudaMemcpyAsync(P.g_loop.p, g_loop.data(), (G + 1) * 4, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(P.g_word.p, g_word.data(), (G + 1) * 8, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(P.g_smd.p, g_smd.data(), (G + 1) * 8, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(P.traj_ptr.p, traj_ptr.data(), traj_ptr.size() * 4, cudaMemcpyHostToDevice, h->stream));
  if (F) {
    PCK(cudaMemcpyAsync(P.traj.p, traj.data(), F * 4, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(P.ego.p, ego.data(), F * 64, cudaMemcpyHostToDevice, h->stream));
  }
  if (n) {
    PCK(cudaMemcpyAsync(P.fa.p, sfa.data(), n * 4, cudaMemcpyHostToDevice, h->stream)); PCK(cudaMemcpyAsync(P.fb.p, sfb.data(), n * 4, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(P.src.p, src.data(), n * 4, cudaMemcpyHostToDevice, h->stream)); PCK(cudaMemcpyAsync(P.flip.p, flip.data(), n, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(P.rel_in.p, rel7, n * 56, cudaMemcpyHostToDevice, h->stream)); PCK(cudaMemcpyAsync(P.sqrt_in.p, sqrt_info36, n * 288, cudaMemcpyHostToDevice, h->stream));
  }
  PcmDev d;
  d.g_loop = P.g_loop.p; d.g_word = P.g_word.p; d.g_smd = P.g_smd.p; d.fa = P.fa.p; d.fb = P.fb.p; d.flip = P.flip.p; d.rel = P.rel.p; d.cov = P.cov.p;
  d.ego = P.ego.p; d.path = P.path.p; d.adj = P.adj.p; d.deg = P.deg.p; d.smd = P.smd.p;
  d.is4 = h->dof == 4; d.thr = thr; d.pos_cov = cfg->pos_covariance_per_meter; d.yaw_cov = cfg->yaw_covariance_per_meter;
  PCK(cudaEventRecord(h->ev0, h->stream));
  if (!trajs.empty()) k_pcm_path<<<((int)trajs.size() * 32 + 255) / 256, 256, 0, h->stream>>>((int)trajs.size(), P.traj_ptr.p, P.traj.p, P.ego.p, P.path.p);
  if (n) {
    k_pcm_loop<<<((int)n + 127) / 128, 128, 0, h->stream>>>((int)n, P.src.p, P.rel_in.p, P.sqrt_in.p, P.rel.p, P.cov.p);
    const long long words = g_word[G];
    k_pcm_pairs<<<(unsigned)((words * 32 + 255) / 256), 256, 0, h->stream>>>(d, G, words);
  }
  PCK(cudaGetLastError());
  PCK(cudaEventRecord(P.ev_pair, h->stream));
  if (int rc = pcm_run_clique(h, G, (int)n, max_w)) return rc;
  PCK(cudaEventRecord(h->ev1, h->stream));
  std::vector<unsigned char> inl(n);
  std::vector<long long> stats(2 * (size_t)G);
  if (n) PCK(cudaMemcpyAsync(inl.data(), P.inlier.p, n, cudaMemcpyDeviceToHost, h->stream));
  if (G) PCK(cudaMemcpyAsync(stats.data(), P.stats.p, 16 * (size_t)G, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  d2pgo_pcm_report R; memset(&R, 0, sizeof R);
  for (size_t s = 0; s < n; s++) { inlier_out[src[s]] = inl[s]; R.inliers += inl[s]; }
  for (int g = 0; g < G; g++) { R.consistent_pairs += stats[2 * g] / 2; R.clique_rounds += stats[2 * g + 1]; }
  R.groups = G; R.pairs_tested = g_smd[G];
  float ms = 0, mp = 0;
  cudaEventElapsedTime(&ms, h->ev0, h->ev1); cudaEventElapsedTime(&mp, h->ev0, P.ev_pair);
  R.device_ms = ms; R.pair_ms = mp; R.clique_ms = ms - mp;
  P.n_smd = g_smd[G];
  if (rep) *rep = R;
  return 0;
}

int d2pgo_debug_pcm_smd(d2pgo_handle *h, double *out, int64_t out_doubles) {
  if (!h) return 1;
  if (!h->pcm || h->pcm->n_smd < 0) return pgo_fail(h, 2, "debug_pcm_smd: no successful d2pgo_pcm call on this handle");
  const PcmBufs &P = *h->pcm;
  if (out_doubles < P.n_smd) return pgo_fail(h, 2, "debug_pcm_smd: buffer too small: " + std::to_string(P.n_smd) + " doubles needed");
  cudaSetDevice(h->cfg.device);
  if (P.n_smd) {
    PCK(cudaMemcpyAsync(out, P.smd.p, (size_t)P.n_smd * 8, cudaMemcpyDeviceToHost, h->stream));
    PCK(cudaStreamSynchronize(h->stream));
  }
  return 0;
}

int d2pgo_debug_pcm_clique(d2pgo_handle *h, int32_t n, const uint32_t *adj, uint8_t *member_out, int32_t *size_out) {
  if (!h) return 1;
  if (n < 0 || (n && (!adj || !member_out))) return pgo_fail(h, 1, "debug_pcm_clique: null argument or negative count");
  if (n > kPcmMaxGroup) return pgo_fail(h, 4, "debug_pcm_clique: at most " + std::to_string(kPcmMaxGroup) + " vertices are supported");
  cudaSetDevice(h->cfg.device);
  if (!h->pcm) h->pcm.reset(new PcmBufs());
  PcmBufs &P = *h->pcm;
  const long long W = (n + 31) / 32;
  const int g_loop[2] = {0, n}; const long long g_word[2] = {0, n * W};
  P.n_smd = -1;   // the buffers below are shared with d2pgo_pcm
  PCK(P.g_loop.alloc(2)); PCK(P.g_word.alloc(2)); PCK(P.adj.alloc(n * W));
  PCK(cudaMemcpyAsync(P.g_loop.p, g_loop, 8, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(P.g_word.p, g_word, 16, cudaMemcpyHostToDevice, h->stream));
  if (n) PCK(cudaMemcpyAsync(P.adj.p, adj, (size_t)(n * W) * 4, cudaMemcpyHostToDevice, h->stream));
  if (int rc = pcm_run_clique(h, n ? 1 : 0, n, (int)std::max(W, 1LL))) return rc;
  if (n) PCK(cudaMemcpyAsync(member_out, P.inlier.p, n, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  int c = 0;
  for (int k = 0; k < n; k++) c += member_out[k];
  if (size_out) *size_out = c;
  return 0;
}

int d2pgo_debug_pcm_clique_inc(d2pgo_handle *h, int32_t n, const uint32_t *adj, int32_t n_new, int32_t prev_size, uint8_t *member_out, int32_t *size_out) {
  if (!h) return 1;
  if (n < 0 || (n && (!adj || !member_out))) return pgo_fail(h, 1, "debug_pcm_clique_inc: null argument or negative count");
  if (n > kPcmMaxGroup) return pgo_fail(h, 4, "debug_pcm_clique_inc: at most " + std::to_string(kPcmMaxGroup) + " vertices are supported");
  if (n_new < 0 || n_new > n || prev_size < 0) return pgo_fail(h, 2, "debug_pcm_clique_inc: n_new must lie in [0, n] and prev_size be non-negative");
  cudaSetDevice(h->cfg.device);
  if (!h->pcm) h->pcm.reset(new PcmBufs());
  PcmBufs &P = *h->pcm;
  const long long W = (n + 31) / 32;
  const int g_loop[2] = {0, n}; const long long g_word[2] = {0, n * W};
  P.n_smd = -1;   // the buffers below are shared with d2pgo_pcm
  PCK(P.g_loop.alloc(2)); PCK(P.g_word.alloc(2)); PCK(P.adj.alloc(n * W)); PCK(P.deg.alloc(n)); PCK(P.inlier.alloc(n)); PCK(P.stats.alloc(2)); PCK(P.jobs.alloc(1));
  const PcmCliqueJob job{P.adj.p, P.deg.p, P.inlier.p, (long long)W, n, n - n_new, prev_size};
  PCK(cudaMemcpyAsync(P.g_loop.p, g_loop, 8, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(P.g_word.p, g_word, 16, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(P.jobs.p, &job, sizeof job, cudaMemcpyHostToDevice, h->stream));
  if (n) {
    PCK(cudaMemcpyAsync(P.adj.p, adj, (size_t)(n * W) * 4, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemsetAsync(P.inlier.p, 0, n, h->stream));   // the flags stay 0 when no seed beats prev_size
    k_pcm_degree<<<(n + 255) / 256, 256, 0, h->stream>>>(1, P.g_loop.p, P.g_word.p, P.adj.p, P.deg.p);
    k_pcm_clique_jobs<<<1, kPcmWarps * 32, (size_t)(1 + kPcmWarps) * std::max(W, 1LL) * 4, h->stream>>>(P.jobs.p, P.stats.p);
    PCK(cudaGetLastError());
    PCK(cudaMemcpyAsync(member_out, P.inlier.p, n, cudaMemcpyDeviceToHost, h->stream));
  }
  PCK(cudaStreamSynchronize(h->stream));
  int c = 0;
  for (int k = 0; k < n; k++) c += member_out[k];
  if (size_out) *size_out = c > 0 ? c : prev_size;   // FMC's return: the clique that beat prev_size, else prev_size
  return 0;
}

int d2pgo_pcm_stream_reset(d2pgo_handle *h, const d2pgo_pcm_config *cfg, int32_t incremental) {
  if (!h) return 1;
  if (!cfg) return pgo_fail(h, 1, "pcm_stream_reset: null argument");
  const double thr = (double)(float)cfg->pcm_thres;   // a float in the reference, as in d2pgo_pcm
  if (!(std::isfinite(thr) && thr > 0.0)) return pgo_fail(h, 2, "pcm_stream_reset: pcm_thres must be finite and positive");
  if (!(std::isfinite(cfg->pos_covariance_per_meter) && cfg->pos_covariance_per_meter >= 0.0 && std::isfinite(cfg->yaw_covariance_per_meter) && cfg->yaw_covariance_per_meter >= 0.0))
    return pgo_fail(h, 2, "pcm_stream_reset: covariance rates must be finite and non-negative");
  if (incremental != 0 && incremental != 1) return pgo_fail(h, 2, "pcm_stream_reset: incremental must be 0 or 1");
  cudaSetDevice(h->cfg.device);
  h->pcm_stream.reset(new d2pgo_host::PcmStream());
  d2pgo_host::PcmStream &S = *h->pcm_stream;
  S.ready = true; S.incremental = incremental; S.is4 = h->dof == 4; S.thr = thr;
  S.pos_cov = cfg->pos_covariance_per_meter; S.yaw_cov = cfg->yaw_covariance_per_meter;
  PCK(cudaEventCreate(&S.ev_pair));
  return 0;
}

int d2pgo_pcm_stream(d2pgo_handle *h, int32_t n_frames, const int64_t *frame_ids, const int32_t *frame_agent, const double *ego_poses7, int32_t n_loops,
                     const int64_t *loop_ids, const int64_t *kf_a, const int64_t *kf_b, const double *rel7, const double *sqrt_info36, uint8_t *inlier_out,
                     d2pgo_pcm_stream_report *rep) {
  if (!h) return 1;
  if (n_frames < 0 || n_loops < 0 || (n_frames && (!frame_ids || !frame_agent || !ego_poses7)) ||
      (n_loops && (!loop_ids || !kf_a || !kf_b || !rel7 || !sqrt_info36 || !inlier_out)))
    return pgo_fail(h, 1, "pcm_stream: null argument or negative count");
  if (!h->pcm_stream || !h->pcm_stream->ready) return pgo_fail(h, 5, "pcm_stream: no d2pgo_pcm_stream_reset on this handle");
  d2pgo_host::PcmStream &S = *h->pcm_stream;
  // ---- checks: nothing of the call is kept until all of them pass
  std::unordered_map<int64_t, int32_t> fnew;   // keyframes first seen in this call -> drone
  std::vector<int> fadd;                       // their positions in the call, in the order given
  for (int f = 0; f < n_frames; f++) {
    auto old = S.fidx.find(frame_ids[f]);
    const int32_t had = old != S.fidx.end() ? S.f_agent[old->second] : (fnew.count(frame_ids[f]) ? fnew[frame_ids[f]] : frame_agent[f]);
    if (had != frame_agent[f])
      return pgo_fail(h, 3, "pcm_stream: keyframe id " + std::to_string(frame_ids[f]) + " was given with drone " + std::to_string(had) + " and now with drone " + std::to_string(frame_agent[f]));
    if (old != S.fidx.end() || fnew.count(frame_ids[f])) continue;
    for (int k = 0; k < 7; k++)
      if (!std::isfinite(ego_poses7[(size_t)f * 7 + k])) return pgo_fail(h, 2, "pcm_stream: non-finite ego pose of keyframe id " + std::to_string(frame_ids[f]));
    fnew.emplace(frame_ids[f], frame_agent[f]); fadd.push_back(f);
  }
  auto agent_of = [&](int64_t id, int32_t *a) {
    auto it = S.fidx.find(id);
    if (it != S.fidx.end()) { *a = S.f_agent[it->second]; return true; }
    auto jt = fnew.find(id);
    if (jt != fnew.end()) { *a = jt->second; return true; }
    return false;
  };
  std::unordered_map<int64_t, int> seen;       // loop id -> position in the call
  std::vector<int> ladd;                       // new loops: positions in the call
  std::unordered_map<uint64_t, int> gnew_size; // loops per group after the call, for the groups that get new loops
  for (int e = 0; e < n_loops; e++) {
    if (!seen.emplace(loop_ids[e], e).second) return pgo_fail(h, 3, "pcm_stream: loop id " + std::to_string(loop_ids[e]) + " appears twice in one call");
    if (S.loop_of.count(loop_ids[e])) continue;
    int32_t x, y;
    if (!agent_of(kf_a[e], &x) || !agent_of(kf_b[e], &y))
      return pgo_fail(h, 3, "pcm_stream: loop id " + std::to_string(loop_ids[e]) + " names unknown keyframe id " + std::to_string(agent_of(kf_a[e], &x) ? kf_b[e] : kf_a[e]));
    for (int k = 0; k < 7; k++)
      if (!std::isfinite(rel7[(size_t)e * 7 + k])) return pgo_fail(h, 2, "pcm_stream: non-finite relative pose of loop id " + std::to_string(loop_ids[e]));
    for (int k = 0; k < 36; k++)
      if (!std::isfinite(sqrt_info36[(size_t)e * 36 + k])) return pgo_fail(h, 2, "pcm_stream: non-finite sqrt_info of loop id " + std::to_string(loop_ids[e]));
    const uint64_t key = (uint64_t)(uint32_t)std::min(x, y) << 32 | (uint32_t)std::max(x, y);
    auto it = gnew_size.find(key);
    if (it == gnew_size.end()) { auto g = S.gid.find(key); it = gnew_size.emplace(key, g == S.gid.end() ? 0 : S.groups[g->second]->L).first; }
    if (++it->second > kPcmMaxGroup)
      return pgo_fail(h, 4, "pcm_stream: the group of drones " + std::to_string(std::min(x, y)) + " and " + std::to_string(std::max(x, y)) + " would hold " +
                                std::to_string(it->second) + " loops; at most " + std::to_string(kPcmMaxGroup) + " are supported");
    ladd.push_back(e);
  }
  cudaSetDevice(h->cfg.device);
  cudaStream_t st = h->stream;
  // ---- frames: appended to their drone's trajectory; ego poses [F][8] stay on the device
  const int F0 = (int)S.f_agent.size(), F = F0 + (int)fadd.size();
  if (!fadd.empty()) {
    PCK(pcm_grow(S.ego, (size_t)F0 * 8, (size_t)F * 8, st)); PCK(pcm_grow(S.path, F0, F, st));
    std::vector<double> ego(fadd.size() * 8, 0.0);
    for (size_t k = 0; k < fadd.size(); k++) {
      const int f = fadd[k];
      memcpy(&ego[k * 8], ego_poses7 + (size_t)f * 7, 56);
      S.fidx.emplace(frame_ids[f], F0 + (int)k); S.f_agent.push_back(frame_agent[f]);
      auto it = S.drone_of.emplace(frame_agent[f], (int)S.trajs.size());
      if (it.second) S.trajs.emplace_back();
      S.trajs[it.first->second].push_back(F0 + (int)k);
    }
    PCK(cudaMemcpyAsync(S.ego.p + (size_t)F0 * 8, ego.data(), ego.size() * 8, cudaMemcpyHostToDevice, st));
    std::vector<int> traj_ptr(1, 0), traj;
    for (auto &t : S.trajs) { traj.insert(traj.end(), t.begin(), t.end()); traj_ptr.push_back((int)traj.size()); }
    PCK(S.traj_ptr.alloc(traj_ptr.size())); PCK(S.traj.alloc(traj.size()));
    PCK(cudaMemcpyAsync(S.traj_ptr.p, traj_ptr.data(), traj_ptr.size() * 4, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(S.traj.p, traj.data(), traj.size() * 4, cudaMemcpyHostToDevice, st));
  }
  // ---- new loops: constants by loop index, rows of their group (groups numbered by their first loop)
  const int n0 = (int)S.l_group.size(), nn = (int)ladd.size(), n1 = n0 + nn;
  std::vector<int> touched, L0_of;   // group indices in ascending order, and their sizes before the call
  std::vector<int> sfa(nn), sfb(nn), iota(nn);
  std::vector<unsigned char> sflip(nn);
  std::vector<double> rin((size_t)nn * 7), sqi((size_t)nn * 36);
  std::vector<std::vector<int>> gslots;   // per touched group: the loop indices of its new rows
  std::unordered_map<int, int> tpos;
  for (int k = 0; k < nn; k++) {
    const int e = ladd[k];
    const int a = S.fidx.at(kf_a[e]), b = S.fidx.at(kf_b[e]);
    const int32_t x = S.f_agent[a], y = S.f_agent[b];
    const uint64_t key = (uint64_t)(uint32_t)std::min(x, y) << 32 | (uint32_t)std::max(x, y);
    auto g = S.gid.emplace(key, (int)S.groups.size());
    if (g.second) { S.groups.emplace_back(new PcmStreamGroup()); S.groups.back()->lo = std::min(x, y); S.groups.back()->hi = std::max(x, y); }
    const int gi = g.first->second;
    auto t = tpos.emplace(gi, (int)touched.size());
    if (t.second) { touched.push_back(gi); L0_of.push_back(S.groups[gi]->L); gslots.emplace_back(); }
    S.loop_of.emplace(loop_ids[e], n0 + k); S.l_group.push_back(gi); S.l_row.push_back(S.groups[gi]->L++);
    gslots[t.first->second].push_back(n0 + k);
    sfa[k] = a; sfb[k] = b; sflip[k] = x > y; iota[k] = k;
    memcpy(&rin[(size_t)k * 7], rel7 + (size_t)e * 7, 56); memcpy(&sqi[(size_t)k * 36], sqrt_info36 + (size_t)e * 36, 288);
  }
  if (nn) {
    PCK(pcm_grow(S.fa, n0, n1, st)); PCK(pcm_grow(S.fb, n0, n1, st)); PCK(pcm_grow(S.flip, n0, n1, st));
    PCK(pcm_grow(S.rel, (size_t)n0 * 8, (size_t)n1 * 8, st)); PCK(pcm_grow(S.cov, (size_t)n0 * 21, (size_t)n1 * 21, st));
    PCK(S.rel_in.alloc((size_t)nn * 7)); PCK(S.sqrt_in.alloc((size_t)nn * 36)); PCK(S.src.alloc(nn));
    PCK(cudaMemcpyAsync(S.fa.p + n0, sfa.data(), nn * 4, cudaMemcpyHostToDevice, st)); PCK(cudaMemcpyAsync(S.fb.p + n0, sfb.data(), nn * 4, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(S.flip.p + n0, sflip.data(), nn, cudaMemcpyHostToDevice, st)); PCK(cudaMemcpyAsync(S.src.p, iota.data(), nn * 4, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(S.rel_in.p, rin.data(), rin.size() * 8, cudaMemcpyHostToDevice, st)); PCK(cudaMemcpyAsync(S.sqrt_in.p, sqi.data(), sqi.size() * 8, cudaMemcpyHostToDevice, st));
  }
  // touched groups in the order of their first loop; each grows its adjacency (pitch doubling, rows copied to the new pitch)
  std::vector<int> order(touched.size());
  for (size_t k = 0; k < order.size(); k++) order[k] = (int)k;
  std::sort(order.begin(), order.end(), [&](int u, int v) { return touched[u] < touched[v]; });
  const int T = (int)touched.size();
  std::vector<PcmPairJob> pj(T); std::vector<PcmCliqueJob> cj(T);
  std::vector<long long> pword(T + 1, 0), smd_off(T + 1, 0); std::vector<int> row_off(T + 1, 0);
  int max_w = 1;
  for (int k = 0; k < T; k++) {
    const int u = order[k];
    PcmStreamGroup &G = *S.groups[touched[u]];
    const int L0 = L0_of[u], L = G.L;
    if (32 * G.pitch < L) {
      int p = std::max(G.pitch, 1);
      while (32 * p < L) p *= 2;
      d2pgo_host::Buf<unsigned> na;
      PCK(na.alloc((size_t)32 * p * p));
      if (L0) PCK(cudaMemcpy2DAsync(na.p, (size_t)p * 4, G.adj.p, (size_t)G.pitch * 4, (size_t)G.pitch * 4, L0, cudaMemcpyDeviceToDevice, st));
      PCK(cudaStreamSynchronize(st));
      std::swap(G.adj.p, na.p); std::swap(G.adj.n, na.n);
      PCK(pcm_grow(G.slot, L0, (size_t)32 * p, st)); PCK(pcm_grow(G.deg, L0, (size_t)32 * p, st)); PCK(pcm_grow(G.member, L0, (size_t)32 * p, st));
      G.pitch = p;
    }
    PCK(cudaMemcpyAsync(G.slot.p + L0, gslots[u].data(), (L - L0) * 4, cudaMemcpyHostToDevice, st));
    const long long W = (L + 31) / 32;
    max_w = std::max(max_w, (int)W);
    pj[k] = PcmPairJob{G.adj.p, G.slot.p, nullptr, G.pitch, L0, L};
    cj[k] = PcmCliqueJob{G.adj.p, G.deg.p, G.member.p, G.pitch, L, S.incremental ? L0 : 0, S.incremental ? G.size : -1};
    pword[k + 1] = pword[k] + (L - L0) * W + (long long)L0 * (W - (L0 >> 5));
    smd_off[k + 1] = smd_off[k] + (long long)L * (L - 1) / 2 - (long long)L0 * (L0 - 1) / 2;
    row_off[k + 1] = row_off[k] + L;
  }
  PCK(S.smd.alloc(smd_off[T]));
  for (int k = 0; k < T; k++) pj[k].smd = S.smd.p + smd_off[k];
  PCK(S.pjobs.alloc(T)); PCK(S.cjobs.alloc(T)); PCK(S.pword.alloc(T + 1)); PCK(S.row_off.alloc(T + 1)); PCK(S.stats.alloc(2 * (size_t)T));
  if (T) {
    PCK(cudaMemcpyAsync(S.pjobs.p, pj.data(), T * sizeof(PcmPairJob), cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(S.cjobs.p, cj.data(), T * sizeof(PcmCliqueJob), cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(S.pword.p, pword.data(), (T + 1) * 8, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(S.row_off.p, row_off.data(), (T + 1) * 4, cudaMemcpyHostToDevice, st));
  }
  // ---- device: path lengths over the whole trajectories (appending frames leaves an earlier frame's value unchanged: the warp
  // scan of k_pcm_path adds lane k's prefix from lanes <= k only, and the carry from whole earlier chunks), loop constants of the
  // new loops, the changed adjacency words, degrees and cliques of the touched groups
  PcmDev d;
  memset(&d, 0, sizeof d);
  d.fa = S.fa.p; d.fb = S.fb.p; d.flip = S.flip.p; d.rel = S.rel.p; d.cov = S.cov.p; d.ego = S.ego.p; d.path = S.path.p;
  d.is4 = S.is4; d.thr = S.thr; d.pos_cov = S.pos_cov; d.yaw_cov = S.yaw_cov;
  PCK(cudaEventRecord(h->ev0, st));
  if (!S.trajs.empty()) k_pcm_path<<<((int)S.trajs.size() * 32 + 255) / 256, 256, 0, st>>>((int)S.trajs.size(), S.traj_ptr.p, S.traj.p, S.ego.p, S.path.p);
  if (nn) k_pcm_loop<<<(nn + 127) / 128, 128, 0, st>>>(nn, S.src.p, S.rel_in.p, S.sqrt_in.p, S.rel.p + (size_t)n0 * 8, S.cov.p + (size_t)n0 * 21);
  if (pword[T]) k_pcm_stream_pairs<<<(unsigned)((pword[T] * 32 + 255) / 256), 256, 0, st>>>(d, S.pjobs.p, S.pword.p, T, pword[T]);
  PCK(cudaGetLastError());
  PCK(cudaEventRecord(S.ev_pair, st));
  if (T) {
    k_pcm_stream_degree<<<(row_off[T] + 255) / 256, 256, 0, st>>>(S.cjobs.p, S.row_off.p, T);
    k_pcm_clique_jobs<<<T, kPcmWarps * 32, (size_t)(1 + kPcmWarps) * max_w * 4, st>>>(S.cjobs.p, S.stats.p);
  }
  PCK(cudaGetLastError());
  PCK(cudaEventRecord(h->ev1, st));
  std::vector<long long> stats(2 * (size_t)T);
  for (int k = 0; k < T; k++) {
    PcmStreamGroup &G = *S.groups[touched[order[k]]];
    G.member_h.resize(G.L);
    PCK(cudaMemcpyAsync(G.member_h.data(), G.member.p, G.L, cudaMemcpyDeviceToHost, st));
  }
  if (T) PCK(cudaMemcpyAsync(stats.data(), S.stats.p, 16 * (size_t)T, cudaMemcpyDeviceToHost, st));
  PCK(cudaStreamSynchronize(st));
  d2pgo_pcm_stream_report R; memset(&R, 0, sizeof R);
  for (int k = 0; k < T; k++) {
    PcmStreamGroup &G = *S.groups[touched[order[k]]];
    int c = 0;
    for (unsigned char m : G.member_h) c += m;
    G.size = c;
    R.consistent_pairs += (stats[2 * k] - G.dsum) / 2; G.dsum = stats[2 * k];
    R.clique_rounds += stats[2 * k + 1];
  }
  // every group the call names has been through the clique, so each loop's pair has an inlier set (:96-111): membership decides
  for (int e = 0; e < n_loops; e++) {
    const int l = S.loop_of.at(loop_ids[e]);
    inlier_out[e] = S.groups[S.l_group[l]]->member_h[S.l_row[l]];
    R.inliers += inlier_out[e];
  }
  R.new_loops = nn; R.total_loops = n1; R.groups = (int32_t)S.groups.size(); R.groups_touched = T; R.pairs_tested = smd_off[T];
  float ms = 0, mp = 0;
  cudaEventElapsedTime(&ms, h->ev0, h->ev1); cudaEventElapsedTime(&mp, h->ev0, S.ev_pair);
  R.device_ms = ms; R.pair_ms = mp; R.clique_ms = ms - mp;
  S.n_smd = smd_off[T];
  if (rep) *rep = R;
  return 0;
}

int d2pgo_debug_pcm_stream_smd(d2pgo_handle *h, double *out, int64_t out_doubles) {
  if (!h) return 1;
  if (!h->pcm_stream || h->pcm_stream->n_smd < 0) return pgo_fail(h, 2, "debug_pcm_stream_smd: no successful d2pgo_pcm_stream call since the last reset");
  const d2pgo_host::PcmStream &S = *h->pcm_stream;
  if (out_doubles < S.n_smd) return pgo_fail(h, 2, "debug_pcm_stream_smd: buffer too small: " + std::to_string(S.n_smd) + " doubles needed");
  cudaSetDevice(h->cfg.device);
  if (S.n_smd) {
    PCK(cudaMemcpyAsync(out, S.smd.p, (size_t)S.n_smd * 8, cudaMemcpyDeviceToHost, h->stream));
    PCK(cudaStreamSynchronize(h->stream));
  }
  return 0;
}

}  // extern "C"
