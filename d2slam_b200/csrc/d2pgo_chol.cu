// d2pgo_chol.cu -- exact Levenberg-Marquardt steps for the pose graph: a supernodal multifrontal sparse Cholesky of
// H = J^T J + damping over the free poses, in binary64, with no floating-point atomics (bitwise reproducible).
//
// Host, once per graph structure: the block graph of the free poses, a nested-dissection ordering (recursive bisection by the
// middle level of a breadth-first level structure; parts of at most kNdLeaf poses in natural order), the elimination tree and
// its column structures, a postorder, fundamental supernodes, relaxed amalgamation (a child that ends right before its parent
// is merged while the explicit zeros stay within kAmalgamateZeros of the stored entries), and the level sets of the
// supernodal tree.  Device, per LM iteration, two CUDA graphs per linearisation buffer:
//   factor: k_chol_pairs (one thread per distinct pose pair: sum of J_lo^T J_hi over its edges in ascending edge order),
//           k_chol_diag (block diagonal D of k_pgo_gD + the self loops' cross terms + lambda diag(D) + 1e-12, and b = -g),
//           k_chol_factor per level, leaves first (one CTA per supernode: assemble the front from the original blocks and the
//           children's update matrices in child order, partial Cholesky of its columns, Schur update into its own corner)
//   solve:  k_chol_fwd per level (L y = b; a CTA pulls its children's update vectors), k_chol_bwd per level, root first
//           (L^T x = y; a CTA gathers x at its rows below from its ancestors), k_chol_scatter (dx per pose, 0 on fixed).
// lambda lives in device memory, so the captured graphs serve every iteration.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <numeric>

#include "d2ba_math.cuh"
#include "d2pgo_chol.cuh"

namespace d2pgo_chol {

// ------------------------------------------------------------------------------------------------ symbolic analysis
namespace {

// nested dissection of the graph (CSR ap / aj over n vertices), deterministic: ties go to the lower index
void nd_order(int n, const std::vector<int> &ap, const std::vector<int> &aj, std::vector<int> &out) {
  std::vector<int> mark(n, -1), dist(n, -1), queue;
  int stamp = 0;
  struct Task { std::vector<int> nodes; bool emit; };
  std::vector<Task> stack;
  std::vector<int> all(n);
  std::iota(all.begin(), all.end(), 0);
  stack.push_back({std::move(all), false});
  // breadth-first search from `src` inside the vertices marked `tag`; dist[], returns the visit order
  auto bfs = [&](int src, int tag, int seen_tag) {
    queue.clear(); queue.push_back(src); mark[src] = seen_tag; dist[src] = 0;
    for (size_t q = 0; q < queue.size(); q++) {
      const int u = queue[q];
      for (int k = ap[u]; k < ap[u + 1]; k++) {
        const int v = aj[k];
        if (mark[v] == tag) { mark[v] = seen_tag; dist[v] = dist[u] + 1; queue.push_back(v); }
      }
    }
    return queue;
  };
  while (!stack.empty()) {
    Task t = std::move(stack.back());
    stack.pop_back();
    std::vector<int> &nodes = t.nodes;   // ascending
    if (t.emit || (int)nodes.size() <= kNdLeaf) { out.insert(out.end(), nodes.begin(), nodes.end()); continue; }
    // connected components, in the order of their lowest vertex
    const int in_set = ++stamp;
    for (int v : nodes) mark[v] = in_set;
    std::vector<std::vector<int>> comps;
    for (int v : nodes) {
      if (mark[v] != in_set) continue;
      const int seen = ++stamp;
      std::vector<int> c = bfs(v, in_set, seen);
      std::sort(c.begin(), c.end());
      comps.push_back(std::move(c));
    }
    if (comps.size() > 1) {
      for (size_t k = comps.size(); k-- > 0;) stack.push_back({std::move(comps[k]), false});
      continue;
    }
    // one component: a pseudo-peripheral vertex (last reached from the lowest vertex), its level structure, and the
    // separator = the level at the median distance (at least 1, at most the depth)
    int tag = ++stamp;
    for (int v : nodes) mark[v] = tag;
    int seen = ++stamp;
    const int far = bfs(nodes[0], tag, seen).back();
    tag = seen; seen = ++stamp;
    bfs(far, tag, seen);
    std::vector<int> ds;
    ds.reserve(nodes.size());
    int depth = 0;
    for (int v : nodes) { ds.push_back(dist[v]); depth = std::max(depth, dist[v]); }
    std::nth_element(ds.begin(), ds.begin() + ds.size() / 2, ds.end());
    const int L = std::min(std::max(ds[ds.size() / 2], 1), depth);
    Task a{{}, false}, b{{}, false}, s{{}, true};
    for (int v : nodes) (dist[v] < L ? a : dist[v] > L ? b : s).nodes.push_back(v);
    stack.push_back(std::move(s));
    if (!b.nodes.empty()) stack.push_back(std::move(b));
    stack.push_back(std::move(a));
  }
}

int find_root(std::vector<int> &alias, int s) {
  while (alias[s] != s) { alias[s] = alias[alias[s]]; s = alias[s]; }
  return s;
}

std::vector<int> tree_levels(const std::vector<int> &parent) {   // children before parents
  std::vector<int> lv(parent.size(), 0);
  for (size_t s = 0; s < parent.size(); s++) if (parent[s] >= 0) lv[parent[s]] = std::max(lv[parent[s]], lv[s] + 1);
  return lv;
}

}  // namespace

int analyse(int N, const unsigned char *fixed, int E, const int *ea, const int *eb, int D, Symbolic &S, std::string &err) {
  S = Symbolic();
  if (D != 4 && D != 6) { err = "cholesky: block size " + std::to_string(D) + " (4 or 6)"; return 2; }
  S.n_pose = N; S.n_edge = E; S.D = D;
  S.fixed.assign(fixed, fixed + N); S.ea.assign(ea, ea + E); S.eb.assign(eb, eb + E);
  for (int e = 0; e < E; e++)
    if (ea[e] < 0 || ea[e] >= N || eb[e] < 0 || eb[e] >= N) { err = "cholesky: edge " + std::to_string(e) + " names a pose out of range"; return 2; }
  std::vector<int> fidx(N, -1), fpose;
  for (int i = 0; i < N; i++) if (!fixed[i]) { fidx[i] = (int)fpose.size(); fpose.push_back(i); }
  const int nf = (int)fpose.size();
  S.n_free = nf;
  // distinct pairs of free poses (by pose index) with their edges ascending; self loops per free pose
  std::vector<std::array<int, 3>> pe;
  std::vector<std::vector<int>> selfs(nf);
  for (int e = 0; e < E; e++) {
    const int a = ea[e], b = eb[e];
    if (fixed[a] || fixed[b]) continue;
    if (a == b) selfs[fidx[a]].push_back(e);
    else pe.push_back({std::min(a, b), std::max(a, b), e});
  }
  std::sort(pe.begin(), pe.end());
  std::vector<int> pair_hi;
  S.pair_ptr.push_back(0);
  for (size_t k = 0; k < pe.size(); k++) {
    if (k == 0 || pe[k][0] != pe[k - 1][0] || pe[k][1] != pe[k - 1][1]) {
      if (k) S.pair_ptr.push_back((int)k);
      S.pair_lo.push_back(pe[k][0]); pair_hi.push_back(pe[k][1]);
    }
    S.pair_edge.push_back(pe[k][2]);
  }
  if (!pe.empty()) S.pair_ptr.push_back((int)pe.size());
  const int P = (int)S.pair_lo.size();
  S.n_pairs = P;
  // adjacency of the free poses (free indices), neighbours ascending
  std::vector<int> ap(nf + 1, 0), aj(2 * (size_t)P);
  for (int p = 0; p < P; p++) { ap[fidx[S.pair_lo[p]] + 1]++; ap[fidx[pair_hi[p]] + 1]++; }
  for (int i = 0; i < nf; i++) ap[i + 1] += ap[i];
  { std::vector<int> fill(ap.begin(), ap.end() - 1);
    for (int p = 0; p < P; p++) { const int u = fidx[S.pair_lo[p]], v = fidx[pair_hi[p]]; aj[fill[u]++] = v; aj[fill[v]++] = u; } }
  for (int i = 0; i < nf; i++) std::sort(aj.begin() + ap[i], aj.begin() + ap[i + 1]);
  std::vector<int> order;
  order.reserve(nf);
  nd_order(nf, ap, aj, order);
  std::vector<int> iperm(nf);
  for (int k = 0; k < nf; k++) iperm[order[k]] = k;
  // column structures of L (below the diagonal) and the elimination tree: struct(j) = the later neighbours of j and the
  // structures of j's children without j; parent(j) = the first row of struct(j)
  std::vector<std::vector<int>> st(nf), kids(nf);
  std::vector<int> parent(nf, -1);
  for (int j = 0; j < nf; j++) {
    std::vector<int> &s = st[j];
    const int u = order[j];
    for (int k = ap[u]; k < ap[u + 1]; k++) if (iperm[aj[k]] > j) s.push_back(iperm[aj[k]]);
    for (int c : kids[j]) for (int r : st[c]) if (r != j) s.push_back(r);
    std::sort(s.begin(), s.end());
    s.erase(std::unique(s.begin(), s.end()), s.end());
    if (!s.empty()) { parent[j] = s[0]; kids[s[0]].push_back(j); }
  }
  // postorder (roots ascending, children ascending): the same fill, and every subtree becomes a range of columns
  std::vector<int> post, newpos(nf);
  post.reserve(nf);
  {
    std::vector<std::pair<int, size_t>> dfs;
    for (int r = 0; r < nf; r++) {
      if (parent[r] >= 0) continue;
      dfs.push_back({r, 0});
      while (!dfs.empty()) {
        auto &top = dfs.back();
        if (top.second < kids[top.first].size()) { const int c = kids[top.first][top.second++]; dfs.push_back({c, 0}); }
        else { post.push_back(top.first); dfs.pop_back(); }
      }
    }
  }
  for (int k = 0; k < nf; k++) newpos[post[k]] = k;
  std::vector<int> par2(nf), cc(nf), nkids(nf, 0);
  std::vector<std::vector<int>> st2(nf);
  S.perm.resize(nf); S.col_of.assign(N, -1);
  for (int k = 0; k < nf; k++) {
    const int o = post[k];
    S.perm[k] = fpose[order[o]];
    S.col_of[S.perm[k]] = k;
    par2[k] = parent[o] >= 0 ? newpos[parent[o]] : -1;
    for (int r : st[o]) st2[k].push_back(newpos[r]);
    std::sort(st2[k].begin(), st2[k].end());
    cc[k] = (int)st2[k].size() + 1;
    S.nnz_L += cc[k];
    if (par2[k] >= 0) nkids[par2[k]]++;
  }
  st.clear(); kids.clear();
  // fundamental supernodes: j continues j - 1's when j is j - 1's parent, its only child, and one row shorter
  struct Sn { int f, l; std::vector<int> rows; int64_t nz; int parent; bool alive; };
  std::vector<Sn> sn;
  std::vector<int> sn_of(nf);
  for (int j = 0; j < nf; j++) {
    if (j > 0 && par2[j - 1] == j && nkids[j] == 1 && cc[j - 1] == cc[j] + 1) { sn.back().l = j + 1; sn.back().nz += cc[j]; }
    else sn.push_back({j, j + 1, {}, cc[j], -1, true});
    sn_of[j] = (int)sn.size() - 1;
  }
  const int S0 = (int)sn.size();
  for (int s = 0; s < S0; s++) {
    sn[s].rows = st2[sn[s].l - 1];
    sn[s].parent = par2[sn[s].l - 1] >= 0 ? sn_of[par2[sn[s].l - 1]] : -1;
  }
  st2.clear();
  {
    std::vector<int> p0(S0);
    for (int s = 0; s < S0; s++) p0[s] = sn[s].parent;
    const std::vector<int> lv = tree_levels(p0);
    S.sn_fundamental = S0;
    S.levels_fundamental = S0 ? *std::max_element(lv.begin(), lv.end()) + 1 : 0;
  }
  // relaxed amalgamation, children before parents: merge the child that ends right before s while the share of explicit
  // zeros stays bounded and the front fits the kernels
  std::vector<int> alias(S0);
  std::iota(alias.begin(), alias.end(), 0);
  for (int s = 0; s < S0; s++) {
    while (sn[s].f > 0) {
      const int c = find_root(alias, sn_of[sn[s].f - 1]);
      if (!sn[c].alive || sn[c].parent < 0 || find_root(alias, sn[c].parent) != s) break;
      const int64_t w = sn[s].l - sn[c].f, r = (int64_t)sn[s].rows.size();
      const int64_t stored = w * (w + 1) / 2 + w * r, nz = sn[c].nz + sn[s].nz;
      if ((double)(stored - nz) > kAmalgamateZeros * (double)stored || (w + r) * D > kMaxFront) break;
      sn[s].f = sn[c].f; sn[s].nz = nz; sn[c].alive = false; alias[c] = s;
    }
  }
  std::vector<int> renum(S0, -1);
  int NS = 0;
  for (int s = 0; s < S0; s++) if (sn[s].alive) renum[s] = NS++;
  S.sn_first.resize(NS); S.sn_width.resize(NS); S.sn_parent.resize(NS);
  S.idx_ptr.assign(1, 0);
  for (int s = 0, k = 0; s < S0; s++) {
    if (!sn[s].alive) continue;
    S.sn_first[k] = sn[s].f; S.sn_width[k] = sn[s].l - sn[s].f;
    S.sn_parent[k] = sn[s].parent >= 0 ? renum[find_root(alias, sn[s].parent)] : -1;
    for (int j = sn[s].f; j < sn[s].l; j++) { S.idx.push_back(j); sn_of[j] = k; }
    S.idx.insert(S.idx.end(), sn[s].rows.begin(), sn[s].rows.end());
    S.idx_ptr.push_back((int)S.idx.size());
    const int64_t w = S.sn_width[k], r = (int64_t)sn[s].rows.size();
    S.nnz_stored += w * (w + 1) / 2 + w * r;
    k++;
  }
  sn.clear();
  S.sn_level = tree_levels(S.sn_parent);
  // the row map of each front into its parent's, children lists, arena offsets, level sets
  S.relmap.assign(S.idx.size(), -1);
  std::vector<int> nch(NS + 1, 0);
  S.sn_off.resize(NS); S.sn_uoff.resize(NS);
  int levels = 0;
  for (int s = 0; s < NS; s++) {
    const int w = S.sn_width[s], m = S.idx_ptr[s + 1] - S.idx_ptr[s], p = S.sn_parent[s];
    if (p >= 0) {
      const int *pb = &S.idx[S.idx_ptr[p]], *pe_ = &S.idx[0] + S.idx_ptr[p + 1];
      for (int q = S.idx_ptr[s] + w; q < S.idx_ptr[s + 1]; q++) S.relmap[q] = (int)(std::lower_bound(pb, pe_, S.idx[q]) - pb);
      nch[p + 1]++;
    }
    S.sn_off[s] = S.arena; S.arena += (long long)m * D * m * D;
    S.sn_uoff[s] = S.uarena; S.uarena += (long long)(m - w) * D;
    S.max_front_rows = std::max(S.max_front_rows, m * D); S.max_front_cols = std::max(S.max_front_cols, w * D);
    levels = std::max(levels, S.sn_level[s] + 1);
  }
  S.ch_ptr.assign(NS + 1, 0);
  for (int s = 0; s < NS; s++) S.ch_ptr[s + 1] = S.ch_ptr[s] + nch[s + 1];
  S.ch.resize(S.ch_ptr[NS]);
  { std::vector<int> fill(S.ch_ptr.begin(), S.ch_ptr.end() - 1);
    for (int s = 0; s < NS; s++) if (S.sn_parent[s] >= 0) S.ch[fill[S.sn_parent[s]]++] = s; }
  S.lvl_ptr.assign(levels + 1, 0);
  for (int s = 0; s < NS; s++) S.lvl_ptr[S.sn_level[s] + 1]++;
  for (int l = 0; l < levels; l++) S.lvl_ptr[l + 1] += S.lvl_ptr[l];
  S.lvl_sn.resize(NS);
  { std::vector<int> fill(S.lvl_ptr.begin(), S.lvl_ptr.end() - 1);
    for (int s = 0; s < NS; s++) S.lvl_sn[fill[S.sn_level[s]]++] = s; }
  // the off-diagonal blocks of H each front takes: pair p at (row of the later column, the earlier column); transposed when
  // the later column is the pair's higher pose (the pair block is sum J_lo^T J_hi)
  std::vector<std::array<int, 5>> po;
  for (int p = 0; p < P; p++) {
    const int jl = S.col_of[S.pair_lo[p]], jh = S.col_of[pair_hi[p]];
    const int j = std::min(jl, jh), i = std::max(jl, jh), s = sn_of[j];
    const int *b = &S.idx[S.idx_ptr[s]], *e = &S.idx[0] + S.idx_ptr[s + 1];
    po.push_back({s, p, (int)(std::lower_bound(b, e, i) - b), j - S.sn_first[s], jh > jl ? 1 : 0});
  }
  std::sort(po.begin(), po.end());
  S.po_ptr.assign(NS + 1, 0);
  for (const auto &q : po) { S.po_ptr[q[0] + 1]++; S.po_pair.push_back(q[1]); S.po_row.push_back(q[2]); S.po_col.push_back(q[3]); S.po_tr.push_back(q[4]); }
  for (int s = 0; s < NS; s++) S.po_ptr[s + 1] += S.po_ptr[s];
  // self loops by block column
  S.self_ptr.assign(nf + 1, 0);
  for (int j = 0; j < nf; j++) {
    const std::vector<int> &v = selfs[fidx[S.perm[j]]];
    S.self_edge.insert(S.self_edge.end(), v.begin(), v.end());
    S.self_ptr[j + 1] = (int)S.self_edge.size();
  }
  return 0;
}

void fill_info(const Symbolic &s, d2pgo_cholesky_info *o) {
  o->free_poses = s.n_free; o->block_pairs = s.n_pairs; o->nnz_L = s.nnz_L; o->nnz_L_stored = s.nnz_stored;
  o->supernodes = (int32_t)s.sn_first.size(); o->levels = (int32_t)s.lvl_ptr.size() - 1;
  o->supernodes_fundamental = s.sn_fundamental; o->levels_fundamental = s.levels_fundamental;
  o->max_front_rows = s.max_front_rows; o->max_front_cols = s.max_front_cols;
}

std::string check_limits(const Symbolic &s, size_t free_bytes) {
  if (s.max_front_rows > kMaxFront)
    return "cholesky: a front of " + std::to_string(s.max_front_rows) + " rows; the kernels take at most " + std::to_string(kMaxFront);
  const double bytes = 8.0 * (double)(s.arena + s.uarena);
  if (bytes > kArenaShare * (double)free_bytes)
    return "cholesky: the fronts need " + std::to_string((long long)(bytes / 1048576.0)) + " MiB, more than " +
           std::to_string((int)(kArenaShare * 100)) + "% of the " + std::to_string((long long)(free_bytes / 1048576)) + " MiB free on the device";
  return "";
}

// ------------------------------------------------------------------------------------------------ device
namespace {

constexpr int kThreads = 256;
constexpr int kPanel = 16;   // columns of one factorisation panel (a multiple of the DMMA depth 4)

// dynamic shared memory of k_chol_factor for a front of M rows
size_t factor_smem(int M) { return (size_t)kPanel * (((M + 7) & ~7) + 8) * 8; }

struct Dev {
  int n_pose, n_free, n_edge, n_pair;
  const double *lin, *Dg, *g; const unsigned char *fixed; const int *ea, *eb; double *dx;
  const int *perm, *col_of, *pair_lo, *pair_ptr, *pair_edge, *self_ptr, *self_edge;
  const int *sn_first, *sn_width, *idx_ptr, *idx, *relmap, *ch_ptr, *ch, *po_ptr, *po_pair, *po_row, *po_col, *po_tr, *lvl_sn;
  const long long *sn_off, *sn_uoff;
  double *pairH, *diagH, *front, *uvec, *b, *y, *x;
  const double *lambda; int *fail;
};

// one thread per distinct pose pair: sum over its edges (ascending) of J_lo^T J_hi
template <int D>
__global__ void __launch_bounds__(128) k_chol_pairs(Dev c) {
  constexpr int DD = D * D;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= c.n_pair) return;
  const int lo = c.pair_lo[p];
  const size_t E = (size_t)c.n_edge;
  double H[DD];
  for (int k = 0; k < DD; k++) H[k] = 0.0;
  for (int q = c.pair_ptr[p]; q < c.pair_ptr[p + 1]; q++) {
    const int e = c.pair_edge[q], sl = c.ea[e] == lo ? 0 : 1;
    const double *Jl = c.lin + (size_t)(D + DD * sl) * E + e, *Jh = c.lin + (size_t)(D + DD * (1 - sl)) * E + e;
    for (int k = 0; k < D; k++) {
      double jl[D], jh[D];
      for (int a = 0; a < D; a++) { jl[a] = Jl[(size_t)(k * D + a) * E]; jh[a] = Jh[(size_t)(k * D + a) * E]; }
      for (int a = 0; a < D; a++) for (int b = 0; b < D; b++) H[a * D + b] += jl[a] * jh[b];
    }
  }
  for (int k = 0; k < DD; k++) c.pairH[(size_t)p * DD + k] = H[k];
}

// one thread per block column: diagonal block D_i + self-loop cross terms + damping (as k_pgo_precond forms it), b = -g
template <int D>
__global__ void __launch_bounds__(128) k_chol_diag(Dev c) {
  constexpr int DD = D * D;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= c.n_free) return;
  const int i = c.perm[j];
  const size_t E = (size_t)c.n_edge;
  double A[DD];
  for (int k = 0; k < DD; k++) A[k] = c.Dg[(size_t)i * DD + k];
  for (int q = c.self_ptr[j]; q < c.self_ptr[j + 1]; q++) {   // a self loop's J_a^T J_b + J_b^T J_a
    const int e = c.self_edge[q];
    const double *J0 = c.lin + (size_t)D * E + e, *J1 = J0 + (size_t)DD * E;
    for (int k = 0; k < D; k++) {
      double j0[D], j1[D];
      for (int a = 0; a < D; a++) { j0[a] = J0[(size_t)(k * D + a) * E]; j1[a] = J1[(size_t)(k * D + a) * E]; }
      for (int a = 0; a < D; a++) for (int b = 0; b < D; b++) A[a * D + b] += j0[a] * j1[b] + j1[a] * j0[b];
    }
  }
  const double lambda = *c.lambda;
  for (int k = 0; k < D; k++) { const double dk = lambda * c.Dg[(size_t)i * DD + k * (D + 1)] + 1e-12; A[k * (D + 1)] += dk; }
  for (int k = 0; k < DD; k++) c.diagH[(size_t)j * DD + k] = A[k];
  for (int k = 0; k < D; k++) c.b[(size_t)j * D + k] = -c.g[(size_t)i * D + k];
}

// k_chol_diag with ceres' Levenberg-Marquardt damping (d2pgo_set_minimizer's CERES_LM) in place of lambda diag(D) + 1e-12:
// mu_k = clamp(s_k^2 D_kk, min_diag, max_diag) / (radius s_k^2), s the Jacobi scale, par = {radius, min_diag, max_diag}
// in device memory (the minimiser's control kernel moves the radius between factorisations)
template <int D>
__global__ void __launch_bounds__(128) k_chol_diag_lm(Dev c, const double *scale, const double *par) {
  constexpr int DD = D * D;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= c.n_free) return;
  const int i = c.perm[j];
  const size_t E = (size_t)c.n_edge;
  double A[DD];
  for (int k = 0; k < DD; k++) A[k] = c.Dg[(size_t)i * DD + k];
  for (int q = c.self_ptr[j]; q < c.self_ptr[j + 1]; q++) {
    const int e = c.self_edge[q];
    const double *J0 = c.lin + (size_t)D * E + e, *J1 = J0 + (size_t)DD * E;
    for (int k = 0; k < D; k++) {
      double j0[D], j1[D];
      for (int a = 0; a < D; a++) { j0[a] = J0[(size_t)(k * D + a) * E]; j1[a] = J1[(size_t)(k * D + a) * E]; }
      for (int a = 0; a < D; a++) for (int b = 0; b < D; b++) A[a * D + b] += j0[a] * j1[b] + j1[a] * j0[b];
    }
  }
  const double radius = par[0], lo = par[1], hi = par[2];
  for (int k = 0; k < D; k++) {
    const double s2 = scale[(size_t)i * D + k] * scale[(size_t)i * D + k];
    A[k * (D + 1)] += fmin(fmax(s2 * c.Dg[(size_t)i * DD + k * (D + 1)], lo), hi) / (radius * s2);
  }
  for (int k = 0; k < DD; k++) c.diagH[(size_t)j * DD + k] = A[k];
  for (int k = 0; k < D; k++) c.b[(size_t)j * D + k] = -c.g[(size_t)i * D + k];
}

struct Front { int s, f, W, M; double *F; };
template <int D>
__device__ Front front_of(const Dev &c, int s) {
  const int w = c.sn_width[s], m = c.idx_ptr[s + 1] - c.idx_ptr[s];
  return Front{s, c.sn_first[s], w * D, m * D, c.front + c.sn_off[s]};
}

// one CTA per supernode of a level: assemble the front (row-major M x M, lower triangle only), factor its W columns
// (L11 L11^T = F11, L21 = F21 L11^-T), and leave the Schur complement F22 - L21 L21^T in its lower-right corner.
// Right-looking in panels of kPanel columns: the panel (rows k0..M-1) is staged column-major in shared memory and factored
// there (left-looking inside the panel), written back, and the trailing lower triangle is updated by it on the fp64 tensor
// cores (8x8 tiles, kPanel / 4 DMMA m8n8k4 per tile, one warp per tile).  Every output element sees its updates in a fixed
// order, so the result is bitwise reproducible.
template <int D>
__global__ void __launch_bounds__(kThreads) k_chol_factor(Dev c, int lvl_off) {
  constexpr int DD = D * D;
  extern __shared__ double Ps[];   // [kPanel][ldp]: panel column q, row k0 + i at Ps[q * ldp + i]
  const Front fr = front_of<D>(c, c.lvl_sn[lvl_off + blockIdx.x]);
  const int M = fr.M, W = fr.W, tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
  double *F = fr.F;
  for (int i = warp; i < M; i += nw) for (int k = lane; k <= i; k += 32) F[(size_t)i * M + k] = 0.0;
  __syncthreads();
  for (int t = tid; t < W * D; t += nt) {   // diagonal blocks of the own columns
    const int k = t / DD, ab = t % DD, a = ab / D, b = ab % D;
    if (b <= a) F[(size_t)(k * D + a) * M + k * D + b] = c.diagH[(size_t)(fr.f + k) * DD + ab];
  }
  const int q0 = c.po_ptr[fr.s], nq = c.po_ptr[fr.s + 1] - q0;
  for (int t = tid; t < nq * DD; t += nt) {   // off-diagonal blocks, each at its own place
    const int q = q0 + t / DD, ab = t % DD, a = ab / D, b = ab % D;
    const double *H = c.pairH + (size_t)c.po_pair[q] * DD;
    F[(size_t)(c.po_row[q] * D + a) * M + c.po_col[q] * D + b] = c.po_tr[q] ? H[b * D + a] : H[a * D + b];
  }
  __syncthreads();
  for (int q = c.ch_ptr[fr.s]; q < c.ch_ptr[fr.s + 1]; q++) {   // extend-add of the children's update matrices, in order
    const Front ch = front_of<D>(c, c.ch[q]);
    const int R = ch.M - ch.W;
    const int *rm = c.relmap + c.idx_ptr[ch.s] + ch.W / D;
    for (int i = warp; i < R; i += nw) {
      const size_t pi = (size_t)(rm[i / D] * D + i % D) * M;
      const double *src = ch.F + (size_t)(ch.W + i) * ch.M + ch.W;
      for (int k = lane; k <= i; k += 32) F[pi + rm[k / D] * D + k % D] += src[k];
    }
    __syncthreads();
  }
  const int ldp = ((M + 7) & ~7) + 8;
  for (int k0 = 0; k0 < W; k0 += kPanel) {
    const int nb = min(kPanel, W - k0), nr = M - k0;
    for (int t = tid; t < ldp * kPanel; t += nt) {   // stage the panel; zero beyond its columns and rows
      const int i = t / kPanel, q = t % kPanel;
      Ps[q * ldp + i] = (q < nb && i < nr && q <= i) ? F[(size_t)(k0 + i) * M + k0 + q] : 0.0;
    }
    __syncthreads();
    for (int j = 0; j < nb; j++) {
      for (int i = j + tid; i < nr; i += nt) {
        double t = Ps[j * ldp + i];
        for (int q = 0; q < j; q++) t -= Ps[q * ldp + i] * Ps[q * ldp + j];
        Ps[j * ldp + i] = t;
      }
      __syncthreads();
      double piv = Ps[j * ldp + j];
      if (!(piv > 0.0 && piv < INFINITY)) {   // not positive definite (or not finite): flag it and go on with a unit pivot
        if (tid == 0) *c.fail = 1;
        piv = 1.0;
      }
      const double sq = sqrt(piv);
      __syncthreads();
      for (int i = j + tid; i < nr; i += nt) Ps[j * ldp + i] = i == j ? sq : Ps[j * ldp + i] / sq;
      __syncthreads();
    }
    for (int t = tid; t < nr * kPanel; t += nt) {   // the panel back into the front (lower part)
      const int i = t / kPanel, q = t % kPanel;
      if (q < nb && q <= i) F[(size_t)(k0 + i) * M + k0 + q] = Ps[q * ldp + i];
    }
    // trailing update C -= P P^T of the lower triangle of rows / columns k0 + nb .. M - 1
    const int n2 = nr - nb, nt8 = (n2 + 7) >> 3, ntiles = nt8 * (nt8 + 1) / 2;
    const int g = lane >> 2, qd = lane & 3;
    for (int tile = warp; tile < ntiles; tile += nw) {
      int bi = (int)((sqrt(8.0 * tile + 1.0) - 1.0) * 0.5);
      while ((bi + 1) * (bi + 2) / 2 <= tile) bi++;
      while (bi * (bi + 1) / 2 > tile) bi--;
      const int bj = tile - bi * (bi + 1) / 2;
      const int ri = nb + 8 * bi, rj = nb + 8 * bj;   // panel-relative rows of the tile's rows / columns
      const int gi = ri + g, gj = rj + 2 * qd;
      const bool rowok = gi < nr, c0ok = rowok && gj < nr && (bi != bj || gj <= gi), c1ok = rowok && gj + 1 < nr && (bi != bj || gj + 1 <= gi);
      double *dst = F + (size_t)(k0 + gi) * M + k0 + gj;
      double c0 = c0ok ? dst[0] : 0.0, c1 = c1ok ? dst[1] : 0.0;
#pragma unroll
      for (int s4 = 0; s4 < kPanel; s4 += 4) d2ba::dmma(c0, c1, -Ps[(s4 + qd) * ldp + ri + g], Ps[(s4 + qd) * ldp + rj + g]);
      if (c0ok) dst[0] = c0;
      if (c1ok) dst[1] = c1;
    }
    __syncthreads();
  }
}

// forward solve L y = b, one CTA per supernode of a level (leaves first): v = [b of the own columns ; 0] plus the children's
// update vectors, then y = L11^-1 v1 and the update vector v2 - L21 y for the parent
template <int D>
__global__ void __launch_bounds__(kThreads) k_chol_fwd(Dev c, int lvl_off) {
  __shared__ double v[kMaxFront];
  const Front fr = front_of<D>(c, c.lvl_sn[lvl_off + blockIdx.x]);
  const int M = fr.M, W = fr.W, tid = threadIdx.x, nt = blockDim.x;
  const double *F = fr.F;
  for (int t = tid; t < M; t += nt) v[t] = t < W ? c.b[(size_t)fr.f * D + t] : 0.0;
  __syncthreads();
  for (int q = c.ch_ptr[fr.s]; q < c.ch_ptr[fr.s + 1]; q++) {
    const Front ch = front_of<D>(c, c.ch[q]);
    const int R = ch.M - ch.W;
    const int *rm = c.relmap + c.idx_ptr[ch.s] + ch.W / D;
    const double *u = c.uvec + c.sn_uoff[ch.s];
    for (int t = tid; t < R; t += nt) v[rm[t / D] * D + t % D] += u[t];
    __syncthreads();
  }
  for (int j = 0; j < W; j++) {
    const double yj = v[j] / F[(size_t)j * M + j];
    if (tid == 0) c.y[(size_t)fr.f * D + j] = yj;
    for (int i = j + 1 + tid; i < M; i += nt) v[i] -= F[(size_t)i * M + j] * yj;
    __syncthreads();
  }
  double *u = c.uvec + c.sn_uoff[fr.s];
  for (int t = W + tid; t < M; t += nt) u[t - W] = v[t];
}

// backward solve L^T x = y, one CTA per supernode of a level (root first): x at the rows below comes from the ancestors,
// t = y1 - L21^T x2, x1 = L11^-T t
template <int D>
__global__ void __launch_bounds__(kThreads) k_chol_bwd(Dev c, int lvl_off) {
  __shared__ double v[kMaxFront];
  const Front fr = front_of<D>(c, c.lvl_sn[lvl_off + blockIdx.x]);
  const int M = fr.M, W = fr.W, tid = threadIdx.x, nt = blockDim.x;
  const double *F = fr.F;
  const int *rows = c.idx + c.idx_ptr[fr.s];
  for (int t = W + tid; t < M; t += nt) v[t] = c.x[(size_t)rows[t / D] * D + t % D];
  __syncthreads();
  for (int i = tid; i < W; i += nt) {
    double t = c.y[(size_t)fr.f * D + i];
    for (int k = W; k < M; k++) t -= F[(size_t)k * M + i] * v[k];
    v[i] = t;
  }
  __syncthreads();
  for (int j = W - 1; j >= 0; j--) {
    const double xj = v[j] / F[(size_t)j * M + j];
    if (tid == 0) c.x[(size_t)fr.f * D + j] = xj;
    for (int i = tid; i < j; i += nt) v[i] -= F[(size_t)j * M + i] * xj;
    __syncthreads();
  }
}

template <int D>
__global__ void k_chol_scatter(Dev c) {   // dx per pose from x in column order; fixed poses 0
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.n_pose) return;
  const int j = c.col_of[i];
  for (int k = 0; k < D; k++) c.dx[(size_t)i * D + k] = j < 0 ? 0.0 : c.x[(size_t)j * D + k];
}

// lm: the damping of k_chol_diag_lm (or null: k_chol_diag's)
template <int D>
void launch_factor(const Dev &c, const Symbolic &S, cudaStream_t st, const LmDamping *lm = nullptr) {
  if (c.n_pair > 0) k_chol_pairs<D><<<(c.n_pair + 127) / 128, 128, 0, st>>>(c);
  if (c.n_free > 0) {
    if (lm) k_chol_diag_lm<D><<<(c.n_free + 127) / 128, 128, 0, st>>>(c, lm->scale, lm->par);
    else k_chol_diag<D><<<(c.n_free + 127) / 128, 128, 0, st>>>(c);
  }
  for (size_t l = 0; l + 1 < S.lvl_ptr.size(); l++) {
    int m = 0;   // the level's largest front sets its shared memory
    for (int k = S.lvl_ptr[l]; k < S.lvl_ptr[l + 1]; k++) m = std::max(m, S.idx_ptr[S.lvl_sn[k] + 1] - S.idx_ptr[S.lvl_sn[k]]);
    k_chol_factor<D><<<S.lvl_ptr[l + 1] - S.lvl_ptr[l], kThreads, factor_smem(m * D), st>>>(c, S.lvl_ptr[l]);
  }
}

template <int D>
void launch_solve(const Dev &c, const Symbolic &S, cudaStream_t st) {
  const int L = (int)S.lvl_ptr.size() - 1;
  for (int l = 0; l < L; l++) k_chol_fwd<D><<<S.lvl_ptr[l + 1] - S.lvl_ptr[l], kThreads, 0, st>>>(c, S.lvl_ptr[l]);
  for (int l = L - 1; l >= 0; l--) k_chol_bwd<D><<<S.lvl_ptr[l + 1] - S.lvl_ptr[l], kThreads, 0, st>>>(c, S.lvl_ptr[l]);
  k_chol_scatter<D><<<(c.n_pose + 127) / 128, 128, 0, st>>>(c);
}

}  // namespace

#define CCK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { err = std::string(#call) + ": " + cudaGetErrorString(e_); return 100 + (int)e_; } } while (0)

void Numeric::drop_graphs() {
  for (int b = 0; b < 2; b++) {
    if (gfac[b]) cudaGraphExecDestroy(gfac[b]);
    if (gsol[b]) cudaGraphExecDestroy(gsol[b]);
    gfac[b] = gsol[b] = nullptr; gkey[b] = Lin{};
  }
}

void Numeric::release() {
  drop_graphs();
  for (void *p : bufs) cudaFree(p);
  bufs.clear();
  for (auto &e : ev) { if (e) cudaEventDestroy(e); e = nullptr; }
  dev_ready = has_system = false;
}

int Numeric::upload(cudaStream_t st, std::string &err) {
  release();
  const Symbolic &S = sym;
  const int D = S.D, DD = D * D;
  std::vector<int> all;
  auto put = [&](const std::vector<int> &v) { const size_t o = all.size(); all.insert(all.end(), v.begin(), v.end()); return o; };
  o_perm = put(S.perm); o_col_of = put(S.col_of); o_pair_lo = put(S.pair_lo); o_pair_ptr = put(S.pair_ptr); o_pair_edge = put(S.pair_edge);
  o_self_ptr = put(S.self_ptr); o_self_edge = put(S.self_edge); o_sn_first = put(S.sn_first); o_sn_width = put(S.sn_width);
  o_idx_ptr = put(S.idx_ptr); o_idx = put(S.idx); o_relmap = put(S.relmap); o_ch_ptr = put(S.ch_ptr); o_ch = put(S.ch);
  o_po_ptr = put(S.po_ptr); o_po_pair = put(S.po_pair); o_po_row = put(S.po_row); o_po_col = put(S.po_col); o_po_tr = put(S.po_tr);
  o_lvl_sn = put(S.lvl_sn);
  std::vector<long long> offs(S.sn_off);
  offs.insert(offs.end(), S.sn_uoff.begin(), S.sn_uoff.end());
  auto alloc = [&](void **p, size_t bytes) { cudaError_t e = cudaMalloc(p, bytes ? bytes : 8); if (e == cudaSuccess) bufs.push_back(*p); return e; };
  const size_t nf = (size_t)S.n_free;
  CCK(alloc((void **)&d_i, all.size() * 4)); CCK(alloc((void **)&d_off, offs.size() * 8));
  CCK(alloc((void **)&d_pairH, (size_t)S.n_pairs * DD * 8)); CCK(alloc((void **)&d_diagH, nf * DD * 8));
  CCK(alloc((void **)&d_front, (size_t)S.arena * 8)); CCK(alloc((void **)&d_uvec, (size_t)S.uarena * 8));
  CCK(alloc((void **)&d_b, nf * D * 8)); CCK(alloc((void **)&d_y, nf * D * 8)); CCK(alloc((void **)&d_x, nf * D * 8));
  CCK(alloc((void **)&d_lambda, 8)); CCK(alloc((void **)&d_fail, 4));
  if (!all.empty()) CCK(cudaMemcpyAsync(d_i, all.data(), all.size() * 4, cudaMemcpyHostToDevice, st));
  if (!offs.empty()) CCK(cudaMemcpyAsync(d_off, offs.data(), offs.size() * 8, cudaMemcpyHostToDevice, st));
  CCK(cudaStreamSynchronize(st));
  for (auto &e : ev) CCK(cudaEventCreate(&e));
  CCK(cudaFuncSetAttribute(k_chol_factor<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)factor_smem(kMaxFront)));
  CCK(cudaFuncSetAttribute(k_chol_factor<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)factor_smem(kMaxFront)));
  static int uploads = 0;   // process-wide, so that a new Numeric never repeats an old one's generation
  dev_ready = true;
  generation = ++uploads;
  return 0;
}

namespace {
// the kernels' view of n's tables and arenas with the linearisation buffers `in`
Dev dev_of(const Numeric &n, const Lin &in) {
  const Symbolic &S = n.sym;
  const int *d_i = n.d_i;
  Dev c;
  memset(&c, 0, sizeof c);
  c.n_pose = S.n_pose; c.n_free = S.n_free; c.n_edge = S.n_edge; c.n_pair = S.n_pairs;
  c.lin = in.lin; c.Dg = in.Dg; c.g = in.g; c.fixed = in.fixed; c.ea = in.ea; c.eb = in.eb; c.dx = in.dx;
  c.perm = d_i + n.o_perm; c.col_of = d_i + n.o_col_of; c.pair_lo = d_i + n.o_pair_lo; c.pair_ptr = d_i + n.o_pair_ptr; c.pair_edge = d_i + n.o_pair_edge;
  c.self_ptr = d_i + n.o_self_ptr; c.self_edge = d_i + n.o_self_edge; c.sn_first = d_i + n.o_sn_first; c.sn_width = d_i + n.o_sn_width;
  c.idx_ptr = d_i + n.o_idx_ptr; c.idx = d_i + n.o_idx; c.relmap = d_i + n.o_relmap; c.ch_ptr = d_i + n.o_ch_ptr; c.ch = d_i + n.o_ch;
  c.po_ptr = d_i + n.o_po_ptr; c.po_pair = d_i + n.o_po_pair; c.po_row = d_i + n.o_po_row; c.po_col = d_i + n.o_po_col; c.po_tr = d_i + n.o_po_tr;
  c.lvl_sn = d_i + n.o_lvl_sn; c.sn_off = n.d_off; c.sn_uoff = n.d_off + S.sn_off.size();
  c.pairH = n.d_pairH; c.diagH = n.d_diagH; c.front = n.d_front; c.uvec = n.d_uvec; c.b = n.d_b; c.y = n.d_y; c.x = n.d_x; c.lambda = n.d_lambda;
  c.fail = n.d_fail;
  return c;
}
}  // namespace

int Numeric::enqueue_lm(cudaStream_t st, const Lin &in, const LmDamping &lm, std::string &err) {
  const Dev c = dev_of(*this, in);
  CCK(cudaMemsetAsync(d_fail, 0, 4, st));
  if (sym.D == 6) { launch_factor<6>(c, sym, st, &lm); launch_solve<6>(c, sym, st); }
  else { launch_factor<4>(c, sym, st, &lm); launch_solve<4>(c, sym, st); }
  CCK(cudaGetLastError());
  return 0;
}

int Numeric::step(cudaStream_t st, int par, const Lin &in, double lambda, bool *failed_out, std::string &err) {
  const Symbolic &S = sym;
  const Dev c = dev_of(*this, in);
  if (memcmp(&gkey[par], &in, sizeof in)) {   // capture this parity's two graphs for these buffers
    if (gfac[par]) cudaGraphExecDestroy(gfac[par]);
    if (gsol[par]) cudaGraphExecDestroy(gsol[par]);
    gfac[par] = gsol[par] = nullptr;
    for (int k = 0; k < 2; k++) {
      cudaGraph_t g;
      CCK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
      if (k == 0) {
        cudaMemsetAsync(d_fail, 0, 4, st);
        if (S.D == 6) launch_factor<6>(c, S, st); else launch_factor<4>(c, S, st);
      } else {
        if (S.D == 6) launch_solve<6>(c, S, st); else launch_solve<4>(c, S, st);
      }
      CCK(cudaStreamEndCapture(st, &g));
      const cudaError_t e = cudaGraphInstantiate(k == 0 ? &gfac[par] : &gsol[par], g, 0);
      cudaGraphDestroy(g);
      CCK(e);
    }
    gkey[par] = in;
  }
  h_lambda = lambda;
  CCK(cudaMemcpyAsync(d_lambda, &h_lambda, 8, cudaMemcpyHostToDevice, st));
  CCK(cudaEventRecord(ev[0], st));
  CCK(cudaGraphLaunch(gfac[par], st));
  CCK(cudaEventRecord(ev[1], st));
  CCK(cudaGraphLaunch(gsol[par], st));
  CCK(cudaEventRecord(ev[2], st));
  CCK(cudaMemcpyAsync(&h_fail, d_fail, 4, cudaMemcpyDeviceToHost, st));
  CCK(cudaStreamSynchronize(st));
  float a = 0.f, b = 0.f;
  cudaEventElapsedTime(&a, ev[0], ev[1]); cudaEventElapsedTime(&b, ev[1], ev[2]);
  factor_ms += a; solve_ms += b; factorizations++; has_system = true;
  if (h_fail) failed++;
  *failed_out = h_fail != 0;
  return 0;
}

int Numeric::system(cudaStream_t st, double *diag, double *b, int max_pairs, int32_t *pair_ab, double *pair_H, std::string &err) {
  const Symbolic &S = sym;
  const int D = S.D, DD = D * D, nf = S.n_free, P = std::min(max_pairs, S.n_pairs);
  std::vector<double> dg((size_t)nf * DD), bv((size_t)nf * D);
  if (nf) {
    CCK(cudaMemcpyAsync(dg.data(), d_diagH, dg.size() * 8, cudaMemcpyDeviceToHost, st));
    CCK(cudaMemcpyAsync(bv.data(), d_b, bv.size() * 8, cudaMemcpyDeviceToHost, st));
  }
  if (P > 0) CCK(cudaMemcpyAsync(pair_H, d_pairH, (size_t)P * DD * 8, cudaMemcpyDeviceToHost, st));
  CCK(cudaStreamSynchronize(st));
  memset(diag, 0, (size_t)S.n_pose * DD * 8);
  memset(b, 0, (size_t)S.n_pose * D * 8);
  for (int j = 0; j < nf; j++) {
    const int i = S.perm[j];
    for (int r = 0; r < D; r++) for (int c = 0; c < D; c++) diag[(size_t)i * DD + r * D + c] = dg[(size_t)j * DD + std::max(r, c) * D + std::min(r, c)];
    for (int r = 0; r < D; r++) b[(size_t)i * D + r] = bv[(size_t)j * D + r];
  }
  for (int p = 0; p < P; p++) {
    const int e = S.pair_edge[S.pair_ptr[p]], lo = S.pair_lo[p];
    pair_ab[2 * p] = lo; pair_ab[2 * p + 1] = S.ea[e] == lo ? S.eb[e] : S.ea[e];
  }
  return 0;
}

}  // namespace d2pgo_chol

// ------------------------------------------------------------------------------------------------ C ABI: the analysis alone
extern "C" int d2pgo_cholesky_symbolic(int32_t n, const uint8_t *fixed, int32_t n_edges, const int32_t *ea, const int32_t *eb, int32_t dof,
                                       int32_t *perm_out, int32_t *sn_ptr_out, int32_t *sn_parent_out, d2pgo_cholesky_info *info) {
  if (n < 0 || n_edges < 0 || (n > 0 && (!perm_out || !sn_ptr_out || !sn_parent_out)) || (n_edges > 0 && (!ea || !eb)) || !info) return 1;
  std::vector<unsigned char> fx(n, 0);
  if (fixed) for (int i = 0; i < n; i++) fx[i] = fixed[i] ? 1 : 0;
  d2pgo_chol::Symbolic S;
  std::string err;
  if (int rc = d2pgo_chol::analyse(n, fx.data(), n_edges, ea, eb, dof, S, err)) return rc;
  memset(info, 0, sizeof *info);
  d2pgo_chol::fill_info(S, info);
  std::copy(S.perm.begin(), S.perm.end(), perm_out);
  const int NS = (int)S.sn_first.size();
  for (int s = 0; s < NS; s++) { sn_ptr_out[s] = S.sn_first[s]; sn_parent_out[s] = S.sn_parent[s]; }
  sn_ptr_out[NS] = S.n_free;
  return 0;
}
