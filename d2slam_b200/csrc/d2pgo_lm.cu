// d2pgo_lm.cu -- the kernels of the pose graph's ceres minimiser (d2pgo_lm.cuh; the solve's graph is built in d2pgo.cu):
// ceres' Levenberg-Marquardt trust region (d2pgo_set_minimizer, include/d2pgo.h) on the device.  Per-pose / per-term kernels
// write per-block partials; one-thread control kernels sum them in block order (bitwise reproducible, no atomics), make every
// decision of TrustRegionMinimizer in LmState and set the conditional nodes of the solve's graph.  Buffer 0 always holds the
// accepted point (poses, lin records, g, D), buffer 1 the candidate's poses and cost.
#include <float.h>
#include <math.h>

#include "d2ba_math.cuh"
#include "d2pgo_lm.cuh"

namespace d2pgo_lm {
using namespace d2ba;
using d2pgo_host::LmState;
namespace {

D2BA_DEV unsigned long long lm_clock() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__global__ void k_lm_start(LmState *s) {   // the solve's first device work: the clock, the trust region and the counters
  s->t0 = s->t_end = lm_clock();
  s->radius = s->radius0; s->decrease_factor = 2.0;
  s->cost = s->cost0 = s->x_norm = s->model = s->step_norm = 0.0;
  s->iter = s->ok = s->bad = s->invalid_run = s->pivot_fail = s->done = s->reason = s->cand = 0;
  s->pending_grad = 1; s->type = -1;
}

// the Jacobi scale s = 1 / (1 + sqrt(H_kk)) per tangent column from the block diagonal of the first linearisation (1 without
// jacobi_scaling)
template <int D>
__global__ void k_lm_scale(int n, const double *Dg, const LmState *s, double *scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int k = 0; k < D; k++) scale[(size_t)i * D + k] = s->jacobi ? 1.0 / (1.0 + sqrt(Dg[(size_t)i * D * D + k * (D + 1)])) : 1.0;
}

// the retraction of the gradient test (PoseLocalParameterization::Plus / PosAngleManifold::Plus, as d2pgo.cu's PgoEdge6 / PgoEdge4)
template <int D>
D2BA_DEV void lm_plus(const double *x, const double *d, double *o) {
  if constexpr (D == 6) {
    pose_plus(x, d, o);
  } else {
    for (int k = 0; k < 3; k++) o[k] = x[k] + d[k];
    const double a = x[3] + d[3];
    o[3] = a - 2.0 * M_PI * floor((a + M_PI) / (2.0 * M_PI));
  }
}

// per free pose at the accepted point: partials of |x|^2 (ambient) and of the gradient test's max |x - x [+] (-g)|
template <int D>
__global__ void __launch_bounds__(128) k_lm_xnorm(View v, double *part) {
  constexpr int NX = D == 6 ? 7 : 4;
  __shared__ double red[40];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double xx = 0.0, gm = 0.0;
  if (i < v.n_pose && !v.fixed[i]) {
    const double *x = v.x + (size_t)i * 8;
    double mg[D], o[NX];
    for (int k = 0; k < D; k++) mg[k] = -v.g[(size_t)i * D + k];
    lm_plus<D>(x, mg, o);
    for (int k = 0; k < NX; k++) { xx += x[k] * x[k]; gm = fmax(gm, fabs(x[k] - o[k])); }
  }
  xx = block_sum(xx, red);
  gm = block_max(gm, red);
  if (threadIdx.x == 0) { part[blockIdx.x] = xx; part[gridDim.x + blockIdx.x] = gm; }
}

// k_lm_xnorm in the perturbation chart (d2pgo_set_chart): the state [p, theta] has no manifold, so |x|^2 and the gradient
// test's max |x - (x + (-g))| run over the six Euclidean components of each free pose
__global__ void __launch_bounds__(128) k_lm_xnorm_chart(View v, double *part) {
  __shared__ double red[40];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double xx = 0.0, gm = 0.0;
  if (i < v.n_pose && !v.fixed[i]) {
    const double *x = v.x + (size_t)i * 8;
    for (int k = 0; k < 6; k++) { xx += x[k] * x[k]; gm = fmax(gm, fabs(x[k] - (x[k] + -v.g[(size_t)i * 6 + k]))); }
  }
  xx = block_sum(xx, red);
  gm = block_max(gm, red);
  if (threadIdx.x == 0) { part[blockIdx.x] = xx; part[gridDim.x + blockIdx.x] = gm; }
}

// the model terms of the step dx: partials of r.(J dx) and |J dx|^2 over the edges (blocks [0, nbe)), the gravity priors (next
// nbg), the proximal terms (next nbk), and of |dx|^2 over the poses (the rest); part = [3][gridDim.x]
template <int D>
__global__ void __launch_bounds__(128) k_lm_model(View v, int nbe, int nbg, int nbk, double *part) {
  constexpr int DD = D * D;
  __shared__ double red[40];
  const int b = blockIdx.x, t = threadIdx.x;
  double rj = 0.0, jj = 0.0, dd = 0.0;
  if (b < nbe) {
    const int e = b * 128 + t;
    if (e < v.n_edge) {
      const size_t E = (size_t)v.n_edge;
      const double *o = v.lin + e, *J0 = o + (size_t)D * E, *J1 = J0 + (size_t)DD * E;
      const double *da = v.dx + (size_t)v.ea[e] * D, *db = v.dx + (size_t)v.eb[e] * D;
      for (int k = 0; k < D; k++) {
        double f = 0.0;
        for (int q = 0; q < D; q++) f += J0[(size_t)(k * D + q) * E] * da[q] + J1[(size_t)(k * D + q) * E] * db[q];
        rj += o[k * E] * f; jj += f * f;
      }
    }
  } else if (b < nbe + nbg) {
    if constexpr (D == 6) {
      const int k = (b - nbe) * 128 + t;
      if (k < v.n_prior) {
        const size_t G = (size_t)v.n_prior;
        const double *o = v.plin + k, *dq = v.dx + (size_t)v.ppose[k] * 6 + 3;
        for (int a = 0; a < 3; a++) {
          double f = 0.0;
          for (int c = 0; c < 3; c++) f += o[(size_t)(3 + a * 3 + c) * G] * dq[c];
          rj += o[a * G] * f; jj += f * f;
        }
      }
    }
  } else if (b < nbe + nbg + nbk) {
    const int k = (b - nbe - nbg) * 128 + t;
    if (k < v.n_dual) {
      const size_t K = (size_t)v.n_dual;
      const double *o = v.alin + k, *di = v.dx + (size_t)v.apose[k] * D;
      for (int a = 0; a < D; a++) {
        double f = 0.0;
        for (int c = 0; c < D; c++) f += o[(size_t)(D + a * D + c) * K] * di[c];
        rj += o[a * K] * f; jj += f * f;
      }
    }
  } else {
    const int i = (b - nbe - nbg - nbk) * 128 + t;
    if (i < v.n_pose) for (int k = 0; k < D; k++) dd += v.dx[(size_t)i * D + k] * v.dx[(size_t)i * D + k];   // 0 on fixed poses
  }
  rj = block_sum(rj, red); jj = block_sum(jj, red); dd = block_sum(dd, red);
  if (t == 0) { part[b] = rj; part[gridDim.x + b] = jj; part[2 * (size_t)gridDim.x + b] = dd; }
}

D2BA_DEV void lm_stop(LmState *s, int type, int reason) { s->done = 1; s->type = type; s->reason = reason; }
// the iteration's trace record (after its trust-region update) and its count: successful only when accepted
D2BA_DEV void lm_record(LmState *s, d2pgo_minimizer_iteration *trace, double cand, double rho, int kind) {
  if (kind == D2PGO_STEP_ACCEPTED) s->ok++; else s->bad++;
  const int k = s->iter - 1;
  if (k >= s->trace_cap) return;
  d2pgo_minimizer_iteration &r = trace[k];
  r.cost = s->cost; r.candidate_cost = cand; r.model_cost_change = s->model; r.relative_decrease = rho; r.step_norm = s->step_norm;
  r.radius = s->radius; r.decrease_factor = s->decrease_factor; r.kind = kind; r.pad_ = 0;
}
// LevenbergMarquardtStrategy::StepRejected (and StepIsInvalid), then the minimum-radius test
D2BA_DEV void lm_reject(LmState *s, d2pgo_minimizer_iteration *trace, double cand, double rho, int kind) {
  s->radius = s->radius / s->decrease_factor;
  s->decrease_factor = 2.0 * s->decrease_factor;
  lm_record(s, trace, cand, rho, kind);
  if (s->radius < s->min_radius) lm_stop(s, D2PGO_TERMINATION_CONVERGENCE, D2PGO_STOP_MIN_RADIUS);
}

// top of an iteration: after a (re)linearisation the gradient test (cost[0] and xpart of buffer 0), then the iteration and
// time limits.  Sets `go` (the iteration's body) and, once done, `loop` to 0.
__global__ void k_lm_begin(LmState *s, const double *cost, const double *xpart, int nbp, cudaGraphConditionalHandle loop,
                           cudaGraphConditionalHandle go) {
  if (!s->done && s->pending_grad) {
    s->pending_grad = 0;
    s->cost = cost[0];
    if (s->iter == 0) s->cost0 = s->cost;
    double xx = 0.0, gm = 0.0;
    for (int b = 0; b < nbp; b++) { xx += xpart[b]; gm = fmax(gm, xpart[nbp + b]); }
    s->x_norm = sqrt(xx);
    if (gm <= s->gtol) lm_stop(s, D2PGO_TERMINATION_CONVERGENCE, D2PGO_STOP_GRADIENT);
  }
  if (!s->done && s->iter >= s->max_iter) lm_stop(s, D2PGO_TERMINATION_NO_CONVERGENCE, D2PGO_STOP_MAX_ITERATIONS);
  if (!s->done && s->budget_s > 0.0 && (double)(lm_clock() - s->t0) * 1e-9 >= s->budget_s)
    lm_stop(s, D2PGO_TERMINATION_NO_CONVERGENCE, D2PGO_STOP_TIME);
  if (!s->done) s->iter++;
  s->t_end = lm_clock();
  cudaGraphSetConditional(loop, s->done ? 0u : 1u);
  cudaGraphSetConditional(go, s->done ? 0u : 1u);
}

// after the step: m, |dx|, validity, the parameter test.  Sets `eval` (the candidate's evaluation).
__global__ void k_lm_mid(LmState *s, const int *fail, const double *part, int nbm, d2pgo_minimizer_iteration *trace,
                         cudaGraphConditionalHandle eval) {
  double rj = 0.0, jj = 0.0, dd = 0.0;
  for (int b = 0; b < nbm; b++) { rj += part[b]; jj += part[nbm + b]; dd += part[2 * nbm + b]; }
  s->model = -(rj + 0.5 * jj);
  s->step_norm = sqrt(dd);
  s->cand = 0;
  if (*fail) s->pivot_fail++;
  if (*fail || !isfinite(s->model) || !(s->model > 0.0) || !isfinite(s->step_norm)) {
    if (++s->invalid_run > s->max_invalid) {
      lm_record(s, trace, NAN, NAN, D2PGO_STEP_INVALID);
      lm_stop(s, D2PGO_TERMINATION_FAILURE, D2PGO_STOP_INVALID_STEPS);
    } else {
      lm_reject(s, trace, NAN, NAN, D2PGO_STEP_INVALID);
    }
  } else {
    s->invalid_run = 0;
    if (s->step_norm <= s->ptol * (s->x_norm + s->ptol)) {
      lm_record(s, trace, NAN, NAN, D2PGO_STEP_CONVERGED);
      lm_stop(s, D2PGO_TERMINATION_CONVERGENCE, D2PGO_STOP_PARAMETER);
    } else {
      s->cand = 1;
    }
  }
  s->t_end = lm_clock();
  cudaGraphSetConditional(eval, (unsigned)s->cand);
}

// after the candidate's cost (cost[1]): the function test, rho, accept or reject.  Sets `accept` (x <- x+ and relinearise).
__global__ void k_lm_end(LmState *s, const double *cost, d2pgo_minimizer_iteration *trace, cudaGraphConditionalHandle accept) {
  unsigned acc = 0;
  if (s->cand) {
    s->cand = 0;
    const double cp = isfinite(cost[1]) ? cost[1] : DBL_MAX;   // ceres' cost of a failed evaluation
    const double dc = s->cost - cp, rho = dc / s->model;
    if (fabs(dc) <= s->ftol * s->cost) {
      lm_record(s, trace, cp, rho, D2PGO_STEP_CONVERGED);
      lm_stop(s, D2PGO_TERMINATION_CONVERGENCE, D2PGO_STOP_FUNCTION);
    } else if (rho > s->min_rel_dec) {   // LevenbergMarquardtStrategy::StepAccepted
      const double t = 2.0 * rho - 1.0;
      s->radius = fmin(s->radius / fmax(1.0 / 3.0, 1.0 - t * t * t), s->max_radius);
      s->decrease_factor = 2.0;
      s->pending_grad = 1;
      acc = 1;
      lm_record(s, trace, cp, rho, D2PGO_STEP_ACCEPTED);
    } else {
      lm_reject(s, trace, cp, rho, D2PGO_STEP_REJECTED);
    }
  }
  s->t_end = lm_clock();
  cudaGraphSetConditional(accept, acc);
}

}  // namespace

void start(cudaStream_t st, LmState *s) { k_lm_start<<<1, 1, 0, st>>>(s); }

void scale(cudaStream_t st, const View &v, const double *Dg, const LmState *s, double *out) {
  const int nb = (v.n_pose + 127) / 128;
  if (v.D == 6) k_lm_scale<6><<<nb, 128, 0, st>>>(v.n_pose, Dg, s, out);
  else k_lm_scale<4><<<nb, 128, 0, st>>>(v.n_pose, Dg, s, out);
}

void xnorm(cudaStream_t st, const View &v, double *part) {
  const int nb = (v.n_pose + 127) / 128;
  if (v.D == 6) k_lm_xnorm<6><<<nb, 128, 0, st>>>(v, part);
  else k_lm_xnorm<4><<<nb, 128, 0, st>>>(v, part);
}

void xnorm_chart(cudaStream_t st, const View &v, double *part) { k_lm_xnorm_chart<<<(v.n_pose + 127) / 128, 128, 0, st>>>(v, part); }

void model(cudaStream_t st, const View &v, int nbe, int nbg, int nbk, double *part) {
  const int nb = nbe + nbg + nbk + (v.n_pose + 127) / 128;
  if (v.D == 6) k_lm_model<6><<<nb, 128, 0, st>>>(v, nbe, nbg, nbk, part);
  else k_lm_model<4><<<nb, 128, 0, st>>>(v, nbe, nbg, nbk, part);
}

void begin(cudaStream_t st, LmState *s, const double *cost, const double *xpart, int nbp, cudaGraphConditionalHandle loop,
           cudaGraphConditionalHandle go) {
  k_lm_begin<<<1, 1, 0, st>>>(s, cost, xpart, nbp, loop, go);
}

void mid(cudaStream_t st, LmState *s, const int *fail, const double *part, int nbm, d2pgo_minimizer_iteration *trace,
         cudaGraphConditionalHandle eval) {
  k_lm_mid<<<1, 1, 0, st>>>(s, fail, part, nbm, trace, eval);
}

void end(cudaStream_t st, LmState *s, const double *cost, d2pgo_minimizer_iteration *trace, cudaGraphConditionalHandle accept) {
  k_lm_end<<<1, 1, 0, st>>>(s, cost, trace, accept);
}

}  // namespace d2pgo_lm
