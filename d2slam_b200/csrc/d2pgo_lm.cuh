// d2pgo_lm.cuh -- the kernels of the pose graph's ceres minimiser (d2pgo_set_minimizer, D2PGO_MINIMIZER_CERES_LM), in
// d2pgo_lm.cu; d2pgo.cu builds the solve's graph from them, its linearisation kernels and the sparse Cholesky's.
#pragma once
#include "d2pgo_handle.cuh"

namespace d2pgo_lm {

// the arrays the minimiser's kernels read, all of linearisation buffer 0 (the accepted point): poses [N][8], gradient [N][D],
// the step dx [N][D] (0 on fixed poses), and the field-major records of the edges ([D + 2 D^2][E]: r, J_a, J_b), the gravity
// priors ([12][G]: r, J_theta; 6-DoF) and the ARock proximal terms ([D + D^2][K]: r, J)
struct View {
  int D, n_pose, n_edge, n_prior, n_dual;
  const double *x, *g, *dx, *lin, *plin, *alin;
  const unsigned char *fixed; const int *ea, *eb, *ppose, *apose;
};

// each enqueues one kernel on st
void start(cudaStream_t st, d2pgo_host::LmState *s);   // the clock, the trust region and the counters
void scale(cudaStream_t st, const View &v, const double *Dg, const d2pgo_host::LmState *s, double *scale);   // Jacobi scale
void xnorm(cudaStream_t st, const View &v, double *part);   // partials of |x|^2 and of the gradient test, [2][(N + 127) / 128]
void xnorm_chart(cudaStream_t st, const View &v, double *part);   // the same in the perturbation chart (6-DoF)
// partials of r.(J dx), |J dx|^2 and |dx|^2, [3][nbe + nbg + nbk + (N + 127) / 128]
void model(cudaStream_t st, const View &v, int nbe, int nbg, int nbk, double *part);
// the one-thread decisions: the top of an iteration, after the step, after the candidate's cost
void begin(cudaStream_t st, d2pgo_host::LmState *s, const double *cost, const double *xpart, int nbp, cudaGraphConditionalHandle loop,
           cudaGraphConditionalHandle go);
void mid(cudaStream_t st, d2pgo_host::LmState *s, const int *fail, const double *part, int nbm, d2pgo_minimizer_iteration *trace,
         cudaGraphConditionalHandle eval);
void end(cudaStream_t st, d2pgo_host::LmState *s, const double *cost, d2pgo_minimizer_iteration *trace, cudaGraphConditionalHandle accept);

}  // namespace d2pgo_lm
