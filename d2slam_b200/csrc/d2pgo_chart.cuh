// d2pgo_chart.cuh -- the kernels of the pose graph's perturbation chart (d2pgo_set_chart, include/d2pgo.h), in d2pgo_chart.cu:
// the factor, prior and ARock proximal linearisations in [p, theta], the Euclidean retraction and the ARock dual update.  d2pgo.cu enqueues them in place of its
// retraction-chart kernels; everything that consumes the 6x6 records is shared.
#pragma once
#include <cuda_runtime.h>

namespace d2pgo_chart {

// each enqueues one kernel on st.  Pose records x [N][8] = [p, theta, 0, 0], q_init [N][4] (xyzw).
// Edges: lin [6 + 72][E] field-major r(6), J_a (6x6 row-major), J_b (6x6), per-block cost partials [(E + 127) / 128];
// the Jacobians only with want_jac (RelPoseFactorPerturbAD, RelPoseFactor.hpp:138-195)
void edges(cudaStream_t st, int n_edge, const int *ea, const int *eb, const double *x, const double *qinit, const double *rel,
           const double *sinfo, double *lin, double *cost_part, int want_jac);
// gravity priors: lin [12][G] field-major r(3), J_theta (3x3 row-major), partials [(G + 127) / 128] (GravityPriorPerturbAD)
void priors(cudaStream_t st, int n_prior, const int *pose, const double *u, const double *S, const double *x, const double *qinit,
            double *lin, double *cost_part, int want_jac);
// x_out = x + dx on the free poses, x on the fixed ones (no manifold); slots 6, 7 zero
void retract(cudaStream_t st, int n_pose, const double *x, const unsigned char *fixed, const double *dx, double *x_out);

// ARock's proximal terms of the synced dual table (K duals on poses pose[K], targets yr [K][6], weights sqrt(rho)):
// lin [6 + 36][K] field-major r, J (constant), partials [(K + 127) / 128]; and updateDualStates on y_l [K][6] at x
void arock_lin(cudaStream_t st, int n_dual, const int *pose, const double *x, const double *yr, double wT, double wR, double *lin,
               double *cost_part);
void arock_update(cudaStream_t st, int n_dual, const int *pose, const double *x, const double *yr, double *yl, double eta);

}  // namespace d2pgo_chart
