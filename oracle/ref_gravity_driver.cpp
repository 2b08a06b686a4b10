// ref_gravity_driver.cpp -- C entry points over the REFERENCE's own perturbation-mode PGO functors
// (oracle/_ref/libd2ref_gravity.so, oracle/Makefile.ref).
//
// TEST INFRASTRUCTURE ONLY.  d2common/include/d2common/solver/GravityPrior.hpp (GravityPriorPerturbAD) and RelPoseFactor.hpp
// (RelPoseFactorPerturbAD), the functors d2pgo builds in its 6-DoF configuration (perturb_mode = true; d2pgo.cpp:427-433,
// :504-507, :530-559), are included unmodified and run with T = double (residual) and T = ceres::Jet (the exact derivatives
// of the reference's residual code, oracle/_shim/ceres).  Parameters are the perturbation blocks [p, theta] with
// q = q0 (x) quatfromRotationVector(theta).  This file only builds the reference's objects from flat arrays and calls them --
// no factor arithmetic of its own.
#include <Eigen/Dense>
#include <d2common/solver/GravityPrior.hpp>
#include <d2common/solver/RelPoseFactor.hpp>

namespace {
// AutoDiffEvaluate drives two parameter blocks; the prior has one, so a second 1-double block is passed and ignored
struct GravityTwoBlocks {
  const D2Common::GravityPriorPerturbAD &f;
  template <typename T> bool operator()(const T *const pose, const T *const, T *r) const { return f(pose, r); }
};
Eigen::Quaterniond quat(const double *q_xyzw) { return Eigen::Quaterniond(q_xyzw[3], q_xyzw[0], q_xyzw[1], q_xyzw[2]); }
}  // namespace

extern "C" {

// GravityPriorPerturbAD(ego_pose, S, q0) at the perturbation block pose6 = [p, theta]: r (3) and J (3 x 6 row-major) or NULL
int ref_gravity_prior_eval(const double *ego7, const double *sqrt_info9, const double *q0_xyzw, const double *pose6, double *r3, double *J3x6) {
  Eigen::Matrix3d S;
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) S(i, j) = sqrt_info9[i * 3 + j];
  const D2Common::GravityPriorPerturbAD f(Swarm::Pose(ego7), S, quat(q0_xyzw));
  const GravityTwoBlocks w{f};
  const double unused = 0.0;
  const double *params[2] = {pose6, &unused};
  double J_unused[3];
  double *jac[2] = {J3x6, J_unused};
  return ceres::AutoDiffEvaluate<3, 6, 1>(w, params, r3, J3x6 ? jac : nullptr) ? 3 : -2;
}

// RelPoseFactorPerturbAD(rel, S, qa0, qb0) at the perturbation blocks a6 = [p_a, theta_a], b6 = [p_b, theta_b]: r (6) and
// J_a, J_b (6 x 6 row-major) or NULL
int ref_relpose_perturb_eval(const double *rel7, const double *sqrt_info36, const double *qa0_xyzw, const double *qb0_xyzw, const double *a6, const double *b6,
                             double *r6, double *Ja6x6, double *Jb6x6) {
  Eigen::Matrix6d S;
  for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) S(i, j) = sqrt_info36[i * 6 + j];
  const D2Common::RelPoseFactorPerturbAD f(Swarm::Pose(rel7), S, quat(qa0_xyzw), quat(qb0_xyzw));
  const double *params[2] = {a6, b6};
  double *jac[2] = {Ja6x6, Jb6x6};
  return ceres::AutoDiffEvaluate<6, 6, 6>(f, params, r6, Ja6x6 ? jac : nullptr) ? 6 : -2;
}

}  // extern "C"
