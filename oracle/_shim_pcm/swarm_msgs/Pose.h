// Stand-in for HKUST-Swarm swarm_msgs (branch D2SLAM, un-vendored) Swarm::Pose -- the PCM reference build only
// (oracle/Makefile.pcm, searched before oracle/_shim): oracle/_shim/swarm_msgs/Pose.h plus what PCM
// (swarm_outlier_rejection.cpp) touches -- Pose::log_map / toStr, DeltaPose's yaw-only branch, and the LoopEdge members id,
// ts_a / ts_b, res_count, getCovariance, same_robot_pair.
// Semantics ASSUMED from the upstream header: pose = (position, unit attitude quaternion); to_vector = [x y z qx qy qz qw];
// a * b composes, DeltaPose(a, b) = a^-1 * b, tangentSpace = [translation ; rotation vector].
#pragma once
#include <Eigen/Dense>
#include <cmath>
#include <istream>
#include <memory>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>
using namespace Eigen;
inline Eigen::Vector3d quat2eulers(const Eigen::Quaterniond &q) {
  Eigen::Vector3d rpy;
  rpy.x() = std::atan2(2 * (q.w() * q.x() + q.y() * q.z()), 1 - 2 * (q.x() * q.x() + q.y() * q.y()));
  rpy.y() = std::asin(2 * (q.w() * q.y() - q.z() * q.x()));
  rpy.z() = std::atan2(2 * (q.w() * q.z() + q.x() * q.y()), 1 - 2 * (q.y() * q.y() + q.z() * q.z()));
  return rpy;
}
inline Eigen::Quaterniond eulers2quat(const Eigen::Vector3d &e) {
  const double cr = std::cos(e.x() / 2), sr = std::sin(e.x() / 2), cp = std::cos(e.y() / 2), sp = std::sin(e.y() / 2), cy = std::cos(e.z() / 2), sy = std::sin(e.z() / 2);
  return Eigen::Quaterniond(cy * cp * cr + sy * sp * sr, cy * cp * sr - sy * sp * cr, sy * cp * sr + cy * sp * cr, sy * cp * cr - cy * sp * sr);
}
namespace Swarm {
class Pose {
  Eigen::Vector3d position; Eigen::Quaterniond attitude;
 public:
  Pose() : position(0, 0, 0) {}
  Pose(const Eigen::Vector3d &p, const Eigen::Quaterniond &q) : position(p), attitude(q.normalized()) {}
  explicit Pose(const std::shared_ptr<double> &v) : Pose(v.get()) {}
  explicit Pose(const Eigen::VectorXd &v) : position(v(0), v(1), v(2)), attitude(v(6), v(3), v(4), v(5)) { attitude.normalize(); }
  explicit Pose(const double *v, bool xyzyaw = false) : position(v[0], v[1], v[2]), attitude(v[6], v[3], v[4], v[5]) { (void)xyzyaw; attitude.normalize(); }
  const Eigen::Vector3d &pos() const { return position; }
  const Eigen::Quaterniond &att() const { return attitude; }
  Eigen::Matrix3d R() const { return attitude.toRotationMatrix(); }
  double yaw() const { return quat2eulers(attitude).z(); }
  void to_vector(std::shared_ptr<double> v) const { to_vector(v.get()); }
  void to_vector(double *v) const { v[0] = position.x(); v[1] = position.y(); v[2] = position.z(); v[3] = attitude.x(); v[4] = attitude.y(); v[5] = attitude.z(); v[6] = attitude.w(); }
  Pose inverse() const { Eigen::Quaterniond qi = attitude.inverse(); return Pose(-(qi * position), qi); }
  Pose operator*(const Pose &b) const { return Pose(attitude * b.position + position, attitude * b.attitude); }
  Eigen::Vector3d operator*(const Eigen::Vector3d &p) const { return attitude * p + position; }
  // use_yaw_only (ASSUMED): (Rz(-yaw_a) (p_b - p_a), Rz(yaw_b - yaw_a)), the 4-DoF relative pose
  static Pose DeltaPose(const Pose &a, const Pose &b, bool use_yaw_only = false) {
    if (!use_yaw_only) return a.inverse() * b;
    const double ya = a.yaw(), yb = b.yaw(), c = std::cos(ya), s = std::sin(ya);
    const Eigen::Vector3d d = b.pos() - a.pos();
    const double dy = yb - ya;
    return Pose(Eigen::Vector3d(c * d.x() + s * d.y(), -s * d.x() + c * d.y(), d.z()), Eigen::Quaterniond(std::cos(dy / 2), 0.0, 0.0, std::sin(dy / 2)));
  }
  // ASSUMED (upstream swarm_msgs/Pose.h): log_map = [translation ; rotation vector], the tangentSpace convention
  Eigen::Matrix<double, 6, 1> log_map() const { return tangentSpace(); }
  std::string toStr() const {
    char b[160];
    snprintf(b, sizeof b, "[%+.3f %+.3f %+.3f | %+.4f %+.4f %+.4f %+.4f]", position.x(), position.y(), position.z(), attitude.x(), attitude.y(), attitude.z(), attitude.w());
    return b;
  }
  // ASSUMED (upstream swarm_msgs/Pose.h): [translation ; angle * axis] with Eigen::AngleAxisd(q) conventions
  // (angle = 2 atan2(|v|, |w|), axis sign follows w) -- the same assumption oracle/orc_factors.c::orc_delta_pose_tangent states
  Eigen::Matrix<double, 6, 1> tangentSpace() const {
    Eigen::Matrix<double, 6, 1> t; t.setZero();
    t(0) = position.x(); t(1) = position.y(); t(2) = position.z();
    const double n = std::sqrt(attitude.x() * attitude.x() + attitude.y() * attitude.y() + attitude.z() * attitude.z());
    if (n > 0) { const double ang = 2.0 * std::atan2(n, std::fabs(attitude.w())), sg = attitude.w() < 0 ? -1.0 : 1.0; t(3) = ang * sg * attitude.x() / n; t(4) = ang * sg * attitude.y() / n; t(5) = ang * sg * attitude.z() / n; }
    return t;
  }
  // ASSUMED: mean position + D2Common::Utility::averageQuaterions (defined in oracle/ref_driver.cpp against the reference's utils.hpp)
  static Pose averagePoses(const std::vector<Pose> &poses);
};
// Stand-in for Swarm::LoopEdge (swarm_msgs, un-vendored): the members RelPoseFactor.hpp's Create() helpers touch.  ASSUMED.
struct LoopEdge {
  int64_t keyframe_id_a = -1, keyframe_id_b = -1; int id_a = -1, id_b = -1;
  Pose relative_pose; Eigen::Matrix<double, 6, 6> sqrt_info, info;
  LoopEdge() {}
  // (keyframe ids, relative pose, INFORMATION matrix) -- the constructor posegraph_g2o.cpp:160 uses; the square root kept beside
  // it is the Cholesky factor transposed (any S with S^T S = info gives the same cost)
  LoopEdge(int64_t a, int64_t b, const Pose &rel, const Eigen::Matrix<double, 6, 6> &information) : keyframe_id_a(a), keyframe_id_b(b), relative_pose(rel), info(information) {
    Eigen::Matrix<double, 6, 6> L = Eigen::LLT<Eigen::Matrix<double, 6, 6>>(information).matrixL(); sqrt_info = L.transpose();
  }
  Eigen::Matrix<double, 6, 6> getInfoMat() const { return info; }
  Eigen::Matrix<double, 6, 6> getSqrtInfoMat() const { return sqrt_info; }
  Eigen::Matrix<double, 4, 4> getSqrtInfoMat4D() const { Eigen::Matrix<double, 4, 4> m; m.setZero(); for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) m(i, j) = sqrt_info(i, j); m(3, 3) = sqrt_info(5, 5); return m; }
  // the members PCM (swarm_outlier_rejection.cpp) touches.  ASSUMED: covariance = (S^T S)^-1 of the square-root information;
  // same_robot_pair = 1 if the drone ids are in the same order, 2 if swapped, 0 otherwise
  int64_t id = -1; double ts_a = 0, ts_b = 0; int res_count = 6;
  Eigen::Matrix<double, 6, 6> getCovariance() const { return (sqrt_info.transpose() * sqrt_info).inverse(); }
  int same_robot_pair(const LoopEdge &o) const {
    if (id_a == o.id_a && id_b == o.id_b) return 1;
    if (id_a == o.id_b && id_b == o.id_a) return 2;
    return 0;
  }
};
}  // namespace Swarm
// ASSUMED (upstream swarm_msgs): a pose streams as x y z qx qy qz qw, the g2o column order
inline std::istream &operator>>(std::istream &is, Swarm::Pose &p) {
  double v[7]; for (int i = 0; i < 7; i++) is >> v[i];
  p = Swarm::Pose(Eigen::Vector3d(v[0], v[1], v[2]), Eigen::Quaterniond(v[6], v[3], v[4], v[5]));
  return is;
}
