// Stand-in for swarm_msgs/drone_trajectory.hpp (un-vendored) -- oracle/_ref build only: the members PCM
// (d2pgo/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp) touches.  ASSUMED semantics:
//   * a trajectory is one drone's keyframes in the order they were pushed, each with its ego (odometry) pose;
//   * get_relative_pose_by_frame_id(a, b, is_4dof) = (DeltaPose(ego_a, ego_b, is_4dof), covariance), the covariance being
//     d2pgo's ego-motion model (d2pgo.cpp:482-493) at the path length along the keyframe ego positions between a and b,
//     without the min_cov_len clamp:
//       cov_pos = (pos_cov_per_meter len + 0.5 yaw_cov_per_meter len^2) I3,   cov_rot = yaw_cov_per_meter len I3.
#pragma once
#include <swarm_msgs/Pose.h>

#include <cmath>
#include <map>
#include <utility>
#include <vector>

namespace Swarm {
class DroneTrajectory {
  std::vector<int64_t> frame_ids;
  std::vector<double> stamps;
  std::vector<Pose> poses;
  std::vector<double> path;            // path[k]: length of the polyline through the positions 0..k
  std::map<int64_t, int> index;
  double pos_cov_per_meter = 4e-3, yaw_cov_per_meter = 4e-5;   // D2PGOConfig defaults (d2pgo_config.h)

 public:
  DroneTrajectory() {}
  DroneTrajectory(double pos_cov, double yaw_cov) : pos_cov_per_meter(pos_cov), yaw_cov_per_meter(yaw_cov) {}
  void push(int64_t frame_id, double stamp, const Pose &ego) {
    index[frame_id] = (int)frame_ids.size();
    path.push_back(poses.empty() ? 0.0 : path.back() + (ego.pos() - poses.back().pos()).norm());
    frame_ids.push_back(frame_id); stamps.push_back(stamp); poses.push_back(ego);
  }
  double trajectory_length_by_frame_id(int64_t a, int64_t b) const { return std::fabs(path[index.at(b)] - path[index.at(a)]); }
  double trajectory_length_by_ts(double ta, double tb) const {
    int ia = 0, ib = 0;
    for (size_t k = 0; k < stamps.size(); k++) { if (stamps[k] <= ta) ia = (int)k; if (stamps[k] <= tb) ib = (int)k; }
    return std::fabs(path[ib] - path[ia]);
  }
  std::pair<Pose, Eigen::Matrix<double, 6, 6>> get_relative_pose_by_frame_id(int64_t a, int64_t b, bool is_4dof) const {
    const double len = trajectory_length_by_frame_id(a, b);
    Eigen::Matrix<double, 6, 6> cov = Eigen::Matrix<double, 6, 6>::Zero();
    for (int k = 0; k < 3; k++) {
      cov(k, k) = pos_cov_per_meter * len + 0.5 * yaw_cov_per_meter * len * len;
      cov(3 + k, 3 + k) = yaw_cov_per_meter * len;
    }
    return std::make_pair(Pose::DeltaPose(poses[index.at(a)], poses[index.at(b)], is_4dof), cov);
  }
};

// test hook: when set, every distance computed below is appended to it, in call order (oracle/ref_pcm_driver.cpp ref_pcm)
inline std::vector<double> *&pcm_smd_hook() { static std::vector<double> *p = nullptr; return p; }

// ASSUMED (upstream swarm_msgs): v^T cov^-1 v
inline double computeSquaredMahalanobisDistance(const Eigen::Matrix<double, 6, 1> &v, const Eigen::Matrix<double, 6, 6> &cov) {
  const Eigen::Matrix<double, 6, 1> w = cov.inverse() * v;
  double s = 0.0;
  for (int k = 0; k < 6; k++) s += v(k) * w(k);
  if (pcm_smd_hook()) pcm_smd_hook()->push_back(s);
  return s;
}
}  // namespace Swarm
