// Stand-in for swarm_msgs/drone_trajectory.hpp (un-vendored), rotation-initialisation reference build: PGOState::addFrame
// (d2pgo/src/pgostate.hpp) pushes every frame's ego pose; rotation initialisation never reads the trajectory back.
#pragma once
#include <swarm_msgs/Pose.h>

#include <cstdint>
#include <vector>

namespace Swarm {
class DroneTrajectory {
  std::vector<int64_t> frame_ids;
  std::vector<Pose> poses;

 public:
  DroneTrajectory() {}
  void push(double stamp, const Pose &ego, int64_t frame_id) { (void)stamp; frame_ids.push_back(frame_id); poses.push_back(ego); }
};
}  // namespace Swarm
