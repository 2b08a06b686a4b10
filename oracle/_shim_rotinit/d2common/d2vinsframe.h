// Stand-in for d2common/d2vinsframe.h -- rotation-initialisation reference build (searched before oracle/_shim's stand-in):
// as that one, with the frame members PGOState (d2pgo/src/pgostate.hpp) touches: odom.att(), T(), R().
#pragma once
#include <mutex>
#include <d2common/d2basetypes.h>
#include <d2common/utils.hpp>
#include <swarm_msgs/Pose.h>
#include <swarm_msgs/Odometry.h>
#include <d2common/d2imu.h>
namespace D2Common {
typedef std::lock_guard<std::recursive_mutex> Guard;   // d2common/d2imu.h:10
struct D2BaseFrame {   // interface of d2common/d2baseframe.h:7-60 as far as d2state.hpp and pgostate.hpp use it
  double stamp = 0; FrameIdType frame_id = -1; int drone_id = -1; int reference_frame_id = -1; bool is_keyframe = false;
  struct Odom {
    Swarm::Pose p;
    Swarm::Pose &pose() { return p; } const Swarm::Pose &pose() const { return p; }
    const Eigen::Quaterniond &att() const { return p.att(); }
  } odom;
  Swarm::Pose initial_ego_pose;
  Eigen::Vector3d T() const { return odom.p.pos(); }
  Eigen::Matrix3d R() const { return odom.p.R(); }
  virtual void moveByPose(int new_ref_frame_id, const Swarm::Pose &delta_pose) { reference_frame_id = new_ref_frame_id; odom.p = delta_pose * odom.p; }
  virtual ~D2BaseFrame() {}
};
using D2BaseFramePtr = std::shared_ptr<D2BaseFrame>;
struct VINSFrame : D2BaseFrame {};
using VINSFramePtr = std::shared_ptr<VINSFrame>;
}  // namespace D2Common
