// Stand-in for the ROS message swarm_msgs/DPGOData (un-vendored), which d2common/d2pgo_types.h names in DPGOData's ROS
// conversions.  The pins never convert: the type only has to exist.
#pragma once
namespace swarm_msgs {
struct DPGOData {};
}  // namespace swarm_msgs
