// Stand-in for swarm_msgs/Odometry.h (un-vendored), rotation-initialisation reference build: oracle/_shim's, over this
// directory's Pose.h.
#pragma once
#include <swarm_msgs/Pose.h>
namespace Swarm { class Odometry { public: Odometry() {} }; }
