// Stand-in for swarm_msgs/relative_measurments.hpp (un-vendored) -- Swarm::LoopEdge and Swarm::PosePrior live in Pose.h.
#pragma once
#include <swarm_msgs/Pose.h>
