// Stand-in for swarm_msgs/relative_measurments.hpp (un-vendored), PCM reference build -- Swarm::LoopEdge lives in Pose.h.
#pragma once
#include <swarm_msgs/Pose.h>
