#pragma once
#include <ceres/ceres.h>
