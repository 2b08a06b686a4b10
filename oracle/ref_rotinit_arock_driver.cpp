// ref_rotinit_arock_driver.cpp -- C entry point over the REFERENCE's own distributed rotation initialisation
// (oracle/_ref/libd2ref_rotinit_arock.so, oracle/ref_rotinit_arock.py).
//
// TEST INFRASTRUCTURE ONLY.  d2pgo/src/rot_init/rotation_initialization_arock.hpp (RotationInitARock<double>, header-only,
// its receive and broadcast included) and d2common/src/solver/ARock.cpp are compiled unmodified; the reference's own
// SimplicialLLT path (the shim's dense-backed stand-in) runs live -- there is no solve hook.  This file builds one PGOState per
// agent from flat arrays, runs the rounds as D2PGO::rotInitial does (reset, addLoops, setFixedFrameId on the main agent,
// solve(); d2pgo.cpp:336-361) with max_steps = 1, routes the broadcast callbacks synchronously (every agent steps, then every
// message goes to every other agent through inputDPGOData), and reads the states back after every round -- no rotation-
// initialisation arithmetic of its own.
//
// Stand-in: the reference calls Swarm::PosePrior(id, Matrix3d M, Matrix3d info) (setDualStateFactors, :52-57), a constructor
// the shim's PosePrior (oracle/_shim/swarm_msgs/Pose.h) does not have, and PosePrior::createFromDelta in its solve_6d branch
// (out of scope here: it aborts).  The shim's struct is renamed on inclusion and a PosePrior derived from it adds both.
// ASSUMED (swarm_msgs is not in the reference tree): getRotMat() returns M unprojected, and info is information whose Cholesky
// factor is the square root (the shim's convention for its 6x6 constructor), so |getSqrtInfoMatRot()|_F = sqrt(3 rho) for
// info = rho I3.  The shim's JacobiSVD (eigenvectors of A^T A) does not give Eigen's U = V = I on a zero M, so the pin's
// attitudes are only meaningful where M is not degenerate.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <vector>

#define PosePrior PosePriorShim
#include <swarm_msgs/Pose.h>
#undef PosePrior
namespace Swarm {
struct PosePrior : PosePriorShim {
  using PosePriorShim::PosePriorShim;
  bool has_M = false; Eigen::Matrix3d M;
  PosePrior(int64_t f, const Eigen::Matrix3d &m, const Eigen::Matrix3d &info3)
      : PosePriorShim(f, Pose(), block_info(info3)), has_M(true), M(m) {}
  Eigen::Matrix3d getRotMat() const { return has_M ? M : PosePriorShim::getRotMat(); }
  static PosePrior createFromDelta(int64_t, const Eigen::VectorXd &, const Eigen::Matrix<double, 6, 6> &) { std::abort(); }
  static Eigen::Matrix<double, 6, 6> block_info(const Eigen::Matrix3d &info3) {
    Eigen::Matrix<double, 6, 6> I = Eigen::Matrix<double, 6, 6>::Identity();
    I.block<3, 3>(3, 3) = info3;
    return I;
  }
};
}  // namespace Swarm

#include "rot_init/rotation_initialization_arock.hpp"

// declared by the shim, defined by ref_arock_driver.cpp for its library: ARock.cpp's SE(3) dual branch, which rotation duals
// (a vector of 9) never take
Swarm::Pose Swarm::Pose::averagePoses(const std::vector<Pose> &) { std::abort(); }

namespace {
struct Agent : D2PGO::RotationInitARock<double> {
  typedef D2PGO::RotationInitARock<double> Base;
  using Base::Base;
  // the dual table as (neighbour, frame id) -> (y_l, y_r), ascending
  std::map<std::pair<int, int64_t>, std::pair<Eigen::VectorXd, Eigen::VectorXd>> table() {
    std::map<std::pair<int, int64_t>, std::pair<Eigen::VectorXd, Eigen::VectorXd>> out;
    for (auto &d : dual_states_local)
      for (auto &kv : d.second) out[{d.first, all_estimating_params.at(kv.first).id}] = {kv.second, dual_states_remote.at(d.first).at(kv.first)};
    return out;
  }
};
}  // namespace

extern "C" {

// A agents (self_ids[A]; self_ids[0] is main_id).  Per agent a, its frames (n_frames[a] entries, concatenated over the agents):
// ids, poses7 [x y z qx qy qz qw], owner drone, ego7 (initial_ego_pose), fixed flag; its loops (n_loops[a], concatenated): kf a,
// kf b, rel7, sqrt_info36 row-major (info = S^T S).  rho_rot_mat, eta_k, gravity rows and gravity_sqrt_info as in
// RotInitConfig / ARockSolverConfig.  After each of `rounds` rounds (steps, then delivery), per agent and frame: the rotation state
// (9, row-major) -> state_out[round][frame][9], the pose state -> pose_out[round][frame][7]; per agent: state_changes ->
// chg_out[round][a], the dual table -> n_duals_out[round][a] entries at [round][a][k] of neighbour_out, frame_out, yl_out (9),
// yr_out (9), k < max_duals.  Returns 0, or 2 when a table holds more than max_duals duals.
int ref_rot_init_arock(int A, const int32_t *self_ids, const int32_t *n_frames, const int64_t *ids, const double *poses7, const int32_t *owner,
                       const double *ego7, const uint8_t *fixed, const int32_t *n_loops, const int64_t *ka, const int64_t *kb, const double *rel7,
                       const double *sqrt36, double rho_rot_mat, double eta_k, int gravity, double gravity_sqrt_info, int rounds,
                       double *state_out, double *pose_out, double *chg_out, int max_duals, int32_t *n_duals_out, int32_t *neighbour_out,
                       int64_t *frame_out, double *yl_out, double *yr_out) {
  std::vector<std::unique_ptr<D2PGO::PGOState>> states;
  std::vector<std::unique_ptr<Agent>> agents;
  std::vector<std::vector<Swarm::LoopEdge>> loops(A);
  std::vector<std::vector<int64_t>> frames(A), fixed_ids(A);
  std::vector<D2Common::DPGOData> outbox;
  int F0 = 0, L0 = 0;
  for (int a = 0; a < A; a++) {
    states.emplace_back(new D2PGO::PGOState(self_ids[a], false));
    for (int i = F0; i < F0 + n_frames[a]; i++) {
      auto f = std::make_shared<D2Common::D2BaseFrame>();
      f->frame_id = ids[i]; f->drone_id = owner[i];
      f->odom.pose() = Swarm::Pose(poses7 + (size_t)i * 7);
      f->initial_ego_pose = Swarm::Pose(ego7 + (size_t)i * 7);
      states[a]->addFrame(f);
      frames[a].push_back(ids[i]);
      if (fixed[i]) fixed_ids[a].push_back(ids[i]);
    }
    for (int e = L0; e < L0 + n_loops[a]; e++) {
      Swarm::LoopEdge l;
      l.keyframe_id_a = ka[e]; l.keyframe_id_b = kb[e];
      l.relative_pose = Swarm::Pose(rel7 + (size_t)e * 7);
      for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) l.sqrt_info(i, j) = sqrt36[(size_t)e * 36 + i * 6 + j];
      l.info = l.sqrt_info.transpose() * l.sqrt_info;
      loops[a].push_back(l);
    }
    D2PGO::RotInitConfig rc;
    rc.enable_gravity_prior = gravity != 0; rc.gravity_sqrt_info = gravity_sqrt_info; rc.enable_float32 = false; rc.self_id = self_ids[a];
    D2Common::ARockSolverConfig ac;
    ac.self_id = self_ids[a]; ac.rho_rot_mat = rho_rot_mat; ac.eta_k = eta_k; ac.max_steps = 1;
    agents.emplace_back(new Agent(states[a].get(), rc, ac, [&outbox](const D2Common::DPGOData &d) { outbox.push_back(d); }));
    F0 += n_frames[a]; L0 += n_loops[a];
  }
  for (int r = 0; r < rounds; r++) {
    outbox.clear();
    for (int a = 0; a < A; a++) {   // D2PGO::rotInitial
      agents[a]->reset();
      agents[a]->addLoops(loops[a]);
      if (a == 0) for (int64_t f : fixed_ids[a]) agents[a]->setFixedFrameId(f);
      chg_out[(size_t)r * A + a] = agents[a]->solve().state_changes;
    }
    for (int a = 0; a < A; a++)
      for (const auto &d : outbox) if (d.drone_id != self_ids[a]) agents[a]->inputDPGOData(d);
    int f0 = 0;
    for (int a = 0; a < A; a++) {
      for (size_t i = 0; i < frames[a].size(); i++, f0++) {
        const size_t o = (size_t)r * F0 + f0;
        memcpy(state_out + o * 9, states[a]->getRotState(frames[a][i]).get(), 72);
        memcpy(pose_out + o * 7, states[a]->getPoseState(frames[a][i]).get(), 56);
      }
      const auto t = agents[a]->table();
      if ((int)t.size() > max_duals) return 2;
      n_duals_out[(size_t)r * A + a] = (int32_t)t.size();
      size_t k = ((size_t)r * A + a) * max_duals;
      for (const auto &kv : t) {
        neighbour_out[k] = kv.first.first; frame_out[k] = kv.first.second;
        memcpy(yl_out + k * 9, kv.second.first.data(), 72); memcpy(yr_out + k * 9, kv.second.second.data(), 72);
        k++;
      }
    }
  }
  return 0;
}

}  // extern "C"
