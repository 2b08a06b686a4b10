// ref_rotinit_driver.cpp -- C entry point over the REFERENCE's own chordal rotation initialisation
// (oracle/_ref/libd2ref_rotinit.so, oracle/Makefile.ref).
//
// TEST INFRASTRUCTURE ONLY.  d2pgo/src/rot_init/rotation_initialization_base.hpp (RotationInitialization<double>, the
// non-distributed RotInit path of rotation_initialization.cpp:21-28) and d2pgo/src/pgostate.hpp are included unmodified.  This
// file builds PGOState frames and Swarm::LoopEdge records from flat arrays, calls setFixedFrameId and solve() as
// D2PGO::rotInitial does (d2pgo.cpp:336-361), and reads back the rotation states, the pose states and the report -- no
// rotation-initialisation arithmetic of its own.  The dropped-edge count replays the reference's own row builders
// (setupRotInitProblembyLoop / setupRotInitProblembyPrior) per loop and prior after the solve.
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#include "rot_init/rotation_initialization_base.hpp"

namespace {
struct Probe : D2PGO::RotationInitialization<double> {
  typedef D2PGO::RotationInitialization<double> Base;
  Probe(D2PGO::PGOState *s, D2PGO::RotInitConfig c) : Base(s, c) {}
  int rows_of_loops_and_priors() {   // loops and priors that give rows (9 each) in solveLinearRot
    std::vector<Tpl> t;
    VecX b(9);
    int used = 0;
    for (auto &l : loops) used += setupRotInitProblembyLoop(0, l, t, b) == 9;
    for (auto &p : pose_priors) used += setupRotInitProblembyPrior(0, p, t, b) == 9;
    return used;
  }
  bool solved(FrameIdType id) { auto it = frame_id_to_idx.find(id); return it != frame_id_to_idx.end() && it->second >= 0; }
  int n_loops() const { return (int)loops.size(); }
};
}  // namespace

extern "C" {

// n frames (ids, poses7 [x y z qx qy qz qw], fixed flags, ego7 = initial_ego_pose), E loops (kf a, kf b, rel7, sqrt_info36
// row-major; info = S^T S).  Outputs per frame: rot state (9, row-major) and pose state (7) after the call, solved (1 = a free
// frame some loop names); the report's state_changes and the loops that gave no rows.  Returns 0.
int ref_rot_init(int n, const int64_t *ids, const double *poses7, const uint8_t *fixed, const double *ego7, int E, const int64_t *ka,
                 const int64_t *kb, const double *rel7, const double *sqrt36, int gravity, double gravity_sqrt_info, double *rot_out,
                 double *pose_out, uint8_t *solved_out, double *state_changes, int32_t *dropped) {
  D2PGO::PGOState state(0, false);
  for (int i = 0; i < n; i++) {
    auto f = std::make_shared<D2Common::D2BaseFrame>();
    f->frame_id = ids[i]; f->drone_id = (int)(ids[i] / 1000000);
    f->odom.pose() = Swarm::Pose(poses7 + (size_t)i * 7);
    f->initial_ego_pose = Swarm::Pose(ego7 + (size_t)i * 7);
    state.addFrame(f);
  }
  std::vector<Swarm::LoopEdge> loops;
  for (int e = 0; e < E; e++) {
    Swarm::LoopEdge l;
    l.keyframe_id_a = ka[e]; l.keyframe_id_b = kb[e];
    l.relative_pose = Swarm::Pose(rel7 + (size_t)e * 7);
    for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) l.sqrt_info(i, j) = sqrt36[(size_t)e * 36 + i * 6 + j];
    l.info = l.sqrt_info.transpose() * l.sqrt_info;
    loops.push_back(l);
  }
  D2PGO::RotInitConfig cfg;
  cfg.enable_gravity_prior = gravity != 0;
  cfg.gravity_sqrt_info = gravity_sqrt_info;
  cfg.enable_float32 = false;
  cfg.self_id = 0;
  Probe ri(&state, cfg);
  ri.addLoops(loops);
  for (int i = 0; i < n; i++) if (fixed[i]) ri.setFixedFrameId(ids[i]);
  const D2Common::SolverReport rep = ri.solve();
  for (int i = 0; i < n; i++) {
    memcpy(rot_out + (size_t)i * 9, state.getRotState(ids[i]).get(), 9 * sizeof(double));
    memcpy(pose_out + (size_t)i * 7, state.getPoseState(ids[i]).get(), 7 * sizeof(double));
    solved_out[i] = ri.solved(ids[i]);
  }
  *state_changes = rep.state_changes;
  *dropped = ri.n_loops() - ri.rows_of_loops_and_priors();
  return 0;
}

}  // extern "C"
