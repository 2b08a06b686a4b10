// oracle/_ref/libd2ref_arock.so: the reference's OWN ARock loop (d2common/src/solver/ARock.cpp, compiled unmodified:
// ARockBase::solve_arock, updateDualStates, createDualState, ARockSolver::scanAndCreateDualStates, setDualStateFactors with
// ConsenusPoseFactor4D (consenus_factor_4d.h) and ceres::NormalPrior) for N agents in one thread, with
//   * receiveAll / broadcastData restating ARockPGO::processPGOData / broadcastData (d2pgo/src/ARockPGO.cpp:13-104: its
//     include chain, d2pgo.h, needs the whole D2PGO node) over an in-process message table, the synchronous schedule: every
//     agent steps, then every message goes to every other agent;
//   * ceres::Solve replaced by the solve hook: it writes a given local solution (the oracle's) into the agent's states and
//     evaluates every proximal factor setDualStateFactors created in this step at that solution;
//   * each step preceded by resetResiduals + addResidual, as D2PGO::solve_multi re-adds the residuals every tick.
// Test infrastructure (tests/test_pgo_arock.py, tests/golden/ref_arock.npz).
#include <unistd.h>

#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <vector>

#include <d2common/solver/ARock.hpp>
#include <d2common/solver/consenus_factor_4d.h>

namespace Swarm {
Pose Pose::averagePoses(const std::vector<Pose> &poses) {   // ASSUMED stand-in (IsSE3 branch only; not taken by ARockPGO's types)
  Eigen::Vector3d p(0, 0, 0);
  std::vector<Eigen::Quaterniond> qs;
  for (const Pose &x : poses) { p += x.pos(); qs.push_back(x.att()); }
  p = p / (double)poses.size();
  return Pose(p, D2Common::Utility::averageQuaterions(qs));
}
}  // namespace Swarm

namespace {
struct ZeroCost : ceres::CostFunction {
  explicit ZeroCost(int nblk, int size) { set_num_residuals(1); for (int i = 0; i < nblk; i++) mutable_parameter_block_sizes()->push_back(size); }
  bool Evaluate(double const *const *, double *res, double **) const override { res[0] = 0.0; return true; }
};
struct ArockResInfo : D2Common::ResidualInfo {
  std::vector<D2Common::ParamInfo> infos;
  ArockResInfo() : D2Common::ResidualInfo(D2Common::NONE) {}
  bool relavant(const std::set<D2Common::FrameIdType> &) const override { return false; }
  std::vector<D2Common::ParamInfo> paramsList(D2Common::D2State *) const override { return infos; }
};
struct ArockState : D2Common::D2State {
  explicit ArockState(int id) : D2Common::D2State(id) {}
  void add(D2Common::FrameIdType f, int drone) {
    auto fr = std::make_shared<D2Common::D2BaseFrame>(); fr->frame_id = f; fr->drone_id = drone; frame_db[f] = fr;
  }
};
struct Msg { int sender, target; std::map<int64_t, Eigen::VectorXd> duals; };

struct Out {   // this step's outputs of one agent
  int D, max_n;
  int *n; int64_t *keys; double *yl, *yr, *fac;
};

class Agent : public D2Common::ARockSolver {
 public:
  int D;
  std::map<int64_t, D2Common::StatePtr> ptr_of;   // frame id -> state
  std::shared_ptr<ArockResInfo> ri;
  std::vector<Msg> inbox, outbox;
  const double *solved = nullptr;                 // this step's local solution, [n_frames][D] in frame order
  std::vector<int64_t> frames;
  Out out;

  Agent(ArockState *st, D2Common::ARockSolverConfig cfg, int D_, int n, const int64_t *ids, const double *init) : D2Common::ARockSolver(st, cfg), D(D_) {
    ri = std::make_shared<ArockResInfo>();
    for (int i = 0; i < n; i++) {
      D2Common::StatePtr p(new double[D], std::default_delete<double[]>());
      memcpy(p.get(), init + (size_t)i * D, sizeof(double) * D);
      D2Common::ParamInfo info; info.pointer = p; info.index = -1; info.size = D; info.eff_size = D;
      info.type = D == 4 ? D2Common::POSE_4D : D2Common::POSE_PERTURB_6D; info.id = ids[i];
      info.data_copied = Map<VectorXd>(p.get(), D);
      ri->infos.push_back(info); ptr_of[ids[i]] = p; frames.push_back(ids[i]);
    }
    ri->cost_function = std::make_shared<ZeroCost>(n, D);
  }
  // ARockPGO::processPGOData (ARockPGO.cpp:13-60) for POSE_4D / POSE_PERTURB_6D states
  void receiveAll() override {
    for (const Msg &m : inbox)
      for (const auto &it : m.duals) {
        auto f = ptr_of.find(it.first);
        if (f == ptr_of.end()) continue;
        const D2Common::StatePtr ptr = f->second;
        if (all_estimating_params.find(ptr) == all_estimating_params.end()) continue;
        if (m.target == self_id || !hasDualState(ptr, m.sender)) {
          updated = true;
          bool create = false;
          auto param_info = all_estimating_params.at(ptr);
          if (!hasDualState(ptr, m.sender)) { createDualState(param_info, m.sender, true); create = true; }
          dual_states_remote[m.sender][ptr] = it.second;
          if (create) dual_states_local[m.sender][ptr] = it.second;
        }
      }
    inbox.clear();
  }
  // ARockPGO::broadcastData (ARockPGO.cpp:72-104): one message per neighbour of dual_states_local, target = that neighbour
  void broadcastData() override {
    for (const auto &it : dual_states_local) {
      Msg m; m.sender = self_id; m.target = it.first;
      for (const auto &it2 : it.second) m.duals[all_estimating_params.at(it2.first).id] = it2.second;
      outbox.push_back(m);
    }
  }
  // the ceres::Solve of solveLocalStep: the given solution, then the proximal factors of this step evaluated at it
  void on_solve(ceres::Problem *problem) {
    for (size_t i = 0; i < frames.size(); i++) memcpy(ptr_of.at(frames[i]).get(), solved + i * D, sizeof(double) * D);
    std::map<std::pair<int, int64_t>, std::vector<double>> rec;
    size_t b = 0;
    const auto &blocks = problem->residual_blocks();
    while (b < blocks.size() && dynamic_cast<ZeroCost *>(blocks[b].cost)) b++;
    for (const auto &pp : dual_states_remote)             // setDualStateFactors' order (ARock.cpp:257-259)
      for (const auto &it : pp.second) {
        const auto &rb = blocks.at(b++);
        std::vector<double> v(D + D * D);
        const double *x = rb.params[0];
        if (D == 6) {
          double J[36]; double *jac[1] = {J}; const double *ps[1] = {x};
          rb.cost->Evaluate(ps, v.data(), jac);
          memcpy(v.data() + 6, J, sizeof J);
        } else {
          const auto *f = dynamic_cast<ceres::AutoDiffCostFunction<D2Common::ConsenusPoseFactor4D, 4, 4> *>(rb.cost);
          typedef ceres::Jet<double, 4> J4;
          J4 p[4], r[4];
          for (int k = 0; k < 4; k++) p[k] = J4(x[k], k);
          f->functor()(p, r);
          for (int k = 0; k < 4; k++) { v[k] = r[k].a; for (int q = 0; q < 4; q++) v[4 + k * 4 + q] = r[k].v[q]; }
        }
        rec[std::make_pair(pp.first, all_estimating_params.at(it.first).id)] = v;
      }
    int k = 0;
    for (const auto &kv : rec) {
      if (k < out.max_n) memcpy(out.fac + (size_t)k * (D + D * D), kv.second.data(), sizeof(double) * (D + D * D));
      k++;
    }
  }
  // the dual table after the step, (neighbour, frame id) ascending
  void dump() {
    std::map<std::pair<int, int64_t>, std::pair<Eigen::VectorXd, Eigen::VectorXd>> tab;
    for (const auto &pp : dual_states_local)
      for (const auto &it : pp.second)
        tab[std::make_pair(pp.first, all_estimating_params.at(it.first).id)] = std::make_pair(it.second, dual_states_remote.at(pp.first).at(it.first));
    *out.n = (int)tab.size();
    int k = 0;
    for (const auto &kv : tab) {
      if (k >= out.max_n) break;
      out.keys[2 * k] = kv.first.first; out.keys[2 * k + 1] = kv.first.second;
      for (int q = 0; q < D; q++) { out.yl[(size_t)k * D + q] = kv.second.first(q); out.yr[(size_t)k * D + q] = kv.second.second(q); }
      k++;
    }
  }
  void step() {
    resetResiduals();
    addResidual(ri);
    ceres::solve_hook() = [this](const ceres::Solver::Options &, ceres::Problem *p, ceres::Solver::Summary *) { on_solve(p); };
    solve();
    ceres::solve_hook() = nullptr;
    dump();
  }
};
}  // namespace

// n_agents agents, dual dimension D (4: POSE_4D, 6: POSE_PERTURB_6D), `rounds` synchronous rounds.  Agent a: self_ids[a],
// n_frames[a] frames (ids, owners, initial states [n][D], concatenated over the agents); solved[r] = every agent's local
// solution of round r, concatenated like the initial states.  Per round r and agent a (slot r * n_agents + a): n_out = the
// number of duals, keys_out [max_n][2] (neighbour, frame id), yl_out / yr_out [max_n][D] after the step, fac_out
// [max_n][D + D^2] = r | J of the step's proximal factor of each dual at the solution (J w.r.t. the D state entries).
extern "C" int ref_arock_run(int n_agents, int D, int rounds, const int *self_ids, double rho_T, double rho_theta, double eta, int init_zero,
                             const int *n_frames, const int64_t *frame_ids, const int *owners, const double *init, const double *solved, int max_n,
                             int *n_out, int64_t *keys_out, double *yl_out, double *yr_out, double *fac_out) {
  if (D != 4 && D != 6) return 1;
  std::vector<std::unique_ptr<ArockState>> states; std::vector<std::unique_ptr<Agent>> agents;
  std::vector<size_t> off(n_agents + 1, 0);
  for (int a = 0; a < n_agents; a++) off[a + 1] = off[a] + n_frames[a];
  for (int a = 0; a < n_agents; a++) {
    D2Common::ARockSolverConfig cfg;
    cfg.self_id = self_ids[a]; cfg.rho_frame_T = rho_T; cfg.rho_frame_theta = rho_theta; cfg.eta_k = eta; cfg.max_steps = 1;
    cfg.dual_state_init_to_zero = init_zero != 0; cfg.skip_iteration_usec = 0; cfg.verbose = false;
    states.emplace_back(new ArockState(self_ids[a]));
    for (size_t i = off[a]; i < off[a + 1]; i++) states.back()->add(frame_ids[i], owners[i]);
    agents.emplace_back(new Agent(states.back().get(), cfg, D, n_frames[a], frame_ids + off[a], init + off[a] * D));
  }
  const size_t F = off[n_agents];
  for (int r = 0; r < rounds; r++) {
    for (int a = 0; a < n_agents; a++) {
      Agent &g = *agents[a];
      const size_t slot = (size_t)r * n_agents + a;
      g.solved = solved + ((size_t)r * F + off[a]) * D;
      g.out = Out{D, max_n, n_out + slot, keys_out + slot * max_n * 2, yl_out + slot * max_n * D, yr_out + slot * max_n * D, fac_out + slot * max_n * (D + D * D)};
      g.step();
    }
    for (int a = 0; a < n_agents; a++) {
      for (const Msg &m : agents[a]->outbox)
        for (int b = 0; b < n_agents; b++) if (b != a) agents[b]->inbox.push_back(m);
      agents[a]->outbox.clear();
    }
  }
  return 0;
}
