// ref_pcm_driver.cpp -- C entry points over the REFERENCE's own PCM code (oracle/_ref/libd2ref_pcm.so, oracle/Makefile.ref).
//
// TEST INFRASTRUCTURE ONLY.  d2pgo/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp (SwarmLocalOutlierRejection) and
// d2pgo/third_party/fast_max-clique_finder/src/*.cpp (FMC) are compiled unmodified; their un-vendored dependencies are the
// stand-ins of oracle/_shim.  This file only builds the reference's objects from flat arrays and calls
// them -- no PCM arithmetic of its own.  ref_pcm feeds every loop once, in the order given, with redundant = true,
// incremental_pcm = false and the debug-file paths off; loop `id` = its index.  The smd of every tested pair is read from the
// Swarm::computeSquaredMahalanobisDistance stand-in (oracle/_shim/swarm_msgs/drone_trajectory.hpp) in the reference's call
// order: groups in std::map order of (max drone id, min drone id), rows i ascending, j ascending.
#include <cstdint>
#include <map>
#include <vector>

#include "swarm_outlier_rejection/swarm_outlier_rejection.hpp"
#include "fast_max-clique_finder/src/findClique.h"

extern "C" int ref_pcm(int is_4dof, double pcm_thres, double pos_cov, double yaw_cov, int n_frames, const int64_t *frame_ids, const int32_t *frame_agent,
                       const double *ego7, int n_loops, const int64_t *kf_a, const int64_t *kf_b, const double *rel7, const double *sqrt_info36,
                       uint8_t *good_out, double *smd_out, int64_t smd_cap, int64_t *n_smd) {
  std::map<int, Swarm::DroneTrajectory> trajs;
  std::map<int64_t, int> agent_of;
  for (int f = 0; f < n_frames; f++) {
    trajs.emplace(frame_agent[f], Swarm::DroneTrajectory(pos_cov, yaw_cov));
    trajs.at(frame_agent[f]).push(frame_ids[f], (double)f, Swarm::Pose(ego7 + 7 * f));
    agent_of[frame_ids[f]] = frame_agent[f];
  }
  std::vector<Swarm::LoopEdge> loops;
  for (int e = 0; e < n_loops; e++) {
    Swarm::LoopEdge l;
    l.id = e; l.keyframe_id_a = kf_a[e]; l.keyframe_id_b = kf_b[e]; l.id_a = agent_of.at(kf_a[e]); l.id_b = agent_of.at(kf_b[e]);
    l.relative_pose = Swarm::Pose(rel7 + 7 * e);
    for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) l.sqrt_info(r, c) = sqrt_info36[36 * e + r * 6 + c];
    l.info = l.sqrt_info.transpose() * l.sqrt_info;
    loops.push_back(l);
  }
  D2PGO::SwarmLocalOutlierRejectionParams p;
  p.pcm_thres = pcm_thres; p.redundant = true; p.incremental_pcm = false; p.is_4dof = is_4dof != 0;
  p.debug_write_pcm_errors = false; p.debug_write_debug = false; p.debug_write_pcm_good = false;
  D2PGO::SwarmLocalOutlierRejection rej(0, p, trajs);
  std::vector<double> smd;
  Swarm::pcm_smd_hook() = &smd;
  std::vector<Swarm::LoopEdge> good = rej.OutlierRejectionLoopEdges(ros::Time(), loops);
  Swarm::pcm_smd_hook() = nullptr;
  for (int e = 0; e < n_loops; e++) good_out[e] = 0;
  for (auto &l : good) good_out[l.id] = 1;
  *n_smd = (int64_t)smd.size();
  if ((int64_t)smd.size() > smd_cap) return -1;
  for (size_t k = 0; k < smd.size(); k++) smd_out[k] = smd[k];
  return (int)good.size();
}

// FMC::maxCliqueHeu on a CSR graph (ascending adjacency lists, as swarm_outlier_rejection.cpp:262-268 builds them)
extern "C" int ref_fmc_heu(int n, const int *ptr, const int *adj, int *clique_out) {
  FMC::CGraphIO g;
  g.m_vi_Vertices.assign(ptr, ptr + n + 1);
  g.m_vi_Edges.assign(adj, adj + ptr[n]);
  g.CalculateVertexDegrees();
  std::vector<int> c;
  FMC::maxCliqueHeu(g, c);
  for (size_t k = 0; k < c.size(); k++) clique_out[k] = c[k];
  return (int)c.size();
}
