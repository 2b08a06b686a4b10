// ref_pcm_stream_driver.cpp -- C entry points over the REFERENCE's own PCM code kept across calls
// (oracle/_ref/libd2ref_pcm_stream.so, oracle/Makefile.ref_pcm_stream).
//
// TEST INFRASTRUCTURE ONLY.  d2pgo/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp (SwarmLocalOutlierRejection) and
// d2pgo/third_party/fast_max-clique_finder/src/*.cpp (FMC) are compiled unmodified against the stand-ins of oracle/_shim, as
// for libd2ref_pcm.so.  This file only builds the reference's objects from flat arrays and calls them -- no PCM arithmetic of
// its own.
//   ref_pcm_stream_*  one SwarmLocalOutlierRejection kept across calls (redundant = true, incremental_pcm = false, the
//                     debug-file paths off), fed as D2PGO::solve_single / solve_multi feed it (d2pgo.cpp:170-186): before each
//                     call the keyframes new since the last one are pushed to their drones' trajectories (the map the object
//                     holds by reference); available_loops = the loops given (every loop so far, as D2PGO passes them).  Per
//                     call: the good mask over the loops given and the smd of the pairs the call tested, read from the
//                     Swarm::computeSquaredMahalanobisDistance stand-in in the reference's call order (groups in std::map
//                     order of (max drone id, min drone id), new rows in arrival order, j ascending).
//   ref_fmc_heu_inc   FMC::maxCliqueHeuIncremental's return value (its clique buffer is not a clique, findCliqueHeuInc.cpp:92-94,
//                     and is not returned).
#include <cstdint>
#include <map>
#include <vector>

#include "swarm_outlier_rejection/swarm_outlier_rejection.hpp"
#include "fast_max-clique_finder/src/findClique.h"

struct RefPcmStream {
  std::map<int, Swarm::DroneTrajectory> trajs;   // declared before rej, which holds it by reference
  std::map<int64_t, int> agent_of;
  double pos_cov, yaw_cov, stamp = 0.0;
  D2PGO::SwarmLocalOutlierRejection rej;
  RefPcmStream(const D2PGO::SwarmLocalOutlierRejectionParams &p, double pc, double yc) : pos_cov(pc), yaw_cov(yc), rej(0, p, trajs) {}
};

extern "C" void *ref_pcm_stream_new(int is_4dof, double pcm_thres, double pos_cov, double yaw_cov) {
  D2PGO::SwarmLocalOutlierRejectionParams p;
  p.pcm_thres = pcm_thres; p.redundant = true; p.incremental_pcm = false; p.is_4dof = is_4dof != 0;
  p.debug_write_pcm_errors = false; p.debug_write_debug = false; p.debug_write_pcm_good = false;
  return new RefPcmStream(p, pos_cov, yaw_cov);
}

extern "C" void ref_pcm_stream_free(void *s) { delete static_cast<RefPcmStream *>(s); }

extern "C" int ref_pcm_stream_call(void *sp, int n_frames, const int64_t *frame_ids, const int32_t *frame_agent, const double *ego7, int n_loops,
                                   const int64_t *loop_ids, const int64_t *kf_a, const int64_t *kf_b, const double *rel7, const double *sqrt_info36,
                                   uint8_t *good_out, double *smd_out, int64_t smd_cap, int64_t *n_smd) {
  RefPcmStream &S = *static_cast<RefPcmStream *>(sp);
  for (int f = 0; f < n_frames; f++) {
    if (S.agent_of.count(frame_ids[f])) continue;
    S.trajs.emplace(frame_agent[f], Swarm::DroneTrajectory(S.pos_cov, S.yaw_cov));
    S.trajs.at(frame_agent[f]).push(frame_ids[f], S.stamp, Swarm::Pose(ego7 + 7 * f));
    S.stamp += 1.0;
    S.agent_of[frame_ids[f]] = frame_agent[f];
  }
  std::vector<Swarm::LoopEdge> loops;
  std::map<int64_t, int> pos;
  for (int e = 0; e < n_loops; e++) {
    Swarm::LoopEdge l;
    l.id = loop_ids[e]; l.keyframe_id_a = kf_a[e]; l.keyframe_id_b = kf_b[e]; l.id_a = S.agent_of.at(kf_a[e]); l.id_b = S.agent_of.at(kf_b[e]);
    l.relative_pose = Swarm::Pose(rel7 + 7 * e);
    for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) l.sqrt_info(r, c) = sqrt_info36[36 * e + r * 6 + c];
    l.info = l.sqrt_info.transpose() * l.sqrt_info;
    loops.push_back(l); pos[l.id] = e;
  }
  std::vector<double> smd;
  Swarm::pcm_smd_hook() = &smd;
  std::vector<Swarm::LoopEdge> good = S.rej.OutlierRejectionLoopEdges(ros::Time(), loops);
  Swarm::pcm_smd_hook() = nullptr;
  for (int e = 0; e < n_loops; e++) good_out[e] = 0;
  for (auto &l : good) good_out[pos.at(l.id)] = 1;
  *n_smd = (int64_t)smd.size();
  if ((int64_t)smd.size() > smd_cap) return -1;
  for (size_t k = 0; k < smd.size(); k++) smd_out[k] = smd[k];
  return (int)good.size();
}

// on a CSR graph (ascending adjacency lists) whose last num_new vertices are new, under the bound prev
extern "C" int ref_fmc_heu_inc(int n, const int *ptr, const int *adj, int num_new, int prev) {
  FMC::CGraphIO g;
  g.m_vi_Vertices.assign(ptr, ptr + n + 1);
  g.m_vi_Edges.assign(adj, adj + ptr[n]);
  g.CalculateVertexDegrees();
  std::vector<int> c;
  return FMC::maxCliqueHeuIncremental(g, (size_t)num_new, (size_t)prev, c);
}
