#!/bin/bash
# Run on the GPU box (gpurun).  Produces the per-launch list and full ncu captures of the hot kernels.
#   bash tools/profile.sh [B]      -> gpurun_out/launches_B$B.csv, gpurun_out/prof_<kernel>_B$B.ncu-rep
set -x
B=${1:-592}
K='regex:k_(lm_gather|lm_gather16|schur|schur_small|sb_elim|chol|chol_smem|sb_back|step|misc_lin|imu_lin|proj_lin|proj_lin_pp|control)'
ncu --metrics gpu__time_duration.sum --clock-control none -k "$K" -s 30 -c 120 --csv --log-file gpurun_out/launches_B${B}.csv python tools/profile_target.py $B 3 > gpurun_out/prof_target.log 2>&1
for kn in proj_lin_pp lm_gather16 chol_smem sb_elim sb_back schur_small step misc_lin imu_lin; do
  ncu --set full --clock-control none --import-source on -k "regex:^k_${kn}\$|^void k_${kn}|d2ba::k_${kn}" -s 4 -c 1 -f -o gpurun_out/prof_${kn}_B${B} python tools/profile_target.py $B 3 >> gpurun_out/prof_target.log 2>&1
done
ls -la gpurun_out/
