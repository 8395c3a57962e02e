#!/bin/bash
# tools/profile_step.sh TAG [CONFIG] - regenerates the ncu evidence bench.py's roofline object cites, for the CURRENT build,
# into $PROFILE_OUT (default profile_out/, git-ignored); copy the summaries into profiles/ and commit them with the build
# they measure to make them the evidence bench.py reads:
#   profiles/TAG_launches.csv   every launch of one step with its device time, DRAM bytes, warp instructions, activity
#   profiles/TAG_traffic.json   per kernel / per stage DRAM bytes (dram__bytes_read.sum + dram__bytes_write.sum)
#   profiles/TAG_inst.json      warp instructions per step (smsp__inst_executed.sum), per kernel
#   profiles/TAG_<kernel>_ncu.txt  `--set full` detail page of the dominant kernels (one launch each)
# Run on a GPU machine with Nsight Compute:  bash tools/profile_step.sh h1
# The sub-batch workers are serialised and cold-cache under ncu: compare SHARES, not absolutes.
set -u
TAG=${1:?usage: profile_step.sh TAG [CONFIG]}
CFG=${2:-1}
OUT=${PROFILE_OUT:-profile_out}
mkdir -p $OUT
CMD="python bench.py --config $CFG --profile --steps 1 --warmup 1"
METRICS=gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum,smsp__inst_executed.sum,smsp__cycles_active.avg,sm__cycles_elapsed.max,sm__warps_active.avg.per_cycle_active,smsp__thread_inst_executed.sum
ncu --metrics $METRICS --clock-control none --csv --log-file $OUT/${TAG}_launches_raw.csv $CMD > $OUT/${TAG}_prof_bench.json 2> $OUT/${TAG}_prof_bench.err
python tools/profile_summary.py $OUT/${TAG}_launches_raw.csv $TAG $OUT
for K in bb_k_node_warp bb_k_node_pair bb_k_window_lane bb_k_mutate bb_k_node_lane bb_k_leaf_lane; do
  # the second step's first launch of the kernel (skip the warm-up step's launches of that kernel)
  SKIP=$(python tools/profile_summary.py --count $OUT/${TAG}_launches_raw.csv $K)
  timeout 600 ncu --set full --clock-control none --import-source on -k regex:$K -s $SKIP -c 1 -f -o $OUT/${TAG}_$K $CMD > /dev/null 2> $OUT/${TAG}_$K.err
  ncu -i $OUT/${TAG}_$K.ncu-rep --page details > $OUT/${TAG}_${K}_ncu.txt 2>/dev/null
done
ls -la $OUT | grep $TAG
