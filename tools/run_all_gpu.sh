#!/bin/bash
# Single-GPU evidence run (from the repo root, after build()); outputs land in $OUT (default gpu_out/).
#   smoke + GPU tests -> reference arm + default bench -> key modes / memory budgets -> C++ replay -> launch list + ncu --set full ->
#   microbenchmarks -> sanitizers.      Multi-GPU: bash tools/r2_mg.sh N   (N = 2, 4, 8; N >= 2 also runs tests/test_multigpu.py).
set -u
OUT=${OUT:-gpu_out}
mkdir -p $OUT
python __graft_entry__.py --smoke 2>&1 | tail -1
timeout 1800 python -m pytest tests -x -q -m gpu 2>&1 | tail -3 | tee $OUT/pytest_gpu.log
python bench.py --impl reference --steps 3 --warmup 1 > $OUT/bench_reference_arm.json 2>/dev/null
python bench.py > $OUT/bench_default.json 2> $OUT/bench_default.err
for mode in indexed cache generic; do
  python bench.py --key-mode $mode --steps 5 --warmup 4 --no-cpu-baseline --no-strong > $OUT/bench_$mode.json 2>/dev/null
done
for cfg in "24 14" "20 12" "16 10"; do set -- $cfg
  python bench.py --base-window $1 --key-window $2 --no-strong --no-cpu-baseline --no-e2e --steps 5 > $OUT/bench_budget_$1_$2.json 2>/dev/null
done
python tools/variants/lastjson.py $OUT/bench_*.json
g++ -O2 -std=c++17 tools/replay_config5.cpp -Iinclude -Ioracle -Lhotstuff_b200 -lhs_crypto -Loracle -lhs_oracle -Wl,-rpath,'$ORIGIN/../hotstuff_b200' -Wl,-rpath,'$ORIGIN/../oracle' -o tools/replay_config5
./tools/replay_config5 1000 > $OUT/replay_config5.json 2>/dev/null
python tools/h2d_bw.py
ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file $OUT/launches.csv python bench.py --steps 3 --warmup 3 --no-cpu-baseline --no-strong > /dev/null 2>&1
ncu --set full --clock-control none --import-source on -k regex:"k_verify_main|k_verify_finish|k_digest32_fixed|k_key_lookup" -s 5 -c 5 -o $OUT/prof python tools/prof_run.py 1048576 committee > $OUT/ncu.log 2>&1
python tools/ncu_traffic.py $OUT/prof.ncu-rep 1048576 $OUT/ncu_summary.md $OUT/traffic.json > /dev/null
for mb in latency fe_warp; do
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/microbench/$mb tools/microbench/$mb.cu 2>/dev/null && ./tools/microbench/$mb > $OUT/microbench_$mb.txt
done
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize_run.py > $OUT/sanitizer_memcheck.log 2>&1; echo "memcheck rc=$?"
timeout 900 compute-sanitizer --tool racecheck --error-exitcode 9 python tools/sanitize_run.py > $OUT/sanitizer_racecheck.log 2>&1; echo "racecheck rc=$?"
