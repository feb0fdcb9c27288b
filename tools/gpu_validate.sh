#!/bin/bash
# One-GPU validation pass used during round 2 (run under gpurun).
#   $1 = none | ncu | final   $2 = file prefix under gpurun_out/
set -u
O=gpurun_out
P=${2:-r2}
M=${1:-none}
mkdir -p $O
timeout 500 python -m pytest tests/test_gpu_tc_gemm.py tests/test_gpu_fullsize.py -q -rs -rf 2>&1 | grep -v "^  \|^E  \|^$" | tail -40 > $O/${P}_tests.log
timeout 900 python -m pytest tests -m gpu -q -rf --deselect tests/test_gpu_tc_gemm.py --deselect tests/test_gpu_fullsize.py 2>&1 | grep -v "^  \|^E  \|^$" | tail -25 > $O/${P}_pytest_gpu.log
timeout 200 python tools/tc_probe.py perf > $O/${P}_tc_perf.jsonl 2>&1
if [ "$M" = "final" ]; then
  timeout 500 python bench.py --steps 20 --warmup 5 2>&1 | tail -1 > $O/${P}_bench_n1.json
  timeout 300 python bench.py --impl reference --steps 4 --warmup 1 2>&1 | tail -1 > $O/${P}_bench_reference_arm.json
  # compute-sanitizer on the smoke step (K1, K2, wgmma tower at a small size, lazy Adam)
  timeout 300 compute-sanitizer --tool memcheck --error-exitcode 9 python -c "import __graft_entry__ as g; g.smoke()" > $O/${P}_sanitizer_memcheck.log 2>&1; echo "memcheck rc=$?" >> $O/${P}_sanitizer_memcheck.log
  B200REC_TEST_EXPERIMENTAL=1 timeout 200 python -m pytest tests/test_gpu_kernels.py -q -k "v2" -rf 2>&1 | tail -5 > $O/${P}_k6_v2.log
  # opt-in paths that have not run on a GPU yet (ahead-of-time grouping; fused push needs >= 2 GPUs)
  B200REC_TEST_EXPERIMENTAL=1 timeout 300 python -m pytest tests/test_gpu_experimental.py -q -rf 2>&1 | tail -8 > $O/${P}_experimental.log
  B200REC_GROUP_AHEAD=1 timeout 200 python bench.py --steps 20 --warmup 5 --no-cpu-baseline 2>&1 | tail -1 > $O/${P}_bench_n1_group_ahead.json
  timeout 200 python tools/config_bench.py --what dcn --iters 6 2>&1 | grep "^{" > $O/${P}_cfg3_dcn_n1.jsonl
  timeout 120 python tools/config_bench.py --what din --B 4096 --iters 6 2>&1 | grep "^{" > $O/${P}_cfg4_din_n1.jsonl
  timeout 300 python tools/config_bench.py --what gather --vocabs 1e6,1e7,1e8,1e9 --dims 16,64,128 --iters 6 2>&1 | grep "^{" > $O/${P}_cfg5_gather_n1.jsonl
else
  timeout 400 python bench.py --steps 20 --warmup 5 --no-cpu-baseline 2>&1 | tail -1 > $O/${P}_bench_n1.json
fi
if [ "$M" = "ncu" ] || [ "$M" = "final" ]; then
  timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -s 300 -c 220 --csv \
      --log-file $O/${P}_launches.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline > $O/${P}_bench_under_ncu.log 2>&1
  timeout 400 ncu --set full --clock-control none --import-source on -k regex:tc_gemm_kmajor2 -c 4 \
      -o $O/${P}_prof_tc_gemm_pair python tools/tc_probe.py perf > $O/${P}_ncu_tc.log 2>&1
fi
tail -3 $O/${P}_sanitizer_memcheck.log 2>/dev/null
cat $O/${P}_k6_v2.log $O/${P}_cfg3_dcn_n1.jsonl $O/${P}_cfg4_din_n1.jsonl $O/${P}_bench_reference_arm.json 2>/dev/null
cat $O/${P}_tests.log; cat $O/${P}_pytest_gpu.log; cat $O/${P}_tc_perf.jsonl | cut -c1-600; cat $O/${P}_bench_n1.json
