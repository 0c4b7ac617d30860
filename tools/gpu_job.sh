#!/bin/bash
# One parametrised GPU job instead of a script per call:
#   gpurun --timeout 1500 -- 'bash tools/gpu_job.sh TAG step [step ...]'
# Every step writes under gpurun_out/TAG_* (merged back by gpurun) and prints a short summary.  Steps:
#   tests         pytest -m gpu (whole suite)            tests:<expr>   pytest -m gpu -k <expr>
#   bench         bench.py (N=1, defaults)               bench_ref      bench.py --impl reference        bench_c4   bench.py --config c4 (N=1)
#   bench_n:<N>[:tag[:args]]   torchrun bench.py --gpus N (needs gpurun --gpus N)
#   launches      ncu launch list of a short bench run   ncu_scan       ncu --set full of scan_kernel (int8 10M x 384)
#   ncu_tc_int8 / ncu_tc_bf16   ncu --set full of tc_scan_kernel (batch 1024)
#   tc_variants   experimental epilogue variants of tc_scan_kernel (timing + correctness)
#   fp_scan       single-query scan timing for f32 / f16 / bf16 (10M x 384)        ncu_fp   ncu --set full of the f32 scan
#   sqlbench      tools/sql_bench.py at n = 1M for both extensions
#   shard8        one or two scan streams on a 1/8 shard (1.25M x 384 int8)
#   stream        f3: single-query scan of a streamed (pinned host -> two device windows) 10M x 384 int8 index
#   sanitizer     compute-sanitizer memcheck + racecheck over small scans / batches
set -u
TAG=$1; shift
mkdir -p gpurun_out
O=gpurun_out/$TAG
NCU="ncu --clock-control none"
# gpurun merges at most 64 MiB back: export what is read afterwards (raw metrics, details, per-line source counters) and drop the report
export_rep() {
  local rep=$1
  [ -f "$rep.ncu-rep" ] || { echo "no report $rep"; return; }
  ncu -i "$rep.ncu-rep" --page raw --csv > "${rep}_raw.csv" 2>/dev/null
  ncu -i "$rep.ncu-rep" --page details > "${rep}_details.txt" 2>/dev/null
  ncu -i "$rep.ncu-rep" --page source --csv > "${rep}_source.csv" 2>/dev/null
  python tools/ncu_summary.py "${rep}_raw.csv" > "${rep}_summary.json" 2>/dev/null
  rm -f "$rep.ncu-rep"
  ls -la ${rep}_* | awk '{print $5, $9}'
}
for step in "$@"; do
  echo "=== [$TAG] $step  ($(date +%T))"
  case "$step" in
    tests)      timeout 1500 python -m pytest tests -q -m gpu 2>&1 | tail -40 | tee ${O}_tests.txt ;;
    tests:*)    timeout 1500 python -m pytest tests -x -q -m gpu -k "${step#tests:}" 2>&1 | tail -15 | tee ${O}_tests_k.txt ;;
    bench)      timeout 900 python bench.py > ${O}_bench_n1.json 2> ${O}_bench_n1.err; tail -3 ${O}_bench_n1.err; python tools/bench_summary.py ${O}_bench_n1.json ;;
    bench_c4)   timeout 900 python bench.py --config c4 --steps 5 --warmup 1 > ${O}_bench_c4_n1.json 2> ${O}_bench_c4_n1.err; tail -2 ${O}_bench_c4_n1.err; python tools/bench_summary.py ${O}_bench_c4_n1.json ;;
    bench_n:*)  # bench_n:<N>[:tag[:extra bench.py args]]  -> torchrun, one rank per GPU
      IFS=: read -r _ NG TAG2 EXTRA <<< "$step"
      TAG2=${TAG2:-peer}
      timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((29700 + NG)) bench.py --gpus $NG $EXTRA > ${O}_bench_n${NG}_${TAG2}.json 2> ${O}_bench_n${NG}_${TAG2}.err
      tail -3 ${O}_bench_n${NG}_${TAG2}.err | cut -c1-300; python tools/bench_summary.py ${O}_bench_n${NG}_${TAG2}.json ;;
    bench_ref)  timeout 600 python bench.py --impl reference --steps 3 --warmup 1 > ${O}_bench_reference.json 2> ${O}_bench_reference.err; cut -c1-400 ${O}_bench_reference.json ;;
    launches)   timeout 600 $NCU --metrics gpu__time_duration.sum -c 400 --csv --log-file ${O}_launches.csv python bench.py --steps 16 --warmup 3 --no-cpu-baseline > /dev/null 2>&1; tail -5 ${O}_launches.csv ;;
    ncu_scan)   timeout 600 $NCU --set full --import-source on -k regex:scan_kernel -s 30 -c 1 -f -o ${O}_scan_full python bench.py --steps 40 --warmup 3 --no-cpu-baseline --no-batched > /dev/null 2>&1; export_rep ${O}_scan_full ;;
    ncu_tc_int8) timeout 600 $NCU --set full --import-source on -k regex:tc_scan_kernel -s 5 -c 1 -f -o ${O}_tc_int8_full python tools/quick_batch.py --n 10000000 --dim 384 --vtype 5 --metric 1 --nq 1024 --iters 2 > /dev/null 2>&1; export_rep ${O}_tc_int8_full ;;
    ncu_tc_bf16) timeout 600 $NCU --set full --import-source on -k regex:tc_scan_kernel -s 5 -c 1 -f -o ${O}_tc_bf16_full python tools/quick_batch.py --n 10000000 --dim 768 --vtype 3 --metric 4 --nq 1024 --iters 2 > /dev/null 2>&1; export_rep ${O}_tc_bf16_full ;;
    tc_variants)
      timeout 300 python tools/quick_batch.py --n 10000000 --dim 384 --vtype 5 --metric 1 --nq 1024 --iters 3 --sweep "${TC_SWEEP:-epi_chunk=0;epi_chunk=1}" 2>&1 | grep -v "iter 0" | tail -8 | tee ${O}_tc_variants.txt ;;
    fp_scan)
      for vt in 1 2 3; do timeout 300 python tools/quick_bench.py --n 10000000 --dim 384 --vtype $vt --metric 1 --iters 30 2>&1 | tail -1; done | tee ${O}_fp_scan.txt
      timeout 300 python tools/quick_bench.py --n 10000000 --dim 384 --vtype 2 --metric 4 --iters 30 2>&1 | tail -1 | tee -a ${O}_fp_scan.txt ;;
    ncu_fp)     timeout 600 $NCU --set full --import-source on -k regex:scan_kernel -s 8 -c 1 -f -o ${O}_scan_f32_full python tools/quick_bench.py --n 10000000 --dim 384 --vtype 1 --metric 1 --iters 10 > /dev/null 2>&1; export_rep ${O}_scan_f32_full ;;
    sqlbench)   timeout 900 python tools/sql_bench.py --n 1000000 --dim 384 --queries 50 --which both 2>&1 | cut -c1-900 | tee ${O}_sql_bench.jsonl ;;
    shard8)     timeout 300 python tools/quick_group.py 2>&1 | tail -2 | tee ${O}_shard8.txt ;;
    stream)     timeout 600 python tools/quick_stream.py 2>&1 | tail -1 | tee ${O}_stream.json ;;
    sanitizer)
      for tool in memcheck racecheck; do
        timeout 900 compute-sanitizer --tool $tool --error-exitcode 9 python tools/sanitizer_workload.py > ${O}_sanitizer_$tool.txt 2>&1
        echo "$tool rc=$?"; grep -E "ERROR SUMMARY|RACECHECK SUMMARY|workload ok" ${O}_sanitizer_$tool.txt | tail -3
      done ;;
    *) echo "unknown step $step" ;;
  esac
done
echo "=== [$TAG] done ($(date +%T))"
