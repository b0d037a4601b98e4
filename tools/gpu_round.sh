#!/bin/bash
# Runs on the GPU machine: parity tests, smoke, bench, ncu launch list + full captures, sanitizers.
# Everything of interest lands in gpurun_out/.   usage: bash tools/gpu_round.sh [all|test,smoke,bench,ncu,race,...]
set -u
mkdir -p gpurun_out
cd "${GRAFT_REPO_ROOT:-/root/repo}"
PH=${1:-all}
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,memory.total --format=csv > gpurun_out/gpu.txt 2>&1
nproc > gpurun_out/nproc.txt; lscpu > gpurun_out/lscpu.txt 2>&1
if [[ $PH == all || $PH == *test* ]]; then
  timeout 1500 python -m pytest tests -m gpu -x -q > gpurun_out/pytest_gpu.log 2>&1; echo "pytest rc=$?" >> gpurun_out/pytest_gpu.log
  tail -15 gpurun_out/pytest_gpu.log
fi
if [[ $PH == all || $PH == *smoke* ]]; then
  timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/smoke.log 2>&1; echo "smoke rc=$?" >> gpurun_out/smoke.log
  tail -3 gpurun_out/smoke.log
fi
if [[ $PH == all || $PH == *quick* ]]; then   # c2 only, no extras: the number to iterate on
  timeout 600 python bench.py --steps 200 --warmup 20 --no-cpu-baseline --no-extra-workloads --e2e-steps 5 > gpurun_out/bench_quick.json 2> gpurun_out/bench_quick.err; echo "bench quick rc=$?"
  python tools/summarize_bench.py gpurun_out/bench_quick.json
fi
if [[ $PH == all || $PH == *bench* ]]; then
  timeout 1200 python bench.py --steps 200 --warmup 20 > gpurun_out/bench.json 2> gpurun_out/bench.err; echo "bench rc=$?"
  python tools/summarize_bench.py gpurun_out/bench.json; tail -5 gpurun_out/bench.err
  timeout 600 python bench.py --impl reference --steps 20 --warmup 5 > gpurun_out/bench_ref.json 2>> gpurun_out/bench.err
  cut -c1-600 gpurun_out/bench_ref.json
fi
for w in c3 c4 c5; do
  if [[ $PH == *$w* ]]; then
    timeout 900 python bench.py --workload $w --steps 60 --warmup 10 --no-cpu-baseline --e2e-steps 3 > gpurun_out/bench_$w.json 2> gpurun_out/bench_$w.err; echo "bench $w rc=$?"
    python tools/summarize_bench.py gpurun_out/bench_$w.json; tail -3 gpurun_out/bench_$w.err
  fi
done
if [[ $PH == all || $PH == *ncu* ]]; then
  B="--no-cpu-baseline --no-extra-workloads --e2e-steps 3 --steps 20 --warmup 5"
  timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -s 1010 -c 80 --csv --log-file gpurun_out/launches.csv \
      python bench.py $B > gpurun_out/ncu_launches.log 2>&1; echo "ncu launches rc=$?"
  timeout 900 ncu --set full --clock-control none --import-source on -k regex:aie_step -s 1030 -c 1 -f -o gpurun_out/prof_step_c2 \
      python bench.py $B > gpurun_out/ncu_step_c2.log 2>&1; echo "ncu step c2 rc=$?"
fi
if [[ $PH == *ncuo* ]]; then   # the stand-alone observation kernel (c2), launched in the bench's per-kernel section
  B="--no-cpu-baseline --no-extra-workloads --e2e-steps 3 --steps 20 --warmup 5"
  timeout 900 ncu --set full --clock-control none --import-source on -k regex:aie_observe -s 4 -c 1 -f -o gpurun_out/prof_observe_c2 \
      python bench.py $B > gpurun_out/ncu_observe_c2.log 2>&1; echo "ncu observe c2 rc=$?"
fi
if [[ $PH == all || $PH == *ncx* ]]; then   # full captures of the other workloads' dominant kernels (dram bytes for `traffic`)
  B="--no-cpu-baseline --no-extra-workloads --e2e-steps 3 --steps 20 --warmup 5"
  timeout 900 ncu --set full --clock-control none --import-source on -k regex:aie_step -s 1030 -c 1 -f -o gpurun_out/prof_step_c3 \
      python bench.py --workload c3 $B > gpurun_out/ncu_step_c3.log 2>&1; echo "ncu step c3 rc=$?"
  timeout 900 ncu --set full --clock-control none --import-source on -k regex:aie_step -s 200 -c 1 -f -o gpurun_out/prof_step_c5 \
      python bench.py --workload c5 $B > gpurun_out/ncu_step_c5.log 2>&1; echo "ncu step c5 rc=$?"
  timeout 900 ncu --set full --clock-control none --import-source on -k regex:aie_covid_step -s 60 -c 1 -f -o gpurun_out/prof_step_c4 \
      python bench.py --workload c4 $B > gpurun_out/ncu_step_c4.log 2>&1; echo "ncu step c4 rc=$?"
fi
if [[ $PH == all || $PH == *race* ]]; then
  timeout 900 compute-sanitizer --tool racecheck --racecheck-report analysis python tools/sanitizer_run.py > gpurun_out/racecheck.log 2>&1; echo "racecheck rc=$?"
  tail -8 gpurun_out/racecheck.log
  timeout 600 compute-sanitizer --tool memcheck python tools/sanitizer_run.py > gpurun_out/memcheck.log 2>&1; echo "memcheck rc=$?"
  tail -5 gpurun_out/memcheck.log
fi
# gpurun_out/ is capped at 64 MiB: keep the CSV pages of every full capture, not the reports
for rep in gpurun_out/prof_*.ncu-rep; do
  [[ -f $rep ]] || continue
  b=${rep%.ncu-rep}
  ncu -i $rep --page raw --csv > ${b}_raw.csv 2>/dev/null
  ncu -i $rep --page source --csv --print-source cuda,sass > ${b}_src.csv 2>/dev/null
  rm -f $rep
done
du -sh gpurun_out; ls -la gpurun_out | head -60
