#!/bin/bash
# c5 / c3 e2e leg vs. number of step chunks (large records: a chunk must still fill the GPU)
for n in 1 2 4 6; do SKIP_TESTS=1 BENCH_ARGS="--e2e-steps 5 --steps 20 --preroll 100" bash tools/gpu_e2e_chunks.sh c5 AIE_E2E_CHUNKS=$n | grep "^c5"; done
for n in 1 2 4 8; do SKIP_TESTS=1 BENCH_ARGS="--e2e-steps 10 --steps 20 --preroll 300" bash tools/gpu_e2e_chunks.sh c3 AIE_E2E_CHUNKS=$n | grep "^c3"; done
