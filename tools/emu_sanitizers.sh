#!/bin/bash
# The device source, compiled for the host (tests/emu), under AddressSanitizer + UndefinedBehaviorSanitizer: every
# emulation-backed test of the suite plus a randomised configuration run.  CPU only.  usage: bash tools/emu_sanitizers.sh [n_fuzz]
set -u
cd "$(dirname "$0")/.."
make -C tests/emu -s libaie_emu_asan.so || exit 1   # (before the preload: the toolchain itself must not run under ASan)
export AIE_EMU_SANITIZE=1
export LD_PRELOAD="$(/usr/bin/gcc -print-file-name=libasan.so):$(/usr/bin/gcc -print-file-name=libubsan.so)"
export ASAN_OPTIONS=detect_leaks=0:halt_on_error=1 UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=1
python -m pytest tests/test_emu_golden.py tests/test_compact_transfer.py tests/test_dynamic_layout.py tests/test_one_step_economy.py \
    tests/test_device_reset.py tests/test_edge_configs.py tests/test_micro_scenarios.py tests/test_covid.py tests/test_sampler.py \
    tests/test_dense_log.py tests/test_metrics.py tests/test_reference_api.py tests/test_unflattened_views.py tests/test_adapters.py \
    tests/test_saez_batch.py tests/test_staging_plan.py tests/test_batched_metrics.py tests/test_reset_on_device.py "tests/test_fuzz_subsets.py::test_fuzz_emulated_device_code_matches_oracle" -q -m "not gpu" -p no:cacheprovider
AIE_EMU_NT=32 python -m pytest tests/test_emu_golden.py -q -m "not gpu" -p no:cacheprovider
AIE_EMU_NT=128 python -m pytest tests/test_emu_golden.py -q -m "not gpu" -p no:cacheprovider
python tools/fuzz_emu_vs_oracle.py "${1:-300}" 4242
