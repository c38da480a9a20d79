#!/bin/bash
# Shared-memory race detection for the kernels, without a GPU: the emulated build of the kernel sources
# (tests/cudaemu: threads of a block are real threads, __syncthreads / warp collectives are barriers) compiled with
# ThreadSanitizer, the emulated-kernel tests run under it.  A kernel that reads shared memory another thread of the
# block wrote without a barrier in between shows up as a TSAN data-race report with the kernel source line.
#   bash tools/race_check.sh            -> expects "0 reports"
#   B200_EMU_DROP_SYNC=1 bash tools/race_check.sh   -> negative control: one __syncthreads of vcs_generic_kernel removed
set -u
cd "$(dirname "$0")/.."
TS=$(g++ -print-file-name=libtsan.so)
LOG=$(mktemp -d)/tsan
B200_EMU_TSAN=1 LD_PRELOAD=$TS TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0 log_path=$LOG" \
  python -m pytest tests/test_emu_kernels.py tests/test_emu_batch.py tests/test_emu_worstcase.py tests/test_ars_packed_formats.py tests/test_comp_convert.py tests/test_comp_domain.py tests/test_comp_fused.py -q -p no:cacheprovider ${1:+-k "$1"} | tail -3
n=$(cat "$LOG".* 2>/dev/null | grep -c "WARNING: ThreadSanitizer")
echo "race_check: $n reports"
cat "$LOG".* 2>/dev/null | grep -A3 "WARNING: ThreadSanitizer: data race" | grep "#0" | sort | uniq -c | sort -rn | head -10
[ "$n" = "0" ]
