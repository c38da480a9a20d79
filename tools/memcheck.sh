#!/bin/bash
# Out-of-bounds detection for the kernels, without a GPU: the emulated build of the kernel sources (tests/cudaemu)
# compiled with AddressSanitizer.  "Device memory" (frames, tap tables, scratch images) is heap memory with red zones,
# the dynamic shared memory of a launch is a heap block of exactly the requested size, static __shared__ arrays are
# instrumented globals - a kernel that reads or writes past any of them is reported with its source line.
#   bash tools/memcheck.sh     -> expects "0 reports"
set -u
cd "$(dirname "$0")/.."
AS=$(g++ -print-file-name=libasan.so)
LOG=$(mktemp -d)/asan
B200_EMU_ASAN=1 LD_PRELOAD=$AS ASAN_OPTIONS="detect_leaks=0:halt_on_error=0:log_path=$LOG" \
  python -m pytest tests/test_emu_kernels.py tests/test_emu_batch.py tests/test_emu_worstcase.py tests/test_ars_packed_formats.py tests/test_comp_convert.py tests/test_comp_domain.py tests/test_comp_fused.py tests/test_host_staging.py -q -p no:cacheprovider ${1:+-k "$1"} | tail -3
n=$(cat "$LOG".* 2>/dev/null | grep -c "ERROR: AddressSanitizer")
echo "memcheck: $n reports"
cat "$LOG".* 2>/dev/null | grep -A3 "ERROR: AddressSanitizer" | grep "#0\|#1" | sort | uniq -c | sort -rn | head -10
[ "$n" = "0" ]
