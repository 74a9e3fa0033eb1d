#!/bin/bash
# tl/nvl kernels in the host emulation under ThreadSanitizer: checks the synchronisation PROTOCOL of every kernel (are all
# cross-"GPU" data accesses ordered by the flag / barrier exchanges?) at the happens-before level.  The kernels validated on
# GPUs are the controls (0 reports); removing the wait of one inter-GPU barrier from nvls_pipe produces reports.
set -e
cd "$(dirname "$0")/.."
K=src/components/tl/nvl/kernels
rc=0
# driver:modes (the complex and swap drivers run everything in one mode)
for spec in "nvl_emu:staged xchg pipe symm push oneshot_rs soak soak2" "nvl_emu_complex:complex" "nvl_emu_swap:swap"; do
  exe=/tmp/ucc_b200_${spec%%:*}_tsan
  /usr/bin/g++ -O1 -g -fsanitize=thread -std=c++17 -pthread -I/usr/local/cuda/include -I$K -Iinclude -Isrc tests/emu/${spec%%:*}.cpp -o $exe
  for w in ${spec#*:}; do
    TSAN_OPTIONS="halt_on_error=0:report_signal_unsafe=0" $exe $w > /tmp/ucc_b200_emu_tsan_$w.log 2>&1 || true
    n=$(grep -c 'WARNING: ThreadSanitizer' /tmp/ucc_b200_emu_tsan_$w.log || true)
    ok=$(grep -c NVL_EMU_OK /tmp/ucc_b200_emu_tsan_$w.log || true)
    echo "$w: tsan reports $n, result $([ "$ok" = 1 ] && echo ok || echo FAILED)"
    if [ "$n" != 0 ] || [ "$ok" != 1 ]; then rc=1; fi
  done
done
exit $rc
