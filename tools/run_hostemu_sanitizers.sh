#!/bin/bash
# The full tl/nvl stack in the host emulation (the workers of tests/test_nvl_hostemu.py, test_nvl_complex.py, test_nvl_swap.py,
# test_nvl_graph.py, test_nvl_int128.py ...) under ThreadSanitizer and AddressSanitizer: the plugin's host code (team creation,
# launch queue, exchange board, ...) cannot be sanitised on a GPU box without the CUDA runtime getting in the way; against the
# emulated runtime it can.
# A run is a scenario of tests/hostemu_worker.py, or worker:scenario for tests/hostemu_<worker>_worker.py (e.g. graph:graphs,
# int128:zcopy); every run uses the one plugin of tests/emu/build_hostemu.sh.
cd "$(dirname "$0")/.."
export EMU_CC=/usr/bin/gcc EMU_CXX=/usr/bin/g++
rc=0
for san in thread address; do
  EMU_EXTRA="-fsanitize=$san -g" tests/emu/build_hostemu.sh > /dev/null 2>&1 || { echo "build failed ($san)"; exit 1; }
  rm -f /tmp/ucc_b200_he_$san.*
  lib=$(/usr/bin/gcc -print-file-name=$([ $san = thread ] && echo libtsan.so || echo libasan.so))
  for s in ${HOSTEMU_SCENARIOS:-allreduce colls_staged colls_zcopy colls_push colls_ce misc triggered p2p memh lanes complex: \
                                swap:zcopy swap:staged swap:persistent swap:memh swap:big_team swap:tune}; do
    case $s in *:*) worker=tests/hostemu_${s%%:*}_worker.py;; *) worker=tests/hostemu_worker.py;; esac
    log=/tmp/ucc_b200_he_${san}_${s/:/_}.log
    LD_PRELOAD=$lib TSAN_OPTIONS="log_path=/tmp/ucc_b200_he_$san:halt_on_error=0:report_signal_unsafe=0" \
      ASAN_OPTIONS="detect_leaks=0:detect_odr_violation=0:log_path=/tmp/ucc_b200_he_$san" timeout 1500 python $worker ${s#*:} > $log 2>&1
    ok=$(grep -c HOSTEMU_WORKER_OK $log)
    echo "$san $s: $([ "$ok" = 1 ] && echo ok || echo FAILED)"; [ "$ok" = 1 ] || rc=1
  done
  n=$(ls /tmp/ucc_b200_he_$san.* 2>/dev/null | wc -l)
  echo "$san: sanitizer report files: $n"; [ "$n" = 0 ] || rc=1
done
tests/emu/build_hostemu.sh > /dev/null 2>&1   # back to the plain build
exit $rc
