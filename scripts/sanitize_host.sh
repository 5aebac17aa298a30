#!/usr/bin/env bash
# AddressSanitizer + UndefinedBehaviorSanitizer (+ ThreadSanitizer for the rank runtime) over the host-only programs (no GPU needed): the OpenMP concurrency
# bench (driver grammar, autotune, verdict, JSON rows, error paths) and the native self-test (rank runtime, topology,
# mapping policies, tile / ring orderings).  The device code has its own check: scripts/sanitize.sh (compute-sanitizer).
set -euo pipefail
cd "$(dirname "$0")/.."
out=${1:-build/sanitize_host}; mkdir -p "$out"
CXX=${HOSTCXX:-/usr/bin/g++}
FLAGS="-O1 -g -std=c++17 -fopenmp -fsanitize=address,undefined -fno-sanitize-recover=undefined -fno-omit-frame-pointer -Icsrc -I/usr/local/cuda/include"
$CXX $FLAGS csrc/concurency/main.cpp csrc/concurency/driver.cpp csrc/concurency/backend_cpu.cpp \
     csrc/concurency/backend_nocuda.cpp -o "$out/omp_con"
$CXX $FLAGS csrc/tests/native_selftest.cpp csrc/concurency/driver.cpp csrc/p2p/topology_core.cpp -o "$out/native_selftest" -ldl
# ThreadSanitizer over the thread-per-rank runtime (barriers, reductions, failure propagation) that every native CLI uses
$CXX -O1 -g -std=c++17 -fopenmp -fsanitize=thread -Icsrc -I/usr/local/cuda/include csrc/tests/native_selftest.cpp \
     csrc/concurency/driver.cpp csrc/p2p/topology_core.cpp -o "$out/native_selftest_tsan" -ldl
if "$out/native_selftest_tsan" 2>&1 | tee "$out/tsan.log" | grep -q "WARNING: ThreadSanitizer"; then
  echo "sanitize_host: FAILED (data race, see $out/tsan.log)"; exit 1
fi
export ASAN_OPTIONS=detect_leaks=1:abort_on_error=0 UBSAN_OPTIONS=print_stacktrace=1
"$out/native_selftest"
"$out/omp_con" host_threads --globalsize_default_memory 200000 --tripcount_C 1000 --commands C M2D \
     --commands M2D D2M --commands A H2D --json "$out/rows.jsonl" > "$out/run.log" 2>&1 || true   # verdicts may be FAILURE
"$out/omp_con" nowait --verbose --repetitions 2 --globalsize_default_memory 50000 --commands C C >> "$out/run.log" 2>&1 || true
"$out/omp_con" nowait --commands HM >> "$out/run.log" 2>&1 || true      # usage errors exit 1 by design
"$out/omp_con" >> "$out/run.log" 2>&1 || true
if grep -E "ERROR: AddressSanitizer|runtime error:|LeakSanitizer" "$out/run.log"; then
  echo "sanitize_host: FAILED (see $out/run.log)"; exit 1
fi
# Optional (SANITIZE_CLI=1, needs nvcc + build/libhpcp.a, ~2 min): the --cpu plumbing paths of the three GPU CLIs under
# ThreadSanitizer (ranks are host threads there) and ASan/UBSan.
if [ "${SANITIZE_CLI:-0}" = 1 ]; then
  make -s build/libhpcp.a >/dev/null
  for san in thread "address,-fsanitize=undefined"; do
    tag=${san%%,*}
    for prog in miniapps/allreduce miniapps/halo p2p/peer2pear; do
      nvcc -ccbin $CXX -gencode arch=compute_90a,code=sm_90a -O1 -g -std=c++17 -Xcompiler -fopenmp,-fsanitize=$san \
           -Icsrc csrc/$prog.cu build/libhpcp.a -o "$out/$(basename $prog)_$tag" -lgomp
    done
    ASAN_OPTIONS=protect_shadow_gap=0 "$out/allreduce_$tag" --cpu -n 6 -p 14 >> "$out/cli.log" 2>&1
    ASAN_OPTIONS=protect_shadow_gap=0 "$out/allreduce_$tag" --cpu -a --type int -p 12 >> "$out/cli.log" 2>&1
    ASAN_OPTIONS=protect_shadow_gap=0 "$out/peer2pear_$tag" label --cpu -n 4 --bytes 1048576 >> "$out/cli.log" 2>&1
    ASAN_OPTIONS=protect_shadow_gap=0 "$out/halo_$tag" --cpu -n 5 --rows 3 --bytes 8192 --steps 6 --iters 2 >> "$out/cli.log" 2>&1
    ASAN_OPTIONS=protect_shadow_gap=0 "$out/halo_$tag" --cpu -n 3 --rows 1 --bytes 4096 --steps 5 --iters 2 --mode push >> "$out/cli.log" 2>&1
  done
  if grep -E "WARNING: ThreadSanitizer|ERROR: AddressSanitizer|runtime error:" "$out/cli.log"; then
    echo "sanitize_host: FAILED (see $out/cli.log)"; exit 1
  fi
fi
grep -c "^## " "$out/run.log" | xargs echo "sanitize_host: OK, verdict lines:"
