#!/bin/sh
# Build the CPU emulation with thread-block clusters (tests only): the kernel lists of build.sh plus the cluster Four-Step
# kernels, on cuda_emu_cluster.h (-DB2_EMU_CLUSTER).  The kernel lists are split over 8 translation units.
set -e
here="$(cd "$(dirname "$0")" && pwd)"
root="$(cd "$here/../.." && pwd)"
mkdir -p "$here/_build"
FLAGS="-std=c++20 -O1 -fPIC -pthread -DB2_EMU -DB2_EMU_CLUSTER -DB2_SHARD=-1 -DB2_EMU_PARTS=8 -I$root/vkfft_b200/csrc -I$here"
pids=""
for p in 0 1 2 3 4 5 6 7; do
  g++ $FLAGS -DB2_EMU_PART=$p -c "$here/emu_cluster_kernels.cpp" -o "$here/_build/emu_cluster_kernels_$p.o" &
  pids="$pids $!"
done
g++ $FLAGS -DB2_EMU_PART=99 -c "$here/emu_cluster_driver.cpp" -o "$here/_build/emu_cluster_driver.o" &
pids="$pids $!"
for pid in $pids; do wait $pid; done
g++ -shared -pthread -o "$here/_build/libb200fft_emu_cluster.so" "$here"/_build/emu_cluster_kernels_*.o "$here/_build/emu_cluster_driver.o" \
    "$root/vkfft_b200/csrc/kernel_registry.cpp" "$root/vkfft_b200/csrc/planner.cpp" -std=c++20 -fPIC -I"$root/vkfft_b200/csrc" -I"$root/include"
