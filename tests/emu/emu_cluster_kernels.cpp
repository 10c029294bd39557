// TEST INFRASTRUCTURE ONLY: the kernel lists of emu_kernels.cpp plus the cluster Four-Step kernels, for the emulation with
// thread-block clusters (cuda_emu_cluster.h, built by build_cluster.sh with -DB2_EMU_CLUSTER).
#include "emu_kernels.cpp"
#include "kernel_list_cluster.def"
