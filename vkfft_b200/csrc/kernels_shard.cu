// One translation unit per shard of kernel_list.def (compile with -DB2_SHARD=<k>).
#include "kernel_inst.cuh"

#ifndef B2_SHARD
#error "compile with -DB2_SHARD=<k>"
#endif

#include "kernel_list.def"
#include "kernel_list_nonpow2.def"
#include "kernel_list_blue1.def"
#include "kernel_list_fused.def"
#include "kernel_list_cluster.def"
