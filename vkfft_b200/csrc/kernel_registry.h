// Registry of kernel instantiations.  The planner looks kernels up by (kind, precision, length, direction, fused-operator
// set).  The hot path -- powers of two, the curated lengths, every Four-Step factor of the BASELINE configurations -- is
// compiled ahead of time for sm_90a.  A length that is 2..31-smooth but not in the ahead-of-time lists gets the SAME
// hand-written templates (stockham.cuh) instantiated for it when its plan is created (jit.cpp, NVRTC -> cubin; the product
// library only) instead of falling back to the runtime-scheduled kernel, which is 3-5x slower.  The reference compiles every
// kernel of every plan that way (vkFFT_CompileKernel.h:299-491); here it is the exception, and B200FFT_NO_JIT=1 turns it off.
#pragma once
#include "pass_params.h"

#ifdef __cplusplus
extern "C" {
#endif

enum {
    B2_KIND_ROWS = 0,       // lines contiguous in HBM on both sides
    B2_KIND_ROWS_TOUT = 1,  // contiguous lines in, neighbouring lines interleaved on the way out (four-step final pass)
    B2_KIND_COLS = 2,       // neighbouring lines interleaved (strided axis / four-step first pass)
    B2_KIND_GENERIC = 3,    // runtime-scheduled kernel (generic.cuh): n = 0 in the registry, any addressing
    B2_KIND_ELEMENTWISE = 4,// elementwise helper passes (ew.cuh)
    B2_KIND_COUNT
};
enum { B2_PREC_F32 = 0, B2_PREC_F64 = 1 };

typedef struct b2_kernel_info {
    int kind, prec, n, inv, ops;       // lookup key
    int variant;                       // 0 = default; further CTA shapes / schedules for the same key (tuning)
    int pipelined;                     // 1: persistent TMA-fed kernel (pipe.cuh): input pointer and line pitch must be 16-byte aligned
    int threads, q, tpl, v, smem_bytes;
    int ns;
    int radices[8];
    int lut_size;                      // complex entries of the stage-twiddle LUT
    // enqueue `grid` CTAs on `stream` (cudaStream_t); returns cudaError_t as int
    int (*launch)(const b2_pass_params* P, unsigned grid, void* stream);
    int (*prepare)(void);              // one-time cudaFuncSetAttribute (max dynamic smem)
    const char* name;
    int regs;                          // register budget per thread the kernel was compiled with (0 = not recorded)
    void* jit;                         // != 0: instantiated at plan time (jit.cpp); launch / prepare are null, use b2_jit_prepare / b2_jit_launch
} b2_kernel_info;

// plan-time instantiation (jit.cpp installs the provider in the product library; absent in the CPU emulation): asked on a
// registry miss, returns a kernel description (not compiled yet) or null when the key is not eligible
typedef const b2_kernel_info* (*b2_kernel_provider)(int kind, int prec, int n, int inv, int ops);
void b2_set_kernel_provider(b2_kernel_provider p);
// jit.cpp (product library only): compile + load the kernel behind a plan-time description / enqueue it
int b2_jit_prepare(const b2_kernel_info* k);
void b2_jit_disable(const b2_kernel_info* k);   // after a failed prepare: stop offering the key (the plan is rebuilt without it)
int b2_jit_launch(const b2_kernel_info* k, const b2_pass_params* P, unsigned grid, void* stream);
long b2_jit_selftest(int kind, int prec, int n, int ops);   // no GPU needed: cubin size, 0 = not eligible, < 0 = compile error
const char* b2_jit_last_log(void);
int b2_jit_available(void);

void b2_register_kernel(const b2_kernel_info* k);
const b2_kernel_info* b2_find_kernel(int kind, int prec, int n, int inv, int ops);   // honours B200FFT_VARIANTS
const b2_kernel_info* b2_find_kernel_variant(int kind, int prec, int n, int inv, int ops, int variant);
int b2_kernel_count(void);
const b2_kernel_info* b2_kernel_at(int i);

// fused Four-Step kernels (fused4.cuh): both passes of n1 x n2 in one persistent launch
typedef struct b2_fused_info {
    int prec, n1, n2, inv;             // lookup key
    int variant;
    int threads, qa, qb, smem_bytes;   // CTA shape, columns per pass-A tile, rows per pass-B tile
    int regs;                          // register budget per thread (bounds the resident CTAs per SM)
    int ns_a, ns_b;
    int radices_a[8], radices_b[8];
    // enqueue the control-block reset + the persistent kernel (at most max_ctas CTAs; 0 = as many as are resident)
    int (*launch)(const b2_fused_params* F, unsigned max_ctas, void* stream);
    int (*prepare)(void);
    const char* name;
} b2_fused_info;
void b2_register_fused(const b2_fused_info* k);
const b2_fused_info* b2_find_fused(int prec, int n1, int n2, int inv);
const b2_fused_info* b2_find_fused_variant(int prec, int n1, int n2, int inv, int variant);
int b2_fused_count(void);
const b2_fused_info* b2_fused_at(int i);

// cluster Four-Step kernels (cluster4.cuh): both passes of n1 x n2 in one launch, one thread-block cluster per sequence
typedef struct b2_cluster_info {
    int prec, n1, n2, inv;             // lookup key
    int variant;
    int cluster, threads, smem_bytes;  // CTAs per cluster, threads per CTA, dynamic shared memory per CTA
    int tpl_a, q_a, tpl_b, q_b;        // CTA shapes of the stand-alone kernels whose stage code the two passes run
    int ns_a, ns_b;
    int radices_a[8], radices_b[8];
    int (*launch)(const b2_cluster_params* K, void* stream);
    int (*prepare)(void);
    // clusters of this kernel the device can hold at once (cudaOccupancyMaxActiveClusters, once per device); 0: cannot run
    int (*max_active)(int device);
    const char* name;
} b2_cluster_info;
void b2_register_cluster(const b2_cluster_info* k);
const b2_cluster_info* b2_find_cluster(int prec, int n1, int n2, int inv);   // honours B200FFT_CLUSTER4_VARIANTS
int b2_cluster_count(void);
const b2_cluster_info* b2_cluster_at(int i);

#ifdef __cplusplus
}
#endif
