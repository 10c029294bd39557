// POD description of ONE kernel launch ("pass") of the engine: a set of FFT lines, how they are addressed
// in HBM on the way in and on the way out, and which pre/post operators are fused into the pass.
// Plain C so the host planner (g++), the CUDA kernels (nvcc) and the CPU emulation tests agree on it.
//
// Replaces the per-axis push-constant / specialization-constant state the reference keeps in
// VkFFTSpecializationConstantsLayout (vkFFT_Structs.h:719-1014) and the stride bookkeeping of
// VkFFTPlanAxis (vkFFT_Plan_FFT.h:252-417).
#pragma once
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
    B2_MAX_OUTER = 3,
};

// fused operators (bit flags)
enum {
    B2_OP_NONE = 0,
    B2_OP_TWIDDLE_OUT = 1,   // four-step phase  W_M^(line*elem) applied on store  (vkFFT_4step.h:31-119)
    B2_OP_SCALE = 2,         // multiply by `scale` on store (normalize=1, vkFFT_Structs.h:220)
    B2_OP_MUL_IN = 4,        // multiply element p by aux0[p] on load   (Bluestein chirp, vkFFT_Bluestein.h:32)
    B2_OP_MUL_OUT = 8,       // multiply element p by aux1[p] on store  (Bluestein filter / post chirp, :201)
    B2_OP_REAL_EVEN = 16,    // specialised kernels: even-length real transform fused into the pass -- forward: Hermitian
                             // post-pass on store (n+1 outputs), inverse: Hermitian pre-pass on load (n+1 inputs); aux0 = e^{-2 pi i k/2n}
    B2_OP_DCT23 = 32,        // specialised kernels: DCT-II (forward FFT: Makhoul gather on load, split + phase on store) or
                             // DCT-III (inverse FFT: phase + merge on load, Makhoul scatter on store); aux0 = e^{-i pi k/2n},
                             // aux_u0 = number of real lines.  Contiguous lines: a complex line is a pair of real lines, aux_u1 =
                             // their distance on the load side, aux_u2 on the store side (out of place the pitches differ)
    B2_OP_PERM_IN = 64,      // strided Four-Step first launch of a long DCT-II: rows are gathered through the Makhoul
                             // permutation of the FULL index p*N2 + n2 (aux_u0 = full length, aux_u1 = N2, n2 = coordinate tw_sel)
    B2_OP_BLUESTEIN = 256,   // specialised kernels: Bluestein launches on contiguous lines.  Forward kernel = first launch (zero-pad to n,
                             // chirp aux0 on load, filter aux1 on store); inverse kernel = second launch (chirp aux0 + truncation to
                             // out_len on store).  P.inverse selects the direction of the WHOLE transform at run time (outer re/im swap)
    B2_OP_CONV = 512,        // specialised kernels, contiguous lines: forward transform, product with the kernel line
                             // (aux0, data offset modulo aux_u0 = features x plane elements; aux_u1 = B2_CONV_* option bits of ew.cuh), inverse
                             // transform, all in one launch -- needs a schedule whose first and last radix agree
    B2_OP_BLUE_FUSED = 1024, // specialised kernels, contiguous lines: the WHOLE Bluestein transform of a line in one launch (stockham.cuh
                             // RMODE 11) -- zero-pad to n + chirp aux0 on load, forward stages, filter aux1 in registers, the stages again
                             // (inverse), chirp aux0 + scale + truncation to out_len on store.  One HBM read and one write of the N-point
                             // line, no scratch.  Needs a schedule whose first and last radix agree; P.inverse = direction at run time
    B2_OP_HALF_IN = 2048,    // the lines this pass READS are stored in half precision (32-bit complex elements, cplx.cuh); plain complex
    B2_OP_HALF_OUT = 4096,   // the lines it WRITES are                                   transforms, FP32 arithmetic, KCfg::ST
    B2_OP_PERM_OUT = 128,    // strided Four-Step last launch of a long DCT-III: result k1 + N1*p is scattered to row makhoul(k)
                             // (aux_u0 = full length, aux_u1 = N1, k1 = coordinate tw_sel)
};

// how the generic kernel fills a line on load / drains it on store (real-data transforms live here)
enum {
    B2_IO_C2C = 0,           // complex line as is (zero-filled beyond in_len / truncated at out_len)
    B2_IO_R2C_EVEN = 1,      // store: Hermitian post-pass of the even-length trick -> n+1 outputs (vkFFT_R2C_even_decomposition.h:181-230)
    B2_IO_C2R_EVEN = 2,      // load : inverse of the above from n+1 inputs
    B2_IO_DCT2 = 3,          // load : Makhoul even/odd permutation of two real lines (vkFFT_R2R.h:193-229); store: split + phase (:784-859)
    B2_IO_DCT3 = 4,          // the transpose of DCT2: phase + merge on load, inverse permutation on store
    B2_IO_DCT1 = 5,          // even extension to 2n-2 on load, real part on store (vkFFT_Scheduler.h:2271-2273)
    B2_IO_DCT4 = 6,          // pre/post phases around a half-length complex transform (vkFFT_Scheduler.h:2277-2280)
    B2_IO_REAL = 7,          // odd-length R2C/C2R fallback: real line <-> complex line with zero imaginary part
    B2_IO_HERM = 8,          // load only: rebuild the full spectrum from the Hermitian half (odd-length C2R)
    B2_IO_DST1 = 9,
    B2_IO_DCT4_ODD = 10,     // odd-length DCT-IV: pre-phase + zero-pad to 2N on load, post-phase + real part of the first N outputs on store          // odd extension to 2n+2 on load, -Im / Re on store (DST-I, API guide :581-583)
};

// DST-II/III/IV are the DCT operators with sign / index-reversal wrappers (vkFFT_R2R.h:769-780):
enum {
    B2_DST_NEG_ODD_IN = 1,   // multiply input sample n by (-1)^n
    B2_DST_REV_IN = 2,       // read input index N-1-n
    B2_DST_REV_OUT = 4,      // write output index N-1-k
    B2_DST_ALT_OUT = 8,      // multiply output k by (-1)^k
};

enum { B2_MAX_STAGES = 16 };

typedef struct b2_pass_params {
    const void* in;
    void* out;
    const void* lut;      // per-stage radix twiddles (complex T), layout documented in lut.h
    const void* tw_hi;    // two-level four-step table: W_M^(hi << tw_shift)
    const void* tw_lo;    // W_M^lo , lo < 2^tw_shift
    // auxiliary tables used by fused real-transform operators (R2C split, DCT phases, Bluestein chirps)
    const void* aux0;
    const void* aux1;

    int64_t in_es, out_es;                 // element stride inside a line (complex elements)
    int64_t in_gs, out_gs;                 // stride between neighbouring lines of the grouped dimension
    int64_t in_bs[B2_MAX_OUTER];           // strides of the outer (batch) dimensions
    int64_t out_bs[B2_MAX_OUTER];
    uint32_t nb[B2_MAX_OUTER];             // extents of the outer dimensions (>=1)
    uint32_t G;                            // number of lines along the grouped dimension
    uint32_t n;                            // FFT length of this pass
    uint32_t tw_shift;                     // log2(size of tw_lo)
    uint32_t tw_line0;                     // offset added to the line index before forming line*elem
    uint32_t ops;                          // B2_OP_* flags
    uint32_t inverse;                      // 1: swap re/im on load+store (inverse transform)
    uint32_t aux_u0, aux_u1;               // operator specific (e.g. logical real length)
    double scale;
    // ---- generic (runtime-scheduled) kernel only -------------------------------------------------------------
    uint32_t nstages;
    uint32_t radix[B2_MAX_STAGES];
    uint32_t tpl, q;                       // threads per line, lines per CTA (blockDim.x = tpl*q)
    uint32_t load_io, store_io;            // B2_IO_*
    uint32_t in_len, out_len;              // elements actually read / written per line (<= n, or n+1 for R2C)
    uint32_t load_qfast, store_qfast;      // 1: neighbouring lanes walk neighbouring lines (unit group stride)
    uint32_t line_stride;                  // smem elements between lines
    uint32_t inner_inverse;                // 1: the FFT inside this pass is an inverse one (swap around the stages only)
    uint32_t tw_sel;                       // which coordinate is the four-step "line": 0 group index, 1..3 outer dim 0..2
    uint32_t dst_flags;                    // B2_DST_* wrappers around the DCT operators
    uint32_t gen_flags;                    // B2_GEN_*: first stage reads its legs from HBM / last stage writes its outputs to HBM
    uint32_t aux_u2;                       // operator specific (B2_OP_DCT23 on contiguous lines: pair distance on the store side)
} b2_pass_params;

enum {
    B2_GEN_FUSE_IN = 1,
    B2_GEN_FUSE_OUT = 2,
};

// One launch of the fused Four-Step kernel (fused4.cuh): both passes of a two-factor split N = n1*n2 in ONE persistent
// launch.  Pass A (strided n1-point transforms + phase) writes into a small ring of scratch "units" that stays in L2,
// pass B (contiguous n2-point transforms, transposed store) consumes a unit as soon as all of its A tiles are done.
// The reference always runs the two uploads as separate dispatches with the whole intermediate going through DRAM
// (vkFFT_Scheduler.h:2582-2893, vkFFT_DispatchPlan.h:157-225).
typedef struct b2_fused_params {
    // TMA descriptor (CUtensorMap, 128 bytes, filled in by the runtime at launch) of pass A's input seen as a 2-D array of
    // floats: [sequences * n1 rows][2 * n2 floats]; a pass-A tile is a box of 2*Q_A floats x n1 rows of it
    unsigned long long tmap_a[16]
#if defined(__GNUC__) || defined(__CUDACC__)
        __attribute__((aligned(64)))
#endif
        ;
    b2_pass_params A, B;       // A.out / B.in = scratch ring base; their outer strides on the scratch side are ignored
    uint32_t* ctl;             // per group 64 words: [0] finished pass-A tiles, [32] finished pass-B tiles; zeroed before every launch
    uint32_t nseq;             // sequences = product of the outer extents (same for A and B)
    uint32_t U, NU;            // K = CTAs per group (planner), number of groups (launch: as many as are resident)
    uint32_t R;                // (unused)
    uint32_t TA, TB;           // tiles per SEQUENCE of pass A / pass B
    uint32_t reserved;
} b2_fused_params;

// One launch of the cluster Four-Step kernel (cluster4.cuh): both passes of N = n1*n2 with the intermediate in the distributed
// shared memory of one thread-block cluster per sequence.  A and B are the two passes of the two-launch plan; A.out and B.in
// (the scratch) are not touched.
typedef struct b2_cluster_params {
    b2_pass_params A, B;
    uint32_t nseq;             // sequences = product of the outer extents (same for A and B); one cluster each
} b2_cluster_params;

enum {
    B2_FCTL_MAX_GROUPS = 1024,
    B2_FCTL_WORDS = 64 * B2_FCTL_MAX_GROUPS,
};

#ifdef __cplusplus
}
#endif
