// Cluster Four-Step: both passes of N = n1 * n2 in ONE launch, one thread-block cluster per sequence, the intermediate in
// the cluster's distributed shared memory (DSMEM).  HBM sees every point once on the way in and once on the way out.
//
// The two-launch plan writes the whole intermediate to HBM and reads it back, which caps these sizes at 0.5 of the copy
// roofline; the L2 variant (fused4.cuh) exchanges tiles through an L2 ring and global counters.  Here a sequence of up to
// 1 MiB fits the shared memory of a cluster of CL CTAs, so the exchange is SM to SM inside the launch:
//   pass A   CTA r owns the columns b in [r*n2/CL, (r+1)*n2/CL).  Its TA thread groups (one per COLS tile of Q_A columns) read
//            them straight from HBM (first-stage legs, rows of Q_A*8 contiguous bytes), run the n1-point stages in their part
//            of the CTA's buffer, and keep the last-stage legs in registers.
//   barrier  every CTA holds its last-stage legs: from here on a peer may overwrite its buffer.
//            The last stage multiplies by the Four-Step phase and stores each output k1 into the buffer of the CTA that owns
//            row k1, in the padded row layout of pass B (st.shared::cluster).
//   barrier  every row is complete.
//   pass B   CTA r owns the rows k1 in [r*n1/CL, (r+1)*n1/CL); groups of its threads run the n2-point stages of Q_B rows at a
//            time, the first stage reading its legs from the buffer, and store X[k1 + n1*k2] to HBM (runs of Q_B points).
// No CTA touches a peer's memory after the second barrier, so a CTA may exit after pass B without a third one.  Each cluster
// reads all of its sequence before the first barrier and writes it only after the second: in-place execution needs no
// scratch.  Both passes run the stage code of the stand-alone kernels (Engine<C>: same radix schedules, LUTs, two-level phase
// table, scale placement), so the result is bit-identical to the two-launch plan with the same kernels.
#pragma once
#include "stockham.cuh"

namespace b200fft {

#if defined(__CUDA_ARCH__)
B2_D void cl_sync() {      // every thread of every CTA of the cluster; release / acquire: shared-memory stores are visible after it
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
B2_D uint32_t cl_smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
template <typename T>
B2_D void cl_store(uint32_t local_addr, uint32_t rank, const cpx<T>& v) {     // the same offset in CTA `rank`'s shared memory
    uint32_t a;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(local_addr), "r"(rank));
    if constexpr (sizeof(T) == 4) asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(v.x), "f"(v.y) : "memory");
    else asm volatile("st.shared::cluster.v2.f64 [%0], {%1, %2};" ::"r"(a), "d"(v.x), "d"(v.y) : "memory");
}
#elif defined(B2_EMU_CLUSTER)
B2_D void cl_sync() { b2emu::cluster_sync(); }
B2_D uint32_t cl_smem_addr(const void*) { return 0; }      // the emulation addresses a CTA's memory by byte offset
template <typename T>
B2_D void cl_store(uint32_t local_addr, uint32_t rank, const cpx<T>& v) { b2emu::dsmem_st(rank, local_addr, v); }
#elif defined(B2_EMU)
#error "cluster kernels run on the emulation with thread-block clusters only (B2_EMU_CLUSTER, cuda_emu_cluster.h)"
#else   // host pass of nvcc: device functions only
B2_D void cl_sync() {}
B2_D uint32_t cl_smem_addr(const void*) { return 0; }
template <typename T>
B2_D void cl_store(uint32_t, uint32_t, const cpx<T>&) {}
#endif

template <class CA, class CB, int CL>
struct Cluster4 {
    using T = typename CA::T;
    using X = cpx<T>;
    // strides known at compile time: pass A reads columns (element stride n2), pass B stores transposed (element stride n1)
    using EA = Engine<CA, XF_DSMEM_OUT, CB::N, CB::N>;
    using EB = Engine<CB, XF_SMEM_IN, 0, CA::N>;
    static constexpr int N1 = CA::N, N2 = CB::N;
    static constexpr int COLS = N2 / CL, ROWS = N1 / CL;          // pass-A columns / pass-B rows per CTA
    static constexpr int TA = COLS / CA::Q;                       // pass-A tiles per CTA, all transformed at once
    static constexpr int THREADS = TA * CA::THREADS;
    static constexpr int TB = ROWS / CB::Q;                       // pass-B tiles per CTA ...
    static constexpr int GB = THREADS / CB::THREADS;              // ... GB of them at a time
    static constexpr int TILE_A = CA::N * CA::Q;                  // elements of a pass-A tile (interleaved columns, no padding)
    static constexpr int ELEMS = (TA * TILE_A > ROWS * CB::LS) ? TA * TILE_A : ROWS * CB::LS;
    static constexpr int SMEM_BYTES = ELEMS * (int)sizeof(X);
    static_assert(CA::LAYOUT == LAY_ELEM && CB::LAYOUT == LAY_LINE, "pass A: interleaved columns, pass B: contiguous rows");
    static_assert(CA::V == 1 && CB::V == 1 && (CA::OPS & B2_OP_TWIDDLE_OUT) != 0 && CA::INV == CB::INV, "plain Four-Step pair");
    static_assert(N2 % CL == 0 && N1 % CL == 0 && COLS % CA::Q == 0 && ROWS % CB::Q == 0, "whole tiles per CTA");
    static_assert(THREADS % CB::THREADS == 0 && TB % GB == 0 && THREADS <= 1024, "pass B runs in whole rounds of the CTA's threads");

    B2_D static void seq_coords(const b2_pass_params& P, uint32_t seq, uint32_t& o0, uint32_t& o1, uint32_t& o2) {
        o0 = seq % P.nb[0]; seq /= P.nb[0];
        o1 = seq % P.nb[1]; seq /= P.nb[1];
        o2 = seq;
    }

    // pass A's last stage: output k1 of column `col` goes to row k1 % ROWS of CTA k1 / ROWS, position col of the padded row
    struct RowSink {
        uint32_t base;     // shared-window address of the buffer (the same in every CTA of the cluster)
        uint32_t pcol;     // col + pad(col)
        B2_D void operator()(int p, const X& v) const {
            const uint32_t idx = (uint32_t)(p % ROWS) * CB::LS + pcol;
            cl_store<T>(base + idx * (uint32_t)sizeof(X), (uint32_t)(p / ROWS), v);
        }
    };

    B2_D static void run(const b2_cluster_params& K, unsigned char* smem_raw) {
        X* sm = reinterpret_cast<X*>(smem_raw);
        const int tid = threadIdx.x;
        const uint32_t rank = blockIdx.x % CL, seq = blockIdx.x / CL;
        // ---- pass A: n1-point transforms of this CTA's columns; last-stage legs stay in registers ----
        {
            const b2_pass_params& P = K.A;
            uint32_t o0, o1, o2;
            seq_coords(P, seq, o0, o1, o2);
            const int64_t obase = (int64_t)o0 * P.in_bs[0] + (int64_t)o1 * P.in_bs[1] + (int64_t)o2 * P.in_bs[2];
            const X* __restrict__ lut = (const X*)P.lut;
            const int g = tid / CA::THREADS, lt = tid % CA::THREADS;
            X* sa = sm + (size_t)g * TILE_A;
            const uint32_t col0 = rank * COLS + g * CA::Q;
            using Sch = typename CA::Sch;
            int ql, tl;
            EA::template tmap<CA::LMAP>(lt, ql, tl);
            {
                X x[EA::template bpt<0>() * Sch::r(0)];
                EA::template load_global<0>(x, (const X*)P.in + obase + (int64_t)(col0 + ql) * P.in_gs, P.in_es, tl, true);
                EA::template compute<0>(x, lut, tl);
                EA::template store_smem<0>(x, sa, ql, tl);
            }
            __syncthreads();
            EA::template middle<1>(sa, lut, lt);
            constexpr int s = Sch::ns - 1;
            int qs, ts;
            EA::template tmap<CA::SMAP>(lt, qs, ts);
            X x[EA::template bpt<s>() * Sch::r(s)];
            EA::template load_smem<s>(x, sa, qs, ts);
            EA::template compute<s>(x, lut, ts);
            cl_sync();          // every CTA holds its last-stage legs: the buffers may be overwritten
            const uint32_t col = col0 + qs;
            EA::template store_global<s>(x, nullptr, 0, ts, true, P, EA::twl(P, col, o0, o1, o2), (uint32_t)qs,
                                         RowSink{cl_smem_addr(sm), col + (col >> CB::PAD_SHIFT)});
        }
        cl_sync();              // every row of every CTA is complete; no CTA touches a peer's memory after this point
        // ---- pass B: n2-point transforms of this CTA's rows, transposed store to HBM ----
        {
            const b2_pass_params& P = K.B;
            uint32_t o0, o1, o2;
            seq_coords(P, seq, o0, o1, o2);
            const int64_t obase = (int64_t)o0 * P.out_bs[0] + (int64_t)o1 * P.out_bs[1] + (int64_t)o2 * P.out_bs[2];
            const X* __restrict__ lut = (const X*)P.lut;
            const int lt = tid % CB::THREADS;
            using Sch = typename CB::Sch;
            constexpr int s = Sch::ns - 1;
            int ql, tl, qs, ts;
            EB::template tmap<CB::LMAP>(lt, ql, tl);
            EB::template tmap<CB::SMAP>(lt, qs, ts);
#pragma unroll 1
            for (int j = tid / CB::THREADS; j < TB; j += GB) {
                X* sb = sm + (size_t)j * CB::Q * CB::LS;
                {
                    X x[EB::template bpt<0>() * Sch::r(0)];
                    EB::template load_first_smem<0>(x, sb, ql, tl);
                    EB::template compute<0>(x, lut, tl);
                    __syncthreads();        // every first-stage read of the tile is done: the stages run in place
                    EB::template store_smem<0>(x, sb, ql, tl);
                }
                __syncthreads();
                EB::template middle<1>(sb, lut, lt);
                const uint32_t gs = rank * ROWS + j * CB::Q + qs;
                X x[EB::template bpt<s>() * Sch::r(s)];
                EB::template load_smem<s>(x, sb, qs, ts);
                EB::template compute<s>(x, lut, ts);
                EB::template store_global<s>(x, (X*)P.out + obase + (int64_t)gs * P.out_gs, P.out_es, ts, true, P,
                                             EB::twl(P, gs, o0, o1, o2), (uint32_t)qs);
            }
        }
    }
};

#if defined(__CUDACC__)
template <class CA, class CB, int CL, int MINB>
__global__ void __launch_bounds__(Cluster4<CA, CB, CL>::THREADS, MINB) cluster4_kernel(const __grid_constant__ b2_cluster_params K) {
    extern __shared__ __align__(128) unsigned char b2_smem_cluster[];
    Cluster4<CA, CB, CL>::run(K, b2_smem_cluster);
}
#endif

}  // namespace b200fft
