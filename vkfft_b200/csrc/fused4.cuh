// Fused Four-Step: both passes of N = n1 * n2 in ONE persistent launch, the intermediate kept in L2.
//
// The reference (and this engine's two-launch plan) writes the whole intermediate to DRAM in the first dispatch and
// reads it back in the second (vkFFT_Scheduler.h:2582-2893: "numAxisUploads = 2"), i.e. two HBM round trips, which caps
// those sizes at 0.5 of the copy roofline.  Here:
//   * sequences are grouped into UNITS; the scratch is a ring of R units (a few MB ... tens of MB, below the H100's 50 MB
//     L2), rewritten over and over, so it lives in L2: pass A's stores and pass B's loads never reach HBM;
//   * persistent CTAs take TILES from two ordered queues.  A tile of pass A (Q_A neighbouring columns of one sequence:
//     strided n1-point transforms + the Four-Step phase) may be taken when its unit's ring slot is free; a tile of pass B
//     (Q_B rows: contiguous n2-point transforms, transposed store to the final place) when ALL A tiles of its unit are
//     done.  The schedule is static: groups of K CTAs own whole sequences and two private scratch slots each and walk them
//     in phases (pass B of the previous sequence, then pass A of the next), synchronised by two tile counters per group;
//     every CTA knows its tile list in advance, so the next tile is always being copied in by TMA while the current one is
//     transformed, and the counter traffic rides behind the first butterflies of the following tile;
//   * pass B reads the scratch with ld.global.cg (it was written by other SMs in this launch) and, once the legs are in
//     registers, drops the lines from L2 (discard.global.L2) so that dead scratch is never written back to HBM.
// Both passes run the very same stage code as the stand-alone kernels (Engine<C>::run_at), so results are identical
// to the two-launch plan bit for bit.
#pragma once
#include "stockham.cuh"
#include "pipe.cuh"

namespace b200fft {

// Memory ordering of the tile protocol.  Producers: the CTA's stores, bar.sync, then thread 0 bumps the unit's done-counter
// with RELEASE semantics (one MEMBAR.GPU per tile: the tile's stores / discards are performed at L2 before the count
// moves).  Consumers: every claim word is read and updated with RELAXED operations at L2 (no fence, no L1 flush --
// an acquire here would put a MEMBAR + CCTL.IVALL on the per-tile path and throw the twiddle tables out of L1), and
// the data itself is then read with ld.global.cg, i.e. from L2, where the producer's fence has already put it; the
// addresses depend on the claimed ticket, so the loads cannot be issued early.  Only the once-per-unit prefix advance
// uses acquire loads.
#if defined(__CUDA_ARCH__)
B2_D uint32_t fz_ld_acquire(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
B2_D uint32_t fz_ld_relaxed(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
B2_D uint32_t fz_add(uint32_t* p, uint32_t v) {       // relaxed fetch-add
    uint32_t o;
    asm volatile("atom.relaxed.gpu.global.add.u32 %0, [%1], %2;" : "=r"(o) : "l"(p), "r"(v) : "memory");
    return o;
}
B2_D uint32_t fz_add_release(uint32_t* p, uint32_t v) {
    uint32_t o;
    asm volatile("atom.release.gpu.global.add.u32 %0, [%1], %2;" : "=r"(o) : "l"(p), "r"(v) : "memory");
    return o;
}
B2_D uint32_t fz_cas(uint32_t* p, uint32_t cmp, uint32_t val) {
    uint32_t o;
    asm volatile("atom.relaxed.gpu.global.cas.b32 %0, [%1], %2, %3;" : "=r"(o) : "l"(p), "r"(cmp), "r"(val) : "memory");
    return o;
}
B2_D uint32_t fz_cas_release(uint32_t* p, uint32_t cmp, uint32_t val) {
    uint32_t o;
    asm volatile("atom.release.gpu.global.cas.b32 %0, [%1], %2, %3;" : "=r"(o) : "l"(p), "r"(cmp), "r"(val) : "memory");
    return o;
}
B2_D void fz_sleep(unsigned ns) { __nanosleep(ns); }
#else
// CPU emulation: one CTA at a time, only thread 0 touches the control words
B2_D uint32_t fz_ld_acquire(const uint32_t* p) { return *p; }
B2_D uint32_t fz_ld_relaxed(const uint32_t* p) { return *p; }
B2_D uint32_t fz_add(uint32_t* p, uint32_t v) { uint32_t o = *p; *p = o + v; return o; }
B2_D uint32_t fz_add_release(uint32_t* p, uint32_t v) { return fz_add(p, v); }
B2_D uint32_t fz_cas(uint32_t* p, uint32_t cmp, uint32_t val) { uint32_t o = *p; if (o == cmp) *p = val; return o; }
B2_D uint32_t fz_cas_release(uint32_t* p, uint32_t cmp, uint32_t val) { return fz_cas(p, cmp, val); }
B2_D void fz_sleep(unsigned) {}
#endif

// NBUF: tile buffers per CTA.  2: the NEXT tile is copied into the other buffer by TMA while this one is transformed;
// 1 (tiles too large to double): the next tile is copied into the same buffer as soon as the last stage has its legs in
// registers, i.e. it overlaps the last butterflies and the global stores.
#if defined(__CUDA_ARCH__)
// 2-D tensor copy global -> shared (TMA, SASS UTMALDG): box of the tensor map at element coordinates (c0, c1)
B2_D void tma_load_2d(void* dst, const void* tmap, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                     smem_u32(dst)),
                 "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar))
                 : "memory");
}
#endif

template <class CA, class CB, int NBUF = 2>
struct Fused4 {
    // strides known at compile time: pass A walks columns of an n1 x n2 matrix (element stride n2 on both sides), pass B
    // stores transposed (element stride n1)
    using EA = Engine<CA, 0, CB::N, CB::N>;
    using EB = Engine<CB, XF_LDCG | XF_DISCARD, 0, CA::N>;
    using T = typename CA::T;
    using X = cpx<T>;
    static_assert(CA::THREADS == CB::THREADS, "both passes run in the same CTA shape");
    static_assert(CA::LAYOUT == LAY_ELEM && CB::LAYOUT == LAY_LINE, "pass A: interleaved columns, pass B: contiguous rows");
    static_assert(CA::V == 1 && CB::V == 1, "one butterfly per thread and step");
    static_assert(NBUF == 1 || NBUF == 2, "one or two tile buffers");
    static constexpr int THREADS = CA::THREADS;
    static constexpr int MINB = CA::MINB < CB::MINB ? CA::MINB : CB::MINB;
    static constexpr int TILE_BYTES = ((CA::SMEM_BYTES > CB::SMEM_BYTES ? CA::SMEM_BYTES : CB::SMEM_BYTES) + 127) / 128 * 128;
    static constexpr int SMEM_BYTES = NBUF * TILE_BYTES + 64;     // + two mbarriers + mailbox: two slots of (kind, unit, tile)
    static constexpr uint32_t BYTES_A = (uint32_t)(CA::N * CA::Q * sizeof(X)), BYTES_B = (uint32_t)(CB::N * CB::Q * sizeof(X));
    static constexpr int BOX_ROWS = CA::N < 256 ? CA::N : 256;      // rows per TMA box (hardware limit 256 per dimension)
    enum { NONE = 0, TILE_A = 1, TILE_B = 2 };

    // ---- schedule: static, per GROUP of K CTAs -------------------------------------------------------------------------------
    // The resident CTAs are split into groups of K (F.U); group g owns the sequences g, g+NG, g+2NG, ... and a private pair
    // of scratch slots, and walks them in phases:
    //      phase j :  pass-B tiles of its (j-1)-th sequence (slot (j-1)&1)   then   pass-A tiles of its j-th sequence (slot j&1)
    // CTA r of the group takes tiles r, r+K, ... of each part, so every CTA knows its whole tile list in advance (the TMA
    // copy of the next tile can always be started early) and nothing is handed out at run time.  Two counters per group
    // count finished tiles:
    //      a pass-B tile of phase j may start when  cntA >= TA*j      (every pass-A tile of that sequence is done)
    //      a pass-A tile of phase j may start when  cntB >= TB*(j-1)  (the slot it overwrites has been read completely)
    // Both conditions refer to work that ended at least half a phase earlier, so CTAs rarely wait; the scratch of all groups
    // together is 2 * NG sequences (tens of MB at most: K is chosen by the planner so that it stays far below the L2 size)
    // and is rewritten in place for the whole launch, so it never leaves L2.  (Three dynamic schedulers -- semaphores,
    // reserved tickets, one ordered queue -- were measured first: every ticket a CTA holds ahead of its work widens the
    // window of units that must stay resident and the CTAs ended up waiting for each other.)
    // The counter updates of a tile (one MEMBAR.GPU + one atomic) and the refresh of the two counters are issued behind the
    // NEXT tile's first butterflies and only looked at after its last store: no memory round trip on the tile path.
    struct Sched {
        uint32_t cntA, cntB;           // last values read of the group's counters
        uint32_t pend_kind;            // finished tile whose completion has not been published yet
    };
    struct Tile { uint32_t kind, m, t; };      // pass, ordinal of the sequence within the group, tile within the sequence

    B2_D static uint32_t* counters(const b2_fused_params& F) { return F.ctl + (size_t)(blockIdx.x / F.U) * 64; }
    B2_D static uint32_t nseq_of_group(const b2_fused_params& F) {
        const uint32_t g = blockIdx.x / F.U;
        return g < F.nseq ? (F.nseq - g + F.NU - 1) / F.NU : 0u;
    }
    // the CTA's next tile after `c` (c.kind == NONE: its first one)
    B2_D static Tile advance(const b2_fused_params& F, Tile c, uint32_t P) {
        const uint32_t K = F.U, r = blockIdx.x % K;
        uint32_t j, part, t;                    // phase, part (0: B of sequence j-1, 1: A of sequence j), tile
        if (c.kind == NONE) { j = 0; part = 0; t = r; }
        else { part = c.kind == TILE_B ? 0u : 1u; j = part ? c.m : c.m + 1; t = c.t + K; }
        for (;;) {
            if (j > P) return Tile{NONE, 0, 0};
            if (part == 0) {
                if (j >= 1 && t < F.TB) return Tile{TILE_B, j - 1, t};
                part = 1; t = r;
            } else {
                if (j < P && t < F.TA) return Tile{TILE_A, j, t};
                part = 0; t = r; ++j;
            }
        }
    }
    B2_D static bool runnable(const b2_fused_params& F, const Sched& S, const Tile& c) {
        if (F.B.aux_u1 & 2u) return true;      // tuning switch: ignore the dependencies (wrong results, upper bound of the tile pipeline)
        if (c.kind == TILE_B) return S.cntA >= F.TA * (c.m + 1);
        return c.m < 2 || S.cntB >= F.TB * (c.m - 1);
    }
    B2_D static void publish(const b2_fused_params& F, Sched& S) {      // release the pending tile (if any)
        if (S.pend_kind != NONE) {
            fz_add_release(counters(F) + (S.pend_kind == TILE_B ? 32 : 0), 1u);
            S.pend_kind = NONE;
        }
    }
    // scheduler traffic of one tile, issued by thread 0 while the tile's first-stage legs are being read
    B2_D static void sched_issue(const b2_fused_params& F, Sched& S) {
        S.cntA = fz_ld_relaxed(counters(F));
        S.cntB = fz_ld_relaxed(counters(F) + 32);
        publish(F, S);
    }

    B2_D static void seq_coords(const b2_pass_params& P, uint32_t seq, uint32_t& o0, uint32_t& o1, uint32_t& o2) {
        o0 = seq % P.nb[0]; seq /= P.nb[0];
        o1 = seq % P.nb[1]; seq /= P.nb[1];
        o2 = seq;
    }
    struct Where { uint32_t grp, seq, o0, o1, o2; int64_t obase_in, obase_out; };
    B2_D static Where locate(const b2_fused_params& F, const Tile& c) {
        constexpr uint64_t NN = (uint64_t)CA::N * (uint64_t)CB::N;              // points per sequence
        const uint32_t g = blockIdx.x / F.U;
        const int64_t slot = (int64_t)(((uint64_t)g * 2 + (c.m & 1u)) * NN);  // this group's scratch slot of that sequence
        Where w;
        w.grp = c.t;
        w.seq = g + F.NU * c.m;
        if (c.kind == TILE_A) {
            seq_coords(F.A, w.seq, w.o0, w.o1, w.o2);
            w.obase_in = (int64_t)w.o0 * F.A.in_bs[0] + (int64_t)w.o1 * F.A.in_bs[1] + (int64_t)w.o2 * F.A.in_bs[2];
            w.obase_out = slot;
        } else {
            seq_coords(F.B, w.seq, w.o0, w.o1, w.o2);
            w.obase_in = slot;
            w.obase_out = (int64_t)w.o0 * F.B.out_bs[0] + (int64_t)w.o1 * F.B.out_bs[1] + (int64_t)w.o2 * F.B.out_bs[2];
        }
        return w;
    }

    // ---- TMA: copy a tile into a shared-memory buffer; completion on the buffer's mbarrier ------------------------------------
    //   pass A: Q_A neighbouring columns = n1 row segments of Q_A*8 bytes, n2*8 bytes apart -> buf[p*Q_A + q]  (the
    //           interleaved-line layout the stages use, so they run in place); the 32 lanes of warp 0 share the row copies
    //   pass B: Q_B contiguous rows of the scratch = ONE contiguous block                   -> buf[q*n2 + p]  (dense; the
    //           first scatter moves it to the padded layout)
    // Called by every lane of warp 0 (emulation: by thread 0 alone); the arguments are taken from lane 0.
    B2_D static void warp_issue(const b2_fused_params& F, bool go, Tile c, X* buf, uint64_t* bar) {
#if defined(__CUDA_ARCH__)
        const int lane = threadIdx.x & 31, nlanes = 32;
        go = __shfl_sync(0xffffffffu, go ? 1 : 0, 0) != 0;
        c.kind = __shfl_sync(0xffffffffu, c.kind, 0); c.m = __shfl_sync(0xffffffffu, c.m, 0); c.t = __shfl_sync(0xffffffffu, c.t, 0);
#else
        const int lane = 0, nlanes = 1;
#endif
        if (!go) return;
        const Where w = locate(F, c);
        if (c.kind == TILE_A) {
#if defined(__CUDA_ARCH__)
            // one tensor copy per box of up to 256 rows: the TMA unit walks the rows (row-by-row bulk copies cost ~50 cycles
            // of the unit each and made the launch several times slower)
            if (lane == 0) {
                mbar_expect_tx(bar, BYTES_A);
#pragma unroll
                for (int r0 = 0; r0 < CA::N; r0 += BOX_ROWS)
                    tma_load_2d(buf + (size_t)r0 * CA::Q, &F.tmap_a, (int)(2 * w.grp * CA::Q), (int)(w.seq * CA::N + r0), bar);
            }
            (void)nlanes;
#else
            if (lane == 0) mbar_expect_tx(bar, BYTES_A);
            const X* src = (const X*)F.A.in + w.obase_in + (int64_t)w.grp * CA::Q * F.A.in_gs;
            for (int p = lane; p < CA::N; p += nlanes)
                tma_load_1d(buf + (size_t)p * CA::Q, src + (int64_t)p * CB::N, (uint32_t)(CA::Q * sizeof(X)), bar);
#endif
        } else if (lane == 0) {
            mbar_expect_tx(bar, BYTES_B);
            const X* src = (const X*)F.B.in + w.obase_in + (int64_t)w.grp * CB::Q * CB::N;
            tma_load_1d(buf, src, BYTES_B, bar);
        }
    }
    // thread 0: hold back nothing, then wait until the tile may run (the slow path: its sequence was not ready when looked at)
    B2_D static void wait_runnable(const b2_fused_params& F, Sched& S, const Tile& c) {
        publish(F, S);
        for (;;) {
            S.cntA = fz_ld_relaxed(counters(F));
            S.cntB = fz_ld_relaxed(counters(F) + 32);
            if (runnable(F, S, c)) return;
            fz_sleep(100);
        }
    }

    // first-stage legs from the tile as TMA delivered it
    template <class E, class C>
    B2_D static void load_raw(X* x, const X* sm, int q, int t) {
        using Sch = typename C::Sch;
        constexpr int r = Sch::r(0), NB = C::N / r, BPT = E::template bpt<0>();
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
            const int b = t + m * C::TPL;
            if (E::template guarded<0>() && b >= NB) continue;
#pragma unroll
            for (int k = 0; k < r; ++k) {
                const int p = b + k * NB;
                X a = B2_SMEM_LD(sm, C::LAYOUT == LAY_ELEM ? p * C::Q + q : q * C::N + p);
                x[m * r + k] = C::INV ? swp(a) : a;
            }
        }
    }

    // one tile of pass `C` from buffer `sm`.  `on_dead` runs (thread 0 .. 31) once every thread has read its last-stage legs
    template <class E, class C, class Dead>
    B2_D static void process(const b2_fused_params& F, const b2_pass_params& P, X* sm, const Where& w, Sched& S, bool discard, Dead on_dead) {
        using Sch = typename C::Sch;
        constexpr int NS = Sch::ns;
        const int tid = threadIdx.x;
        const X* __restrict__ lut = (const X*)P.lut;
        int ql, tl;
        E::template tmap<C::LMAP>(tid, ql, tl);
        {
            X x[E::template bpt<0>() * Sch::r(0)];
            load_raw<E, C>(x, sm, ql, tl);
            if (tid == 0) sched_issue(F, S);         // atomics + limit loads in flight behind the first butterflies
            E::template compute<0>(x, lut, tl);
            __syncthreads();                         // every raw read of the buffer is done: switch to the stage layout
            if constexpr (C::LAYOUT == LAY_LINE) { if (discard) E::discard_tile(P, w.obase_in, w.grp, tid); }   // pass B: the scratch lines are dead in L2 as well
            E::template store_smem<0>(x, sm, ql, tl);
        }
        __syncthreads();
        E::template middle<1>(sm, lut, tid);
        {
            constexpr int s = NS - 1;
            int qs, ts;
            E::template tmap<C::SMAP>(tid, qs, ts);
            const uint32_t gs = w.grp * C::Q + qs;
            X x[E::template bpt<s>() * Sch::r(s)];
            E::template load_smem<s>(x, sm, qs, ts);
            if constexpr (NBUF == 1) {
                fence_proxy_async_smem();
                __syncthreads();                     // the buffer is dead: refill it while the last stage runs
                on_dead();
            }
            E::template compute<s>(x, lut, ts);
            X* out_line = (X*)P.out + w.obase_out + (int64_t)gs * P.out_gs;
            E::template store_global<s>(x, out_line, P.out_es, ts, gs < P.G, P, E::twl(P, gs, w.o0, w.o1, w.o2), (uint32_t)qs);
        }
    }

    B2_D static void run(const b2_fused_params& F, unsigned char* smem_raw) {
        uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + (size_t)NBUF * TILE_BYTES);
        volatile uint32_t* mail = reinterpret_cast<volatile uint32_t*>(smem_raw + (size_t)NBUF * TILE_BYTES + 16);   // [slot][kind, m, t]
        const int tid = threadIdx.x;
#if defined(__CUDA_ARCH__)
        const bool w0 = tid < 32;                    // warp 0 issues the copies
#else
        const bool w0 = tid == 0;
#endif
        auto bufp = [&](uint32_t i) { return reinterpret_cast<X*>(smem_raw + (size_t)(i % NBUF) * TILE_BYTES); };
        const uint32_t P = nseq_of_group(F);
        Sched S;
        S.cntA = S.cntB = 0; S.pend_kind = NONE;
        // thread 0: the tile being transformed and the one after it (whose copy may already be running)
        Tile cur{NONE, 0, 0}, nxt{NONE, 0, 0};
        bool cissued = false, nissued = false;
        if (tid == 0) {
            for (int i = 0; i < NBUF; ++i) mbar_init(&bars[i], 1);
            mbar_init_fence();
            cur = advance(F, Tile{NONE, 0, 0}, P);
            nxt = cur.kind != NONE ? advance(F, cur, P) : cur;
            mail[0] = cur.kind; mail[1] = cur.m; mail[2] = cur.t;
            if (cur.kind != NONE) wait_runnable(F, S, cur);
        }
        __syncthreads();                             // mbarriers initialised, mailbox written
        if (w0) { warp_issue(F, cur.kind != NONE, cur, bufp(0), &bars[0]); cissued = true; }
        for (uint32_t it = 0;; ++it) {
            const uint32_t slot = it & 1u;
            const Tile c{mail[3 * slot], mail[3 * slot + 1], mail[3 * slot + 2]};
            if (c.kind == NONE) break;
            X* sm = bufp(it);
            uint64_t* bar = &bars[it % NBUF];
            if (w0) {
                // this tile's copy could not be started ahead (its sequence was not ready): wait for it now
                if (tid == 0 && !cissued) wait_runnable(F, S, cur);
                warp_issue(F, !cissued, cur, sm, bar);
                cissued = true;
                if constexpr (NBUF == 2) {           // the other buffer is free: start the next tile's copy if it may run
                    const bool go = nxt.kind != NONE && runnable(F, S, nxt);
                    warp_issue(F, go, nxt, bufp(it + 1), &bars[(it + 1) % NBUF]);
                    nissued = go;
                }
            }
            mbar_wait(bar, (it / NBUF) & 1u);
            const Where w = locate(F, c);
            auto dead = [&]() {                      // one buffer: refill it as soon as the last stage has its legs
                if (w0) {
                    const bool go = nxt.kind != NONE && runnable(F, S, nxt);
                    warp_issue(F, go, nxt, sm, bar);
                    nissued = go;
                }
            };
            if (c.kind == TILE_A) process<EA, CA>(F, F.A, sm, w, S, false, dead);
            else process<EB, CB>(F, F.B, sm, w, S, !(F.B.aux_u1 & 1u), dead);
            if (tid == 0) {
                S.pend_kind = c.kind;                // published behind the next tile's first stage (or on the wait / exit path)
                volatile uint32_t* m = mail + 3 * (slot ^ 1);
                m[0] = nxt.kind; m[1] = nxt.m; m[2] = nxt.t;
                cur = nxt; cissued = nissued;
                nxt = cur.kind != NONE ? advance(F, cur, P) : cur;
                nissued = false;
            }
            fence_proxy_async_smem();
            __syncthreads();      // stores issued; this buffer may be refilled; the next mailbox slot is visible
        }
        if (tid == 0) publish(F, S);
    }
};

#if defined(__CUDACC__)
template <class CA, class CB, int NBUF>
__global__ void __launch_bounds__(CA::THREADS, Fused4<CA, CB, NBUF>::MINB) fused4_kernel(const __grid_constant__ b2_fused_params F) {
    extern __shared__ __align__(128) unsigned char b2_smem_fused[];
    Fused4<CA, CB, NBUF>::run(F, b2_smem_fused);
}
// control block: ticket counters, unit prefixes and per-unit done counters all start at zero
template <int DUMMY = 0>
__global__ void fused4_init_kernel(uint32_t* ctl, uint32_t words) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < words; i += gridDim.x * blockDim.x) ctl[i] = 0u;
}
#endif

}  // namespace b200fft
