// Compile-time specialised Stockham autosort FFT: one CTA transforms Q lines of length N that live in
// shared memory between radix stages; first-stage legs come straight from HBM into registers and the
// last stage stores straight from registers (one HBM read + one HBM write per element).
//
// Algorithm (what the reference's generated VkFFT_main does, vkFFT_FFT.h:97-239 / vkFFT_RadixStage.h:35):
//   stage s has radix r and stageSize S = prod(previous radices); butterfly b in [0, N/r), j = b mod S:
//     leg k  = x[b + k*N/r] * W_{S*r}^{j*k}          (DIT twiddle before the butterfly)
//     y[(b-j)*r + j + k*S] = DFT_r(legs)[k]           (autosort scatter, vkFFT_RadixShuffle.h:34)
//   so the output of the last stage is in natural order with no bit reversal.
// What is different from the reference: twiddles are correctly-rounded LUT entries (never __sincosf),
// thread<->line mapping can differ between the load side and the store side (so the four-step transposed
// write is coalesced), all shapes are template constants (compiled ahead of time for sm_90a; lengths outside those lists get
// the same templates instantiated when their plan is created, jit.cpp -- there is no code GENERATOR), and the
// inverse transform is the forward code with re/im swapped at the HBM boundary.
#pragma once
#include <math.h>

#include "pass_params.h"
#include "radix.cuh"

#if defined(B2_EMU_CLUSTER)
#include "cuda_emu_cluster.h"       // the emulation with thread-block clusters (tests/emu/build_cluster.sh)
#elif defined(B2_EMU)
#include "cuda_emu.h"
#else
#define B2_SMEM_LD(sm, i) ((sm)[(i)])
#define B2_SMEM_ST(sm, i, v) ((sm)[(i)] = (v))
#endif

namespace b200fft {

// ------------------------------------------------------------------------------------------------
// radix schedule
template <int... Rs>
struct RList {
    static constexpr int ns = sizeof...(Rs);
    B2_HD static constexpr int r(int s) {
        const int a[] = {Rs...};
        return a[s];
    }
    B2_HD static constexpr int S(int s) {  // stage size before stage s
        int p = 1;
        for (int i = 0; i < s; ++i) p *= r(i);
        return p;
    }
    static constexpr int N = (Rs * ... * 1);
    B2_HD static constexpr int lut_off(int s) {  // offset of stage s in the stage-twiddle LUT
        int o = 0;
        for (int i = 1; i < s; ++i) o += (r(i) - 1) * S(i);
        return o;
    }
    static constexpr int lut_size = lut_off(ns);
    B2_HD static constexpr int rmax() {
        int m = 1;
        for (int i = 0; i < ns; ++i) m = r(i) > m ? r(i) : m;
        return m;
    }
};

enum { MAP_TFAST = 0, MAP_QFAST = 1 };      // which of (t = thread-in-line, q = line) is the fast lane index
enum { LAY_LINE = 0, LAY_ELEM = 1 };        // smem[q][pad(p)]  or  smem[p][q]

B2_HD constexpr int cdiv(int a, int b) { return (a + b - 1) / b; }

// ------------------------------------------------------------------------------------------------
// global-memory access helpers (vector width W complex elements)
template <typename T, int W>
struct gvec;
template <> struct gvec<float, 1> { using type = float2; };
template <> struct gvec<float, 2> { using type = float4; };
template <> struct gvec<double, 1> { using type = double2; };

#if defined(__CUDA_ARCH__)
template <typename T> B2_D cpx<T> ld_lut(const cpx<T>* p) {
    if constexpr (sizeof(T) == 4) {
        float2 v = __ldg(reinterpret_cast<const float2*>(p));
        return mk<T>(v.x, v.y);
    } else {
        double2 v = __ldg(reinterpret_cast<const double2*>(p));
        return mk<T>(v.x, v.y);
    }
}
#else
template <typename T> B2_D cpx<T> ld_lut(const cpx<T>* p) { return *p; }
#endif

// (Streaming / evict-first hints -- __ldcs/__stcs -- on the transformed data were measured and rejected: the transposed
//  128-byte stores lose L2 write combining and every kernel got slower.)
// two-level table lookup of W_M^m  (m = hi*2^shift + lo):  one complex multiply, error <= ~1.5 ulp
template <typename T>
B2_D cpx<T> twiddle2(const cpx<T>* hi, const cpx<T>* lo, uint32_t shift, uint64_t m) {
    cpx<T> a = ld_lut(hi + (m >> shift));
    cpx<T> b = ld_lut(lo + (m & ((1ull << shift) - 1)));
    return a * b;
}

// ------------------------------------------------------------------------------------------------
// Kernel configuration (all compile-time)
template <typename T_, class Sch_, int TPL_, int Q_, int V_, int LMAP_, int SMAP_, int LAYOUT_, bool INV_,
          int OPS_, bool IN_UNIT_, bool OUT_UNIT_, int REGS_ = 128, int RMODE_ = 0, int ST_ = 0>
struct KCfg {
    // storage in HBM: 0 = elements of T on both sides; bit 0 = the lines READ are half precision (32-bit complex elements),
    // bit 1 = the lines WRITTEN are (cplx.cuh; plain complex transforms, and even-length R2C / C2R with both bits set, where a
    // pair of half reals is one 32-bit element).  Strides and offsets count elements either way
    static constexpr int ST = ST_;
    using T = T_;
    using Sch = Sch_;
    static constexpr int N = Sch::N;
    static constexpr int TPL = TPL_;      // threads cooperating on one line
    static constexpr int Q = Q_;          // lines per CTA
    static constexpr int V = V_;          // adjacent butterflies per thread (vector width of HBM access)
    static constexpr int LMAP = LMAP_;    // thread mapping used on the HBM-load side
    static constexpr int SMAP = SMAP_;    // thread mapping used on the HBM-store side
    static constexpr int LAYOUT = LAYOUT_;
    static constexpr bool INV = INV_;
    static constexpr int OPS = OPS_;
    static constexpr bool IN_UNIT = IN_UNIT_;    // in_es == 1 guaranteed
    static constexpr bool OUT_UNIT = OUT_UNIT_;  // out_es == 1 guaranteed
    // 0: complex in/out; 1: real-to-complex (even length 2N): Hermitian post-pass fused into the store;
    // 2: complex-to-real: Hermitian pre-pass fused into the load (vkFFT_R2C_even_decomposition.h:181-230 as a fused stage)
    static constexpr int RMODE = RMODE_;
    static constexpr int THREADS = TPL * Q;
    // register budget per thread -> resident CTAs per SM the compiler must make room for
    static constexpr int MINB = (65536 / (THREADS * REGS_)) < 1 ? 1 : ((65536 / (THREADS * REGS_)) > 32 ? 32 : (65536 / (THREADS * REGS_)));
    // line-major layout: every 16 B*8 = 128 B of a line is followed by one pad element; lines start on
    // an odd multiple so that the column access of the transposed store is conflict free as well.
    static constexpr int PAD_SHIFT = (sizeof(T) == 4) ? 4 : 3;
    static constexpr int NPAD = N + (N >> PAD_SHIFT);
    static constexpr int LS = (LAYOUT == LAY_LINE) ? (Q == 1 ? NPAD : (NPAD | 1)) : 0;
    static constexpr int QP = Q;  // elem-major row pitch
    // 3: DCT-II, 4: DCT-III with two real lines per complex line (contiguous real lines, or neighbouring real columns
    //    viewed as one complex column on strided axes) -- vkFFT_R2R.h:193-229, :784-859 as fused load/store stages
    // 10: short contiguous lines, one thread per line, staged through shared memory so that HBM is read and written in
    //     whole consecutive segments (thread q alone would walk its line in 8-byte steps N*8 bytes apart from its neighbour)
    static constexpr int SMEM_ELEMS = RMODE == 10 ? Q * (N + 1)
                                    : ((Sch::ns <= 1 && RMODE != 1 && RMODE != 3 && RMODE != 4) ? 0 : ((LAYOUT == LAY_LINE) ? Q * LS : N * QP));
    static constexpr int SMEM_BYTES = SMEM_ELEMS * 2 * (int)sizeof(T);
    // stage twiddles w^k generated from w^1, w^2, w^4, w^8 (Engine::compute): 4 table loads instead of 15 per radix-16
    // butterfly; every kernel generates them.
    static constexpr bool TWCHAIN = true;
};

// XF (extra flags, fused Four-Step kernel):
//   XF_LDCG      first-stage legs are read with ld.global.cg (L2 only): the data was written by other SMs during this launch
//   XF_DISCARD   after the first-stage legs of a tile are in registers its lines are dropped from L2 without write-back
//                (discard.global.L2): scratch that is never read again must not cost HBM write bandwidth
// XF (cluster Four-Step kernel, cluster4.cuh):
//   XF_SMEM_IN   first-stage legs come from the CTA's own shared-memory tile (load_first_smem), where other CTAs of the
//                cluster put exactly what the first launch of the two-launch plan would have written to HBM
//   XF_DSMEM_OUT the last stage hands every output (natural-order index p, after phase / scale / inverse swap) to a sink
//                that stores it into the shared memory of the CTA owning row p, instead of writing HBM
enum { XF_LDCG = 1, XF_DISCARD = 2, XF_SMEM_IN = 4, XF_DSMEM_OUT = 8 };

#if defined(__CUDA_ARCH__)
// the value becomes opaque to the optimiser (it stays in its register): keeps address chains additive without losing
// the address space of the pointer they are added to
#define B2_OPAQUE64(v) asm("" : "+l"(v))
#else
#define B2_OPAQUE64(v) ((void)0)
#endif

#if defined(__CUDA_ARCH__)
template <typename T> B2_D cpx<T> ld_cg(const cpx<T>* p) {
    if constexpr (sizeof(T) == 4) { float2 v = __ldcg(reinterpret_cast<const float2*>(p)); return mk<T>(v.x, v.y); }
    else { double2 v = __ldcg(reinterpret_cast<const double2*>(p)); return mk<T>(v.x, v.y); }
}
#else
template <typename T> B2_D cpx<T> ld_cg(const cpx<T>* p) { return *p; }
#endif

struct NoHook { B2_D void operator()() const {} };
struct NoSink { template <class X> B2_D void operator()(int, const X&) const {} };

// ESI / ESO: compile-time element strides of the input / output lines (0 = the runtime values of the pass descriptor).
// The fused Four-Step kernel knows both (n2 on both sides of pass A, n1 on the store side of pass B), which turns the
// per-access 64-bit address arithmetic into immediate offsets.
template <class C, int XF = 0, int ESI = 0, int ESO = 0>
struct Engine {
    using T = typename C::T;
    using X = cpx<T>;
    using Sch = typename C::Sch;
    static constexpr int N = C::N, TPL = C::TPL, Q = C::Q, V = C::V, NS = Sch::ns;
    static constexpr bool RUNNING_IN = !C::IN_UNIT && ESI == 0;      // strides only known at run time
    static constexpr bool RUNNING_OUT = !C::OUT_UNIT && ESO == 0;
    // element types in HBM (half-precision storage: one 32-bit word per complex element, converted in the load / store)
    static constexpr bool HIN = (C::ST & 1) != 0, HOUT = (C::ST & 2) != 0;
    // (even-length R2C / C2R: half on both sides only -- the real pairs and the spectrum are both 32-bit elements)
    static_assert(C::ST == 0 || ((C::RMODE == 0 || ((C::RMODE == 1 || C::RMODE == 2) && C::ST == 3)) && V == 1 && sizeof(T) == 4 && XF == 0),
                  "half storage: FP32 complex transforms and even-length real transforms");
    template <bool H, class A, class B> struct Sel { using type = A; };
    template <class A, class B> struct Sel<true, A, B> { using type = B; };
    using XI = typename Sel<HIN, X, uint32_t>::type;
    using XO = typename Sel<HOUT, X, uint32_t>::type;
    B2_D static X ldx(const X* p) { return *p; }
    B2_D static X ldx(const uint32_t* p) { float re, im; b2_h2_to_f2(*p, re, im); return mk<T>((T)re, (T)im); }
    B2_D static void stx(X* p, X a) { *p = a; }
    B2_D static void stx(uint32_t* p, X a) { *p = b2_f2_to_h2((float)a.x, (float)a.y); }

    B2_D static int sidx(int q, int p) {
        if constexpr (C::LAYOUT == LAY_LINE) return q * C::LS + p + (p >> C::PAD_SHIFT);
        else return p * C::QP + q;
    }
    template <int MAP> B2_D static void tmap(int tid, int& q, int& t) {
        if constexpr (MAP == MAP_TFAST) { t = tid % TPL; q = tid / TPL; }
        else { q = tid % Q; t = tid / Q; }
    }
    template <int s> B2_HD static constexpr int nbut() { return N / Sch::r(s); }
    template <int s> B2_HD static constexpr int bpt() { return cdiv(nbut<s>(), V * TPL); }
    template <int s> B2_HD static constexpr bool guarded() { return (nbut<s>() % (V * TPL)) != 0; }

    // ---- HBM load of first-stage legs --------------------------------------------------------------
    template <int s>
    B2_D static void load_global(X* x, const XI* __restrict__ line, int64_t es_rt, int t, bool valid) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
        // element stride: 1 (contiguous kinds), a compile-time constant (fused kernel) or the descriptor's value; the legs
        // of one butterfly are `step` apart, so one multiply per butterfly and additions from there (the per-leg 64-bit
        // multiply + LEA pair this replaces was a fifth of the instructions of the strided kernels)
        const int64_t es = C::IN_UNIT ? 1 : (ESI ? (int64_t)ESI : es_rt);
        const int64_t step = (int64_t)NB * es;
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
            const int b0 = V * (t + m * TPL);
            const bool ok = valid && (!guarded<s>() || b0 < NB);
            const XI* src = line + (int64_t)b0 * es;
#pragma unroll
            for (int k = 0; k < r; ++k) {
                // runtime stride: walk the legs with a running pointer the compiler may not re-associate into
                // (b0 + k*NB) * es (it does otherwise: a 64-bit multiply + two LEA per leg); constant stride: immediates
                const XI* lp = src;
                if constexpr (RUNNING_IN) { if (k + 1 < r) { int64_t st = step; B2_OPAQUE64(st); src += st; } }
                else lp = src + k * step;
                if constexpr (V == 2 && C::IN_UNIT && !HIN) {
                    using G = typename gvec<T, 2>::type;
                    G g = ok ? *reinterpret_cast<const G*>(lp) : G{};
                    X a = mk<T>(g.x, g.y), c = mk<T>(g.z, g.w);
                    x[(m * V + 0) * r + k] = C::INV ? swp(a) : a;
                    x[(m * V + 1) * r + k] = C::INV ? swp(c) : c;
                } else {
#pragma unroll
                    for (int v = 0; v < V; ++v) {
                        X a = mk<T>(T(0), T(0));
                        if (ok) {
                            const XI* q = lp + (int64_t)v * es;
                            if constexpr ((XF & XF_LDCG) != 0 && !HIN) a = ld_cg(q); else a = ldx(q);
                        }
                        x[(m * V + v) * r + k] = C::INV ? swp(a) : a;
                    }
                }
            }
        }
    }

    // ---- C2R: first-stage legs assembled from the Hermitian half spectrum (n+1 inputs per line) ---------------------
    //  Zin[p] = (X[p] + conj X[n-p]) + i conj(w_p) (X[p] - conj X[n-p]),  w_p = e^{-2 pi i p/2n};  then the inverse FFT
    template <int s>
    B2_D static void load_global_c2r(X* x, const XI* __restrict__ line, const X* __restrict__ w, int t, bool valid) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int b = V * (t + m * TPL) + v;
                const bool ok = valid && (!guarded<s>() || b < NB);
#pragma unroll
                for (int k = 0; k < r; ++k) {
                    const int p = b + k * NB;
                    X z = mk<T>(T(0), T(0));
                    if (ok) {
                        const X a = ldx(line + p), bc = conj(ldx(line + (N - p)));
                        const X sm = a + bc, d = mulc(a - bc, ld_lut(w + p));
                        z = mk<T>(sm.x - d.y, sm.y + d.x);
                    }
                    x[(m * V + v) * r + k] = swp(z);          // RMODE 2 is always an inverse transform
                }
            }
        }
    }

    B2_D static int makhoul(int p) { return (p < (N + 1) / 2) ? 2 * p : 2 * (N - 1 - p) + 1; }

    B2_D static int64_t makhoul_full(int64_t i, int64_t nfull) { return (i < (nfull + 1) / 2) ? 2 * i : 2 * (nfull - 1 - i) + 1; }

    // ---- long strided DCT-II, first Four-Step launch (RMODE 5): rows gathered through the permutation of the full index ----
    template <int s>
    B2_D static void load_global_perm(X* x, const X* __restrict__ base, int64_t es0, uint32_t n2, uint32_t N2, uint32_t nfull,
                                      int t, bool valid) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int b = V * (t + m * TPL) + v;
                const bool ok = valid && (!guarded<s>() || b < NB);
#pragma unroll
                for (int k = 0; k < r; ++k) {
                    const int p = b + k * NB;
                    X a = mk<T>(T(0), T(0));
                    if (ok) a = base[makhoul_full((int64_t)p * N2 + n2, nfull) * es0];
                    x[(m * V + v) * r + k] = C::INV ? swp(a) : a;
                }
            }
        }
    }

    // ---- long strided DCT-III, last Four-Step launch (RMODE 6): scatter through the permutation of k1 + N1*p ---------------
    template <int s>
    B2_D static void store_global_perm(const X* x, X* __restrict__ base, int64_t es0, uint32_t k1, uint32_t N1, uint32_t nfull,
                                       int t, bool valid, const b2_pass_params& P) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
        const bool do_scale = (P.ops & B2_OP_SCALE) != 0;
        const T sc = (T)P.scale;
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int b = V * (t + m * TPL) + v;
                if (!valid || (guarded<s>() && b >= NB)) continue;
#pragma unroll
                for (int k = 0; k < r; ++k) {
                    X a = x[(m * V + v) * r + k];
                    if (do_scale) a = a * sc;
                    if (C::INV) a = swp(a);
                    const int p = b + k * NB;
                    base[makhoul_full((int64_t)k1 + (int64_t)N1 * p, nfull) * es0] = a;
                }
            }
        }
    }

    // ---- Bluestein, first launch (RMODE 7): zero-pad + chirp on load, filter on store ---------------------------------
    template <int s>
    B2_D static void load_global_blue(X* x, const X* __restrict__ line, const b2_pass_params& P, int t, bool valid) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
        const X* __restrict__ chirp = (const X*)P.aux0;
        const bool oswap = P.inverse != 0;
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int b = V * (t + m * TPL) + v;
                const bool ok = valid && (!guarded<s>() || b < NB);
#pragma unroll
                for (int k = 0; k < r; ++k) {
                    const int p = b + k * NB;
                    X a = mk<T>(T(0), T(0));
                    if (ok && p < (int)P.in_len) {
                        a = line[p];
                        if (oswap) a = swp(a);
                        a = a * ld_lut(chirp + p);
                    }
                    x[(m * V + v) * r + k] = a;
                }
            }
        }
    }
    // RMODE 7 store: x * filter -> packed scratch line;  RMODE 8 store: inner un-swap, chirp, scale, outer swap, truncation
    template <int s>
    B2_D static void store_global_blue(const X* x, X* __restrict__ line, const b2_pass_params& P, int t, bool valid) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
        const bool do_scale = (P.ops & B2_OP_SCALE) != 0;
        const T sc = (T)P.scale;
        const bool oswap = P.inverse != 0;
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int b = V * (t + m * TPL) + v;
                if (!valid || (guarded<s>() && b >= NB)) continue;
#pragma unroll
                for (int k = 0; k < r; ++k) {
                    const int p = b + k * NB;
                    X a = x[(m * V + v) * r + k];
                    if constexpr (C::RMODE == 7) {
                        line[p] = a * ld_lut((const X*)P.aux1 + p);
                    } else {
                        if (p < (int)P.out_len) {
                            a = swp(a) * ld_lut((const X*)P.aux0 + p);
                            if (do_scale) a = a * sc;
                            line[p] = oswap ? swp(a) : a;
                        }
                    }
                }
            }
        }
    }

    // ---- DCT-II / DCT-III on contiguous real lines: HBM -> shared memory staging -----------------------------------
    // Two real lines (a, b) travel as one complex line a + i b.  Reading them straight into the first-stage legs
    // costs four loads per element for DCT-III (it needs p and N-p of both lines).  Instead the CTA copies both lines
    // with fully coalesced loads into the tile and the legs come from shared memory.
    // Staging both the loads and the stores measured fastest for the DCT-III rows; the DCT-II kernel keeps its direct
    // Makhoul gather, which measured faster than staging its input as well.
#ifndef B2_TW_CHAIN
#define B2_TW_CHAIN 1
#endif
#ifndef B2_DCT3_STAGE_IN
#define B2_DCT3_STAGE_IN 1
#endif
#ifndef B2_DCT3_STAGE_OUT
#define B2_DCT3_STAGE_OUT 1
#endif
    B2_D static int unmakhoul(int j) { return (j & 1) ? N - 1 - (j >> 1) : (j >> 1); }

    B2_D static void stage_in_dct(X* sm, const b2_pass_params& P, int64_t obase_in, uint32_t gl, int q, int t, bool valid) {
        if (!valid) return;
        const T* __restrict__ la = (const T*)P.in + obase_in + (int64_t)gl * P.in_gs;
        const T* __restrict__ lb = la + P.aux_u1;
        const bool vb = (2 * gl + 1 < P.aux_u0);
#pragma unroll 8
        for (int j = t; j < N; j += TPL) {
            const T a = la[j];
            const T b = vb ? lb[j] : T(0);
            B2_SMEM_ST(sm, sidx(q, C::RMODE == 3 ? unmakhoul(j) : j), mk<T>(a, b));
        }
    }
    // DCT-III legs from the raw staged lines:  z_p = swap( (a_p + b_{N-p}, b_p - a_{N-p}) * conj-phase_p )
    template <int s>
    B2_D static void load_smem_dct3(X* x, const X* sm, const X* __restrict__ c, int q, int t) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int b = V * (t + m * TPL) + v;
                if (guarded<s>() && b >= NB) continue;
#pragma unroll
                for (int k = 0; k < r; ++k) {
                    const int p = b + k * NB;
                    const X u = B2_SMEM_LD(sm, sidx(q, p));
                    X w2 = mk<T>(T(0), T(0));
                    if (p != 0) w2 = B2_SMEM_LD(sm, sidx(q, N - p));
                    x[(m * V + v) * r + k] = swp(mulc(mk<T>(u.x + w2.y, u.y - w2.x), ld_lut(c + p)));
                }
            }
        }
    }

    // ---- DCT-II / DCT-III: first-stage legs (RMODE 3 / 4) --------------------------------------------------------------
    template <int s>
    B2_D static void load_global_dct(X* x, const b2_pass_params& P, int64_t obase_in, uint32_t gl, int t, bool valid) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
        const X* __restrict__ c = (const X*)P.aux0;
        const T* la = nullptr; const T* lb = nullptr; const X* lc = nullptr;
        bool vb = false;
        if constexpr (C::LAYOUT == LAY_LINE) {
            la = (const T*)P.in + obase_in + (int64_t)gl * P.in_gs;
            lb = la + P.aux_u1;
            vb = valid && (2 * gl + 1 < P.aux_u0);
        } else {
            lc = (const X*)P.in + obase_in + (int64_t)gl * P.in_gs;
        }
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int b = V * (t + m * TPL) + v;
                const bool ok = valid && (!guarded<s>() || b < NB);
#pragma unroll
                for (int k = 0; k < r; ++k) {
                    const int p = b + k * NB;
                    X z = mk<T>(T(0), T(0));
                    if (ok) {
                        if constexpr (C::RMODE == 3) {
                            const int src = makhoul(p);
                            if constexpr (C::LAYOUT == LAY_LINE) { z.x = la[src]; if (vb) z.y = lb[src]; }
                            else z = lc[(int64_t)src * P.in_es];
                        } else {
                            T a0, a1 = T(0), b0, b1 = T(0);
                            if constexpr (C::LAYOUT == LAY_LINE) {
                                a0 = la[p]; b0 = vb ? lb[p] : T(0);
                                if (p != 0) { a1 = la[N - p]; b1 = vb ? lb[N - p] : T(0); }
                            } else {
                                const X u = lc[(int64_t)p * P.in_es];
                                a0 = u.x; b0 = u.y;
                                if (p != 0) { const X w2 = lc[(int64_t)(N - p) * P.in_es]; a1 = w2.x; b1 = w2.y; }
                            }
                            z = swp(mulc(mk<T>(a0 + b1, b0 - a1), ld_lut(c + p)));
                        }
                    }
                    x[(m * V + v) * r + k] = z;
                }
            }
        }
    }

    // ---- DCT-II store: split + phase through shared memory;  DCT-III store: Makhoul scatter from registers ----------
    template <int s>
    B2_D static void store_global_dct(const X* x, X* sm, const b2_pass_params& P, int64_t obase_out, uint32_t gl, int q,
                                      int t, bool valid) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
        const bool do_scale = (P.ops & B2_OP_SCALE) != 0;
        const T sc = (T)P.scale;
        T* oa = nullptr; T* ob = nullptr; X* oc = nullptr;
        bool vb = false;
        if constexpr (C::LAYOUT == LAY_LINE) {
            oa = (T*)P.out + obase_out + (int64_t)gl * P.out_gs;
            ob = oa + P.aux_u2;
            vb = (2 * gl + 1 < P.aux_u0);
        } else {
            oc = (X*)P.out + obase_out + (int64_t)gl * P.out_gs;
        }
        if constexpr (C::RMODE == 4 && C::LAYOUT == LAY_LINE && B2_DCT3_STAGE_OUT) {
            // Makhoul scatter through the tile: natural-order spectrum in, coalesced 4-byte stores out
#pragma unroll
            for (int m = 0; m < BPT; ++m) {
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    const int b = V * (t + m * TPL) + v;
                    if (guarded<s>() && b >= NB) continue;
#pragma unroll
                    for (int k = 0; k < r; ++k) {
                        X u = swp(x[(m * V + v) * r + k]);
                        if (do_scale) u = u * sc;
                        B2_SMEM_ST(sm, sidx(q, b + k * NB), u);
                    }
                }
            }
            __syncthreads();
            if (!valid) return;
#pragma unroll 8
            for (int j = t; j < N; j += TPL) {
                const X u = B2_SMEM_LD(sm, sidx(q, unmakhoul(j)));
                oa[j] = u.x;
                if (vb) ob[j] = u.y;
            }
        } else if constexpr (C::RMODE == 4) {
#pragma unroll
            for (int m = 0; m < BPT; ++m) {
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    const int b = V * (t + m * TPL) + v;
                    if (!valid || (guarded<s>() && b >= NB)) continue;
#pragma unroll
                    for (int k = 0; k < r; ++k) {
                        X u = swp(x[(m * V + v) * r + k]);
                        if (do_scale) u = u * sc;
                        const int dst = makhoul(b + k * NB);
                        if constexpr (C::LAYOUT == LAY_LINE) { oa[dst] = u.x; if (vb) ob[dst] = u.y; }
                        else oc[(int64_t)dst * P.out_es] = u;
                    }
                }
            }
        } else {
            const X* __restrict__ c = (const X*)P.aux0;
#pragma unroll
            for (int m = 0; m < BPT; ++m) {
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    const int b = V * (t + m * TPL) + v;
                    if (guarded<s>() && b >= NB) continue;
#pragma unroll
                    for (int k = 0; k < r; ++k) B2_SMEM_ST(sm, sidx(q, b + k * NB), x[(m * V + v) * r + k]);
                }
            }
            __syncthreads();
            if (!valid) return;
            for (int k = t; k < N; k += TPL) {
                const X a = B2_SMEM_LD(sm, sidx(q, k));
                const X bc = conj(B2_SMEM_LD(sm, sidx(q, k == 0 ? 0 : N - k)));
                const X ck = ld_lut(c + k);
                const X su = ck * (a + bc), d = ck * (a - bc);
                T ya = su.x, yb = d.y;
                if (do_scale) { ya *= sc; yb *= sc; }
                if constexpr (C::LAYOUT == LAY_LINE) { oa[k] = ya; if (vb) ob[k] = yb; }
                else oc[(int64_t)k * P.out_es] = mk<T>(ya, yb);
            }
        }
    }

    // ---- R2C: Hermitian post-pass through shared memory, n+1 outputs per line ---------------------------------------
    //  X[k] = 1/2 (Z[k] + conj Z[n-k]) - i/2 w_k (Z[k] - conj Z[n-k])
    template <int s>
    B2_D static void store_global_r2c(const X* x, X* sm, XO* __restrict__ line, const X* __restrict__ w, int q, int t,
                                      bool valid, const b2_pass_params& P) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
        const bool do_scale = (P.ops & B2_OP_SCALE) != 0;
        const T sc = (T)P.scale;
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int b = V * (t + m * TPL) + v;
                if (guarded<s>() && b >= NB) continue;
#pragma unroll
                for (int k = 0; k < r; ++k) B2_SMEM_ST(sm, sidx(q, b + k * NB), x[(m * V + v) * r + k]);
            }
        }
        __syncthreads();
        if (!valid) return;
        for (int k = t; k <= N; k += TPL) {
            const X a = B2_SMEM_LD(sm, sidx(q, k == N ? 0 : k));
            const X bc = conj(B2_SMEM_LD(sm, sidx(q, k == 0 ? 0 : N - k)));
            const X sum = a + bc, d = (a - bc) * ld_lut(w + k);
            X o = mk<T>(T(0.5) * (sum.x + d.y), T(0.5) * (sum.y - d.x));
            if (do_scale) o = o * sc;
            stx(line + k, o);
        }
    }

    // ---- smem read of stage legs ---------------------------------------------------------------------
    template <int s>
    B2_D static void load_smem(X* x, const X* sm, int q, int t) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int b = V * (t + m * TPL) + v;
                if (guarded<s>() && b >= NB) continue;
#pragma unroll
                for (int k = 0; k < r; ++k) x[(m * V + v) * r + k] = B2_SMEM_LD(sm, sidx(q, b + k * NB));
            }
        }
    }

    // ---- XF_SMEM_IN: first-stage legs from the tile, which holds the values HBM would hold (load_global's swap included) ----
    template <int s>
    B2_D static void load_first_smem(X* x, const X* sm, int q, int t) {
        static_assert((XF & XF_SMEM_IN) != 0 && s == 0 && V == 1, "first stage from shared memory");
        load_smem<s>(x, sm, q, t);
        if constexpr (C::INV) {
#pragma unroll
            for (int i = 0; i < bpt<s>() * Sch::r(s); ++i) x[i] = swp(x[i]);
        }
    }

    // ---- twiddle + butterfly ---------------------------------------------------------------------------
    template <int s>
    B2_D static void compute(X* x, const X* __restrict__ lut, int t) {
        constexpr int r = Sch::r(s), S = Sch::S(s), NB = nbut<s>(), BPT = bpt<s>();
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int b = V * (t + m * TPL) + v;
                if (guarded<s>() && b >= NB) continue;
                X* xb = x + (m * V + v) * r;
                if constexpr (s > 0) {
                    const int j = b % S;
                    const X* l = lut + Sch::lut_off(s) + j;
                    if constexpr (B2_TW_CHAIN && C::TWCHAIN) {
                    // only w^1, w^2, w^4, ... come from the table; w^k = w^(lowest set bit of k) * w^(rest), <= 3
                    // multiplies deep for r <= 16: 4 loads instead of 15 per radix-16 butterfly (the LSU pipe, not
                    // the FMA pipe, is what these kernels run out of)
                    X w[r];
#pragma unroll
                    for (int k = 1; k < r; ++k) {
                        if ((k & (k - 1)) == 0) w[k] = ld_lut(l + (k - 1) * S);
                        else w[k] = w[k & -k] * w[k - (k & -k)];
                        xb[k] = xb[k] * w[k];
                    }
                    } else {
#pragma unroll
                    for (int k = 1; k < r; ++k) xb[k] = xb[k] * ld_lut(l + (k - 1) * S);
                    }
                }
                dft<r, T>(xb);
            }
        }
    }

    // ---- autosort scatter into smem ------------------------------------------------------------------
    template <int s>
    B2_D static void store_smem(const X* x, X* sm, int q, int t) {
        constexpr int r = Sch::r(s), S = Sch::S(s), NB = nbut<s>(), BPT = bpt<s>();
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const int b = V * (t + m * TPL) + v;
                if (guarded<s>() && b >= NB) continue;
                const int j = b % S;
                const int base = (b - j) * r + j;
#pragma unroll
                for (int k = 0; k < r; ++k) B2_SMEM_ST(sm, sidx(q, base + k * S), x[(m * V + v) * r + k]);
            }
        }
    }

    // ---- HBM store of last-stage outputs (+ fused post operators) --------------------------------------
    // Four-step phase on store: W_M^(line*p).  A thread's outputs are p = p0 + k*NB, k = 0..r-1, so the phases form a
    // geometric sequence: one two-level lookup (two small L1-resident loads + one complex multiply) per group of 8
    // outputs, three more for the step W^(line*NB) and its 2nd / 4th power, and every phase of the group is the group's
    // first one times at most three of those (error <= ~7 ulp worst case, ~2 ulp rms).  This replaced a lookup per
    // output (64 scattered 8-byte loads + 64-bit index arithmetic per 32 outputs), which kept the LSU pipe the limiter
    // of these kernels.  Also measured and rejected: a tile-factored scheme with coalesced table reads and the
    // reference-style full M-entry table.
    // XF_DSMEM_OUT: `line` is unused and sink(p, value) receives every output instead.
    template <int s, class Sink = NoSink>
    B2_D static void store_global(const X* x, XO* __restrict__ line, int64_t es_rt, int t, bool valid,
                                  const b2_pass_params& P, uint32_t gline, uint32_t qline, const Sink& sink = Sink{}) {
        constexpr int r = Sch::r(s), NB = nbut<s>(), BPT = bpt<s>();
        static_assert(s == NS - 1, "global store only after the last stage");
        constexpr bool TW = (C::OPS & B2_OP_TWIDDLE_OUT) != 0;
        const bool do_scale = (P.ops & B2_OP_SCALE) != 0;   // runtime: normalize=1 on the last inverse pass
        const T sc = (T)P.scale;
        const int64_t es = C::OUT_UNIT ? 1 : (ESO ? (int64_t)ESO : es_rt);
        const int64_t step = (int64_t)NB * es;
        X s1 = mk<T>(T(1), T(0)), s2 = s1, s4 = s1;
        if constexpr (TW) {
            const uint64_t e1 = (uint64_t)gline * (uint64_t)NB;     // 4*e1 < M for r >= 4; unused otherwise
            if constexpr (r > 1) s1 = twiddle2<T>((const X*)P.tw_hi, (const X*)P.tw_lo, P.tw_shift, e1);
            if constexpr (r > 2) s2 = twiddle2<T>((const X*)P.tw_hi, (const X*)P.tw_lo, P.tw_shift, 2 * e1);
            if constexpr (r > 4) s4 = twiddle2<T>((const X*)P.tw_hi, (const X*)P.tw_lo, P.tw_shift, 4 * e1);
        }
#pragma unroll
        for (int m = 0; m < BPT; ++m) {
            const int b0 = V * (t + m * TPL);
            const bool ok = valid && (!guarded<s>() || b0 < NB);
            if (!ok) continue;                     // one branch per butterfly, not one per output
            XO* dst = line + (int64_t)b0 * es;
            X w0[V], w2[V], w4[V], w6[V];
#pragma unroll
            for (int k = 0; k < r; ++k) {
                XO* sp = dst;
                if constexpr (RUNNING_OUT) { if (k + 1 < r) { int64_t st = step; B2_OPAQUE64(st); dst += st; } }
                else sp = dst + k * step;
                X o[V];
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    X a = x[(m * V + v) * r + k];
                    const int p = b0 + v + k * NB;  // natural-order output index (S == NB in the last stage)
                    if constexpr (TW) {
                        const int tt = k & 7;
                        X w;
                        if (tt == 0) { w0[v] = twiddle2<T>((const X*)P.tw_hi, (const X*)P.tw_lo, P.tw_shift, (uint64_t)gline * (uint64_t)p); w = w0[v]; }
                        else if (tt == 1) w = w0[v] * s1;
                        else if (tt == 2) { w2[v] = w0[v] * s2; w = w2[v]; }
                        else if (tt == 3) w = w2[v] * s1;
                        else if (tt == 4) { w4[v] = w0[v] * s4; w = w4[v]; }
                        else if (tt == 5) w = w4[v] * s1;
                        else if (tt == 6) { w6[v] = w4[v] * s2; w = w6[v]; }
                        else w = w6[v] * s1;
                        a = a * w;
                    }
                    if (do_scale) a = a * sc;
                    o[v] = C::INV ? swp(a) : a;
                }
                if constexpr ((XF & XF_DSMEM_OUT) != 0) {
                    static_assert(V == 1 && !HOUT, "one output per butterfly leg, FP32 / FP64 elements");
                    sink(b0 + k * NB, o[0]);
                } else if constexpr (V == 2 && C::OUT_UNIT && !HOUT) {
                    using G = typename gvec<T, 2>::type;
                    G g;
                    g.x = o[0].x; g.y = o[0].y; g.z = o[1].x; g.w = o[1].y;
                    *reinterpret_cast<G*>(sp) = g;
                } else {
#pragma unroll
                    for (int v = 0; v < V; ++v) stx(sp + (int64_t)v * es, o[v]);
                }
            }
        }
    }

    // drop the (contiguous-line) input tile from L2 without write-back: every thread of the CTA has its legs in registers
    B2_D static void discard_tile(const b2_pass_params& P, int64_t obase_in, uint32_t grp, int tid) {
#if defined(__CUDA_ARCH__)
        static_assert(C::LAYOUT == LAY_LINE && C::IN_UNIT, "discard: contiguous input lines");
        constexpr int LINES_PER_ROW = (N * 2 * (int)sizeof(T)) / 128;      // 128-byte cache lines per FFT line
        static_assert(LINES_PER_ROW * 128 == N * 2 * (int)sizeof(T), "whole cache lines");
        const uint32_t g0 = grp * Q;
        const uint32_t nrows = (P.G - g0) < (uint32_t)Q ? (P.G - g0) : (uint32_t)Q;
        const char* base = (const char*)((const X*)P.in + obase_in + (int64_t)g0 * P.in_gs);
        if ((((uintptr_t)base) | (uintptr_t)(P.in_gs * 2 * (int64_t)sizeof(T))) & 127) return;   // unaligned scratch: keep the lines
        for (uint32_t i = tid; i < nrows * LINES_PER_ROW; i += C::THREADS) {
            const char* a = base + (int64_t)(i / LINES_PER_ROW) * P.in_gs * 2 * (int64_t)sizeof(T) + (size_t)(i % LINES_PER_ROW) * 128;
            asm volatile("discard.global.L2 [%0], 128;" ::"l"(a) : "memory");
        }
#endif
    }

    // coordinate that multiplies the element index in the four-step phase
    B2_D static uint32_t twl(const b2_pass_params& P, uint32_t g, uint32_t o0, uint32_t o1, uint32_t o2) {
        const uint32_t sel = P.tw_sel;
        return P.tw_line0 + (sel == 0 ? g : (sel == 1 ? o0 : (sel == 2 ? o1 : o2)));
    }

    // ---- middle stages (recursive over the schedule) --------------------------------------------------
    template <int s>
    B2_D static void middle(X* sm, const X* lut, int tid) {
        if constexpr (s < NS - 1) {
            int q, t;
            tmap<C::LMAP>(tid, q, t);
            X x[bpt<s>() * V * Sch::r(s)];
            load_smem<s>(x, sm, q, t);
            compute<s>(x, lut, t);
            __syncthreads();
            store_smem<s>(x, sm, q, t);
            __syncthreads();
            middle<s + 1>(sm, lut, tid);
        }
    }

    B2_D static void run(const b2_pass_params& P, unsigned char* smem_raw) {
        // decode CTA -> (line group, outer batch coordinates)
        const uint32_t ngrp = (P.G + Q - 1) / Q;
        uint32_t rest = blockIdx.x;
        const uint32_t grp = rest % ngrp; rest /= ngrp;
        const uint32_t o0 = rest % P.nb[0]; rest /= P.nb[0];
        const uint32_t o1 = rest % P.nb[1]; rest /= P.nb[1];
        const uint32_t o2 = rest;
        const int64_t obase_in = (int64_t)o0 * P.in_bs[0] + (int64_t)o1 * P.in_bs[1] + (int64_t)o2 * P.in_bs[2];
        const int64_t obase_out = (int64_t)o0 * P.out_bs[0] + (int64_t)o1 * P.out_bs[1] + (int64_t)o2 * P.out_bs[2];
        run_at(P, smem_raw, grp, o0, o1, o2, obase_in, obase_out, NoHook{});
    }

    // one tile: line group `grp` of the lines at (o0, o1, o2); obase_* = element offsets of those coordinates.
    // `hook` runs once, after the first-stage loads have been issued and before their values are used (the fused
    // Four-Step kernel claims its next tile there, hidden behind the HBM latency)
    template <class Hook>
    B2_D static void run_at(const b2_pass_params& P, unsigned char* smem_raw, uint32_t grp, uint32_t o0, uint32_t o1, uint32_t o2,
                            int64_t obase_in, int64_t obase_out, Hook hook) {
        const int tid = threadIdx.x;
        const X* __restrict__ lut = (const X*)P.lut;
        X* sm = reinterpret_cast<X*>(smem_raw);

        int ql, tl;
        tmap<C::LMAP>(tid, ql, tl);
        const uint32_t gl = grp * Q + ql;
        const XI* in_line = (const XI*)P.in + obase_in + (int64_t)gl * P.in_gs;

        const X* __restrict__ rw = (const X*)P.aux0;   // e^{-2 pi i k/2n} for the fused real transforms
        const uint32_t psel = (P.tw_sel == 1 ? o0 : (P.tw_sel == 2 ? o1 : o2));   // n2 / k1 of the long strided DCT launches
        if constexpr (C::RMODE == 10) {
            // ---- short lines (N <= 32), one thread per line --------------------------------------------------------------------
            // A warp reading "its" 32 lines directly touches 32 segments N*8 bytes apart with every load instruction; here the
            // CTA copies its Q lines as ONE contiguous run (consecutive lanes, consecutive elements) into the tile, every thread
            // transforms the line it owns out of shared memory (line pitch N+1: conflict free), and the run goes back the same way.
            static_assert(NS == 1 && TPL == 1 && V == 1 && C::LAYOUT == LAY_LINE && C::IN_UNIT && C::OUT_UNIT, "staged short lines");
            const uint32_t g0 = grp * Q;
            const uint32_t nv = (P.G - g0) < (uint32_t)Q ? (P.G - g0) : (uint32_t)Q;
            const X* __restrict__ src = (const X*)P.in + obase_in + (int64_t)g0 * P.in_gs;
            X* __restrict__ dst = (X*)P.out + obase_out + (int64_t)g0 * P.out_gs;
            const bool dense_in = P.in_gs == (int64_t)N, dense_out = P.out_gs == (int64_t)N;
            for (uint32_t i = tid; i < nv * (uint32_t)N; i += C::THREADS) {
                const uint32_t l = i / N, p = i % N;
                X a = dense_in ? src[i] : src[(int64_t)l * P.in_gs + p];
                B2_SMEM_ST(sm, l * (N + 1) + p, C::INV ? swp(a) : a);
            }
            __syncthreads();
            if ((uint32_t)tid < nv) {
                X x[N];
#pragma unroll
                for (int p = 0; p < N; ++p) x[p] = B2_SMEM_LD(sm, tid * (N + 1) + p);
                dft<N, T>(x);
#pragma unroll
                for (int p = 0; p < N; ++p) B2_SMEM_ST(sm, tid * (N + 1) + p, x[p]);
            }
            __syncthreads();
            const bool do_scale = (P.ops & B2_OP_SCALE) != 0;
            const T sc = (T)P.scale;
            for (uint32_t i = tid; i < nv * (uint32_t)N; i += C::THREADS) {
                const uint32_t l = i / N, p = i % N;
                X a = B2_SMEM_LD(sm, l * (N + 1) + p);
                if (do_scale) a = a * sc;
                if (C::INV) a = swp(a);
                if (dense_out) dst[i] = a; else dst[(int64_t)l * P.out_gs + p] = a;
            }
        } else if constexpr (C::RMODE == 9) {
            // ---- fused convolution (vkFFT_Convolution.h:125 fuses the same three steps into the last-axis kernel) ----------
            // forward transform; the last stage leaves element p = b + k*NB in the registers of the thread that would read
            // exactly these legs for the first stage of another transform, because the schedule starts and ends with the
            // same radix.  So: multiply by the kernel line in registers, swap re/im (inverse = swap, forward, swap) and run
            // the stages again.  One HBM read and one write of the data for FFT -> product -> iFFT.
            static_assert(Sch::r(0) == Sch::r(NS - 1), "fused convolution needs a schedule with equal first and last radix");
            static_assert(C::LMAP == C::SMAP && V == 1, "same thread map on both sides");
            constexpr int s = NS - 1, r = Sch::r(0), NB = nbut<0>(), BPT = bpt<0>();
            const bool valid = gl < P.G;
            const uint32_t flags = P.aux_u1;
            // kernel operand: same offsets as the data inside one block of aux_u0 elements (features x plane), shared by
            // every batch -- a line never leaves its feature plane, so one modulo per line is enough
            const int64_t es = C::IN_UNIT ? 1 : P.in_es;
            const X* __restrict__ kline = (const X*)P.aux0 + (int64_t)((uint64_t)(obase_in + (int64_t)gl * P.in_gs) % (uint64_t)(P.aux_u0 ? P.aux_u0 : 1));
            X* out_line = (X*)P.out + obase_out + (int64_t)gl * P.out_gs;
            X x[BPT * r];
            load_global<0>(x, in_line, P.in_es, tl, valid);
            compute<0>(x, lut, tl);
            if constexpr (NS > 1) {
                store_smem<0>(x, sm, ql, tl);
                __syncthreads();
                middle<1>(sm, lut, tid);
                load_smem<s>(x, sm, ql, tl);
                compute<s>(x, lut, tl);
            }
#pragma unroll
            for (int m = 0; m < BPT; ++m) {
                const int b = tl + m * TPL;
#pragma unroll
                for (int k = 0; k < r; ++k) {
                    X w = mk<T>(T(1), T(0));
                    if (valid && (!guarded<0>() || b < NB)) w = ld_lut(kline + (int64_t)(b + k * NB) * es);
                    X a = x[m * r + k];
                    if (flags & (1u << 13)) a = conj(a);      // B2_CONV_CONJ_SEQ
                    if (flags & (1u << 14)) w = conj(w);      // B2_CONV_CONJ_KER
                    a = a * w;
                    if (flags & (1u << 15)) {                  // B2_CONV_XPS
                        const T mag = sqrt(a.x * a.x + a.y * a.y);
                        if (mag > T(0)) a = a * (T(1) / mag);
                    }
                    x[m * r + k] = swp(a);
                }
            }
            compute<0>(x, lut, tl);
            if constexpr (NS > 1) {
                __syncthreads();       // every last-stage read of the forward transform is done
                store_smem<0>(x, sm, ql, tl);
                __syncthreads();
                middle<1>(sm, lut, tid);
                load_smem<s>(x, sm, ql, tl);
                compute<s>(x, lut, tl);
            }
            const bool do_scale = (P.ops & B2_OP_SCALE) != 0;
            const T sc = (T)P.scale;
#pragma unroll
            for (int m = 0; m < BPT; ++m) {
                const int b = tl + m * TPL;
                if (!valid || (guarded<0>() && b >= NB)) continue;
#pragma unroll
                for (int k = 0; k < r; ++k) {
                    X a = swp(x[m * r + k]);
                    if (do_scale) a = a * sc;
                    out_line[C::OUT_UNIT ? (int64_t)(b + k * NB) : (int64_t)(b + k * NB) * P.out_es] = a;
                }
            }
        } else if constexpr (C::RMODE == 11) {
            // ---- the whole Bluestein transform of a line in ONE launch -----------------------------------------------------
            //   X[k] = conj(b_k) sum_n (x_n conj(b_n)) b_{k-n}:  chirp + zero-pad to the padded length on load, forward stages,
            //   product with the filter spectrum (aux1, one table for every line) in registers, swap, the stages again (= inverse),
            //   chirp + scale + truncation on store.  Same register hand-over as the fused convolution above (equal first and last
            //   radix); the two-launch form (RMODE 7 then 8) writes and re-reads a padded scratch line of n >= 2N-1 points in between,
            //   here HBM sees the N-point line once in and once out.  The reference runs Bluestein as separate FFT / multiply / iFFT
            //   dispatches through its temp buffer as well (vkFFT_Bluestein.h:32,201; vkFFT_Scheduler.h:2493-2578).
            static_assert(Sch::r(0) == Sch::r(NS - 1), "fused Bluestein needs a schedule with equal first and last radix");
            static_assert(C::LMAP == C::SMAP && V == 1 && C::IN_UNIT && C::OUT_UNIT, "contiguous lines, same thread map on both sides");
            constexpr int s = NS - 1, r = Sch::r(0), NB = nbut<0>(), BPT = bpt<0>();
            const bool valid = gl < P.G;
            const X* __restrict__ filt = (const X*)P.aux1;
            X* out_line = (X*)P.out + obase_out + (int64_t)gl * P.out_gs;
            X x[BPT * r];
            load_global_blue<0>(x, in_line, P, tl, valid);
            compute<0>(x, lut, tl);
            if constexpr (NS > 1) {
                store_smem<0>(x, sm, ql, tl);
                __syncthreads();
                middle<1>(sm, lut, tid);
                load_smem<s>(x, sm, ql, tl);
                compute<s>(x, lut, tl);
            }
#pragma unroll
            for (int m = 0; m < BPT; ++m) {
                const int b = tl + m * TPL;
                const bool ok = valid && (!guarded<0>() || b < NB);
#pragma unroll
                for (int k = 0; k < r; ++k) {
                    X w = mk<T>(T(0), T(0));
                    if (ok) w = ld_lut(filt + (b + k * NB));
                    x[m * r + k] = swp(x[m * r + k] * w);
                }
            }
            compute<0>(x, lut, tl);
            if constexpr (NS > 1) {
                __syncthreads();       // every last-stage read of the forward transform is done
                store_smem<0>(x, sm, ql, tl);
                __syncthreads();
                middle<1>(sm, lut, tid);
                load_smem<s>(x, sm, ql, tl);
                compute<s>(x, lut, tl);
            }
            {
                const bool do_scale = (P.ops & B2_OP_SCALE) != 0;
                const T sc = (T)P.scale;
                const bool oswap = P.inverse != 0;
                const X* __restrict__ chirp = (const X*)P.aux0;
#pragma unroll
                for (int m = 0; m < BPT; ++m) {
                    const int b = tl + m * TPL;
                    if (!valid || (guarded<0>() && b >= NB)) continue;
#pragma unroll
                    for (int k = 0; k < r; ++k) {
                        const int p = b + k * NB;
                        if (p < (int)P.out_len) {
                            X a = swp(x[m * r + k]) * ld_lut(chirp + p);
                            if (do_scale) a = a * sc;
                            out_line[p] = oswap ? swp(a) : a;
                        }
                    }
                }
            }
        } else if constexpr (C::RMODE == 4 && C::LAYOUT == LAY_LINE && B2_DCT3_STAGE_IN) {
            // real lines staged through the tile (see stage_in_dct); every stage reads its legs from shared memory
            stage_in_dct(sm, P, obase_in, gl, ql, tl, gl < P.G);
            __syncthreads();
            if constexpr (NS == 1) {
                X x[bpt<0>() * V * Sch::r(0)];
                if constexpr (C::RMODE == 3) load_smem<0>(x, sm, ql, tl);
                else load_smem_dct3<0>(x, sm, rw, ql, tl);
                compute<0>(x, lut, tl);
                __syncthreads();
                store_global_dct<0>(x, sm, P, obase_out, gl, ql, tl, gl < P.G);
            } else {
                {
                    X x[bpt<0>() * V * Sch::r(0)];
                    if constexpr (C::RMODE == 3) load_smem<0>(x, sm, ql, tl);
                    else load_smem_dct3<0>(x, sm, rw, ql, tl);
                    compute<0>(x, lut, tl);
                    __syncthreads();
                    store_smem<0>(x, sm, ql, tl);
                }
                __syncthreads();
                middle<1>(sm, lut, tid);
                constexpr int s = NS - 1;
                int qs, ts;
                tmap<C::SMAP>(tid, qs, ts);
                const uint32_t gs = grp * Q + qs;
                X x[bpt<s>() * V * Sch::r(s)];
                load_smem<s>(x, sm, qs, ts);
                compute<s>(x, lut, ts);
                __syncthreads();
                store_global_dct<s>(x, sm, P, obase_out, gs, qs, ts, gs < P.G);
            }
        } else if constexpr (NS == 1) {
            X x[bpt<0>() * V * Sch::r(0)];
            if constexpr (C::RMODE == 2) load_global_c2r<0>(x, in_line, rw, tl, gl < P.G);
            else if constexpr (C::RMODE == 3 || C::RMODE == 4) load_global_dct<0>(x, P, obase_in, gl, tl, gl < P.G);
            else if constexpr (C::RMODE == 5) load_global_perm<0>(x, in_line, P.in_es / P.aux_u1, psel, P.aux_u1, P.aux_u0, tl, gl < P.G);
            else if constexpr (C::RMODE == 7) load_global_blue<0>(x, in_line, P, tl, gl < P.G);
            else load_global<0>(x, in_line, P.in_es, tl, gl < P.G);
            compute<0>(x, lut, tl);
            XO* out_line = (XO*)P.out + obase_out + (int64_t)gl * P.out_gs;
            if constexpr (C::RMODE == 1) store_global_r2c<0>(x, sm, out_line, rw, ql, tl, gl < P.G, P);
            else if constexpr (C::RMODE == 3 || C::RMODE == 4) store_global_dct<0>(x, sm, P, obase_out, gl, ql, tl, gl < P.G);
            else if constexpr (C::RMODE == 6) store_global_perm<0>(x, out_line, P.out_es / P.aux_u1, psel, P.aux_u1, P.aux_u0, tl, gl < P.G, P);
            else if constexpr (C::RMODE >= 7) store_global_blue<0>(x, out_line, P, tl, gl < P.G);
            else store_global<0>(x, out_line, P.out_es, tl, gl < P.G, P, twl(P, gl, o0, o1, o2), (uint32_t)ql);
        } else {
            {
                X x[bpt<0>() * V * Sch::r(0)];
                if constexpr (C::RMODE == 2) load_global_c2r<0>(x, in_line, rw, tl, gl < P.G);
                else if constexpr (C::RMODE == 3 || C::RMODE == 4) load_global_dct<0>(x, P, obase_in, gl, tl, gl < P.G);
                else if constexpr (C::RMODE == 5) load_global_perm<0>(x, in_line, P.in_es / P.aux_u1, psel, P.aux_u1, P.aux_u0, tl, gl < P.G);
                else if constexpr (C::RMODE == 7) load_global_blue<0>(x, in_line, P, tl, gl < P.G);
                else load_global<0>(x, in_line, P.in_es, tl, gl < P.G);
                hook();
                compute<0>(x, lut, tl);
                store_smem<0>(x, sm, ql, tl);
            }
            __syncthreads();
            if constexpr ((XF & XF_DISCARD) != 0) { if (!(P.aux_u1 & 1u)) discard_tile(P, obase_in, grp, tid); }   // aux_u1 bit 0: tuning switch
            middle<1>(sm, lut, tid);
            {
                constexpr int s = NS - 1;
                int qs, ts;
                tmap<C::SMAP>(tid, qs, ts);
                const uint32_t gs = grp * Q + qs;
                X x[bpt<s>() * V * Sch::r(s)];
                load_smem<s>(x, sm, qs, ts);
                compute<s>(x, lut, ts);
                XO* out_line = (XO*)P.out + obase_out + (int64_t)gs * P.out_gs;
                if constexpr (C::RMODE == 1) {
                    __syncthreads();     // every last-stage read of the tile is done before it is overwritten
                    store_global_r2c<s>(x, sm, out_line, rw, qs, ts, gs < P.G, P);
                } else if constexpr (C::RMODE == 3 || C::RMODE == 4) {
                    if constexpr (C::RMODE == 3 || C::LAYOUT == LAY_LINE) __syncthreads();   // the store goes through the tile
                    store_global_dct<s>(x, sm, P, obase_out, gs, qs, ts, gs < P.G);
                } else if constexpr (C::RMODE == 6) {
                    store_global_perm<s>(x, out_line, P.out_es / P.aux_u1, psel, P.aux_u1, P.aux_u0, ts, gs < P.G, P);
                } else if constexpr (C::RMODE >= 7) {
                    store_global_blue<s>(x, out_line, P, ts, gs < P.G);
                } else {
                    store_global<s>(x, out_line, P.out_es, ts, gs < P.G, P, twl(P, gs, o0, o1, o2), (uint32_t)qs);
                }
            }
        }
    }
};

#if defined(__CUDACC__)
template <class C>
__global__ void __launch_bounds__(C::THREADS, C::MINB) stockham_kernel(const __grid_constant__ b2_pass_params P) {
    extern __shared__ __align__(16) unsigned char b2_smem_raw[];
    Engine<C>::run(P, b2_smem_raw);
}
#endif

}  // namespace b200fft
