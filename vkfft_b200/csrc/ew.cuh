// Elementwise passes used when an operator cannot be fused into a shared-memory pass because the line does not
// fit on chip: Bluestein chirp / zero-pad, filter multiply and post-chirp around a multi-launch Four-Step
// (the reference runs its upload chain twice for this case, vkFFT_RunApp.h:158-204), and the Hermitian post-/pre-pass
// of long even-length R2C / C2R (the reference's separate VkFFT_main_R2C kernel,
// vkFFT_R2C_even_decomposition.h:40-241, launched at vkFFT_RunApp.h:205-231).
#pragma once
#include <math.h>

#include "pass_params.h"
#include "stockham.cuh"

namespace b200fft {

enum { B2_EW_COPY_MUL = 0, B2_EW_R2C_POST = 1, B2_EW_C2R_PRE = 2,
       B2_EW_DCT2_POST_COLS = 3,   // long strided DCT-II: split + phase of rows (k, N-k); items = neighbouring columns
       B2_EW_DCT3_PRE_COLS = 4,    // long strided DCT-III: phase + merge of rows (k, N-k)
       B2_EW_CONV = 5,             // convolution: spectrum (x) kernel, per feature or as a 2x2 / 3x3 matrix-vector product
       // odd-length R2C / C2R of lengths the single-launch kernel cannot take (composed with a C2C plan on scratch):
       B2_EW_REAL_TO_CPLX = 6,     // real line (scalar strides) -> complex line with zero imaginary part
       B2_EW_HERM_EXPAND = 7,      // half spectrum (n/2+1 points) -> full spectrum of n points, X[n-k] = conj X[k]
       B2_EW_CPLX_TO_REAL = 8,     // real part of a complex line -> real line (scalar strides), optional scale
       // DCT / DST of lengths the single-launch kernel cannot take: the operator's load side and store side as launches of
       // their own around a C2C plan on scratch (one real line per complex line).  store_io = B2_IO_DCT1/2/3/DCT4_ODD/DST1,
       // aux_u0 = logical real length N, aux_u1 = complex length, dst_flags as in generic.cuh
       B2_EW_R2R_PRE = 9, B2_EW_R2R_POST = 10,
       B2_EW_ZERO = 11,            // clear P.n items of every line (aux_u0 = 1: items and strides count scalars, not complex elements)
       B2_EW_CONV_REAL = 12 };     // B2_EW_CONV on real elements (DCT / DST spectra): offsets and strides count scalars
// B2_EW_CONV packs its options into aux_u0: bits 0-7 features per vector, 8-11 matrix size (0 = per-feature product),
// 12 symmetric kernel, 13-14 conjugation (1 sequence, 2 kernel), 15 cross-power-spectrum normalisation; aux_u1 = kernels
enum { B2_CONV_SYM = 1u << 12, B2_CONV_CONJ_SEQ = 1u << 13, B2_CONV_CONJ_KER = 1u << 14, B2_CONV_XPS = 1u << 15 };
enum { B2_EW_THREADS = 256, B2_EW_PER_THREAD = 8 };

// HALF: half-precision storage on both sides (32-bit complex elements, cplx.cuh), FP32 arithmetic -- the Hermitian passes only
// (B2_EW_R2C_POST / B2_EW_C2R_PRE of a long even-length R2C / C2R whose buffers are all half)
template <typename T, bool HALF = false>
struct Elementwise {
    using X = cpx<T>;
    B2_D static X ldx(const X* p) { return *p; }
    B2_D static X ldx(const uint32_t* p) { float re, im; b2_h2_to_f2(*p, re, im); return mk<T>((T)re, (T)im); }
    B2_D static void stx(X* p, X a) { *p = a; }
    B2_D static void stx(uint32_t* p, X a) { *p = b2_f2_to_h2((float)a.x, (float)a.y); }

    // pairs (k, n-k), k = 0 .. n/2 ; n = P.n complex points of the half-length transform, aux0[k] = e^{-2 pi i k/(2n)}
    template <class XS>
    B2_D static void hermitian(const b2_pass_params& P, const XS* in, XS* out, uint32_t j0, bool do_scale, T sc) {
        const uint32_t n = P.n;
        const X* w = (const X*)P.aux0;
#pragma unroll
        for (int i = 0; i < B2_EW_PER_THREAD; ++i) {
            const uint32_t k = j0 + i * B2_EW_THREADS;
            if (k > n / 2) break;
            const uint32_t kc = n - k;                    // partner index (n for k = 0)
            if (P.load_io == B2_EW_R2C_POST) {
                const X zk = ldx(in + (int64_t)k * P.in_es), zc = ldx(in + (int64_t)(kc == n ? 0 : kc) * P.in_es);
                // X[k] = 1/2 (Zk + conj Zc) - i/2 w_k (Zk - conj Zc)
                auto f = [&](X a, X bconj, X wk) {
                    const X s = a + bconj, d = (a - bconj) * wk;
                    X r = mk<T>(T(0.5) * (s.x + d.y), T(0.5) * (s.y - d.x));
                    return do_scale ? r * sc : r;
                };
                const X xk = f(zk, conj(zc), ld_lut(w + k));
                const X xc = f(zc, conj(zk), ld_lut(w + kc));
                stx(out + (int64_t)k * P.out_es, xk);
                if (kc != k) stx(out + (int64_t)kc * P.out_es, xc);
            } else {
                const X xk = ldx(in + (int64_t)k * P.in_es), xc = ldx(in + (int64_t)kc * P.in_es);
                // Zin[k] = (Xk + conj Xc) + i conj(w_k) (Xk - conj Xc)
                auto f = [&](X a, X bconj, X wk) {
                    const X s = a + bconj, d = mulc(a - bconj, wk);
                    return mk<T>(s.x - d.y, s.y + d.x);
                };
                const X zk = f(xk, conj(xc), ld_lut(w + k));
                const X zc = f(xc, conj(xk), ld_lut(w + kc));
                stx(out + (int64_t)k * P.out_es, zk);
                if (kc != k && kc != n) stx(out + (int64_t)kc * P.out_es, zc);
            }
        }
    }

    // B2_EW_CONV on real elements (DCT / DST spectra): the same layout rules, offsets and strides in scalars, and no
    // conjugation or normalisation options.  The vector is held in named registers rather than an array, so that this
    // operation adds no stack frame to the kernel the other operations share.
    B2_D static void conv_real(const b2_pass_params& P, int64_t in_off, int64_t out_off, uint32_t j0) {
        const T* rin = (const T*)P.in + in_off;
        T* rout = (T*)P.out + out_off;
        const uint32_t C = P.aux_u0 & 0xff, M = (P.aux_u0 >> 8) & 0xf, NK = P.aux_u1 ? P.aux_u1 : 1;
        const bool sym = (P.aux_u0 & B2_CONV_SYM) != 0;
        const int64_t batch_stride = (int64_t)C * P.in_es;
        const T* __restrict__ ker = (const T*)P.aux0 + in_off % batch_stride;
        const uint32_t kplanes = M >= 2 ? (sym ? M * (M + 1) / 2 : M * M) : C;
#pragma unroll 2
        for (int i = 0; i < B2_EW_PER_THREAD; ++i) {
            const uint32_t j = j0 + i * B2_EW_THREADS;
            if (j >= P.n) break;
            if (M >= 2) {
                const T x0 = rin[j], x1 = rin[P.in_es + j], x2 = M > 2 ? rin[2 * P.in_es + j] : T(0);
                for (uint32_t k = 0; k < NK; ++k) {
                    const T* kk = ker + (int64_t)k * kplanes * P.out_es + j;
                    auto w = [&](uint32_t r, uint32_t c) {
                        uint32_t idx;
                        if (sym) { const uint32_t a = r < c ? r : c, b = r < c ? c : r; idx = a * M - a * (a - 1) / 2 + (b - a); }
                        else idx = r * M + c;
                        return kk[(int64_t)idx * P.out_es];
                    };
                    for (uint32_t r = 0; r < M; ++r) {
                        T acc = w(r, 0) * x0 + w(r, 1) * x1;
                        if (M > 2) acc += w(r, 2) * x2;
                        rout[(int64_t)k * batch_stride + (int64_t)r * P.in_es + j] = acc;
                    }
                }
            } else {
                for (uint32_t c = 0; c < C; ++c) {
                    const T xv = rin[(int64_t)c * P.in_es + j];
                    for (uint32_t k = 0; k < NK; ++k)
                        rout[(int64_t)k * batch_stride + (int64_t)c * P.in_es + j] = ker[(int64_t)(k * kplanes + c) * P.out_es + j] * xv;
                }
            }
        }
    }

    // P.load_io = operation, P.n = items per line (elements, or pairs for the R2C passes), P.tpl = chunks per line,
    // P.inverse = swap re/im right after the load, P.inner_inverse = swap right before the store.
    B2_D static void run(const b2_pass_params& P) {
        const uint32_t chunks = P.tpl;
        uint32_t rest = blockIdx.x;
        const uint32_t chunk = rest % chunks; rest /= chunks;
        const uint32_t gl = rest % P.G; rest /= P.G;
        const uint32_t o0 = rest % P.nb[0]; rest /= P.nb[0];
        const uint32_t o1 = rest % P.nb[1]; rest /= P.nb[1];
        const uint32_t o2 = rest;
        const int64_t in_off = (int64_t)o0 * P.in_bs[0] + (int64_t)o1 * P.in_bs[1] + (int64_t)o2 * P.in_bs[2] + (int64_t)gl * P.in_gs;
        const int64_t out_off = (int64_t)o0 * P.out_bs[0] + (int64_t)o1 * P.out_bs[1] + (int64_t)o2 * P.out_bs[2] + (int64_t)gl * P.out_gs;
        const T sc = (T)P.scale;
        const bool do_scale = (P.ops & B2_OP_SCALE) != 0;
        const uint32_t j0 = chunk * (B2_EW_THREADS * B2_EW_PER_THREAD) + threadIdx.x;
        if constexpr (HALF) {
            hermitian(P, (const uint32_t*)P.in + in_off, (uint32_t*)P.out + out_off, j0, do_scale, sc);
            return;
        }
        const X* in = (const X*)P.in + in_off;
        X* out = (X*)P.out + out_off;
        if (P.load_io == B2_EW_COPY_MUL) {
#pragma unroll
            for (int i = 0; i < B2_EW_PER_THREAD; ++i) {
                const uint32_t j = j0 + i * B2_EW_THREADS;
                if (j >= P.out_len) break;
                X v = mk<T>(T(0), T(0));
                if (j < P.in_len) {
                    v = in[(int64_t)j * P.in_es];
                    if (P.inverse) v = swp(v);
                    if (P.ops & B2_OP_MUL_IN) v = v * ld_lut((const X*)P.aux0 + j);
                }
                if (do_scale) v = v * sc;
                if (P.inner_inverse) v = swp(v);
                out[(int64_t)j * P.out_es] = v;
            }
        } else if (P.load_io == B2_EW_REAL_TO_CPLX || P.load_io == B2_EW_CPLX_TO_REAL || P.load_io == B2_EW_HERM_EXPAND) {
            // the real side is addressed in scalars: in_off / out_off were accumulated from scalar strides
            const T* rin = (const T*)P.in + in_off;
            T* rout = (T*)P.out + out_off;
#pragma unroll
            for (int i = 0; i < B2_EW_PER_THREAD; ++i) {
                const uint32_t j = j0 + i * B2_EW_THREADS;
                if (j >= P.n) break;
                if (P.load_io == B2_EW_REAL_TO_CPLX) {
                    out[j] = mk<T>(rin[(int64_t)j * P.in_es], T(0));
                } else if (P.load_io == B2_EW_CPLX_TO_REAL) {
                    T v = in[j].x;
                    if (do_scale) v *= sc;
                    rout[(int64_t)j * P.out_es] = v;
                } else {
                    // j runs over the n/2+1 stored points; P.aux_u0 = n
                    const X v = in[j];
                    out[j] = v;
                    if (j != 0 && 2 * j != P.aux_u0) out[P.aux_u0 - j] = conj(v);
                }
            }
        } else if (P.load_io == B2_EW_ZERO) {
            T* rout = (T*)P.out + out_off;
#pragma unroll
            for (int i = 0; i < B2_EW_PER_THREAD; ++i) {
                const uint32_t j = j0 + i * B2_EW_THREADS;
                if (j >= P.n) break;
                if (P.aux_u0) rout[(int64_t)j * P.out_es] = T(0);
                else out[(int64_t)j * P.out_es] = mk<T>(T(0), T(0));
            }
        } else if (P.load_io == B2_EW_R2R_PRE || P.load_io == B2_EW_R2R_POST) {
            const T* rin = (const T*)P.in + in_off;       // real side in scalars
            T* rout = (T*)P.out + out_off;
            const int N = (int)P.aux_u0, nc = (int)P.aux_u1, type = (int)P.store_io;
            const X* __restrict__ tab = (const X*)P.aux0;
            auto mak = [&](int p2) { return (p2 < (nc + 1) / 2) ? 2 * p2 : 2 * (nc - 1 - p2) + 1; };
            auto src_i = [&](int i2, int L) { return (P.dst_flags & B2_DST_REV_IN) ? L - 1 - i2 : i2; };
            auto sg_in = [&](int i2) { return ((P.dst_flags & B2_DST_NEG_ODD_IN) && (i2 & 1)) ? T(-1) : T(1); };
            auto dst_i = [&](int k2, int L) { return (P.dst_flags & B2_DST_REV_OUT) ? L - 1 - k2 : k2; };
            auto sg_out = [&](int k2) { return ((P.dst_flags & B2_DST_ALT_OUT) && (k2 & 1)) ? T(-1) : T(1); };
#pragma unroll 2
            for (int i = 0; i < B2_EW_PER_THREAD; ++i) {
                const int j = (int)(j0 + i * B2_EW_THREADS);
                if ((uint32_t)j >= P.n) break;
                if (P.load_io == B2_EW_R2R_PRE) {            // j runs over the nc complex points
                    X v = mk<T>(T(0), T(0));
                    if (type == B2_IO_DCT2) {
                        const int sidx = mak(j);
                        v.x = sg_in(sidx) * rin[(int64_t)src_i(sidx, N) * P.in_es];
                    } else if (type == B2_IO_DCT3) {
                        const T a0 = rin[(int64_t)src_i(j, N) * P.in_es];
                        const T a1 = j == 0 ? T(0) : rin[(int64_t)src_i(N - j, N) * P.in_es];
                        v = mulc(mk<T>(a0, -a1), ld_lut(tab + j));
                    } else if (type == B2_IO_DCT1) {
                        v.x = rin[(int64_t)(j < N ? j : nc - j) * P.in_es];
                    } else if (type == B2_IO_DST1) {
                        if (j != 0 && j != N + 1) v.x = (j <= N ? T(1) : T(-1)) * rin[(int64_t)(j <= N ? j - 1 : nc - j - 1) * P.in_es];
                    } else {                                  // B2_IO_DCT4_ODD (any N)
                        if (j < N) v = ld_lut(tab + j) * rin[(int64_t)src_i(j, N) * P.in_es];
                    }
                    out[j] = v;
                } else {                                       // j runs over the N real outputs (DCT-III: over the nc points)
                    T y;
                    int o = j;
                    if (type == B2_IO_DCT2) {
                        const X a = in[j], b = conj(in[j == 0 ? 0 : nc - j]);
                        y = (ld_lut(tab + j) * (a + b)).x;
                        o = dst_i(j, N);
                    } else if (type == B2_IO_DCT3) {
                        o = mak(j);
                        y = sg_out(o) * in[j].x;
                    } else if (type == B2_IO_DCT1) {
                        y = in[j].x;
                    } else if (type == B2_IO_DST1) {
                        y = -in[j + 1].y;
                    } else {
                        y = sg_out(j) * T(2) * (in[j] * ld_lut((const X*)P.aux1 + j)).x;
                    }
                    if (do_scale) y *= sc;
                    rout[(int64_t)o * P.out_es] = y;
                }
            }
        } else if (P.load_io == B2_EW_CONV) {
            // (vkFFT_Convolution.h:125 does this inside the last-axis kernel)  One thread = one frequency point j of
            // input batch gl: every feature of the point is read before anything is written, so the product runs in place.
            //   in_es / out_es = distance between feature planes of the buffer / of the kernel, C * in_es = batch stride.
            // A line is a whole plane (packed layout) or one row of it (padded pitches: the gaps between rows are not the
            // transform's to touch); its place inside the batch is also its place inside every plane of the kernel.
            const uint32_t C = P.aux_u0 & 0xff, M = (P.aux_u0 >> 8) & 0xf, NK = P.aux_u1 ? P.aux_u1 : 1;
            const bool sym = (P.aux_u0 & B2_CONV_SYM) != 0, cseq = (P.aux_u0 & B2_CONV_CONJ_SEQ) != 0,
                       cker = (P.aux_u0 & B2_CONV_CONJ_KER) != 0, xps = (P.aux_u0 & B2_CONV_XPS) != 0;
            const int64_t batch_stride = (int64_t)C * P.in_es;
            const X* __restrict__ ker = (const X*)P.aux0 + in_off % batch_stride;
            const uint32_t kplanes = M >= 2 ? (sym ? M * (M + 1) / 2 : M * M) : C;
            auto finish = [&](X v) {
                if (xps) {
                    const T a = sqrt(v.x * v.x + v.y * v.y);
                    if (a > T(0)) v = v * (T(1) / a);
                }
                return v;
            };
#pragma unroll 2
            for (int i = 0; i < B2_EW_PER_THREAD; ++i) {
                const uint32_t j = j0 + i * B2_EW_THREADS;
                if (j >= P.n) break;
                if (M >= 2) {
                    X x[3];
                    for (uint32_t c = 0; c < M; ++c) { x[c] = in[(int64_t)c * P.in_es + j]; if (cseq) x[c] = conj(x[c]); }
                    for (uint32_t k = 0; k < NK; ++k) {
                        const X* kk = ker + (int64_t)k * kplanes * P.out_es + j;
                        for (uint32_t r = 0; r < M; ++r) {
                            X acc = mk<T>(T(0), T(0));
                            for (uint32_t c = 0; c < M; ++c) {
                                uint32_t idx;
                                if (sym) { const uint32_t a = r < c ? r : c, b = r < c ? c : r; idx = a * M - a * (a - 1) / 2 + (b - a); }
                                else idx = r * M + c;
                                X w = kk[(int64_t)idx * P.out_es];
                                if (cker) w = conj(w);
                                acc = acc + w * x[c];
                            }
                            out[(int64_t)k * batch_stride + (int64_t)r * P.in_es + j] = finish(acc);
                        }
                    }
                } else {
                    for (uint32_t c = 0; c < C; ++c) {
                        X xv = in[(int64_t)c * P.in_es + j];
                        if (cseq) xv = conj(xv);
                        for (uint32_t k = 0; k < NK; ++k) {
                            X w = ker[(int64_t)(k * kplanes + c) * P.out_es + j];
                            if (cker) w = conj(w);
                            out[(int64_t)k * batch_stride + (int64_t)c * P.in_es + j] = finish(w * xv);
                        }
                    }
                }
            }
        } else if (P.load_io == B2_EW_CONV_REAL) {
            conv_real(P, in_off, out_off, j0);
        } else if (P.load_io == B2_EW_DCT2_POST_COLS || P.load_io == B2_EW_DCT3_PRE_COLS) {
            // this CTA's "line" is row k = gl of a complex-view column block; its partner is row N-k (N = aux_u0);
            // items are the columns (unit stride).  aux0[k] = e^{-i pi k/2N}
            const int64_t N = (int64_t)P.aux_u0, k = (int64_t)gl, kc = N - k;
            const X ck = ld_lut((const X*)P.aux0 + k);
            const X cc = (k == 0) ? ck : ld_lut((const X*)P.aux0 + kc);
            const int64_t pin = (kc - k) * P.in_gs, pout = (kc - k) * P.out_gs;
#pragma unroll
            for (int i = 0; i < B2_EW_PER_THREAD; ++i) {
                const uint32_t j = j0 + i * B2_EW_THREADS;
                if (j >= P.n) break;
                const X a = in[j];
                if (P.load_io == B2_EW_DCT2_POST_COLS) {
                    const X b = (k == 0) ? a : in[pin + j];
                    const X s1 = ck * (a + conj(b)), d1 = ck * (a - conj(b));
                    X xk = mk<T>(s1.x, d1.y);
                    if (do_scale) xk = xk * sc;
                    out[j] = xk;
                    if (k != 0 && kc != k) {
                        const X s2 = cc * (b + conj(a)), d2 = cc * (b - conj(a));
                        X xc = mk<T>(s2.x, d2.y);
                        if (do_scale) xc = xc * sc;
                        out[pout + j] = xc;
                    }
                } else {
                    const X b = (k == 0) ? mk<T>(T(0), T(0)) : in[pin + j];
                    out[j] = mulc(mk<T>(a.x + b.y, a.y - b.x), ck);
                    if (k != 0 && kc != k) out[pout + j] = mulc(mk<T>(b.x + a.y, b.y - a.x), cc);
                }
            }
        } else {
            hermitian(P, in, out, j0, do_scale, sc);
        }
    }
};

#if defined(__CUDACC__)
template <typename T, bool HALF = false>
__global__ void __launch_bounds__(B2_EW_THREADS) elementwise_kernel(const __grid_constant__ b2_pass_params P) {
    Elementwise<T, HALF>::run(P);
}
#endif

}  // namespace b200fft
