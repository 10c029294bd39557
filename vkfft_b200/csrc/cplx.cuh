// Complex arithmetic + host/device portability macros shared by every kernel in the engine.
//
// The same headers are compiled three ways:
//   * nvcc for sm_90a             -> the product (libb200fft.so)
//   * g++ with tests/emu/cuda_emu.h -> a CPU "one OS thread per CUDA thread" emulation used only by
//                                    the CPU test-suite to check index maps / bank conflicts
//   * g++ for the host planner (only the POD parts)
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2_HD __host__ __device__ __forceinline__
#define B2_D __device__ __forceinline__
#else
#define B2_HD inline
#define B2_D inline
#endif

namespace b200fft {

template <typename T>
struct alignas(2 * sizeof(T)) cpx {
    T x, y;
};
using cf32 = cpx<float>;
using cf64 = cpx<double>;

template <typename T> B2_HD cpx<T> mk(T a, T b) { cpx<T> r; r.x = a; r.y = b; return r; }

// Half-precision STORAGE (the reference's halfPrecision / halfPrecisionMemoryOnly, vkFFT_Structs.h:210-211: "data is read and
// written as half, all computations are float"): one complex element in HBM is 32 bits, (re, im) as two IEEE binary16 values,
// re in the low half.  Conversion happens in the HBM load / store of the first / last stage, everything in between is FP32.
#if defined(__CUDA_ARCH__)
B2_D void b2_h2_to_f2(uint32_t h, float& re, float& im) {
    asm("{\n\t.reg .b16 lo, hi;\n\tmov.b32 {lo, hi}, %2;\n\tcvt.f32.f16 %0, lo;\n\tcvt.f32.f16 %1, hi;\n\t}" : "=f"(re), "=f"(im) : "r"(h));
}
B2_D uint32_t b2_f2_to_h2(float re, float im) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(im), "f"(re));     // d = {hi: first operand, lo: second operand}
    return r;
}
#else
// host / emulation: plain software conversion (round to nearest even, overflow to infinity)
inline float b2_half_bits_to_float(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000) << 16, ex = (h >> 10) & 31, man = h & 1023;
    uint32_t bits;
    if (ex == 0) {
        if (man == 0) bits = sign;
        else { int e = -1; uint32_t m = man; do { ++e; m <<= 1; } while (!(m & 1024)); bits = sign | ((uint32_t)(112 - e) << 23) | ((m & 1023) << 13); }
    } else if (ex == 31) bits = sign | 0x7f800000u | (man << 13);
    else bits = sign | ((ex + 112) << 23) | (man << 13);
    float f; __builtin_memcpy(&f, &bits, 4); return f;
}
inline uint16_t b2_float_to_half_bits(float f) {
    uint32_t x; __builtin_memcpy(&x, &f, 4);
    const uint32_t sign = (x >> 16) & 0x8000; x &= 0x7fffffff;
    if (x >= 0x7f800000u) return (uint16_t)(sign | 0x7c00 | (x > 0x7f800000u ? 0x200 : 0));
    if (x >= 0x477ff000u) return (uint16_t)(sign | 0x7c00);                 // rounds to infinity
    if (x < 0x33000001u) return (uint16_t)sign;                              // rounds to zero
    if (x < 0x38800000u) {                                                   // subnormal half: units of 2^-24, ties to even
        const double scaled = (double)(f < 0 ? -f : f) * 16777216.0;
        uint32_t n = (uint32_t)scaled;
        const double fr = scaled - n;
        if (fr > 0.5 || (fr == 0.5 && (n & 1))) ++n;
        return (uint16_t)(sign | n);
    }
    uint32_t m = x + 0xc8000000u + 0xfff + ((x >> 13) & 1);                  // rebias exponent, round to nearest even
    return (uint16_t)(sign | (m >> 13));
}
inline void b2_h2_to_f2(uint32_t h, float& re, float& im) { re = b2_half_bits_to_float((uint16_t)(h & 0xffff)); im = b2_half_bits_to_float((uint16_t)(h >> 16)); }
inline uint32_t b2_f2_to_h2(float re, float im) { return (uint32_t)b2_float_to_half_bits(re) | ((uint32_t)b2_float_to_half_bits(im) << 16); }
#endif

// FP32 complex arithmetic on the device is spelled out with the round-to-nearest intrinsics, which the compiler never
// contracts or reorders: every kernel that runs the same stage code -- a stand-alone pass or the same pass inside the
// fused Four-Step launch -- then rounds identically, whatever code surrounds it.  The product rounds a.x*b.x (a.y*b.x)
// before the fused multiply-add.  Host code, the CPU emulation and FP64 use the plain component-wise form.
template <typename T> B2_HD cpx<T> operator+(cpx<T> a, cpx<T> b) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) return mk<T>(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
#endif
    return mk<T>(a.x + b.x, a.y + b.y);
}
template <typename T> B2_HD cpx<T> operator-(cpx<T> a, cpx<T> b) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) return mk<T>(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y));
#endif
    return mk<T>(a.x - b.x, a.y - b.y);
}
template <typename T> B2_HD cpx<T> operator*(cpx<T> a, cpx<T> b) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) return mk<T>(__fmaf_rn(-a.y, b.y, __fmul_rn(a.x, b.x)), __fmaf_rn(a.x, b.y, __fmul_rn(a.y, b.x)));
#endif
    return mk<T>(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
template <typename T> B2_HD cpx<T> operator*(cpx<T> a, T s) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) return mk<T>(__fmul_rn(a.x, s), __fmul_rn(a.y, s));
#endif
    return mk<T>(a.x * s, a.y * s);
}
// a * conj(b)
template <typename T> B2_HD cpx<T> mulc(cpx<T> a, cpx<T> b) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) return mk<T>(__fmaf_rn(a.y, b.y, __fmul_rn(a.x, b.x)), __fmaf_rn(-a.x, b.y, __fmul_rn(a.y, b.x)));
#endif
    return mk<T>(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y);
}
// c + a * s  (real scalar s)
template <typename T> B2_HD cpx<T> fma_s(cpx<T> a, T s, cpx<T> c) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) return mk<T>(__fmaf_rn(a.x, s, c.x), __fmaf_rn(a.y, s, c.y));
#endif
    return mk<T>(c.x + a.x * s, c.y + a.y * s);
}
template <typename T> B2_HD cpx<T> conj(cpx<T> a) { return mk<T>(a.x, -a.y); }
// multiply by -i  (forward-transform quarter turn):  (x + iy)(-i) = y - ix
template <typename T> B2_HD cpx<T> mul_mi(cpx<T> a) { return mk<T>(a.y, -a.x); }
// multiply by +i
template <typename T> B2_HD cpx<T> mul_pi(cpx<T> a) { return mk<T>(-a.y, a.x); }
// swap real/imag: IFFT(x) = swap(FFT(swap(x)))  -- how every inverse plan runs forward code
template <typename T> B2_HD cpx<T> swp(cpx<T> a) { return mk<T>(a.y, a.x); }

}  // namespace b200fft
