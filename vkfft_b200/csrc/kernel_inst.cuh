// Expands kernel_list.def into registry entries.  Included by the CUDA shard translation units (product)
// and, with B2_EMU defined, by the CPU emulation used in tests.
#pragma once
#include <cstdio>

#include "kernel_registry.h"
#include "stockham.cuh"
#include "generic.cuh"
#include "pipe.cuh"
#include "fused4.cuh"
#if !defined(B2_EMU) || defined(B2_EMU_CLUSTER)
#include "cluster4.cuh"
#endif
#include "ew.cuh"

#if !defined(B2_EMU)
#include <cuda_runtime.h>
#endif

namespace b200fft {

#if !defined(B2_EMU)
// cudaLaunchKernel reports THIS launch's status; `kernel<<<>>>` + cudaGetLastError() would also pick up a stale
// non-sticky error some other library left behind in the calling process (seen with NCCL's peer-access setup)
inline int launch_checked(const void* kernel, unsigned grid, unsigned threads, size_t smem, void* stream, const b2_pass_params* P) {
    void* args[] = {const_cast<b2_pass_params*>(P)};
    return (int)cudaLaunchKernel(kernel, dim3(grid), dim3(threads), args, smem, (cudaStream_t)stream);
}
#endif

template <int KIND> struct KindTraits;
template <> struct KindTraits<B2_KIND_ROWS> {
    static constexpr int LMAP = MAP_TFAST, SMAP = MAP_TFAST, LAYOUT = LAY_LINE;
    static constexpr bool IN_UNIT = true, OUT_UNIT = true;
};
template <> struct KindTraits<B2_KIND_ROWS_TOUT> {
    static constexpr int LMAP = MAP_TFAST, SMAP = MAP_QFAST, LAYOUT = LAY_LINE;
    static constexpr bool IN_UNIT = true, OUT_UNIT = false;
};
template <> struct KindTraits<B2_KIND_COLS> {
    static constexpr int LMAP = MAP_QFAST, SMAP = MAP_QFAST, LAYOUT = LAY_ELEM;
    static constexpr bool IN_UNIT = false, OUT_UNIT = false;
};

template <typename T> struct PrecOf;
template <> struct PrecOf<float> { static constexpr int value = B2_PREC_F32; };
template <> struct PrecOf<double> { static constexpr int value = B2_PREC_F64; };

#if defined(B2_EMU)
// the emulation refuses what cudaLaunchKernel would refuse (block size, shared memory, grid): report it like a failed launch
inline int emu_refused() {
    const bool r = b2emu::st().launch_refused || b2emu::st().smem_oob || b2emu::st().hazards.load() != 0;
    if (b2emu::st().hazards.load())
        fprintf(stderr, "b2emu racecheck: %d shared-memory hazards, first at byte %u (kind %u: 1 WAW, 2 WAR, 3 RAW)\n",
                b2emu::st().hazards.load(), b2emu::st().hazard_addr, b2emu::st().hazard_kind);
    b2emu::st().launch_refused = false;
    b2emu::st().smem_oob = false;
    b2emu::st().hazards = 0;
    return r ? 1 : 0;
}
template <class C>
int launch_impl(const b2_pass_params* P, unsigned grid, void*) {
    const b2_pass_params PP = *P;
    b2emu::launch(grid, C::THREADS, C::SMEM_BYTES, [&](unsigned char* sm) { Engine<C>::run(PP, sm); },
                  b2emu::st().log);
    return emu_refused();
}
template <class C> int prepare_impl() { return 0; }
#else
template <class C>
int launch_impl(const b2_pass_params* P, unsigned grid, void* stream) {
    return launch_checked((const void*)stockham_kernel<C>, grid, C::THREADS, C::SMEM_BYTES, stream, P);
}
template <class C>
int prepare_impl() {
    if (C::SMEM_BYTES > 48 * 1024)
        return (int)cudaFuncSetAttribute(stockham_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         C::SMEM_BYTES);
    return 0;
}
#endif

// ---- generic (runtime-scheduled) kernel: one entry per precision ------------------------------------------------
template <typename T> inline size_t generic_smem_bytes(const b2_pass_params* P) {
    return (size_t)2 * P->q * P->line_stride * 2 * sizeof(T);
}
#if defined(B2_EMU)
template <typename T, int RMAX>
int generic_launch(const b2_pass_params* P, unsigned grid, void*) {
    const b2_pass_params PP = *P;
    b2emu::launch(grid, PP.tpl * PP.q, generic_smem_bytes<T>(P), [&](unsigned char* sm) { Generic<T, RMAX>::run(PP, sm); },
                  b2emu::st().log);
    return emu_refused();
}
template <typename T, int RMAX> int generic_prepare() { return 0; }
#else
template <typename T, int RMAX>
int generic_launch(const b2_pass_params* P, unsigned grid, void* stream) {
    return launch_checked((const void*)generic_kernel<T, RMAX>, grid, P->tpl * P->q, generic_smem_bytes<T>(P), stream, P);
}
template <typename T, int RMAX>
int generic_prepare() {
    return (int)cudaFuncSetAttribute(generic_kernel<T, RMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
}
#endif
// registry key n = radix class (8, 11, 16)
template <typename T, int RMAX>
struct GenericRegistrar {
    b2_kernel_info info;
    explicit GenericRegistrar(const char* name) {
        info = b2_kernel_info{};
        info.kind = B2_KIND_GENERIC; info.prec = PrecOf<T>::value; info.n = RMAX; info.inv = 0; info.ops = 0;
        info.launch = &generic_launch<T, RMAX>;
        info.prepare = &generic_prepare<T, RMAX>;
        info.name = name;
        b2_register_kernel(&info);
    }
};

// ---- elementwise helper kernel ---------------------------------------------------------------------------------------
#if defined(B2_EMU)
template <typename T, bool HALF>
int ew_launch(const b2_pass_params* P, unsigned grid, void*) {
    const b2_pass_params PP = *P;
    b2emu::launch(grid, B2_EW_THREADS, 0, [&](unsigned char*) { Elementwise<T, HALF>::run(PP); }, false);
    return emu_refused();
}
#else
template <typename T, bool HALF>
int ew_launch(const b2_pass_params* P, unsigned grid, void* stream) {
    return launch_checked((const void*)elementwise_kernel<T, HALF>, grid, B2_EW_THREADS, 0, stream, P);
}
#endif
// HALF: the half-storage Hermitian passes of long even-length R2C / C2R, registered with ops = B2_OP_HALF_IN | B2_OP_HALF_OUT
template <typename T, bool HALF = false>
struct ElementwiseRegistrar {
    b2_kernel_info info;
    explicit ElementwiseRegistrar(const char* name) {
        info = b2_kernel_info{};
        info.kind = B2_KIND_ELEMENTWISE; info.prec = PrecOf<T>::value;
        info.ops = HALF ? (B2_OP_HALF_IN | B2_OP_HALF_OUT) : 0;
        info.threads = B2_EW_THREADS;
        info.launch = &ew_launch<T, HALF>;
        info.name = name;
        b2_register_kernel(&info);
    }
};

template <int KIND, typename T, int TPL, int Q, int V, int MINB, bool INV, int OPS, int... Rs>
struct Registrar {
    using KT = KindTraits<KIND>;
    using Sch = RList<Rs...>;
    static constexpr int RMODE = (OPS & B2_OP_REAL_EVEN) ? (INV ? 2 : 1)
                               : ((OPS & B2_OP_DCT23) ? ((OPS & B2_OP_CONV) ? 12 : (INV ? 4 : 3)) : ((OPS & B2_OP_PERM_IN) ? 5 : ((OPS & B2_OP_PERM_OUT) ? 6 : ((OPS & B2_OP_BLUESTEIN) ? (INV ? 8 : 7) : ((OPS & B2_OP_CONV) ? 9 : ((OPS & B2_OP_BLUE_FUSED) ? 11 : 0))))));
    static constexpr int ST = ((OPS & B2_OP_HALF_IN) ? 1 : 0) | ((OPS & B2_OP_HALF_OUT) ? 2 : 0);   // half-precision storage
    using C = KCfg<T, Sch, TPL, Q, V, KT::LMAP, KT::SMAP, KT::LAYOUT, INV, (OPS & B2_OP_TWIDDLE_OUT), KT::IN_UNIT, KT::OUT_UNIT,
                   MINB, RMODE, ST>;
    b2_kernel_info info;
    explicit Registrar(const char* name) {
        info = b2_kernel_info{};
        info.kind = KIND; info.prec = PrecOf<T>::value; info.n = Sch::N; info.inv = INV; info.ops = OPS;
        info.threads = C::THREADS; info.q = Q; info.tpl = TPL; info.v = V; info.smem_bytes = C::SMEM_BYTES;
        info.ns = Sch::ns;
        for (int s = 0; s < Sch::ns; ++s) info.radices[s] = Sch::r(s);
        info.lut_size = Sch::lut_size;
        info.regs = MINB;                  // (the template parameter is the register budget; KCfg turns it into min blocks per SM)
        info.launch = &launch_impl<C>;
        info.prepare = &prepare_impl<C>;
        info.name = name;
        b2_register_kernel(&info);
    }
};

// ---- persistent TMA-fed variants (pipe.cuh) ------------------------------------------------------------------------
#if defined(B2_EMU)
template <class C, int NBUF>
int pipe_launch_impl(const b2_pass_params* P, unsigned grid, void*) {
    const b2_pass_params PP = *P;
    const unsigned g = grid < 3 ? grid : 3;       // few persistent CTAs so that the buffer ring wraps
    b2emu::launch(g, C::THREADS, PipeEngine<C, NBUF>::SMEM_BYTES, [&](unsigned char* sm) { PipeEngine<C, NBUF>::run(PP, sm); },
                  b2emu::st().log);
    return emu_refused();
}
template <class C, int NBUF> int pipe_prepare_impl() { return 0; }
#else
template <class C, int NBUF>
int pipe_launch_impl(const b2_pass_params* P, unsigned grid, void* stream) {
    static int resident = 0;
    if (!resident) {
        int dev = 0, sms = 0, per_sm = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, stockham_pipe_kernel<C, NBUF>, C::THREADS,
                                                      PipeEngine<C, NBUF>::SMEM_BYTES);
        resident = sms * (per_sm > 0 ? per_sm : 1);
    }
    const unsigned g = grid < (unsigned)resident ? grid : (unsigned)resident;
    return launch_checked((const void*)stockham_pipe_kernel<C, NBUF>, g, C::THREADS, PipeEngine<C, NBUF>::SMEM_BYTES, stream, P);
}
template <class C, int NBUF>
int pipe_prepare_impl() {
    return (int)cudaFuncSetAttribute(stockham_pipe_kernel<C, NBUF>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     PipeEngine<C, NBUF>::SMEM_BYTES);
}
#endif

template <int KIND, typename T, int TPL, int Q, int V, int REGS, int NBUF, bool INV, int... Rs>
struct PipeRegistrar {
    using KT = KindTraits<KIND>;
    using Sch = RList<Rs...>;
    using C = KCfg<T, Sch, TPL, Q, V, KT::LMAP, KT::SMAP, KT::LAYOUT, INV, 0, KT::IN_UNIT, KT::OUT_UNIT, REGS>;
    b2_kernel_info info;
    explicit PipeRegistrar(const char* name) {
        info = b2_kernel_info{};
        info.kind = KIND; info.prec = PrecOf<T>::value; info.n = Sch::N; info.inv = INV; info.ops = 0;
        info.threads = C::THREADS; info.q = Q; info.tpl = TPL; info.v = V; info.smem_bytes = PipeEngine<C, NBUF>::SMEM_BYTES;
        info.ns = Sch::ns;
        for (int s = 0; s < Sch::ns; ++s) info.radices[s] = Sch::r(s);
        info.lut_size = Sch::lut_size;
        info.pipelined = 1;
        info.launch = &pipe_launch_impl<C, NBUF>;
        info.prepare = &pipe_prepare_impl<C, NBUF>;
        info.name = name;
        b2_register_kernel(&info);
    }
};
template <bool EN, int KIND, typename T, int TPL, int Q, int V, int REGS, int NBUF, int... Rs>
struct MaybePipe {
    explicit MaybePipe(const char*) {}
};
template <int KIND, typename T, int TPL, int Q, int V, int REGS, int NBUF, int... Rs>
struct MaybePipe<true, KIND, T, TPL, Q, V, REGS, NBUF, Rs...> {
    PipeRegistrar<KIND, T, TPL, Q, V, REGS, NBUF, false, Rs...> f;
    PipeRegistrar<KIND, T, TPL, Q, V, REGS, NBUF, true, Rs...> i;
    explicit MaybePipe(const char* n) : f(n), i(n) {}
};

// every kind gets forward+inverse; COLS additionally gets the four-step twiddle-on-store variant
template <int KIND, typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct RegistrarSet {
    Registrar<KIND, T, TPL, Q, V, MINB, false, 0, Rs...> f;
    Registrar<KIND, T, TPL, Q, V, MINB, true, 0, Rs...> i;
    explicit RegistrarSet(const char* n) : f(n), i(n) {}
};
// contiguous lines additionally get the fused even-length real transforms (R2C on the forward kernel, C2R on the inverse)
template <typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct RegistrarSet<B2_KIND_ROWS, T, TPL, Q, V, MINB, Rs...> {
    Registrar<B2_KIND_ROWS, T, TPL, Q, V, MINB, false, 0, Rs...> f;
    Registrar<B2_KIND_ROWS, T, TPL, Q, V, MINB, true, 0, Rs...> i;
    Registrar<B2_KIND_ROWS, T, TPL, Q, V, MINB, false, B2_OP_REAL_EVEN, Rs...> fr;
    Registrar<B2_KIND_ROWS, T, TPL, Q, V, MINB, true, B2_OP_REAL_EVEN, Rs...> ir;
    explicit RegistrarSet(const char* n) : f(n), i(n), fr(n), ir(n) {}
};
template <typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct RegistrarSet<B2_KIND_COLS, T, TPL, Q, V, MINB, Rs...> {
    Registrar<B2_KIND_COLS, T, TPL, Q, V, MINB, false, 0, Rs...> f;
    Registrar<B2_KIND_COLS, T, TPL, Q, V, MINB, true, 0, Rs...> i;
    Registrar<B2_KIND_COLS, T, TPL, Q, V, MINB, false, B2_OP_TWIDDLE_OUT, Rs...> ft;
    Registrar<B2_KIND_COLS, T, TPL, Q, V, MINB, true, B2_OP_TWIDDLE_OUT, Rs...> it;
    explicit RegistrarSet(const char* n) : f(n), i(n), ft(n), it(n) {}
};

}  // namespace b200fft

namespace b200fft {
template <bool EN, int KIND, typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeSet {
    explicit MaybeSet(const char*) {}
};
template <int KIND, typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeSet<true, KIND, T, TPL, Q, V, MINB, Rs...> : RegistrarSet<KIND, T, TPL, Q, V, MINB, Rs...> {
    explicit MaybeSet(const char* n) : RegistrarSet<KIND, T, TPL, Q, V, MINB, Rs...>(n) {}
};
}  // namespace b200fft

#define B2_KP(shard, KIND, T, TPL, Q, V, REGS, NBUF, ...)                                                  \
    static ::b200fft::MaybePipe<B2_SHARD_ON(shard), B2_KIND_##KIND, T, TPL, Q, V, REGS, NBUF, \
                                __VA_ARGS__>                                                              \
        B2_CAT(b2_regp_, __COUNTER__)("PIPE" #NBUF "_" #KIND "<" #T "," #TPL "x" #Q ",V" #V ";" #__VA_ARGS__ ">");

// DCT-II/III variants of a line of the list (explicit, only where the shapes are worth it)
namespace b200fft {
template <bool EN, int KIND, typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeDct {
    explicit MaybeDct(const char*) {}
};
template <int KIND, typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeDct<true, KIND, T, TPL, Q, V, MINB, Rs...> {
    Registrar<KIND, T, TPL, Q, V, MINB, false, B2_OP_DCT23, Rs...> d2;
    Registrar<KIND, T, TPL, Q, V, MINB, true, B2_OP_DCT23, Rs...> d3;
    Registrar<KIND, T, TPL, Q, V, MINB, false, B2_OP_DCT23 | B2_OP_CONV, Rs...> cv;   // DCT / DST convolution (RMODE 12)
    explicit MaybeDct(const char* n) : d2(n), d3(n), cv(n) {}
};
}  // namespace b200fft
// factor kernels of the long strided DCT-II/III Four-Step: (forward, phase + permuted gather) and (inverse, permuted scatter)
namespace b200fft {
template <bool EN, typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeDctLong {
    explicit MaybeDctLong(const char*) {}
};
template <typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeDctLong<true, T, TPL, Q, V, MINB, Rs...> {
    Registrar<B2_KIND_COLS, T, TPL, Q, V, MINB, false, B2_OP_TWIDDLE_OUT | B2_OP_PERM_IN, Rs...> a;
    Registrar<B2_KIND_COLS, T, TPL, Q, V, MINB, true, B2_OP_PERM_OUT, Rs...> b;
    explicit MaybeDctLong(const char* n) : a(n), b(n) {}
};
}  // namespace b200fft
#define B2_KDL(shard, T, TPL, Q, V, MINB, ...)                                                             \
    static ::b200fft::MaybeDctLong<B2_SHARD_ON(shard), T, TPL, Q, V, MINB, __VA_ARGS__>                   \
        B2_CAT(b2_regdl_, __COUNTER__)("DCTLONG_COLS<" #T "," #TPL "x" #Q ",V" #V ";" #__VA_ARGS__ ">");

// Bluestein launches on a contiguous-line schedule
namespace b200fft {
template <bool EN, typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeBlue {
    explicit MaybeBlue(const char*) {}
};
template <typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeBlue<true, T, TPL, Q, V, MINB, Rs...> {
    Registrar<B2_KIND_ROWS, T, TPL, Q, V, MINB, false, B2_OP_BLUESTEIN, Rs...> a;
    Registrar<B2_KIND_ROWS, T, TPL, Q, V, MINB, true, B2_OP_BLUESTEIN, Rs...> b;
    explicit MaybeBlue(const char* n) : a(n), b(n) {}
};
}  // namespace b200fft
#define B2_KB(shard, T, TPL, Q, V, MINB, ...)                                                              \
    static ::b200fft::MaybeBlue<B2_SHARD_ON(shard), T, TPL, Q, V, MINB, __VA_ARGS__>                      \
        B2_CAT(b2_regb_, __COUNTER__)("BLUESTEIN_ROWS<" #T "," #TPL "x" #Q ",V" #V ";" #__VA_ARGS__ ">");

// half-precision storage variants of one schedule: (half in, half out), (half in, float out), (float in, half out); forward and
// inverse; OPS = 0 or B2_OP_TWIDDLE_OUT.  The product library instantiates these at plan time (jit.cpp); the CPU emulation
// registers a handful ahead of time so that the load / store conversions are exercised by the CPU suite
namespace b200fft {
template <bool EN, int KIND, typename T, int TPL, int Q, int V, int MINB, int OPS, int... Rs>
struct MaybeHalf {
    explicit MaybeHalf(const char*) {}
};
template <int KIND, typename T, int TPL, int Q, int V, int MINB, int OPS, int... Rs>
struct MaybeHalf<true, KIND, T, TPL, Q, V, MINB, OPS, Rs...> {
    Registrar<KIND, T, TPL, Q, V, MINB, false, OPS | B2_OP_HALF_IN | B2_OP_HALF_OUT, Rs...> a;
    Registrar<KIND, T, TPL, Q, V, MINB, true, OPS | B2_OP_HALF_IN | B2_OP_HALF_OUT, Rs...> b;
    Registrar<KIND, T, TPL, Q, V, MINB, false, OPS | B2_OP_HALF_IN, Rs...> c;
    Registrar<KIND, T, TPL, Q, V, MINB, true, OPS | B2_OP_HALF_IN, Rs...> d;
    Registrar<KIND, T, TPL, Q, V, MINB, false, OPS | B2_OP_HALF_OUT, Rs...> e;
    Registrar<KIND, T, TPL, Q, V, MINB, true, OPS | B2_OP_HALF_OUT, Rs...> f;
    explicit MaybeHalf(const char* n) : a(n), b(n), c(n), d(n), e(n), f(n) {}
};
}  // namespace b200fft
#define B2_KH(shard, KIND, OPS, TPL, Q, V, MINB, ...)                                                      \
    static ::b200fft::MaybeHalf<B2_SHARD_ON(shard), B2_KIND_##KIND, float, TPL, Q, V, MINB, OPS, __VA_ARGS__> \
        B2_CAT(b2_regh_, __COUNTER__)("HALF_" #KIND "<float," #TPL "x" #Q ",V" #V ";" #__VA_ARGS__ ">");
// even-length R2C (forward) / C2R (inverse) on contiguous lines with half storage on both sides (the real pairs and the spectrum)
namespace b200fft {
template <bool EN, typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeHalfReal {
    explicit MaybeHalfReal(const char*) {}
};
template <typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeHalfReal<true, T, TPL, Q, V, MINB, Rs...> {
    Registrar<B2_KIND_ROWS, T, TPL, Q, V, MINB, false, B2_OP_REAL_EVEN | B2_OP_HALF_IN | B2_OP_HALF_OUT, Rs...> a;
    Registrar<B2_KIND_ROWS, T, TPL, Q, V, MINB, true, B2_OP_REAL_EVEN | B2_OP_HALF_IN | B2_OP_HALF_OUT, Rs...> b;
    explicit MaybeHalfReal(const char* n) : a(n), b(n) {}
};
}  // namespace b200fft
#define B2_KHR(shard, TPL, Q, V, MINB, ...)                                                                \
    static ::b200fft::MaybeHalfReal<B2_SHARD_ON(shard), float, TPL, Q, V, MINB, __VA_ARGS__>               \
        B2_CAT(b2_reghr_, __COUNTER__)("HALF_R2C_ROWS<float," #TPL "x" #Q ",V" #V ";" #__VA_ARGS__ ">");

// the whole Bluestein transform in one launch (stockham.cuh RMODE 11) on a palindromic schedule
namespace b200fft {
template <bool EN, typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeBlue1 {
    explicit MaybeBlue1(const char*) {}
};
template <typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeBlue1<true, T, TPL, Q, V, MINB, Rs...> {
    Registrar<B2_KIND_ROWS, T, TPL, Q, V, MINB, false, B2_OP_BLUE_FUSED, Rs...> a;
    explicit MaybeBlue1(const char* n) : a(n) {}
};
}  // namespace b200fft
#define B2_KB1(shard, T, TPL, Q, V, MINB, ...)                                                             \
    static ::b200fft::MaybeBlue1<B2_SHARD_ON(shard), T, TPL, Q, V, MINB, __VA_ARGS__>                     \
        B2_CAT(b2_regb1_, __COUNTER__)("BLUESTEIN1_ROWS<" #T "," #TPL "x" #Q ",V" #V ";" #__VA_ARGS__ ">");

// fused convolution (forward transform, kernel product, inverse transform in one launch) on a palindromic schedule
namespace b200fft {
template <bool EN, typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeConv {
    explicit MaybeConv(const char*) {}
};
template <typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeConv<true, T, TPL, Q, V, MINB, Rs...> {
    Registrar<B2_KIND_ROWS, T, TPL, Q, V, MINB, false, B2_OP_CONV, Rs...> a;
    explicit MaybeConv(const char* n) : a(n) {}
};
template <bool EN, typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeConvCols {
    explicit MaybeConvCols(const char*) {}
};
template <typename T, int TPL, int Q, int V, int MINB, int... Rs>
struct MaybeConvCols<true, T, TPL, Q, V, MINB, Rs...> {
    Registrar<B2_KIND_COLS, T, TPL, Q, V, MINB, false, B2_OP_CONV, Rs...> a;
    explicit MaybeConvCols(const char* n) : a(n) {}
};
}  // namespace b200fft
#define B2_KCC(shard, T, TPL, Q, V, MINB, ...)                                                             \
    static ::b200fft::MaybeConvCols<B2_SHARD_ON(shard), T, TPL, Q, V, MINB, __VA_ARGS__>                  \
        B2_CAT(b2_regcc_, __COUNTER__)("CONV_COLS<" #T "," #TPL "x" #Q ",V" #V ";" #__VA_ARGS__ ">");
#define B2_KC(shard, T, TPL, Q, V, MINB, ...)                                                              \
    static ::b200fft::MaybeConv<B2_SHARD_ON(shard), T, TPL, Q, V, MINB, __VA_ARGS__>                      \
        B2_CAT(b2_regc_, __COUNTER__)("CONV_ROWS<" #T "," #TPL "x" #Q ",V" #V ";" #__VA_ARGS__ ">");

// ---- fused Four-Step (fused4.cuh) -----------------------------------------------------------------------------------
namespace b200fft {
#if defined(B2_EMU)
// two tile buffers (the next tile is copied in while this one is transformed) when three such CTAs still fit an SM
template <class CA, class CB> struct FusedNbuf { static constexpr int value = (Fused4<CA, CB, 1>::TILE_BYTES <= 36 * 1024) ? 2 : 1; };

template <class CA, class CB>
int fused_launch_impl(const b2_fused_params* F, unsigned, void*) {
    constexpr int NBUF = FusedNbuf<CA, CB>::value;
    b2_fused_params FF = *F;
    FF.U = 1; FF.NU = 1;                       // one group of one CTA walks every tile of every sequence in phase order
    for (uint32_t i = 0; i < 64; ++i) FF.ctl[i] = 0;
    b2emu::launch(1, CA::THREADS, Fused4<CA, CB, NBUF>::SMEM_BYTES, [&](unsigned char* sm) { Fused4<CA, CB, NBUF>::run(FF, sm); }, b2emu::st().log);
    return emu_refused();
}
template <class CA, class CB> int fused_prepare_impl() { return 0; }
#else
template <class CA, class CB> struct FusedNbuf { static constexpr int value = (Fused4<CA, CB, 1>::TILE_BYTES <= 36 * 1024) ? 2 : 1; };

template <class CA, class CB>
int fused_launch_impl(const b2_fused_params* F, unsigned max_ctas, void* stream) {
    constexpr int NBUF = FusedNbuf<CA, CB>::value;
    static int resident = 0;
    if (!resident) {
        int dev = 0, sms = 0, per_sm = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fused4_kernel<CA, CB, NBUF>, CA::THREADS, Fused4<CA, CB, NBUF>::SMEM_BYTES);
        resident = sms * (per_sm > 0 ? per_sm : 1);
    }
    // groups of K = F->U CTAs, all resident at once (they synchronise with each other); at most nseq/2 groups so that the two
    // scratch slots of every group fit the sequences' own footprint in the temp buffer
    b2_fused_params FF = *F;
    const uint32_t K = FF.U ? FF.U : 1;
    uint32_t cap = (uint32_t)resident;
    if (max_ctas && cap > max_ctas) cap = max_ctas;
    uint32_t NG = cap / K;
    const uint32_t ng_max = FF.nseq >= 2 ? FF.nseq / 2 : 1;
    if (NG > ng_max) NG = ng_max;
    if (NG > B2_FCTL_MAX_GROUPS) NG = B2_FCTL_MAX_GROUPS;
    if (NG < 1) return (int)cudaErrorLaunchOutOfResources;        // a group does not fit the device: the plan must not be fused
    FF.NU = NG;
    const uint32_t words = NG * 64;
    fused4_init_kernel<0><<<(words + 255) / 256 < 64 ? (words + 255) / 256 : 64, 256, 0, (cudaStream_t)stream>>>(FF.ctl, words);
    void* args[] = {&FF};
    return (int)cudaLaunchKernel((const void*)fused4_kernel<CA, CB, NBUF>, dim3(NG * K), dim3(CA::THREADS), args, Fused4<CA, CB, NBUF>::SMEM_BYTES,
                                 (cudaStream_t)stream);
}
template <class CA, class CB>
int fused_prepare_impl() {
    return (int)cudaFuncSetAttribute(fused4_kernel<CA, CB, FusedNbuf<CA, CB>::value>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     Fused4<CA, CB, FusedNbuf<CA, CB>::value>::SMEM_BYTES);
}
#endif

template <typename T, bool INV, int TPLA, int QA, class SchA, int TPLB, int QB, class SchB, int REGS>
struct FusedRegistrar {
    using KA = KindTraits<B2_KIND_COLS>;
    using KB = KindTraits<B2_KIND_ROWS_TOUT>;
    using CA = KCfg<T, SchA, TPLA, QA, 1, KA::LMAP, KA::SMAP, KA::LAYOUT, INV, B2_OP_TWIDDLE_OUT, KA::IN_UNIT, KA::OUT_UNIT, REGS, 0>;
    using CB = KCfg<T, SchB, TPLB, QB, 1, KB::LMAP, KB::SMAP, KB::LAYOUT, INV, 0, KB::IN_UNIT, KB::OUT_UNIT, REGS, 0>;
    static_assert(SchA::ns >= 2 && SchB::ns >= 2, "both passes exchange through shared memory");
    b2_fused_info info;
    explicit FusedRegistrar(const char* name) {
        info = b2_fused_info{};
        info.prec = PrecOf<T>::value; info.n1 = SchA::N; info.n2 = SchB::N; info.inv = INV;
        info.threads = CA::THREADS; info.qa = QA; info.qb = QB; info.smem_bytes = Fused4<CA, CB, FusedNbuf<CA, CB>::value>::SMEM_BYTES; info.regs = REGS;
        info.ns_a = SchA::ns; info.ns_b = SchB::ns;
        for (int s = 0; s < SchA::ns; ++s) info.radices_a[s] = SchA::r(s);
        for (int s = 0; s < SchB::ns; ++s) info.radices_b[s] = SchB::r(s);
        info.launch = &fused_launch_impl<CA, CB>;
        info.prepare = &fused_prepare_impl<CA, CB>;
        info.name = name;
        b2_register_fused(&info);
    }
};
template <bool EN, typename T, int TPLA, int QA, class SchA, int TPLB, int QB, class SchB, int REGS>
struct MaybeFused {
    explicit MaybeFused(const char*) {}
};
template <typename T, int TPLA, int QA, class SchA, int TPLB, int QB, class SchB, int REGS>
struct MaybeFused<true, T, TPLA, QA, SchA, TPLB, QB, SchB, REGS> {
    FusedRegistrar<T, false, TPLA, QA, SchA, TPLB, QB, SchB, REGS> f;
    FusedRegistrar<T, true, TPLA, QA, SchA, TPLB, QB, SchB, REGS> i;
    explicit MaybeFused(const char* n) : f(n), i(n) {}
};
}  // namespace b200fft
#define B2_R(...) ::b200fft::RList<__VA_ARGS__>
//   B2_KF(shard, type, REGS, TPL_A, Q_A, B2_R(radices of n1), TPL_B, Q_B, B2_R(radices of n2))
#define B2_KF(shard, T, REGS, TPLA, QA, SA, TPLB, QB, SB)                                                  \
    static ::b200fft::MaybeFused<B2_SHARD_ON(shard), T, TPLA, QA, SA, TPLB, QB, SB, REGS>                  \
        B2_CAT(b2_regf_, __COUNTER__)("FUSED4<" #T ";A " #TPLA "x" #QA " " #SA ";B " #TPLB "x" #QB " " #SB ">");

// ---- cluster Four-Step (cluster4.cuh) --------------------------------------------------------------------------------
// (the CPU emulation runs these kernels only in its build with thread-block clusters, B2_EMU_CLUSTER)
#if !defined(B2_EMU) || defined(B2_EMU_CLUSTER)
namespace b200fft {
#if defined(B2_EMU)
template <class CA, class CB, int CL, int MINB>
int cluster_launch_impl(const b2_cluster_params* K, void*) {
    using CK = Cluster4<CA, CB, CL>;
    const b2_cluster_params KK = *K;
    b2emu::launch_cluster(KK.nseq * CL, CL, CK::THREADS, CK::SMEM_BYTES, [&](unsigned char* sm) { CK::run(KK, sm); }, b2emu::st().log);
    return emu_refused();
}
template <class CA, class CB, int CL, int MINB> int cluster_prepare_impl() { return 0; }
template <class CA, class CB, int CL, int MINB> int cluster_max_active_impl(int) { return b2emu::st().cluster_capable ? 1 : 0; }
#else
template <class CA, class CB, int CL, int MINB>
cudaLaunchConfig_t cluster_config(unsigned grid, cudaLaunchAttribute* at, void* stream) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(Cluster4<CA, CB, CL>::THREADS);
    cfg.dynamicSmemBytes = Cluster4<CA, CB, CL>::SMEM_BYTES;
    cfg.stream = (cudaStream_t)stream;
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = CL; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    return cfg;
}
template <class CA, class CB, int CL, int MINB>
int cluster_launch_impl(const b2_cluster_params* K, void* stream) {
    cudaLaunchAttribute at[1];
    const cudaLaunchConfig_t cfg = cluster_config<CA, CB, CL, MINB>(K->nseq * CL, at, stream);
    return (int)cudaLaunchKernelEx(&cfg, cluster4_kernel<CA, CB, CL, MINB>, *K);
}
template <class CA, class CB, int CL, int MINB>
int cluster_prepare_impl() {
    int rc = (int)cudaFuncSetAttribute(cluster4_kernel<CA, CB, CL, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       Cluster4<CA, CB, CL>::SMEM_BYTES);
    if (rc == 0 && CL > 8) rc = (int)cudaFuncSetAttribute(cluster4_kernel<CA, CB, CL, MINB>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    return rc;
}
// clusters the device can hold at once; 0 when it cannot run this shape at all (or there is no device)
template <class CA, class CB, int CL, int MINB>
int cluster_max_active_impl(int device) {
    static int known[64] = {0};       // per device: 0 not asked yet, else 1 + the answer
    if (device < 0 || device >= 64) return 0;
    if (known[device]) return known[device] - 1;
    int prev = -1;
    if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); return 0; }
    if (prev != device && cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return 0; }
    int n = 0;
    cudaLaunchAttribute at[1];
    const cudaLaunchConfig_t cfg = cluster_config<CA, CB, CL, MINB>(132 * CL, at, nullptr);
    if (cluster_prepare_impl<CA, CB, CL, MINB>() != 0 ||
        cudaOccupancyMaxActiveClusters(&n, (const void*)cluster4_kernel<CA, CB, CL, MINB>, &cfg) != cudaSuccess)
        n = 0;
    cudaGetLastError();
    if (prev != device) cudaSetDevice(prev);
    known[device] = 1 + (n > 0 ? n : 0);
    return n > 0 ? n : 0;
}
#endif

template <typename T, bool INV, int CL, int MINB, int TPLA, int QA, class SchA, int TPLB, int QB, class SchB>
struct ClusterRegistrar {
    using KA = KindTraits<B2_KIND_COLS>;
    using KB = KindTraits<B2_KIND_ROWS_TOUT>;
    using CA = KCfg<T, SchA, TPLA, QA, 1, KA::LMAP, KA::SMAP, KA::LAYOUT, INV, B2_OP_TWIDDLE_OUT, KA::IN_UNIT, KA::OUT_UNIT, 128, 0>;
    using CB = KCfg<T, SchB, TPLB, QB, 1, KB::LMAP, KB::SMAP, KB::LAYOUT, INV, 0, KB::IN_UNIT, KB::OUT_UNIT, 128, 0>;
    using CK = Cluster4<CA, CB, CL>;
    b2_cluster_info info;
    explicit ClusterRegistrar(const char* name) {
        info = b2_cluster_info{};
        info.prec = PrecOf<T>::value; info.n1 = SchA::N; info.n2 = SchB::N; info.inv = INV;
        info.cluster = CL; info.threads = CK::THREADS; info.smem_bytes = CK::SMEM_BYTES;
        info.tpl_a = TPLA; info.q_a = QA; info.tpl_b = TPLB; info.q_b = QB;
        info.ns_a = SchA::ns; info.ns_b = SchB::ns;
        for (int s = 0; s < SchA::ns; ++s) info.radices_a[s] = SchA::r(s);
        for (int s = 0; s < SchB::ns; ++s) info.radices_b[s] = SchB::r(s);
        info.launch = &cluster_launch_impl<CA, CB, CL, MINB>;
        info.prepare = &cluster_prepare_impl<CA, CB, CL, MINB>;
        info.max_active = &cluster_max_active_impl<CA, CB, CL, MINB>;
        info.name = name;
        b2_register_cluster(&info);
    }
};
template <bool EN, typename T, int CL, int MINB, int TPLA, int QA, class SchA, int TPLB, int QB, class SchB>
struct MaybeCluster {
    explicit MaybeCluster(const char*) {}
};
template <typename T, int CL, int MINB, int TPLA, int QA, class SchA, int TPLB, int QB, class SchB>
struct MaybeCluster<true, T, CL, MINB, TPLA, QA, SchA, TPLB, QB, SchB> {
    ClusterRegistrar<T, false, CL, MINB, TPLA, QA, SchA, TPLB, QB, SchB> f;
    ClusterRegistrar<T, true, CL, MINB, TPLA, QA, SchA, TPLB, QB, SchB> i;
    explicit MaybeCluster(const char* n) : f(n), i(n) {}
};
}  // namespace b200fft
//   B2_KCL(shard, type, CTAs per cluster, min CTAs per SM, TPL_A, Q_A, B2_R(radices of n1), TPL_B, Q_B, B2_R(radices of n2))
#define B2_KCL(shard, T, CL, MINB, TPLA, QA, SA, TPLB, QB, SB)                                               \
    static ::b200fft::MaybeCluster<B2_SHARD_ON(shard), T, CL, MINB, TPLA, QA, SA, TPLB, QB, SB>              \
        B2_CAT(b2_regcl_, __COUNTER__)("CLUSTER4<" #T ";" #CL " CTAs;A " #TPLA "x" #QA " " #SA ";B " #TPLB "x" #QB " " #SB ">");
#endif

// short contiguous lines staged through shared memory (stockham.cuh RMODE 10): same registry key as the plain kernels
namespace b200fft {
template <typename T, int Q, int REGS, bool INV, int N>
struct StagedRegistrar {
    using KT = KindTraits<B2_KIND_ROWS>;
    using C = KCfg<T, RList<N>, 1, Q, 1, KT::LMAP, KT::SMAP, KT::LAYOUT, INV, 0, KT::IN_UNIT, KT::OUT_UNIT, REGS, 10>;
    b2_kernel_info info;
    explicit StagedRegistrar(const char* name) {
        info = b2_kernel_info{};
        info.kind = B2_KIND_ROWS; info.prec = PrecOf<T>::value; info.n = N; info.inv = INV; info.ops = 0;
        info.threads = C::THREADS; info.q = Q; info.tpl = 1; info.v = 1; info.smem_bytes = C::SMEM_BYTES;
        info.ns = 1; info.radices[0] = N; info.lut_size = 0;
        info.launch = &launch_impl<C>;
        info.prepare = &prepare_impl<C>;
        info.name = name;
        b2_register_kernel(&info);
    }
};
template <bool EN, typename T, int Q, int REGS, int N>
struct MaybeStaged {
    explicit MaybeStaged(const char*) {}
};
template <typename T, int Q, int REGS, int N>
struct MaybeStaged<true, T, Q, REGS, N> {
    StagedRegistrar<T, Q, REGS, false, N> f;
    StagedRegistrar<T, Q, REGS, true, N> i;
    explicit MaybeStaged(const char* n) : f(n), i(n) {}
};
}  // namespace b200fft
//   B2_KS(shard, type, Q lines per CTA (= threads), REGS, N)
#define B2_KS(shard, T, Q, REGS, N)                                                                        \
    static ::b200fft::MaybeStaged<B2_SHARD_ON(shard), T, Q, REGS, N>                                       \
        B2_CAT(b2_regs_, __COUNTER__)("STAGED_ROWS<" #T "," #Q " lines;" #N ">");

#define B2_KD(shard, KIND, T, TPL, Q, V, MINB, ...)                                                       \
    static ::b200fft::MaybeDct<B2_SHARD_ON(shard), B2_KIND_##KIND, T, TPL, Q, V, MINB, __VA_ARGS__>       \
        B2_CAT(b2_regd_, __COUNTER__)("DCT_" #KIND "<" #T "," #TPL "x" #Q ",V" #V ";" #__VA_ARGS__ ">");

// B2_SHARD < 0: CPU emulation build -- everything, optionally split over B2_EMU_PARTS translation units
#ifndef B2_EMU_PARTS
#define B2_EMU_PARTS 1
#define B2_EMU_PART 0
#endif
#define B2_SHARD_ON(shard) ((B2_SHARD) < 0 ? (((shard) % B2_EMU_PARTS) == B2_EMU_PART) : ((shard) == (B2_SHARD)))
#define B2_CAT2(a, b) a##b
#define B2_CAT(a, b) B2_CAT2(a, b)
#define B2_K(shard, KIND, T, TPL, Q, V, MINB, ...)                                                        \
    static ::b200fft::MaybeSet<B2_SHARD_ON(shard), B2_KIND_##KIND, T, TPL, Q, V, MINB, \
                               __VA_ARGS__>                                                               \
        B2_CAT(b2_reg_, __COUNTER__)(#KIND "<" #T "," #TPL "x" #Q ",V" #V ";" #__VA_ARGS__ ">");

// the CPU emulation (without thread-block clusters) also registers a few half-precision real kernels ahead of time
#if defined(B2_EMU) && !defined(B2_EMU_CLUSTER)
#include "kernel_list_emu_half.def"
#endif
