// CUDA runtime side of the engine + the C ABI declared in include/b200fft.h.
//
// Replaces the reference's L1 "API handles" layer for the CUDA backend: table upload
// (vkFFT_ManageLUT.h:901-915), kernel launch (vkFFT_DispatchPlan.h:157-225), buffer selection
// (vkFFT_UpdateBuffers.h:776-1199) and teardown (vkFFT_DeletePlan.h:59-69, vkFFT_DeleteApp.h:28-324).
// Kernels are found through the registry: compiled ahead of time for sm_90a, or -- smooth lengths outside those lists --
// instantiated from the same templates when the plan is created (jit.cpp).  There is no CPU fallback: if the device or
// the kernels are missing the call fails.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "lut.h"
#include "plan.h"

using namespace b200fft;

struct TwDev {
    void* hi = nullptr;
    void* lo = nullptr;
    uint32_t shift = 0;
};

struct b200fft_plan {
    PlanGraph g;
    int device = 0;
    cudaStream_t stream = nullptr;
    std::vector<void*> d_luts;
    std::vector<TwDev> d_tws;
    std::vector<void*> d_auxs;
    void* d_temp = nullptr;
    uint64_t temp_bytes = 0;
    void* d_ctl = nullptr;          // control block of the fused Four-Step launches
    uint64_t lut_bytes = 0;
    // exec_host staging
    void* d_stage = nullptr;
    uint64_t stage_bytes = 0;
    // distributed plans: the peer window of `buffer` (not owned)
    b200fft_window* window = nullptr;
};

namespace {

// cuTensorMapEncodeTiled through the runtime's driver entry-point lookup (the library links the CUDA runtime only)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            p = nullptr;
        return (EncodeTiledFn)p;
    }();
    return fn;
}
// pass A of a fused Four-Step: the input as [sequences * n1 rows][2 * n2 floats], tiles = boxes of 2*qa floats x min(n1,256) rows
bool encode_pass_a_map(b2_fused_params& F, uint32_t n1, uint32_t n2, uint32_t qa) {
    EncodeTiledFn enc = encode_tiled();
    if (!enc) return false;
    static_assert(sizeof(CUtensorMap) == sizeof(F.tmap_a), "CUtensorMap is 128 bytes");
    const cuuint64_t dims[2] = {2ull * n2, (cuuint64_t)F.nseq * n1};
    const cuuint64_t strides[1] = {(cuuint64_t)n2 * 8};                  // bytes between rows
    const cuuint32_t box[2] = {2u * qa, n1 < 256 ? n1 : 256u};
    const cuuint32_t estr[2] = {1, 1};
    return enc((CUtensorMap*)F.tmap_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(F.A.in), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
        if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
    }
    ~DeviceGuard() {
        int cur = -1;
        if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
    }
};

template <typename T>
int upload(const std::vector<T>& h, void** d, uint64_t& total) {
    *d = nullptr;
    size_t bytes = h.size() * sizeof(T);
    if (bytes == 0) bytes = 16;
    if (cudaMalloc(d, bytes) != cudaSuccess) return R_FAILED_TO_ALLOCATE;
    if (!h.empty() && cudaMemcpy(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess)
        return R_FAILED_TO_COPY;
    total += bytes;
    return R_SUCCESS;
}

void free_plan(b200fft_plan* p) {
    if (!p) return;
    DeviceGuard dg(p->device);
    for (void* d : p->d_luts) if (d) cudaFree(d);
    for (TwDev& t : p->d_tws) { if (t.hi) cudaFree(t.hi); if (t.lo) cudaFree(t.lo); }
    for (void* d : p->d_auxs) if (d) cudaFree(d);
    if (p->d_temp) cudaFree(p->d_temp);
    if (p->d_ctl) cudaFree(p->d_ctl);
    if (p->d_stage) cudaFree(p->d_stage);
    delete p;
}

}  // namespace

extern "C" int b200fft_plan_create(const b200fft_desc* desc, b200fft_plan** out) {
    if (!out) return R_EMPTY_APP;
    *out = nullptr;
    if (!desc) return R_EMPTY_APP;
    if (b2_kernel_count() == 0) return R_PLAN_NOT_INITIALIZED;  // library built without kernels: fail loudly
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return R_INVALID_DEVICE;
    if (desc->device < 0 || desc->device >= ndev) return R_INVALID_DEVICE;
    b200fft_plan* p = new (std::nothrow) b200fft_plan();
    if (!p) return R_MALLOC_FAILED;
    p->device = desc->device;
    p->stream = (cudaStream_t)desc->stream;
    // callers built against an older header pass a shorter struct: everything beyond struct_size reads as zero
    b200fft_desc full;
    memset(&full, 0, sizeof full);
    {
        const size_t have = (desc->struct_size >= 64 && desc->struct_size <= sizeof full) ? desc->struct_size : sizeof full;
        memcpy(&full, desc, have);
    }
    int rc = build_plan(full, p->g);
    if (rc != R_SUCCESS) { delete p; return rc; }
    DeviceGuard dg(p->device);
    if (!dg.ok) { delete p; return R_INVALID_DEVICE; }
    const PlanGraph& g = p->g;
    p->d_luts.assign(g.luts.size(), nullptr);
    p->d_tws.assign(g.tws.size(), TwDev{});
    for (size_t i = 0; i < g.luts.size() && rc == R_SUCCESS; ++i) {
        const LutSpec& ls = g.luts[i];
        if (ls.prec == B2_PREC_F32) rc = upload(make_stage_lut<float>(ls.radices.data(), (int)ls.radices.size()), &p->d_luts[i], p->lut_bytes);
        else rc = upload(make_stage_lut<double>(ls.radices.data(), (int)ls.radices.size()), &p->d_luts[i], p->lut_bytes);
    }
    for (size_t i = 0; i < g.tws.size() && rc == R_SUCCESS; ++i) {
        const TwSpec& ts = g.tws[i];
        if (ts.prec == B2_PREC_F32) {
            std::vector<float> hi, lo;
            make_twolevel<float>(ts.M, p->d_tws[i].shift, hi, lo);
            rc = upload(hi, &p->d_tws[i].hi, p->lut_bytes);
            if (rc == R_SUCCESS) rc = upload(lo, &p->d_tws[i].lo, p->lut_bytes);
        } else {
            std::vector<double> hi, lo;
            make_twolevel<double>(ts.M, p->d_tws[i].shift, hi, lo);
            rc = upload(hi, &p->d_tws[i].hi, p->lut_bytes);
            if (rc == R_SUCCESS) rc = upload(lo, &p->d_tws[i].lo, p->lut_bytes);
        }
    }
    p->d_auxs.assign(g.auxs.size(), nullptr);
    for (size_t i = 0; i < g.auxs.size() && rc == R_SUCCESS; ++i) {
        const AuxSpec& a = g.auxs[i];
        if (a.prec == B2_PREC_F32) rc = upload(make_aux<float>(a.kind, a.a, a.b), &p->d_auxs[i], p->lut_bytes);
        else rc = upload(make_aux<double>(a.kind, a.a, a.b), &p->d_auxs[i], p->lut_bytes);
    }
    // plan-time instantiated kernels (jit.cpp): compile + load.  One that fails is withdrawn from the registry and the plan is
    // built again without it (the length then runs on the runtime-scheduled kernel): never an error of its own
    if (rc == R_SUCCESS) {
        bool withdrawn = false;
        for (int dir = 0; dir < 2; ++dir)
            for (const PassPlan& pp : (dir ? g.inv : g.fwd))
                if (pp.k && pp.k->jit && b2_jit_prepare(pp.k) != 0) { b2_jit_disable(pp.k); withdrawn = true; }
        if (withdrawn) { cudaGetLastError(); free_plan(p); return b200fft_plan_create(desc, out); }
    }
    // one-time kernel attributes (dynamic shared memory above 48 KiB)
    for (int dir = 0; dir < 2 && rc == R_SUCCESS; ++dir)
        for (const PassPlan& pp : (dir ? g.inv : g.fwd))
            if ((pp.k->prepare && pp.k->prepare() != 0) ||
                (pp.k_unaligned && pp.k_unaligned->prepare && pp.k_unaligned->prepare() != 0)) {
                rc = R_FAILED_TO_SET_DYNAMIC_SHARED_MEMORY;
                break;
            }
    for (int dir = 0; dir < 2 && rc == R_SUCCESS; ++dir)
        for (const PassPlan& pp : (dir ? g.inv : g.fwd))
            if ((pp.fused && pp.fused->prepare && pp.fused->prepare() != 0) || (pp.cluster && pp.cluster->prepare() != 0)) {
                rc = R_FAILED_TO_SET_DYNAMIC_SHARED_MEMORY;
                break;
            }
    if (rc == R_SUCCESS && g.ctl_words && cudaMalloc(&p->d_ctl, g.ctl_words * 4) != cudaSuccess) rc = R_FAILED_TO_ALLOCATE;
    // scratch for Four-Step (the reference auto-allocates tempBuffer the same way, vkFFT_InitializeApp.h:1603-1637)
    if (rc == R_SUCCESS && g.temp_elems && !g.desc.user_temp_buffer) {
        p->temp_bytes = g.temp_elems * (g.role_half[ROLE_TEMP] ? 4 : (g.prec == B2_PREC_F64 ? 16 : 8));
        if (cudaMalloc(&p->d_temp, p->temp_bytes) != cudaSuccess) rc = R_FAILED_TO_ALLOCATE;
    }
    if (rc != R_SUCCESS) { cudaGetLastError(); free_plan(p); return rc; }
    *out = p;
    return R_SUCCESS;
}

static int exec_impl(b200fft_plan* p, int inverse, const b200fft_buffers* b, std::vector<cudaEvent_t>* marks, std::vector<int>* kinds);

extern "C" int b200fft_exec(b200fft_plan* p, int inverse, const b200fft_buffers* b) { return exec_impl(p, inverse, b, nullptr, nullptr); }

// tuning hook: one execution with an event after every launch; ms[i] = duration of interval i, kind[i] = 0 barrier / 1 kernel
extern "C" int b200fft_debug_exec_timed(b200fft_plan* p, int inverse, const b200fft_buffers* b, float* ms, int* kind, int cap, int* count) {
    std::vector<cudaEvent_t> marks;
    std::vector<int> kinds;
    int rc = exec_impl(p, inverse, b, &marks, &kinds);
    if (rc == R_SUCCESS && cudaDeviceSynchronize() != cudaSuccess) rc = R_FAILED_TO_SYNCHRONIZE;
    int n = 0;
    for (size_t i = 0; i + 1 < marks.size() && rc == R_SUCCESS; ++i, ++n) {
        float t = 0;
        cudaEventElapsedTime(&t, marks[i], marks[i + 1]);
        if ((int)i < cap) { ms[i] = t; kind[i] = kinds[i]; }
    }
    for (cudaEvent_t e : marks) cudaEventDestroy(e);
    if (count) *count = n;
    return rc;
}

static int exec_impl(b200fft_plan* p, int inverse, const b200fft_buffers* b, std::vector<cudaEvent_t>* marks, std::vector<int>* kinds) {
    if (!p) return R_EMPTY_APP;
    if (!b) return R_EMPTY_BUFFER;
    const PlanGraph& g = p->g;
    if (inverse == 1 && !g.has_inv) return R_ONLY_FORWARD;
    if (inverse != 1 && !g.has_fwd) return R_ONLY_INVERSE;
    const std::vector<PassPlan>& list = (inverse == 1) ? g.inv : g.fwd;
    const size_t esz = g.prec == B2_PREC_F64 ? 16 : 8;
    unsigned char* base[ROLE_COUNT];
    base[ROLE_BUFFER] = (unsigned char*)b->buffer + b->buffer_offset;
    base[ROLE_TEMP] = g.desc.user_temp_buffer ? (unsigned char*)b->temp_buffer + b->temp_buffer_offset
                                              : (unsigned char*)p->d_temp;
    base[ROLE_INPUT] = (unsigned char*)b->input_buffer + b->input_buffer_offset;
    base[ROLE_OUTPUT] = (unsigned char*)b->output_buffer + b->output_buffer_offset;
    base[ROLE_KERNEL] = g.desc.perform_convolution ? (unsigned char*)b->kernel + b->kernel_offset : nullptr;
    bool used[ROLE_COUNT] = {false, false, false, false, false};
    for (const PassPlan& pp : list) { used[pp.in_role] = true; used[pp.out_role] = true; if (pp.aux0_role >= 0) used[pp.aux0_role] = true; }
    if (used[ROLE_KERNEL] && !b->kernel) return R_EMPTY_KERNEL;
    if (used[ROLE_BUFFER] && !b->buffer) return R_EMPTY_BUFFER;
    if (used[ROLE_TEMP] && !(g.desc.user_temp_buffer ? b->temp_buffer : p->d_temp)) return R_EMPTY_TEMPBUFFER;
    if (used[ROLE_INPUT] && !b->input_buffer) return R_EMPTY_INPUTBUFFER;
    if (used[ROLE_OUTPUT] && !b->output_buffer) return R_EMPTY_OUTPUTBUFFER;
    DeviceGuard dg(p->device);
    if (!dg.ok) return R_INVALID_DEVICE;
    cudaStream_t st = b->stream ? (cudaStream_t)b->stream : p->stream;
    if (g.distributed && !p->window) return R_PLAN_NOT_INITIALIZED;
    // timed mode: events created so far are released on every failure path
    auto fail = [&](int code) {
        if (marks) { for (cudaEvent_t e : *marks) cudaEventDestroy(e); marks->clear(); }
        return code;
    };
    auto mark = [&](int kind_of_next) {
        if (!marks) return;
        cudaEvent_t e;
        cudaEventCreate(&e);
        cudaEventRecord(e, st);
        marks->push_back(e);
        if (kind_of_next >= 0) kinds->push_back(kind_of_next);
    };
    auto resolve = [&](const PassPlan& pp, b2_pass_params& P) {
        P = pp.P;
        const size_t esz_in = g.role_half[pp.in_role] ? 4 : esz, esz_out = g.role_half[pp.out_role] ? 4 : esz;   // half-precision storage
        P.in = base[pp.in_role] + pp.in_off * (int64_t)(pp.in_scalar ? esz_in / 2 : esz_in);
        P.out = base[pp.out_role] + pp.out_off * (int64_t)(pp.out_scalar ? esz_out / 2 : esz_out);
        if (pp.aux0_id >= 0) P.aux0 = p->d_auxs[pp.aux0_id];
        if (pp.aux1_id >= 0) P.aux1 = p->d_auxs[pp.aux1_id];
        if (pp.aux0_role >= 0) P.aux0 = base[pp.aux0_role];
        P.lut = p->d_luts[pp.lut_id];
        if (pp.tw_id >= 0) {
            P.tw_hi = p->d_tws[pp.tw_id].hi;
            P.tw_lo = p->d_tws[pp.tw_id].lo;
            P.tw_shift = p->d_tws[pp.tw_id].shift;
        }
    };
    const unsigned fused_max_ctas = [] { const char* e = getenv("B200FFT_FUSED_CTAS"); return e ? (unsigned)strtoul(e, nullptr, 10) : 0u; }();   // tuning knob
    for (size_t ip = 0; ip < list.size(); ++ip) {
        const PassPlan& pp = list[ip];
        if (pp.fused && ip + 1 < list.size()) {
            // both passes of a two-factor Four-Step in one persistent launch (fused4.cuh)
            mark(1);
            b2_fused_params F;
            memset(&F, 0, sizeof F);
            resolve(pp, F.A);
            resolve(list[ip + 1], F.B);
            if (const char* e = getenv("B200FFT_FUSED_FLAGS")) F.B.aux_u1 |= (uint32_t)strtoul(e, nullptr, 10);   // tuning: 1 = no discard
            F.ctl = (uint32_t*)p->d_ctl;
            F.nseq = pp.fz_nseq; F.U = pp.fz_U; F.NU = pp.fz_NU; F.R = pp.fz_R; F.TA = pp.fz_TA; F.TB = pp.fz_TB; F.reserved = pp.fz_L;
            // the tiles arrive by TMA: 16-byte aligned sources and a dense batch (checked at plan time); otherwise the two
            // launches run on their own
            const bool aligned = ((((uintptr_t)F.A.in) | ((uintptr_t)F.B.in)) & 15) == 0;
            if (aligned && F.ctl && encode_pass_a_map(F, F.A.n, F.B.n, (uint32_t)pp.fused->qa)) {
                if (pp.fused->launch(&F, fused_max_ctas, (void*)st) != 0) return fail(R_FAILED_TO_LAUNCH_KERNEL);
                ++ip;
                continue;
            }
        }

        if (pp.cluster && ip + 1 < list.size()) {
            // both passes of a two-factor Four-Step in one launch of thread-block clusters (cluster4.cuh)
            mark(1);
            b2_cluster_params K;
            memset(&K, 0, sizeof K);
            resolve(pp, K.A);
            resolve(list[ip + 1], K.B);
            K.nseq = pp.cl_nseq;
            if (pp.cluster->launch(&K, (void*)st) != 0) return fail(R_FAILED_TO_LAUNCH_KERNEL);
            ++ip;
            continue;
        }

        if (pp.sync_before) {
            mark(0);
            int brc = b200fft_window_barrier(p->window, (void*)st);
            if (brc != R_SUCCESS) return fail(brc);
        }
        mark(1);
        b2_pass_params P;
        resolve(pp, P);
        // un-fused execution of a fusable pair (unaligned buffers): the stand-alone kernels use their own stage tables
        if (pp.lut_id_plain >= 0) P.lut = p->d_luts[pp.lut_id_plain];
        const b2_kernel_info* k = pp.k;
        if (k->pipelined && ((((uintptr_t)P.in) | (uintptr_t)(P.in_gs * (int64_t)esz) | (uintptr_t)(P.in_bs[0] * (int64_t)esz) |
                              (uintptr_t)(P.in_bs[1] * (int64_t)esz) | (uintptr_t)(P.in_bs[2] * (int64_t)esz)) & 15))
        {
            k = pp.k_unaligned;
            if (pp.lut_id_unaligned >= 0) P.lut = p->d_luts[pp.lut_id_unaligned];
        }
        if (!k || (k->jit ? b2_jit_launch(k, &P, pp.grid, (void*)st) : k->launch(&P, pp.grid, (void*)st)) != 0) {
            // a distributed plan that stops half way would leave the peers spinning in their next barrier until the device-side
            // time-out: keep the barrier sequence complete (the data is lost either way, the error code says so)
            if (g.distributed) {
                for (size_t jp = ip + 1; jp < list.size(); ++jp)
                    if (list[jp].sync_before) b200fft_window_barrier(p->window, (void*)st);
                b200fft_window_barrier(p->window, (void*)st);
            }
            return fail(R_FAILED_TO_LAUNCH_KERNEL);
        }
    }
    // every rank's stores into this rank's slab have landed once all ranks passed this point
    if (g.distributed) {
        mark(0);
        int brc = b200fft_window_barrier(p->window, (void*)st);
        mark(-1);
        return brc;
    }
    mark(-1);
    return R_SUCCESS;
}

extern "C" int b200fft_plan_attach_window(b200fft_plan* p, b200fft_window* w) {
    if (!p) return R_EMPTY_APP;
    p->window = w;
    return R_SUCCESS;
}

extern "C" void b200fft_plan_destroy(b200fft_plan* p) { free_plan(p); }

extern "C" int b200fft_plan_get_info(const b200fft_plan* p, b200fft_plan_info* info) {
    if (!p || !info) return R_EMPTY_APP;
    info->num_passes_forward = (uint32_t)p->g.fwd.size();
    info->num_passes_inverse = (uint32_t)p->g.inv.size();
    info->temp_bytes = p->g.temp_elems * (p->g.role_half[ROLE_TEMP] ? 4 : (p->g.prec == B2_PREC_F64 ? 16 : 8));   // required scratch, whoever owns it
    info->lut_bytes = p->lut_bytes;
    info->algorithmic_bytes = p->g.algorithmic_bytes;
    info->flops = p->g.flops;
    return R_SUCCESS;
}

extern "C" int b200fft_plan_axis_uploads(const b200fft_plan* p, int inverse, uint32_t uploads[B200FFT_MAX_DIMS]) {
    if (!p || !uploads) return R_EMPTY_APP;
    for (int a = 0; a < B200FFT_MAX_DIMS; ++a) uploads[a] = p->g.axis_uploads[inverse == 1 ? 1 : 0][a];
    return R_SUCCESS;
}

extern "C" size_t b200fft_plan_describe(const b200fft_plan* p, int inverse, char* dst, size_t cap) {
    if (!p || !dst || cap == 0) return 0;
    std::string s;
    const std::vector<PassPlan>& list = (inverse == 1) ? p->g.inv : p->g.fwd;
    static const char* role[] = {"buffer", "temp", "input", "output", "kernel"};
    for (size_t i = 0; i < list.size(); ++i) {
        s += "pass " + std::to_string(i) + ": " + list[i].note + "  " + role[list[i].in_role] + " -> " +
             role[list[i].out_role] + "\n";
    }
    size_t n = s.size() < cap - 1 ? s.size() : cap - 1;
    memcpy(dst, s.data(), n);
    dst[n] = 0;
    return n;
}

// Planner only, no device: the launch list the engine WOULD build for `desc` (same text as b200fft_plan_describe), with the
// plan-time kernel descriptions of jit.cpp offered but nothing compiled.  Lets the CPU tests check the product library's
// planning -- which, unlike the emulation's, sees the plan-time kernels.  Returns the planner's VkFFTResult code.
extern "C" int b200fft_debug_plan_text(const b200fft_desc* desc, int inverse, char* dst, size_t cap) {
    if (!desc || !dst || cap == 0) return R_EMPTY_APP;
    b200fft_desc full;
    memset(&full, 0, sizeof full);
    const size_t have = (desc->struct_size >= 64 && desc->struct_size <= sizeof full) ? desc->struct_size : sizeof full;
    memcpy(&full, desc, have);
    PlanGraph g;
    const int rc = build_plan(full, g);
    dst[0] = 0;
    if (rc != R_SUCCESS) return rc;
    std::string s;
    const std::vector<PassPlan>& list = (inverse == 1) ? g.inv : g.fwd;
    static const char* role[] = {"buffer", "temp", "input", "output", "kernel"};
    for (size_t i = 0; i < list.size(); ++i)
        s += "pass " + std::to_string(i) + ": " + list[i].note + "  " + role[list[i].in_role] + " -> " + role[list[i].out_role] + "\n";
    const size_t n = s.size() < cap - 1 ? s.size() : cap - 1;
    memcpy(dst, s.data(), n);
    dst[n] = 0;
    return R_SUCCESS;
}

extern "C" int b200fft_exec_host(b200fft_plan* p, int inverse, const void* host_in, void* host_out,
                                 uint64_t bytes_in, uint64_t bytes_out) {
    if (!p) return R_EMPTY_APP;
    if (!host_in || !host_out) return R_EMPTY_BUFFER;
    if (p->g.desc.is_input_formatted || p->g.desc.is_output_formatted) return R_EMPTY_INPUTBUFFER;
    if (p->g.distributed) return R_UNSUPPORTED_FFT_LENGTH;
    DeviceGuard dg(p->device);
    if (!dg.ok) return R_INVALID_DEVICE;
    // the staging buffer always covers the plan's own layout (strides x batches, counted in complex elements: an upper
    // bound for the real-data layouts), whatever byte counts the caller passes: a short count can then neither make a
    // kernel read or write past the allocation nor leave uninitialised input behind (the tail is cleared)
    const uint64_t extent = p->g.batch_stride * p->g.batches * (p->g.role_half[ROLE_BUFFER] ? 4 : (p->g.prec == B2_PREC_F64 ? 16 : 8));
    uint64_t need = bytes_in > bytes_out ? bytes_in : bytes_out;
    if (extent > need) need = extent;
    if (need > p->stage_bytes) {
        if (p->d_stage) cudaFree(p->d_stage);
        p->d_stage = nullptr;
        p->stage_bytes = 0;
        if (cudaMalloc(&p->d_stage, need) != cudaSuccess) { cudaGetLastError(); return R_FAILED_TO_ALLOCATE; }
        p->stage_bytes = need;
    }
    cudaStream_t st = p->stream;
    if (cudaMemcpyAsync(p->d_stage, host_in, bytes_in, cudaMemcpyHostToDevice, st) != cudaSuccess) return R_FAILED_TO_COPY;
    if (bytes_in < extent && cudaMemsetAsync((char*)p->d_stage + bytes_in, 0, extent - bytes_in, st) != cudaSuccess) return R_FAILED_TO_COPY;
    b200fft_buffers b;
    memset(&b, 0, sizeof b);
    b.buffer = p->d_stage;
    int rc = b200fft_exec(p, inverse, &b);
    if (rc != R_SUCCESS) return rc;
    if (cudaMemcpyAsync(host_out, p->d_stage, bytes_out, cudaMemcpyDeviceToHost, st) != cudaSuccess) return R_FAILED_TO_COPY;
    if (cudaStreamSynchronize(st) != cudaSuccess) return R_FAILED_TO_SYNCHRONIZE;
    return R_SUCCESS;
}

extern "C" void* b200fft_host_alloc(uint64_t bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
extern "C" void b200fft_host_free(void* p) { if (p) cudaFreeHost(p); }

extern "C" const char* b200fft_error_string(int code) {
    switch (code) {
        case R_SUCCESS: return "VKFFT_SUCCESS";
        case R_MALLOC_FAILED: return "VKFFT_ERROR_MALLOC_FAILED";
        case R_PLAN_NOT_INITIALIZED: return "VKFFT_ERROR_PLAN_NOT_INITIALIZED";
        case R_NULL_TEMP_PASSED: return "VKFFT_ERROR_NULL_TEMP_PASSED";
        case R_FFTDIM_GT_MAX: return "VKFFT_ERROR_FFTdim_GT_MAX_FFT_DIMENSIONS";
        case 8: return "VKFFT_ERROR_NONZERO_APP_INITIALIZATION";
        case R_INVALID_DEVICE: return "VKFFT_ERROR_INVALID_DEVICE";
        case R_ONLY_FORWARD: return "VKFFT_ERROR_ONLY_FORWARD_FFT_INITIALIZED";
        case R_ONLY_INVERSE: return "VKFFT_ERROR_ONLY_INVERSE_FFT_INITIALIZED";
        case R_EMPTY_FFTDIM: return "VKFFT_ERROR_EMPTY_FFTdim";
        case R_EMPTY_SIZE: return "VKFFT_ERROR_EMPTY_size";
        case R_EMPTY_BUFFER: return "VKFFT_ERROR_EMPTY_buffer";
        case R_EMPTY_TEMPBUFFER: return "VKFFT_ERROR_EMPTY_tempBuffer";
        case R_EMPTY_INPUTBUFFER: return "VKFFT_ERROR_EMPTY_inputBuffer";
        case R_EMPTY_OUTPUTBUFFER: return "VKFFT_ERROR_EMPTY_outputBuffer";
        case R_EMPTY_KERNEL: return "VKFFT_ERROR_EMPTY_kernel";
        case R_EMPTY_APP: return "VKFFT_ERROR_EMPTY_app";
        case R_USER_TEMP_TOO_SMALL: return "VKFFT_ERROR_INVALID_user_tempBuffer_too_small";
        case R_UNSUPPORTED_RADIX: return "VKFFT_ERROR_UNSUPPORTED_RADIX";
        case R_UNSUPPORTED_FFT_LENGTH: return "VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH";
        case R_UNSUPPORTED_FFT_LENGTH_R2C: return "VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH_R2C";
        case R_UNSUPPORTED_FFT_LENGTH_R2R: return "VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH_R2R";
        case R_UNSUPPORTED_FFT_OMIT: return "VKFFT_ERROR_UNSUPPORTED_FFT_OMIT";
        case R_FAILED_TO_ALLOCATE: return "VKFFT_ERROR_FAILED_TO_ALLOCATE";
        case R_FAILED_TO_SYNCHRONIZE: return "VKFFT_ERROR_FAILED_TO_SYNCHRONIZE";
        case R_FAILED_TO_COPY: return "VKFFT_ERROR_FAILED_TO_COPY";
        case R_FAILED_TO_SET_DYNAMIC_SHARED_MEMORY: return "VKFFT_ERROR_FAILED_TO_SET_DYNAMIC_SHARED_MEMORY";
        case R_FAILED_TO_LAUNCH_KERNEL: return "VKFFT_ERROR_FAILED_TO_LAUNCH_KERNEL";
        default: return "VKFFT_ERROR_UNKNOWN";
    }
}
extern "C" int b200fft_version(void) { return B200FFT_VERSION; }
extern "C" int b200fft_kernel_count(void) { return b2_kernel_count(); }

// ---- tuning hook (not part of the drop-in API): time one registered kernel on a synthetic full-buffer pass ----------
// kind ROWS: total/n contiguous lines; COLS: four-step first pass shape (n x `other` lines interleaved, phase
// multiply if the kernel has it); ROWS_TOUT: four-step last pass shape (transposed store).  `in` != `out` for
// ROWS_TOUT.  Returns 0 and the mean ms per launch.
extern "C" int b200fft_debug_time_kernel(int index, void* in, void* out, uint64_t total, uint32_t other, int reps,
                                         float* ms_out, char* name, int name_cap) {
    if (index < 0 || index >= b2_kernel_count()) return -1;
    const b2_kernel_info* k = b2_kernel_at(index);
    if (k->kind == B2_KIND_GENERIC) return -2;
    if (name) snprintf(name, name_cap, "%s", k->name);
    const uint64_t n = (uint64_t)k->n;
    b2_pass_params P;
    memset(&P, 0, sizeof P);
    void *d_lut = nullptr, *d_hi = nullptr, *d_lo = nullptr, *d_tile = nullptr;
    uint64_t dummy = 0;
    int rc;
    if (k->prec == B2_PREC_F32) rc = upload(make_stage_lut<float>(k->radices, k->ns), &d_lut, dummy);
    else rc = upload(make_stage_lut<double>(k->radices, k->ns), &d_lut, dummy);
    if (rc) return rc;
    P.in = in; P.out = out; P.lut = d_lut; P.n = (uint32_t)n; P.scale = 1.0; P.ops = k->ops; P.inverse = k->inv;
    for (int d = 0; d < B2_MAX_OUTER; ++d) P.nb[d] = 1;
    uint64_t grid;
    if (k->kind == B2_KIND_ROWS) {
        P.in_es = P.out_es = 1; P.in_gs = P.out_gs = (int64_t)n; P.G = (uint32_t)(total / n);
        grid = (P.G + k->q - 1) / k->q;
    } else {
        uint64_t o = other;
        while (o * n > total) o >>= 1;
        const uint64_t nouter = total / (n * o);
        P.nb[0] = (uint32_t)nouter; P.in_bs[0] = P.out_bs[0] = (int64_t)(n * o);
        P.G = (uint32_t)o;
        if (k->kind == B2_KIND_COLS) {
            P.in_es = P.out_es = (int64_t)o; P.in_gs = P.out_gs = 1;
        } else {
            P.in_es = 1; P.in_gs = (int64_t)n; P.out_es = (int64_t)o; P.out_gs = 1;
        }
        grid = ((o + k->q - 1) / k->q) * nouter;
        if (k->ops & B2_OP_TWIDDLE_OUT) {
            if (k->prec == B2_PREC_F32) {
                std::vector<float> hi, lo; make_twolevel<float>(n * o, P.tw_shift, hi, lo);
                rc = upload(hi, &d_hi, dummy); if (!rc) rc = upload(lo, &d_lo, dummy);
            } else {
                std::vector<double> hi, lo; make_twolevel<double>(n * o, P.tw_shift, hi, lo);
                rc = upload(hi, &d_hi, dummy); if (!rc) rc = upload(lo, &d_lo, dummy);
            }
            P.tw_hi = d_hi; P.tw_lo = d_lo;
        }
    }
    if (!rc && k->jit && b2_jit_prepare(k) != 0) rc = R_FAILED_TO_SET_DYNAMIC_SHARED_MEMORY;
    if (!rc && k->prepare && k->prepare() != 0) rc = R_FAILED_TO_SET_DYNAMIC_SHARED_MEMORY;
    auto launch1 = [&]() { return k->jit ? b2_jit_launch(k, &P, (unsigned)grid, nullptr) : k->launch(&P, (unsigned)grid, nullptr); };
    float ms = 0;
    if (!rc) {
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        for (int i = 0; i < 2 && !rc; ++i) rc = launch1();
        cudaEventRecord(e0, 0);
        for (int i = 0; i < reps && !rc; ++i) rc = launch1();
        cudaEventRecord(e1, 0);
        if (cudaDeviceSynchronize() != cudaSuccess) rc = R_FAILED_TO_SYNCHRONIZE;
        cudaEventElapsedTime(&ms, e0, e1);
        cudaEventDestroy(e0); cudaEventDestroy(e1);
        cudaGetLastError();
    }
    if (ms_out) *ms_out = ms / (reps > 0 ? reps : 1);
    cudaFree(d_lut); if (d_hi) cudaFree(d_hi); if (d_lo) cudaFree(d_lo); if (d_tile) cudaFree(d_tile);
    return rc;
}
extern "C" int b200fft_debug_kernel_info(int index, int* v /*kind,prec,n,inv,ops,variant,threads,q,tpl,smem*/) {
    if (index < 0 || index >= b2_kernel_count()) return -1;
    const b2_kernel_info* k = b2_kernel_at(index);
    int a[] = {k->kind, k->prec, k->n, k->inv, k->ops, k->variant, k->threads, k->q, k->tpl, k->smem_bytes};
    for (int i = 0; i < 10; ++i) v[i] = a[i];
    return 0;
}
