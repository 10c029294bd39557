// Plan-time instantiation of the hand-written kernel templates for lengths outside the ahead-of-time lists.
//
// The ahead-of-time registry (kernel_list*.def) covers the powers of two, ~230 curated lengths and every Four-Step factor
// the BASELINE configurations need.  Any other 2..31-smooth length used to fall back to the runtime-scheduled kernel
// (generic.cuh), which is several times slower than a specialised one.  Here such a length gets `Engine<KCfg<...>>` of stockham.cuh -- the very code
// of the ahead-of-time kernels, with its own radix schedule and CTA shape as template constants -- compiled for the
// device's architecture when the plan that needs it is created: NVRTC -> cubin -> cuModuleLoadData.  ~2 s per length, once
// per process.  The reference compiles EVERY kernel of EVERY plan like that (vkFFT_CompileKernel.h:299-491: NVRTC,
// cuModuleLoadDataEx); here it is the exception for lengths nobody curated, nothing on the BASELINE path depends on it,
// and B200FFT_NO_JIT=1 (or a missing libnvrtc) simply leaves those lengths on the runtime-scheduled kernel.
//
// libnvrtc and libcuda are opened with dlopen: the library itself links neither.
#include <dlfcn.h>
#include <stdint.h>
#include <unistd.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "kernel_registry.h"

extern "C" const char* const b2_jit_header_names[];
extern "C" const char* const b2_jit_header_sources[];
extern "C" const int b2_jit_header_count;

namespace {

// ---- the slice of the NVRTC / driver API this file uses ----------------------------------------------------------
typedef struct _nvrtcProgram* nvrtcProgram;
typedef int nvrtcResult;
typedef int CUresult;
typedef void* CUmodule;
typedef void* CUfunction;
typedef void* CUstream;
struct Api {
    bool tried = false, have_nvrtc = false, have_cuda = false;
    nvrtcResult (*CreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
    nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char* const*) = nullptr;
    nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t*) = nullptr;
    nvrtcResult (*GetCUBIN)(nvrtcProgram, char*) = nullptr;
    nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t*) = nullptr;
    nvrtcResult (*GetProgramLog)(nvrtcProgram, char*) = nullptr;
    nvrtcResult (*DestroyProgram)(nvrtcProgram*) = nullptr;
    CUresult (*ModuleLoadData)(CUmodule*, const void*) = nullptr;
    CUresult (*ModuleGetFunction)(CUfunction*, CUmodule, const char*) = nullptr;
    CUresult (*LaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, CUstream, void**, void**) = nullptr;
    CUresult (*FuncSetAttribute)(CUfunction, int, int) = nullptr;
    CUresult (*CtxGetDevice)(int*) = nullptr;
    CUresult (*DeviceGetAttribute)(int*, int, int) = nullptr;
};
Api& api() {
    static Api a;
    if (a.tried) return a;
    a.tried = true;
    void* n = nullptr;
    for (const char* name : {"libnvrtc.so.12", "libnvrtc.so", "libnvrtc.so.13"})
        if ((n = dlopen(name, RTLD_NOW | RTLD_LOCAL))) break;
    if (n) {
#define B2_SYM(field, sym) a.field = (decltype(a.field))dlsym(n, sym)
        B2_SYM(CreateProgram, "nvrtcCreateProgram"); B2_SYM(CompileProgram, "nvrtcCompileProgram");
        B2_SYM(GetCUBINSize, "nvrtcGetCUBINSize"); B2_SYM(GetCUBIN, "nvrtcGetCUBIN");
        B2_SYM(GetProgramLogSize, "nvrtcGetProgramLogSize"); B2_SYM(GetProgramLog, "nvrtcGetProgramLog");
        B2_SYM(DestroyProgram, "nvrtcDestroyProgram");
#undef B2_SYM
        a.have_nvrtc = a.CreateProgram && a.CompileProgram && a.GetCUBINSize && a.GetCUBIN && a.DestroyProgram;
    }
    void* c = dlopen("libcuda.so.1", RTLD_NOW | RTLD_LOCAL);
    if (c) {
#define B2_SYM(field, sym) a.field = (decltype(a.field))dlsym(c, sym)
        B2_SYM(ModuleLoadData, "cuModuleLoadData"); B2_SYM(ModuleGetFunction, "cuModuleGetFunction");
        B2_SYM(LaunchKernel, "cuLaunchKernel"); B2_SYM(FuncSetAttribute, "cuFuncSetAttribute");
        B2_SYM(CtxGetDevice, "cuCtxGetDevice"); B2_SYM(DeviceGetAttribute, "cuDeviceGetAttribute");
#undef B2_SYM
        a.have_cuda = a.ModuleLoadData && a.ModuleGetFunction && a.LaunchKernel && a.FuncSetAttribute && a.CtxGetDevice && a.DeviceGetAttribute;
    }
    return a;
}

// ---- schedule and CTA shape of a length: the rules of tools/gen_nonpow2_kernels.py (what the curated kernels were built with) ----
std::vector<int> factor(int n, bool primes) {
    // fewest stages, then the smallest largest radix; radices in descending order
    static const int cands[] = {31, 29, 23, 19, 17, 16, 15, 14, 13, 12, 11, 10, 9, 8, 7, 6, 5, 4, 3, 2};
    std::vector<int> best, acc;
    auto vmax = [](const std::vector<int>& v) { int m = 0; for (int r : v) m = r > m ? r : m; return m; };
    std::function<void(int, int)> go = [&](int v, int start) {
        if (v == 1) {
            if (best.empty() || acc.size() < best.size() || (acc.size() == best.size() && vmax(acc) < vmax(best))) best = acc;
            return;
        }
        if (!best.empty() && acc.size() >= best.size()) return;
        for (int i = start; i < 20; ++i) {
            const int c = cands[i];
            if (c > 16 && !primes) continue;
            if (v % c == 0) { acc.push_back(c); go(v / c, i); acc.pop_back(); }
        }
    };
    go(n, 0);
    return best;
}

struct Shape {
    std::vector<int> r;
    int tpl = 0, q = 0, regs = 0, smem = 0, smem_i = 0, lut = 0, rmode_f = 0, rmode_i = 0, st = 0;   // smem: launch size (forward kernel), smem_i: inverse kernel's own
};

// the tuned ahead-of-time kernel of the same transform (half-storage variants copy its schedule and CTA shape)
const b2_kernel_info* tuned_base(int kind, int prec, int n, int ops) {
    const b2_kernel_info* best = nullptr;
    for (int i = 0; i < b2_kernel_count(); ++i) {
        const b2_kernel_info* k = b2_kernel_at(i);
        if (k->kind != kind || k->prec != prec || k->n != n || k->inv != 0 || k->ops != ops) continue;
        if (k->pipelined || k->v != 1 || k->regs <= 0 || k->jit || !k->name || !strncmp(k->name, "STAGED", 6)) continue;
        if (!best || k->variant < best->variant) best = k;
    }
    return best;
}

bool choose(int kind, int prec, int n, int ops_all, Shape& s) {
    const bool dbl = prec == B2_PREC_F64;
    // half-precision storage (B2_OP_HALF_IN / _OUT -> KCfg::ST): FP32 plain complex transforms, and the even-length R2C / C2R
    // with half on both sides; no ahead-of-time kernel exists for it, so every length from 2 up comes from here (one-radix
    // kernels included)
    const int half = ops_all & (B2_OP_HALF_IN | B2_OP_HALF_OUT), ops = ops_all & ~half;
    if (half && (dbl || (ops & ~(B2_OP_TWIDDLE_OUT | B2_OP_REAL_EVEN)))) return false;
    if (half && (ops & B2_OP_REAL_EVEN) && (kind != B2_KIND_ROWS || half != (B2_OP_HALF_IN | B2_OP_HALF_OUT))) return false;
    s.st = ((half & B2_OP_HALF_IN) ? 1 : 0) | ((half & B2_OP_HALF_OUT) ? 2 : 0);
    const b2_kernel_info* base = half ? tuned_base(kind, prec, n, ops) : nullptr;
    // contiguous FP32 lines up to 8192 points in one launch (64 KiB tile, up to 32 points per thread), everything else up to 4096
    if (n < (half ? 2 : 18) || n > ((kind == B2_KIND_ROWS && !dbl && (base || !half)) ? 8192 : 4096)) return false;
    // B2_OP_DCT23: DCT-II (forward kernel) / DCT-III (inverse kernel) fused into the load and store, two real lines (or two
    // neighbouring real columns) per complex line -- the B2_KD variants of the curated lists, same shapes
    if (kind == B2_KIND_ROWS) { if (ops != 0 && ops != B2_OP_REAL_EVEN && ops != B2_OP_DCT23) return false; }
    else if (kind == B2_KIND_COLS) { if (ops != 0 && ops != B2_OP_TWIDDLE_OUT && ops != B2_OP_DCT23) return false; if (n > (dbl ? 1024 : 2048)) return false; }
    else if (kind == B2_KIND_ROWS_TOUT) { if (ops != 0) return false; if (n > (dbl ? 1024 : 2048)) return false; }
    else return false;
    s.r = factor(n, kind == B2_KIND_ROWS && !dbl);
    if (s.r.size() < (half ? 1u : 2u) || s.r.size() > 8) return false;
    int rmax = 0;
    for (int r : s.r) rmax = r > rmax ? r : rmax;
    const int esz = dbl ? 16 : 8;
    if (kind == B2_KIND_ROWS) {
        int tpl = n / rmax;
        while (tpl > 256) tpl = (tpl + 1) / 2;
        const int e = (n + tpl - 1) / tpl;
        int q = 128 / tpl < 1 ? 1 : 128 / tpl;
        while (q > 1 && q * n * 8 > 48 * 1024) q /= 2;
        int regs = e * 2 > 40 ? 128 : (e * 2 > 24 ? 96 : 80);
        if (dbl) { regs = regs * 2 > 168 ? 168 : regs * 2; q = q / 2 < 1 ? 1 : q / 2; }
        s.tpl = tpl; s.q = q; s.regs = regs;
    } else {
        int tpl = n / rmax;
        while (tpl > 64) tpl = (tpl + 1) / 2;
        const int e = (n + tpl - 1) / tpl;
        int regs = e * 2 > 40 ? 128 : (e * 2 > 24 ? 96 : 80);
        int q = n <= 256 ? 16 : 8;
        if (dbl) { regs = regs * 2 > 168 ? 168 : regs * 2; q /= 2; }
        // half-precision storage: q neighbouring lines are q * 4 bytes in HBM -- twice the lines for the same 64...128-byte runs
        if (half) q = n <= 128 ? 32 : (n <= 512 ? 16 : 8);
        s.tpl = tpl; s.q = q; s.regs = regs;
    }
    if (base) {
        // powers of two and curated lengths: the measured-best schedule and CTA shape of the FP32-storage kernel; along strided /
        // transposed sides at least the tile width of the half rule above (64...128-byte runs) where the tile still fits
        const int qh = s.q;
        s.r.assign(base->radices, base->radices + base->ns);
        s.tpl = base->tpl; s.q = base->q; s.regs = base->regs;
        if (kind != B2_KIND_ROWS && qh > s.q && s.tpl * qh <= 512 && n * qh * esz <= 96 * 1024) s.q = qh;
    }
    // tuning experiments (tools/jit_shape_sweep.py): B200FFT_JIT_SHAPE="tpl,q,regs[,r0,r1,...]" overrides the rule for contiguous lines
    if (const char* ov = getenv("B200FFT_JIT_SHAPE")) {
        if (kind == B2_KIND_ROWS && !half) {
            std::vector<int> v;
            for (const char* p = ov; *p;) { char* e; long x = strtol(p, &e, 10); if (e == p) break; v.push_back((int)x); p = (*e == ',') ? e + 1 : e; }
            if (v.size() >= 3) {
                s.tpl = v[0]; s.q = v[1]; s.regs = v[2];
                if (v.size() > 3) {
                    long prod = 1;
                    for (size_t i = 3; i < v.size(); ++i) prod *= v[i];
                    if (prod != n || v.size() - 3 > 8) return false;
                    s.r.assign(v.begin() + 3, v.end());
                }
            }
        }
    }
    if (s.tpl < 1 || s.q < 1 || s.tpl * s.q > 1024) return false;
    s.rmode_f = (ops & B2_OP_REAL_EVEN) ? 1 : ((ops & B2_OP_DCT23) ? 3 : 0);
    s.rmode_i = (ops & B2_OP_REAL_EVEN) ? 2 : ((ops & B2_OP_DCT23) ? 4 : 0);
    // KCfg::SMEM_BYTES and RList::lut_size (stockham.cuh); the generated source static_asserts both
    const int pad_shift = dbl ? 3 : 4, npad = n + (n >> pad_shift);
    const bool line = kind != B2_KIND_COLS;
    const int ls = s.q == 1 ? npad : (npad | 1);
    s.smem = s.r.size() <= 1 && !(ops & B2_OP_REAL_EVEN) ? 0 : (line ? s.q * ls : n * s.q) * esz;
    s.smem_i = s.r.size() <= 1 ? 0 : s.smem;          // a one-radix C2R needs no tile (its Hermitian pass is in the load)
    int S = 1, lut = 0;
    for (size_t i = 0; i < s.r.size(); ++i) { if (i > 0) lut += (s.r[i] - 1) * S; S *= s.r[i]; }
    s.lut = lut;
    return s.smem <= 200 * 1024;
}

struct Program {            // one compiled (kind, prec, n, ops): forward + inverse kernel
    std::string source, log;
    std::vector<char> cubin;
    int compiled = 0;       // 0 not yet, 1 ok, -1 failed
    std::map<int, std::pair<CUfunction, CUfunction>> per_device;   // device ordinal -> (forward, inverse)
};
struct Entry {
    b2_kernel_info info;
    Shape shape;
    Program* prog;
    std::string name;
};
typedef std::tuple<int, int, int, int> PKey;          // kind, prec, n, ops
std::mutex g_mu;
std::map<PKey, Program*> g_programs;
std::map<std::tuple<int, int, int, int, int>, Entry*> g_entries;
std::string g_last_log;

std::string make_source(int kind, int prec, int ops, const Shape& s) {
    const char* T = prec == B2_PREC_F64 ? "double" : "float";
    const int lmap = kind == B2_KIND_COLS ? 1 : 0, smap = kind == B2_KIND_ROWS ? 0 : 1, layout = kind == B2_KIND_COLS ? 1 : 0;
    const char* in_unit = kind == B2_KIND_COLS ? "false" : "true";
    const char* out_unit = kind == B2_KIND_ROWS ? "true" : "false";
    std::string rl;
    for (size_t i = 0; i < s.r.size(); ++i) rl += (i ? ", " : "") + std::to_string(s.r[i]);
    char buf[4096];
    snprintf(buf, sizeof buf,
             "#include \"stockham.cuh\"\n"
             "using namespace b200fft;\n"
             "using Sch = RList<%s>;\n"
             "using CF = KCfg<%s, Sch, %d, %d, 1, %d, %d, %d, false, %d, %s, %s, %d, %d, %d>;\n"
             "using CI = KCfg<%s, Sch, %d, %d, 1, %d, %d, %d, true, %d, %s, %s, %d, %d, %d>;\n"
             "static_assert(CF::SMEM_BYTES == %d && CI::SMEM_BYTES == %d, \"host copy of KCfg::SMEM_BYTES\");\n"
             "static_assert(Sch::lut_size == %d, \"host copy of RList::lut_size\");\n"
             "extern \"C\" __global__ void __launch_bounds__(CF::THREADS, CF::MINB) b2_jit_fwd(const __grid_constant__ b2_pass_params P) {\n"
             "    extern __shared__ __align__(16) unsigned char b2_smem_raw[];\n"
             "    Engine<CF>::run(P, b2_smem_raw);\n"
             "}\n"
             "extern \"C\" __global__ void __launch_bounds__(CI::THREADS, CI::MINB) b2_jit_inv(const __grid_constant__ b2_pass_params P) {\n"
             "    extern __shared__ __align__(16) unsigned char b2_smem_raw[];\n"
             "    Engine<CI>::run(P, b2_smem_raw);\n"
             "}\n",
             rl.c_str(), T, s.tpl, s.q, lmap, smap, layout, ops & B2_OP_TWIDDLE_OUT, in_unit, out_unit, s.regs, s.rmode_f, s.st, T, s.tpl, s.q,
             lmap, smap, layout, ops & B2_OP_TWIDDLE_OUT, in_unit, out_unit, s.regs, s.rmode_i, s.st, s.smem, s.smem_i, s.lut);
    return buf;
}

// optional on-disk cache of the compiled kernels (B200FFT_JIT_CACHE=<directory>): one file per (templates, translation unit,
// architecture, options), so that a second process does not pay the ~1-2 s per length again.  The reference offers the same
// saving through saveApplicationToString / loadApplicationFromString (vkFFT_InitializeApp.h:1603-1637).
uint64_t fnv1a(const char* s, uint64_t h = 1469598103934665603ull) {
    for (; *s; ++s) { h ^= (unsigned char)*s; h *= 1099511628211ull; }
    return h;
}
std::string cache_path(const Program& p, const char* arch, bool lineinfo) {
    const char* dir = getenv("B200FFT_JIT_CACHE");
    if (!dir || !*dir) return std::string();
    static uint64_t hdr = 0;
    if (!hdr) { hdr = 1469598103934665603ull; for (int i = 0; i < b2_jit_header_count; ++i) hdr = fnv1a(b2_jit_header_sources[i], hdr); }
    uint64_t h = fnv1a(p.source.c_str(), hdr);
    h = fnv1a(arch, h);
    h = fnv1a(lineinfo ? "L" : "-", h);
    char name[64];
    snprintf(name, sizeof name, "/b200fft_%016llx.cubin", (unsigned long long)h);
    return std::string(dir) + name;
}

// NVRTC -> cubin for `arch` ("sm_90a"); no GPU needed
int compile(Program& p, const char* arch) {
    Api& a = api();
    const bool lineinfo = getenv("B200FFT_JIT_LINEINFO") != nullptr;
    const std::string cached = cache_path(p, arch, lineinfo);
    if (!cached.empty()) {
        if (FILE* f = fopen(cached.c_str(), "rb")) {
            fseek(f, 0, SEEK_END);
            const long sz = ftell(f);
            fseek(f, 0, SEEK_SET);
            bool ok = sz > 0;
            if (ok) { p.cubin.resize((size_t)sz); ok = fread(p.cubin.data(), 1, (size_t)sz, f) == (size_t)sz; }
            fclose(f);
            if (ok) { p.log = "from " + cached; return 0; }
            p.cubin.clear();
        }
    }
    if (!a.have_nvrtc) { p.log = "libnvrtc not found"; return -1; }
    nvrtcProgram prog = nullptr;
    if (a.CreateProgram(&prog, p.source.c_str(), "b200fft_jit.cu", b2_jit_header_count, b2_jit_header_sources, b2_jit_header_names) != 0) {
        p.log = "nvrtcCreateProgram failed";
        return -1;
    }
    const std::string archopt = std::string("--gpu-architecture=") + arch;
    // B200FFT_JIT_LINEINFO=1: line tables so that ncu's source page maps to the templates (cubins grow from ~70 KB to 0.3-1 MB)
    const char* opts[] = {archopt.c_str(), "-std=c++17", "-w", "-lineinfo"};
    const nvrtcResult rc = a.CompileProgram(prog, lineinfo ? 4 : 3, opts);
    size_t ln = 0;
    if (a.GetProgramLogSize && a.GetProgramLog && a.GetProgramLogSize(prog, &ln) == 0 && ln > 1) {
        p.log.resize(ln);
        a.GetProgramLog(prog, &p.log[0]);
    }
    int ret = -1;
    size_t sz = 0;
    if (rc == 0 && a.GetCUBINSize(prog, &sz) == 0 && sz > 0) {
        p.cubin.resize(sz);
        if (a.GetCUBIN(prog, p.cubin.data()) == 0) ret = 0;
    }
    a.DestroyProgram(&prog);
    if (ret == 0 && !cached.empty()) {          // write next to the final name, then rename: readers never see a partial file
        const std::string tmp = cached + ".tmp" + std::to_string((long)getpid());
        if (FILE* f = fopen(tmp.c_str(), "wb")) {
            const bool ok = fwrite(p.cubin.data(), 1, p.cubin.size(), f) == p.cubin.size();
            fclose(f);
            if (!ok || rename(tmp.c_str(), cached.c_str()) != 0) remove(tmp.c_str());
        }
    }
    return ret;
}

const b2_kernel_info* provide(int kind, int prec, int n, int inv, int ops) {
    if (getenv("B200FFT_NO_JIT")) return nullptr;
    if (!api().have_nvrtc) return nullptr;
    std::lock_guard<std::mutex> lk(g_mu);
    // (tuning experiments: descriptions and programs are kept per value of B200FFT_JIT_SHAPE, so a sweep over shapes in one process
    // gets a fresh kernel per shape while the forward and inverse kernel of one plan still share a program)
    const char* ov = getenv("B200FFT_JIT_SHAPE");
    static std::map<std::string, std::pair<std::map<std::tuple<int, int, int, int, int>, Entry*>, std::map<PKey, Program*>>> per_override;
    auto& entries = ov ? per_override[ov].first : g_entries;
    auto& programs = ov ? per_override[ov].second : g_programs;
    auto ek = std::make_tuple(kind, prec, n, inv, ops);
    auto it = entries.find(ek);
    if (it != entries.end()) return it->second ? &it->second->info : nullptr;
    Shape s;
    if (!choose(kind, prec, n, ops, s)) { entries[ek] = nullptr; return nullptr; }
    PKey pk = std::make_tuple(kind, prec, n, ops);
    Program*& prog = programs[pk];
    if (!prog) { prog = new Program; prog->source = make_source(kind, prec, ops, s); }
    Entry* e = new Entry;
    e->shape = s; e->prog = prog;
    std::string rl;
    for (size_t i = 0; i < s.r.size(); ++i) rl += (i ? ", " : "") + std::to_string(s.r[i]);
    const char* kn = kind == B2_KIND_ROWS ? "ROWS" : (kind == B2_KIND_COLS ? "COLS" : "ROWS_TOUT");
    const char* stn[] = {"", ",half in+out", ",half in", ",half out"};
    e->name = std::string("JIT_") + kn + "<" + (prec == B2_PREC_F64 ? "double" : "float") + "," + std::to_string(s.tpl) + "x" + std::to_string(s.q) + ",V1;" + rl +
              stn[s.st == 3 ? 1 : (s.st == 1 ? 2 : (s.st == 2 ? 3 : 0))] + ">";
    b2_kernel_info& k = e->info;
    memset(&k, 0, sizeof k);
    k.kind = kind; k.prec = prec; k.n = n; k.inv = inv; k.ops = ops;
    k.threads = s.tpl * s.q; k.q = s.q; k.tpl = s.tpl; k.v = 1; k.smem_bytes = s.smem;
    k.ns = (int)s.r.size();
    for (size_t i = 0; i < s.r.size(); ++i) k.radices[i] = s.r[i];
    k.lut_size = s.lut;
    k.name = e->name.c_str();
    k.jit = e;
    entries[ek] = e;
    return &k;
}

struct Install { Install() { b2_set_kernel_provider(&provide); } } g_install;

}  // namespace

// compile (once per process) and load (once per device) the kernel behind a plan-time kernel description
extern "C" int b2_jit_prepare(const b2_kernel_info* k) {
    if (!k || !k->jit) return -1;
    Entry* e = (Entry*)k->jit;
    Api& a = api();
    if (!a.have_cuda) return -1;
    std::lock_guard<std::mutex> lk(g_mu);
    int dev = 0;
    if (a.CtxGetDevice(&dev) != 0) return -1;
    Program& p = *e->prog;
    if (p.compiled == 0) {
        int major = 9, minor = 0;
        a.DeviceGetAttribute(&major, 75 /* CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MAJOR */, dev);
        a.DeviceGetAttribute(&minor, 76 /* ..._MINOR */, dev);
        char arch[32];
        snprintf(arch, sizeof arch, major >= 9 ? "sm_%d%da" : "sm_%d%d", major, minor);
        p.compiled = compile(p, arch) == 0 ? 1 : -1;
        if (p.compiled < 0) { g_last_log = p.log; fprintf(stderr, "b200fft: plan-time kernel %s failed to compile:\n%s\n", k->name, p.log.c_str()); }
    }
    if (p.compiled < 0) return -1;
    if (!p.per_device.count(dev)) {
        CUmodule mod = nullptr;
        CUfunction f = nullptr, i = nullptr;
        if (a.ModuleLoadData(&mod, p.cubin.data()) != 0 || a.ModuleGetFunction(&f, mod, "b2_jit_fwd") != 0 || a.ModuleGetFunction(&i, mod, "b2_jit_inv") != 0)
            return -1;
        if (e->shape.smem > 48 * 1024) {
            a.FuncSetAttribute(f, 8 /* CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES */, e->shape.smem);
            a.FuncSetAttribute(i, 8, e->shape.smem);
        }
        p.per_device[dev] = std::make_pair(f, i);
    }
    return 0;
}

// a kernel that failed to compile or load: the registry stops offering it, the caller re-plans (runtime.cu)
extern "C" void b2_jit_disable(const b2_kernel_info* k) {
    if (!k || !k->jit) return;
    std::lock_guard<std::mutex> lk(g_mu);
    for (int inv = 0; inv < 2; ++inv) g_entries[std::make_tuple(k->kind, k->prec, k->n, inv, k->ops)] = nullptr;
}

extern "C" int b2_jit_launch(const b2_kernel_info* k, const b2_pass_params* P, unsigned grid, void* stream) {
    Entry* e = (Entry*)k->jit;
    Api& a = api();
    int dev = 0;
    CUfunction fn = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        if (a.CtxGetDevice(&dev) != 0) return -1;
        auto it = e->prog->per_device.find(dev);
        if (it == e->prog->per_device.end()) return -1;
        fn = k->inv ? it->second.second : it->second.first;
    }
    void* args[] = {const_cast<b2_pass_params*>(P)};
    return a.LaunchKernel(fn, grid, 1, 1, (unsigned)k->threads, 1, 1, (unsigned)e->shape.smem, (CUstream)stream, args, nullptr);
}

// CPU-side self test (no GPU): describe + compile the kernel for (kind, prec, n, ops) to a cubin for sm_90a.
// Returns the cubin size, 0 if the key is not eligible, < 0 on a compile error (log through b2_jit_last_log).
extern "C" long b2_jit_selftest(int kind, int prec, int n, int ops) {
    const b2_kernel_info* k = provide(kind, prec, n, 0, ops);
    if (!k) return 0;
    Entry* e = (Entry*)k->jit;
    std::lock_guard<std::mutex> lk(g_mu);
    Program& p = *e->prog;
    if (p.compiled == 0) p.compiled = compile(p, "sm_90a") == 0 ? 1 : -1;
    if (p.compiled < 0) { g_last_log = p.log; return -1; }
    return (long)p.cubin.size();
}
extern "C" const char* b2_jit_last_log(void) { return g_last_log.c_str(); }
extern "C" int b2_jit_available(void) { return (api().have_nvrtc && !getenv("B200FFT_NO_JIT")) ? 1 : 0; }
