// Planner: turns a b200fft_desc into an ordered list of kernel launches (see plan.h).
//
// Decisions the reference makes in VkFFTScheduler (vkFFT_Scheduler.h:2223-3299: algorithm choice :2288-2578,
// number of uploads :2582-2650, axis split :2651-2893, temp buffer :2902-2944) and VkFFTPlanAxis
// (vkFFT_Plan_FFT.h:252-417 strides, :582-645 grid) are made here against the table of ahead-of-time compiled
// kernels:
//   * a line length with a specialised single-pass kernel     -> one launch of it (1 HBM read + 1 write);
//   * any other 2..13-smooth length that fits shared memory   -> one launch of the runtime-scheduled kernel;
//   * longer contiguous lines                                 -> Four-Step with 2 or 3 launches (strided
//     sub-FFTs + phase multiply, then contiguous sub-FFTs with a transposed, coalesced store so the result is in
//     natural order -- the reference's reorderFourStep=1 behaviour, vkFFT_4step.h:31-119);
//   * lengths with a prime factor > 13                         -> Bluestein through a power-of-two length
//     (chirp / zero-pad fused into the first launch's load, filter and post-chirp into the stores);
//   * R2C / C2R: half-length complex transform of the (even, odd) samples with the Hermitian pass fused into
//     the store / load of the same launch; DCT-I..IV: permutation / phase passes fused the same way.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "lut.h"
#include "plan.h"

namespace b200fft {
namespace {

struct Dim {
    uint64_t n;
    int64_t is, os;  // input / output stride (complex elements, or scalars for the real-data operators)
};

int lut_for(PlanGraph& g, const std::vector<int>& r) {
    for (size_t i = 0; i < g.luts.size(); ++i)
        if (g.luts[i].prec == g.prec && g.luts[i].radices == r) return (int)i;
    g.luts.push_back(LutSpec{g.prec, r});
    return (int)g.luts.size() - 1;
}
int tw_for(PlanGraph& g, uint64_t M) {
    for (size_t i = 0; i < g.tws.size(); ++i)
        if (g.tws[i].prec == g.prec && g.tws[i].M == M) return (int)i;
    g.tws.push_back(TwSpec{g.prec, M});
    return (int)g.tws.size() - 1;
}
int aux_for(PlanGraph& g, int kind, uint64_t a, uint64_t b = 0) {
    for (size_t i = 0; i < g.auxs.size(); ++i)
        if (g.auxs[i].prec == g.prec && g.auxs[i].kind == kind && g.auxs[i].a == a && g.auxs[i].b == b) return (int)i;
    g.auxs.push_back(AuxSpec{g.prec, kind, a, b});
    return (int)g.auxs.size() - 1;
}

// merge neighbouring dims that are contiguous in both the input and the output addressing
std::vector<Dim> merge_dims(const std::vector<Dim>& d) {
    std::vector<Dim> out;
    for (const Dim& x : d) {
        if (x.n == 1) continue;
        if (!out.empty()) {
            Dim& b = out.back();
            if ((int64_t)b.n * b.is == x.is && (int64_t)b.n * b.os == x.os) {
                b.n *= x.n;
                continue;
            }
        }
        out.push_back(x);
    }
    return out;
}

// greedy radix list for the runtime-scheduled kernel (largest radix first).  Prime factors 17..127 become Rader
// stages (the reference inlines Rader kernels for radix primes from 17, vkFFT_InitializeApp.h:1257-1292); empty if
// n has a prime factor above that (-> Bluestein).
const int RADER_MAX_PRIME = 127;
const int RADER_DEFAULT_MAX_PRIME = 127;
// largest prime factor the runtime-scheduled kernel takes as a Rader stage; lengths with a larger one go through Bluestein.
// B200FFT_RADER_MAX_PRIME overrides it (tuning)
int rader_max_prime() {
    if (const char* e = getenv("B200FFT_RADER_MAX_PRIME")) { const int v = atoi(e); return v < 13 ? 13 : (v > RADER_MAX_PRIME ? RADER_MAX_PRIME : v); }
    return RADER_DEFAULT_MAX_PRIME;
}
std::vector<int> generic_radices(uint64_t n) {
    std::vector<int> r, primes;
    static const int cand16[] = {16, 15, 14, 13, 12, 11, 10, 9, 8, 7, 6, 5, 4, 3, 2};
    static const int cand11[] = {11, 10, 9, 8, 7, 6, 5, 4, 3, 2};
    static const int cand8[] = {8, 7, 6, 5, 4, 3, 2};
    // split off prime factors > 13 first
    uint64_t m = n;
    for (int f : {2, 3, 5, 7, 11, 13}) while (m % f == 0) m /= f;
    for (uint64_t f = 17; m > 1 && f <= (uint64_t)rader_max_prime(); f += 2)
        while (m % f == 0) { primes.push_back((int)f); m /= f; n /= f; }
    if (m != 1) return {};
    // greedy factorisation per radix class; keep the leanest class that does not need more stages than the widest one
    auto greedy = [](uint64_t v, const int* c, int nc) {
        std::vector<int> out;
        while (v > 1) {
            bool found = false;
            for (int i = 0; i < nc; ++i)
                if (v % c[i] == 0) { out.push_back(c[i]); v /= c[i]; found = true; break; }
            if (!found) return std::vector<int>{};
        }
        return out;
    };
    if (n > 1) {
        std::vector<int> r16 = greedy(n, cand16, 15), r11 = greedy(n, cand11, 10), r8 = greedy(n, cand8, 7);
        if (r16.empty()) return {};
        r = r16;
        if (!r11.empty() && r11.size() <= r16.size()) r = r11;
        if (!r8.empty() && r8.size() <= r.size()) r = r8;
    }
    // Rader stages last: their legs are already twiddled by a large stageSize, outputs land in natural order as usual
    r.insert(r.end(), primes.begin(), primes.end());
    if (r.size() > B2_MAX_STAGES) return {};
    return r;
}

uint64_t esize(const PlanGraph& g) { return g.prec == B2_PREC_F64 ? 16 : 8; }      // element size of the ARITHMETIC (tiles in shared memory)
uint64_t role_esize(const PlanGraph& g, int role) { return g.role_half[role] ? 4 : esize(g); }   // element size in HBM
bool half_plan(const PlanGraph& g) { return g.role_half[ROLE_BUFFER] || g.role_half[ROLE_INPUT]; }   // some launch converts: plan-time kernels only
int pad_of(const PlanGraph& g, uint64_t n) { return (int)(n + (n >> (g.prec == B2_PREC_F64 ? 3 : 4))); }
const uint64_t GENERIC_SMEM_LIMIT = 200 * 1024;

bool generic_fits(const PlanGraph& g, uint64_t n) {
    if (n < 2 || n > (1u << 20)) return false;
    if (generic_radices(n).empty()) return false;
    return 2ull * (uint64_t)(pad_of(g, n) | 1) * esize(g) <= GENERIC_SMEM_LIMIT;
}

struct PassReq {
    int kind = B2_KIND_ROWS, n = 0, inv = 0, ops = 0;
    int64_t in_es = 1, out_es = 1;
    Dim group{1, 0, 0};          // lines handled Q at a time by one CTA
    std::vector<Dim> outer;      // remaining line dimensions
    int in_role = ROLE_BUFFER, out_role = ROLE_BUFFER;
    uint64_t twM = 0;
    int tw_outer = -1;           // >= 0: index into `outer` (before merging) of the four-step line coordinate
    uint32_t tw_line0 = 0;       // first line coordinate of this launch (a rank's slice of a distributed sequence)
    bool sync_before = false;    // distributed plans: every rank must have finished its previous launch first
    double scale = 1.0;
    const char* what = "";
    // generic-kernel extras
    bool force_generic = false;
    int load_io = B2_IO_C2C, store_io = B2_IO_C2C;
    int inner_inverse = 0;
    uint32_t in_len = 0, out_len = 0;   // 0 -> n
    int aux0 = -1, aux1 = -1;
    uint32_t aux_u0 = 0, aux_u1 = 0, aux_u2 = 0;
    bool real_pairs = false;     // group dim counts REAL lines; two of them form one complex line
    uint32_t dst_flags = 0;
    bool scalar_units = false;   // specialised real-data kernels addressing real lines: offsets/strides count scalars
    int runtime_inverse = -1;    // >= 0: value of P.inverse when it differs from the kernel's compile-time direction
    int64_t in_base = 0, out_base = 0;   // element offsets into the role's buffer (scratch regions)
    // elementwise helper passes (ew.cuh)
    bool elementwise = false;
    int ew_op = 0;
    uint32_t ew_items = 0;       // items per line (elements or pairs)
};

// Emit the launches for one PassReq (more than one only if there are more than B2_MAX_OUTER outer dims).
int emit(PlanGraph& g, std::vector<PassPlan>& list, const PassReq& rq) {
    const b2_kernel_info* k = nullptr;
    const bool plain = !rq.force_generic && rq.load_io == B2_IO_C2C && rq.store_io == B2_IO_C2C &&
                       !(rq.ops & (B2_OP_MUL_IN | B2_OP_MUL_OUT)) &&
                       ((rq.in_len == 0 && rq.out_len == 0) || (rq.ops & (B2_OP_BLUESTEIN | B2_OP_BLUE_FUSED))) && !rq.inner_inverse;
    // half-precision storage on either side: the conversion lives in the specialised kernels' HBM load / store (KCfg::ST),
    // instantiated at plan time (jit.cpp); the runtime-scheduled kernel and the operator launches have no such variant
    const int hops = (g.role_half[rq.in_role] ? B2_OP_HALF_IN : 0) | (g.role_half[rq.out_role] ? B2_OP_HALF_OUT : 0);
    const int key_ops = (rq.ops & (B2_OP_TWIDDLE_OUT | B2_OP_REAL_EVEN | B2_OP_DCT23 | B2_OP_PERM_IN | B2_OP_PERM_OUT | B2_OP_BLUESTEIN | B2_OP_CONV | B2_OP_BLUE_FUSED)) | hops;
    if (plain) k = b2_find_kernel(rq.kind, g.prec, rq.n, rq.inv, key_ops);
    if (hops && !k) return R_UNSUPPORTED_FFT_LENGTH;
    std::vector<int> radices;
    bool generic = false;
    if (!k) {
        if (!generic_fits(g, rq.n)) return R_UNSUPPORTED_FFT_LENGTH;
        radices = generic_radices(rq.n);
        int rmax = 2;
        for (int r : radices) if (r <= 16) rmax = std::max(rmax, r);
        k = b2_find_kernel(B2_KIND_GENERIC, g.prec, rmax <= 8 ? 8 : (rmax <= 11 ? 11 : 16), 0, 0);
        if (!k) return R_UNSUPPORTED_FFT_LENGTH;
        generic = true;
    } else {
        radices.assign(k->radices, k->radices + k->ns);
    }
    // the four-step line coordinate must survive dim merging: keep that dim separate
    std::vector<Dim> outer;
    int tw_sel = 0;
    if (rq.tw_outer >= 0) {
        std::vector<Dim> a(rq.outer.begin(), rq.outer.begin() + rq.tw_outer), b(rq.outer.begin() + rq.tw_outer + 1, rq.outer.end());
        a = merge_dims(a); b = merge_dims(b);
        outer = a;
        tw_sel = 1 + (int)outer.size();
        outer.push_back(rq.outer[rq.tw_outer]);
        outer.insert(outer.end(), b.begin(), b.end());
    } else {
        outer = merge_dims(rq.outer);
    }
    // peel outermost dims into separate launches until at most B2_MAX_OUTER remain
    std::vector<Dim> peeled;
    while (outer.size() > B2_MAX_OUTER) {
        peeled.push_back(outer.back());
        outer.pop_back();
    }
    if (tw_sel > B2_MAX_OUTER) return R_UNSUPPORTED_FFT_LENGTH;
    uint64_t npeel = 1;
    for (const Dim& p : peeled) npeel *= p.n;
    const uint64_t glines = rq.real_pairs ? (rq.group.n + 1) / 2 : rq.group.n;

    // CTA shape
    uint32_t tpl = 0, q = 0, ls = 0;
    const bool qfast_l = (rq.kind == B2_KIND_COLS), qfast_s = (rq.kind != B2_KIND_ROWS);
    if (generic) {
        tpl = 1;
        while (tpl < 256 && tpl * 16 < (uint32_t)rq.n) tpl <<= 1;
        ls = (uint32_t)(pad_of(g, rq.n) | 1);
        const uint64_t per_line = 2ull * ls * esize(g);
        uint32_t qmax = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(GENERIC_SMEM_LIMIT / per_line, 256 / tpl));
        uint32_t want = (qfast_l || qfast_s) ? (g.prec == B2_PREC_F64 ? 8u : 16u) : std::max(1u, 128u / tpl);
        // keep at least two CTAs per SM resident when lines are short
        while (want > 1 && want * per_line > 96 * 1024) want >>= 1;
        q = std::max(1u, std::min(want, qmax));
        if (q > glines) q = (uint32_t)std::max<uint64_t>(1, glines);
    } else {
        tpl = k->tpl; q = k->q;
    }

    for (uint64_t pi = 0; pi < npeel; ++pi) {
        int64_t ioff = 0, ooff = 0;
        uint64_t rem = pi;
        for (const Dim& p : peeled) {
            uint64_t c = rem % p.n;
            rem /= p.n;
            ioff += (int64_t)c * p.is;
            ooff += (int64_t)c * p.os;
        }
        PassPlan pp;
        pp.k = k;
        if (k->pipelined) {   // TMA needs 16-byte aligned sources: keep the first non-pipelined kernel of the same key as a stand-in
            for (int v = 0; v < 16 && !pp.k_unaligned; ++v) {
                const b2_kernel_info* alt = b2_find_kernel_variant(rq.kind, g.prec, rq.n, rq.inv, key_ops, v);
                if (alt && !alt->pipelined && alt->q == k->q) pp.k_unaligned = alt;
            }
            if (!pp.k_unaligned) {    // no drop-in with the same tile height: do not use the pipelined kernel at all
                for (int v = 0; v < 16; ++v) {
                    const b2_kernel_info* alt = b2_find_kernel_variant(rq.kind, g.prec, rq.n, rq.inv, key_ops, v);
                    if (alt && !alt->pipelined) { pp.k = k = alt; break; }
                }
                tpl = k->tpl; q = k->q;
            }
        }
        b2_pass_params& P = pp.P;
        P.in_es = rq.in_es; P.out_es = rq.out_es;
        P.in_gs = rq.group.is; P.out_gs = rq.group.os;
        P.G = (uint32_t)glines;
        uint64_t grid = (glines + q - 1) / q;
        for (int d = 0; d < B2_MAX_OUTER; ++d) {
            if (d < (int)outer.size()) {
                P.nb[d] = (uint32_t)outer[d].n; P.in_bs[d] = outer[d].is; P.out_bs[d] = outer[d].os;
            } else {
                P.nb[d] = 1; P.in_bs[d] = 0; P.out_bs[d] = 0;
            }
            grid *= P.nb[d];
        }
        if (grid == 0 || grid > 0x7fffffffull) return R_UNSUPPORTED_FFT_LENGTH;
        pp.grid = (unsigned)grid;
        P.n = rq.n;
        P.ops = rq.ops;
        P.inverse = rq.runtime_inverse >= 0 ? rq.runtime_inverse : rq.inv;
        P.inner_inverse = rq.inner_inverse;
        P.scale = rq.scale;
        P.tw_sel = tw_sel;
        P.tw_line0 = rq.tw_line0;
        pp.sync_before = rq.sync_before && pi == 0;
        P.nstages = (uint32_t)radices.size();
        for (size_t s = 0; s < radices.size(); ++s) P.radix[s] = radices[s];
        P.tpl = tpl; P.q = q; P.line_stride = ls;
        P.load_io = rq.load_io; P.store_io = rq.store_io;
        if (generic && getenv("B200FFT_GENERIC_FUSED_IO")) {
            // plain complex lines: the first butterflies read HBM and the last ones write it (generic.cuh stage_io) instead of
            // separate copy phases through shared memory.  Measured slower and REJECTED as the default (the strided
            // first-stage legs of a runtime radix cost more than the two shared-memory passes they save); opt-in
            if ((rq.load_io == B2_IO_C2C || rq.load_io == B2_IO_R2C_EVEN) && radices.front() <= 16) P.gen_flags |= B2_GEN_FUSE_IN;
            if ((rq.store_io == B2_IO_C2C || rq.store_io == B2_IO_C2R_EVEN) && radices.back() <= 16) P.gen_flags |= B2_GEN_FUSE_OUT;
        }
        P.in_len = rq.in_len ? rq.in_len : rq.n;
        P.out_len = rq.out_len ? rq.out_len : rq.n;
        P.load_qfast = qfast_l; P.store_qfast = qfast_s;
        P.aux_u0 = rq.aux_u0; P.aux_u1 = rq.aux_u1; P.aux_u2 = rq.aux_u2;
        P.dst_flags = rq.dst_flags;
        pp.in_role = rq.in_role; pp.out_role = rq.out_role;
        pp.in_off = ioff + rq.in_base; pp.out_off = ooff + rq.out_base;
        pp.lut_id = lut_for(g, radices);
        if (pp.k_unaligned)
            pp.lut_id_unaligned = lut_for(g, std::vector<int>(pp.k_unaligned->radices, pp.k_unaligned->radices + pp.k_unaligned->ns));
        if (rq.ops & B2_OP_TWIDDLE_OUT) pp.tw_id = tw_for(g, rq.twM);
        pp.aux0_id = rq.aux0; pp.aux1_id = rq.aux1;
        // specialised kernels: intra-tile factor of the four-step phase (coalesced table, see stockham.cuh)
        auto scalar_io = [](int io) { return io == B2_IO_DCT1 || io == B2_IO_DCT2 || io == B2_IO_DCT3 || io == B2_IO_DCT4 || io == B2_IO_DCT4_ODD || io == B2_IO_REAL || io == B2_IO_DST1; };
        pp.in_scalar = scalar_io(rq.load_io) || rq.scalar_units; pp.out_scalar = scalar_io(rq.store_io) || rq.scalar_units;
        char buf[320];
        std::string rs;
        for (int r : radices) rs += (rs.empty() ? "" : "x") + std::to_string(r);
        snprintf(buf, sizeof buf, "%s n=%d %s[%s] grid=%u threads=%u %s", rq.what, rq.n, generic ? "generic" : k->name,
                 rs.c_str(), pp.grid, tpl * q, rq.inv ? "inverse" : "forward");
        pp.note = buf;
        list.push_back(pp);
    }
    return R_SUCCESS;
}

// can a single launch transform lines of length n (kind only matters for the specialised kernels)?
bool single_ok(const PlanGraph& g, int kind, uint64_t n, int ops) {
    if (n > 0x7fffffffull) return false;
    if (n == 1) return false;
    // half-precision storage: only the specialised kernels convert, and only as plan-time variants (jit.cpp) -- their limits
    // differ from the FP32 kernels' (e.g. a non-curated 5000-point line is one FP32 launch but has no half variant: Four-Step)
    if (half_plan(g)) return b2_find_kernel(kind, g.prec, (int)n, 0, ops | B2_OP_HALF_IN | B2_OP_HALF_OUT) != nullptr;
    if (b2_find_kernel(kind, g.prec, (int)n, 0, ops)) return true;
    return generic_fits(g, n);
}

// Fused Four-Step (fused4.cuh).  DRAM traffic is exactly one read + one write (the ring stays in L2), but each SM now has to
// turn every tile over twice in the time HBM delivers it once, and with the loads of a tile on its critical path the
// resident CTAs do not keep enough bytes in flight: it measured slower than the two launches.  Opt-in (B200FFT_FUSED4=1).
bool fused4_enabled() {
    const char* e = getenv("B200FFT_FUSED4");        // read per plan: tests and tuning scripts switch it between plans
    return e && *e && *e != '0' && !getenv("B200FFT_NO_FUSED4");
}

uint64_t max_single_env() {
    if (const char* e = getenv("B200FFT_MAX_SINGLE_PASS")) return strtoull(e, nullptr, 10);
    return ~0ull;
}

// Factor N for Four-Step.  All factors but the last run as interleaved-line passes with the phase multiply,
// the last one runs on contiguous lines with a transposed store.  Returns empty if impossible.
std::vector<uint64_t> split_four_step(const PlanGraph& g, uint64_t N, bool dist = false) {
    // test hook: B200FFT_FOUR_STEP_SPLIT="n1,n2[,n3]" forces a factorisation (used by the CPU tests to reach
    // the three-pass code with small transforms)
    if (const char* e = getenv("B200FFT_FOUR_STEP_SPLIT")) {
        std::vector<uint64_t> f;
        uint64_t prod = 1;
        for (const char* p = e; *p;) {
            char* end;
            uint64_t v = strtoull(p, &end, 10);
            if (end == p) break;
            f.push_back(v); prod *= v;
            p = (*end == ',') ? end + 1 : end;
        }
        if (prod == N && f.size() >= 2 && f.size() <= 3) return f;
    }
    const uint64_t cap = std::min<uint64_t>(max_single_env(), half_plan(g) ? 512 : 4096);   // (half storage: factors up to 512 keep 16+ lines = 64-byte runs per tile of the strided / transposed side)
    auto fast = [&](int kind, uint64_t n, int ops) { return b2_find_kernel(kind, g.prec, (int)n, 0, ops) != nullptr; };
    // measured cost of one full pass over a 2 GiB FP32 buffer, microseconds (tools/ktune.py, default variant of each kernel;
    // H100 80GB HBM3 SXM at a 400 W power limit); used to rank factorizations.  Unknown sizes / FP64 fall back to
    // "balanced factors".
    auto pass_us = [&](int kind, uint64_t n) -> uint64_t {
        if (g.prec != B2_PREC_F32) return 0;
        static const struct { uint64_t n; uint64_t cols, tout; } t[] = {
            {16, 1434, 1491}, {32, 2220, 1465}, {64, 1439, 1456}, {128, 1431, 1454}, {256, 1472, 1448},
            {512, 1471, 1460}, {1024, 2507, 1468}, {2048, 1660, 2373}};
        for (const auto& e : t)
            if (e.n == n) return kind == B2_KIND_COLS ? e.cols : e.tout;
        return 0;
    };
    // distributed plans: the first launch's stores and the last launch's transposed stores cross NVLink in runs of
    // q elements; 64-byte runs (q = 8) reach markedly less bandwidth per direction than 128-byte runs -> rank kernels with
    // q < 16 as if their pass were 300 us slower
    auto short_runs = [&](int kind, uint64_t n, int ops) -> uint64_t {
        if (!dist) return 0;
        const b2_kernel_info* k = b2_find_kernel(kind, g.prec, (int)n, 0, ops);
        return (k && k->q < 16) ? 300 * 16 : 0;
    };
    std::vector<uint64_t> best;
    uint64_t best_cost = ~0ull;
    for (uint64_t n2 = 2; n2 * 2 <= N && n2 <= cap; ++n2) {
        if (N % n2) continue;
        uint64_t n1 = N / n2;
        if (n1 > cap) continue;
        if (!single_ok(g, B2_KIND_ROWS_TOUT, n2, 0) || !single_ok(g, B2_KIND_COLS, n1, B2_OP_TWIDDLE_OUT)) continue;
        // prefer specialised kernels, then measured pass costs, then balanced factors (contiguous one not smaller)
        uint64_t cost = std::max(n1, n2) * 4 + (n2 < n1 ? 2 : 0);
        if (pass_us(B2_KIND_COLS, n1) && pass_us(B2_KIND_ROWS_TOUT, n2))
            cost = (pass_us(B2_KIND_COLS, n1) + pass_us(B2_KIND_ROWS_TOUT, n2)) * 16 + (cost & 15);
        else cost += 1u << 16;
        if (!fast(B2_KIND_ROWS_TOUT, n2, 0)) cost += 1u << 20;
        if (!fast(B2_KIND_COLS, n1, B2_OP_TWIDDLE_OUT)) cost += 1u << 20;
        cost += short_runs(B2_KIND_COLS, n1, B2_OP_TWIDDLE_OUT) + short_runs(B2_KIND_ROWS_TOUT, n2, 0);
        // splits that run as one fused launch (one HBM round trip instead of two) win over every two-launch split;
        // among them the first registered pair of a length is the measured default (kernel_list_fused.def)
        if (!dist && fused4_enabled()) {
            const b2_fused_info* fk = b2_find_fused(g.prec, (int)n1, (int)n2, 0);
            if (fk) {
                int order = 0;
                for (int i = 0; i < b2_fused_count() && b2_fused_at(i) != fk; ++i)
                    if (b2_fused_at(i)->prec == g.prec && !b2_fused_at(i)->inv && (uint64_t)b2_fused_at(i)->n1 * b2_fused_at(i)->n2 == N) ++order;
                cost = 1 + order;
            }
        }
        if (cost < best_cost) { best_cost = cost; best = {n1, n2}; }
    }
    // from 2^22 on, three launches of fast 128/256-point factors (a 4096-point factor has no fast strided kernel)
    const uint64_t two_level_limit = 1ull << 21;
    if (!best.empty() && N <= two_level_limit) return best;
    std::vector<uint64_t> best3;
    uint64_t best3_cost = ~0ull;
    for (uint64_t n3 = 2; n3 * 4 <= N && n3 <= cap; ++n3) {
        if (N % n3 || !single_ok(g, B2_KIND_ROWS_TOUT, n3, 0)) continue;
        uint64_t rest = N / n3;
        for (uint64_t n2 = 2; n2 * 2 <= rest && n2 <= cap; ++n2) {
            if (rest % n2 || !single_ok(g, B2_KIND_COLS, n2, B2_OP_TWIDDLE_OUT)) continue;
            uint64_t n1 = rest / n2;
            if (n1 > cap || !single_ok(g, B2_KIND_COLS, n1, B2_OP_TWIDDLE_OUT)) continue;
            uint64_t cost = std::max(n1, std::max(n2, n3)) * 4 + (n3 < n1 ? 1 : 0) + (n3 < n2 ? 1 : 0);
            if (pass_us(B2_KIND_COLS, n1) && pass_us(B2_KIND_COLS, n2) && pass_us(B2_KIND_ROWS_TOUT, n3))
                cost = (pass_us(B2_KIND_COLS, n1) + pass_us(B2_KIND_COLS, n2) + pass_us(B2_KIND_ROWS_TOUT, n3)) * 16 + (cost & 15);
            else cost += 1u << 16;
            if (!fast(B2_KIND_ROWS_TOUT, n3, 0)) cost += 1u << 20;
            if (!fast(B2_KIND_COLS, n2, B2_OP_TWIDDLE_OUT)) cost += 1u << 20;
            if (!fast(B2_KIND_COLS, n1, B2_OP_TWIDDLE_OUT)) cost += 1u << 20;
            cost += short_runs(B2_KIND_COLS, n1, B2_OP_TWIDDLE_OUT) + short_runs(B2_KIND_ROWS_TOUT, n3, 0);
            if (cost < best3_cost) { best3_cost = cost; best3 = {n1, n2, n3}; }
        }
    }
    if (!best3.empty()) return best3;
    return best;
}

bool is_smooth(uint64_t n) { return !generic_radices(n).empty() || n == 1; }

// ----------------------------------------------------------------------------------------------------------------
// One C2C transform of length N along lines with element stride (es_in, es_out); `lines` lists every other
// dimension (first entry = the preferred grouped dimension).  unit_lines: lines[0] has unit stride on both sides
// (strided axis: neighbouring lanes walk neighbouring lines).
struct C2CJob {
    uint64_t N;
    int inv;
    int64_t es_in, es_out;
    std::vector<Dim> lines;
    bool unit_lines;
    int in_role, out_role;
    double scale;
    int64_t in_base = 0, out_base = 0, tmp_base = 0;   // element offsets into the roles' buffers
    // distributed sequence: this plan covers rank `rank` of `world` (buffer and temp are peer windows, plan.h)
    uint32_t world = 1, rank = 0;
    // distributed N-D transform, the axis that crosses the slabs: this rank transforms 1/line_world of the lines (a slice
    // of the outermost line dimension); its strided loads and stores reach into every rank's slab of the peer window
    uint32_t line_world = 1, line_rank = 0;
    // R2C slab plans: when no line dimension divides by line_world, the first one (the H = nx/2+1 spectrum columns) is cut
    // into contiguous ranges on multiples of 8 columns and the last rank takes the remainder
    bool line_ragged = false;
    bool sync_first = false;            // a barrier over all ranks precedes the first launch of this job
    // fused convolution along this axis (single launch only): B2_OP_CONV + its operands
    int extra_ops = 0;
    uint32_t aux_u0 = 0, aux_u1 = 0;
};

// keep rank `rank`'s share of dimension d (contiguous block of d.n/world coordinates); returns the first coordinate
bool slice_dim(Dim& d, uint32_t world, uint32_t rank, int64_t& in_base, int64_t& out_base, uint64_t& first) {
    if (world <= 1) { first = 0; return true; }
    if (d.n % world) return false;
    d.n /= world;
    first = (uint64_t)rank * d.n;
    in_base += (int64_t)first * d.is;
    out_base += (int64_t)first * d.os;
    return true;
}

// distributed N-D plan, the axis that crosses the slabs: keep rank `rank`'s share of the line dimensions `lines` -- a contiguous
// block of the outermost dimension with more than one line that `world` divides (never the batch entry, which is 1 here), or,
// when none does and `ragged` is set, a range of lines[0] whose boundaries fall on multiples of 8 lines (neighbouring lanes of
// one CTA), the last rank taking the remainder.  Moves the bases to the share's first line.
int share_lines(std::vector<Dim>& lines, uint32_t world, uint32_t rank, bool ragged, int64_t& in_base, int64_t& out_base) {
    for (size_t i = lines.size(); i-- > 0;) {
        uint64_t first;
        if (lines[i].n > 1 && lines[i].n % world == 0 && slice_dim(lines[i], world, rank, in_base, out_base, first)) return R_SUCCESS;
    }
    if (!ragged || lines.empty()) return R_UNSUPPORTED_FFT_LENGTH;
    Dim& c = lines[0];
    uint64_t per = c.n / world;
    if (per >= 8) per &= ~7ull;
    if (per == 0) return R_UNSUPPORTED_FFT_LENGTH;
    const uint64_t first = (uint64_t)rank * per;
    c.n = (rank + 1 == world) ? c.n - first : per;
    in_base += (int64_t)first * c.is;
    out_base += (int64_t)first * c.os;
    return R_SUCCESS;
}

int plan_c2c(PlanGraph& g, std::vector<PassPlan>& list, const C2CJob& job);

// elementwise helper launch over `lines` (every line dimension, any order)
int emit_ew(PlanGraph& g, std::vector<PassPlan>& list, PassReq rq, const std::vector<Dim>& lines) {
    // half-precision storage: only the Hermitian passes of a long even-length R2C / C2R, half on both sides
    const bool half_in = g.role_half[rq.in_role], half_out = g.role_half[rq.out_role];
    const bool half = half_in && half_out && (rq.ew_op == 1 || rq.ew_op == 2);   // B2_EW_R2C_POST, B2_EW_C2R_PRE
    if ((half_in || half_out) && !half) return R_UNSUPPORTED_FFT_LENGTH;
    const b2_kernel_info* k = b2_find_kernel(B2_KIND_ELEMENTWISE, g.prec, 0, 0, half ? (B2_OP_HALF_IN | B2_OP_HALF_OUT) : 0);
    if (!k) return R_UNSUPPORTED_FFT_LENGTH;
    std::vector<Dim> m = merge_dims(lines);
    if (m.size() > 1 + B2_MAX_OUTER) return R_UNSUPPORTED_FFT_LENGTH;
    PassPlan pp;
    pp.k = k;
    b2_pass_params& P = pp.P;
    P.in_es = rq.in_es; P.out_es = rq.out_es;
    Dim grp = m.empty() ? Dim{1, 0, 0} : m[0];
    P.G = (uint32_t)grp.n; P.in_gs = grp.is; P.out_gs = grp.os;
    uint64_t grid = grp.n;
    for (int d = 0; d < B2_MAX_OUTER; ++d) {
        if (d + 1 < (int)m.size()) { P.nb[d] = (uint32_t)m[d + 1].n; P.in_bs[d] = m[d + 1].is; P.out_bs[d] = m[d + 1].os; }
        else { P.nb[d] = 1; P.in_bs[d] = 0; P.out_bs[d] = 0; }
        grid *= P.nb[d];
    }
    const uint32_t per_cta = 256 * 8;   // B2_EW_THREADS * B2_EW_PER_THREAD
    const uint32_t chunks = (rq.ew_items + per_cta - 1) / per_cta;
    grid *= chunks;
    if (grid == 0 || grid > 0x7fffffffull) return R_UNSUPPORTED_FFT_LENGTH;
    pp.grid = (unsigned)grid;
    P.tpl = chunks;
    P.n = rq.n; P.load_io = rq.ew_op; P.store_io = rq.store_io; P.dst_flags = rq.dst_flags; P.ops = rq.ops; P.scale = rq.scale;
    P.inverse = rq.inv; P.inner_inverse = rq.inner_inverse;
    P.in_len = rq.in_len; P.out_len = rq.out_len;
    P.aux_u0 = rq.aux_u0; P.aux_u1 = rq.aux_u1;
    pp.in_role = rq.in_role; pp.out_role = rq.out_role;
    pp.in_off = rq.in_base; pp.out_off = rq.out_base;
    pp.lut_id = lut_for(g, std::vector<int>{});
    pp.aux0_id = rq.aux0; pp.aux1_id = rq.aux1;
    char buf[200];
    snprintf(buf, sizeof buf, "%s elementwise op=%d items=%u grid=%u%s", rq.what, rq.ew_op, rq.ew_items, pp.grid, half ? " half in+out" : "");
    pp.note = buf;
    list.push_back(pp);
    return R_SUCCESS;
}

// total number of lines and a packed scratch layout for them ([line][M])
uint64_t count_lines(const std::vector<Dim>& lines) {
    uint64_t c = 1;
    for (const Dim& d : lines) c *= d.n;
    return c;
}

// smallest padded length >= 2N-1 with a one-launch Bluestein kernel (stockham.cuh RMODE 11), 0 if there is none
uint64_t blue1_length(const PlanGraph& g, uint64_t N) {
    if (getenv("B200FFT_NO_FUSED_BLUESTEIN")) return 0;
    // measured against the two-launch Bluestein transform: one launch wins up to a padded length of 3584 in FP32 and ties
    // or loses above (32 points per thread at 2 CTAs per SM); in FP64 it wins at every length it exists for
    const uint64_t limit = getenv("B200FFT_FORCE_BLUESTEIN") ? ~0ull : (g.prec == B2_PREC_F32 ? 3584 : 4096);
    if (2 * N - 1 > limit) return 0;
    uint64_t M1 = 0;
    for (int i = 0; i < b2_kernel_count(); ++i) {
        const b2_kernel_info* k = b2_kernel_at(i);
        if (k->kind != B2_KIND_ROWS || k->prec != g.prec || k->ops != B2_OP_BLUE_FUSED || k->inv != 0) continue;
        const uint64_t n = (uint64_t)k->n;
        if (n >= 2 * N - 1 && (M1 == 0 || n < M1)) M1 = n;
    }
    return M1;
}

// is there a pair of specialised two-launch Bluestein kernels (RMODE 7 / 8) for some padded length >= 2N-1 ?
bool blue2_available(const PlanGraph& g, uint64_t N) {
    for (int i = 0; i < b2_kernel_count(); ++i) {
        const b2_kernel_info* k = b2_kernel_at(i);
        if (k->kind != B2_KIND_ROWS || k->prec != g.prec || k->ops != B2_OP_BLUESTEIN || k->inv != 0) continue;
        if ((uint64_t)k->n >= 2 * N - 1 && b2_find_kernel(B2_KIND_ROWS, g.prec, k->n, 1, B2_OP_BLUESTEIN)) return true;
    }
    return false;
}

int plan_bluestein(PlanGraph& g, std::vector<PassPlan>& list, const C2CJob& job) {
    // X[k] = conj(b_k) * sum_n (x_n conj(b_n)) b_{k-n},  b_n = e^{i pi n^2/N}   (API guide :465-493)
    const uint64_t N = job.N;
    uint64_t M = 1;
    while (M < 2 * N - 1) M <<= 1;
    // contiguous lines: a smooth padded length between the powers of two when both specialised Bluestein launches exist for it
    if (!job.unit_lines && job.es_in == 1 && job.es_out == 1 && !getenv("B200FFT_BLUESTEIN_POW2")) {
        for (int i = 0; i < b2_kernel_count(); ++i) {
            const b2_kernel_info* k = b2_kernel_at(i);
            if (k->kind != B2_KIND_ROWS || k->prec != g.prec || k->ops != B2_OP_BLUESTEIN || k->inv != 0) continue;
            const uint64_t n = (uint64_t)k->n;
            if (n >= 2 * N - 1 && n < M && b2_find_kernel(B2_KIND_ROWS, g.prec, k->n, 1, B2_OP_BLUESTEIN)) M = n;
        }
    }
    // contiguous lines: the whole transform in ONE launch (stockham.cuh RMODE 11: chirp, FFT_M, filter, IFFT_M, chirp with the
    // padded line never leaving the SM) on the smallest padded length that has such a kernel.  No scratch, one HBM read and one
    // write of the N-point line instead of 2 + 2 padded ones.  B200FFT_NO_FUSED_BLUESTEIN=1 keeps the two launches (A/B timing).
    if (!job.unit_lines && job.es_in == 1 && job.es_out == 1) {
        const uint64_t M1 = blue1_length(g, N);
        if (M1) {
            PassReq f1;
            f1.kind = B2_KIND_ROWS; f1.n = (int)M1; f1.inv = 0; f1.runtime_inverse = job.inv;
            f1.ops = B2_OP_BLUE_FUSED | (job.scale != 1.0 ? B2_OP_SCALE : 0); f1.scale = job.scale;
            f1.in_es = f1.out_es = 1;
            if (job.lines.empty()) f1.group = Dim{1, 0, 0};
            else { f1.group = job.lines[0]; f1.outer.assign(job.lines.begin() + 1, job.lines.end()); }
            f1.in_role = job.in_role; f1.out_role = job.out_role; f1.in_base = job.in_base; f1.out_base = job.out_base;
            f1.in_len = (uint32_t)N; f1.out_len = (uint32_t)N;
            f1.aux0 = aux_for(g, AUX_BLUE_CHIRP, N); f1.aux1 = aux_for(g, AUX_BLUE_FILTER, N, M1);
            f1.what = "bluestein in one launch: chirp+fft+filter+ifft+chirp (specialised)";
            return emit(g, list, f1);
        }
    }
    const uint64_t L = count_lines(job.lines);
    if (!generic_fits(g, M)) {
        // padded length beyond one shared-memory pass: chirp/zero-pad, FFT_M (Four-Step), filter, IFFT_M, post-chirp as
        // separate launches on packed scratch lines; scratch = [lines][M] twice (data + Four-Step scratch)
        if (M > (1ull << 26) || L * M > (1ull << 32)) return R_UNSUPPORTED_FFT_LENGTH;
        const int chirp_l = aux_for(g, AUX_BLUE_CHIRP, N), filt_l = aux_for(g, AUX_BLUE_FILTER, N, M);
        std::vector<Dim> to_tmp = job.lines, from_tmp = job.lines, packed;
        int64_t run = (int64_t)M;
        for (size_t i = 0; i < job.lines.size(); ++i) {
            to_tmp[i].os = run; from_tmp[i].is = run;
            packed.push_back(Dim{job.lines[i].n, run, run});
            run *= (int64_t)job.lines[i].n;
        }
        const int64_t r0 = job.tmp_base, r1 = job.tmp_base + (int64_t)(L * M);
        PassReq pre;
        pre.elementwise = true; pre.ew_op = 0; pre.ew_items = (uint32_t)M; pre.n = (int)M;
        pre.in_len = (uint32_t)N; pre.out_len = (uint32_t)M; pre.ops = B2_OP_MUL_IN; pre.aux0 = chirp_l;
        pre.inv = job.inv; pre.in_es = job.es_in; pre.out_es = 1;
        pre.in_role = job.in_role; pre.out_role = ROLE_TEMP; pre.in_base = job.in_base; pre.out_base = r0;
        pre.what = "bluestein chirp+pad";
        int rcl = emit_ew(g, list, pre, to_tmp);
        if (rcl != R_SUCCESS) return rcl;
        C2CJob f;
        f.N = M; f.inv = 0; f.es_in = f.es_out = 1; f.lines = packed; f.unit_lines = false;
        f.in_role = f.out_role = ROLE_TEMP; f.in_base = f.out_base = r0; f.tmp_base = r1; f.scale = 1.0;
        if ((rcl = plan_c2c(g, list, f)) != R_SUCCESS) return rcl;
        PassReq mid;
        mid.elementwise = true; mid.ew_op = 0; mid.ew_items = (uint32_t)M; mid.n = (int)M;
        mid.in_len = mid.out_len = (uint32_t)M; mid.ops = B2_OP_MUL_IN; mid.aux0 = filt_l;
        mid.in_es = mid.out_es = 1; mid.in_role = mid.out_role = ROLE_TEMP; mid.in_base = mid.out_base = r0;
        mid.what = "bluestein filter";
        if ((rcl = emit_ew(g, list, mid, packed)) != R_SUCCESS) return rcl;
        f.inv = 1;
        if ((rcl = plan_c2c(g, list, f)) != R_SUCCESS) return rcl;
        PassReq post;
        post.elementwise = true; post.ew_op = 0; post.ew_items = (uint32_t)N; post.n = (int)M;
        post.in_len = (uint32_t)M; post.out_len = (uint32_t)N; post.ops = B2_OP_MUL_IN | (job.scale != 1.0 ? B2_OP_SCALE : 0);
        post.aux0 = chirp_l; post.scale = job.scale; post.inner_inverse = job.inv;
        post.in_es = 1; post.out_es = job.es_out;
        post.in_role = ROLE_TEMP; post.out_role = job.out_role; post.in_base = r0; post.out_base = job.out_base;
        post.what = "bluestein post-chirp";
        g.temp_elems = std::max<uint64_t>(g.temp_elems, (uint64_t)r1 + L * M);
        return emit_ew(g, list, post, from_tmp);
    }
    g.temp_elems = std::max<uint64_t>(g.temp_elems, (uint64_t)job.tmp_base + L * M);
    const int chirp = aux_for(g, AUX_BLUE_CHIRP, N), filt = aux_for(g, AUX_BLUE_FILTER, N, M);
    // scratch lines are packed [.. outer ..][group][M]
    std::vector<Dim> in_lines = job.lines, out_lines = job.lines;
    int64_t run = (int64_t)M;
    for (size_t i = 0; i < job.lines.size(); ++i) {
        in_lines[i].os = run;            // pass 1 writes packed scratch
        out_lines[i].is = run;           // pass 2 reads packed scratch
        run *= (int64_t)job.lines[i].n;
    }
    auto mk = [&](const std::vector<Dim>& ln, PassReq& rq) {
        if (ln.empty()) rq.group = Dim{1, 0, 0};
        else { rq.group = ln[0]; rq.outer.assign(ln.begin() + 1, ln.end()); }
    };
    // contiguous lines: both launches on the specialised kernels (chirp / filter fused into their load / store)
    if (!job.unit_lines && job.es_in == 1 && job.es_out == 1 && M <= 0x7fffffff &&
        b2_find_kernel(B2_KIND_ROWS, g.prec, (int)M, 0, B2_OP_BLUESTEIN) && b2_find_kernel(B2_KIND_ROWS, g.prec, (int)M, 1, B2_OP_BLUESTEIN)) {
        PassReq fa;
        fa.kind = B2_KIND_ROWS; fa.n = (int)M; fa.inv = 0; fa.runtime_inverse = job.inv; fa.ops = B2_OP_BLUESTEIN;
        fa.in_es = fa.out_es = 1;
        mk(in_lines, fa);
        fa.in_role = job.in_role; fa.out_role = ROLE_TEMP; fa.in_base = job.in_base; fa.out_base = job.tmp_base;
        fa.in_len = (uint32_t)N; fa.aux0 = chirp; fa.aux1 = filt;
        fa.what = "bluestein 1/2 chirp+fft+filter (specialised)";
        int rcf = emit(g, list, fa);
        if (rcf != R_SUCCESS) return rcf;
        PassReq fb;
        fb.kind = B2_KIND_ROWS; fb.n = (int)M; fb.inv = 1; fb.runtime_inverse = job.inv;
        fb.ops = B2_OP_BLUESTEIN | (job.scale != 1.0 ? B2_OP_SCALE : 0); fb.scale = job.scale;
        fb.in_es = fb.out_es = 1;
        mk(out_lines, fb);
        fb.in_role = ROLE_TEMP; fb.out_role = job.out_role; fb.in_base = job.tmp_base; fb.out_base = job.out_base;
        fb.out_len = (uint32_t)N; fb.aux0 = chirp;
        fb.what = "bluestein 2/2 ifft+chirp (specialised)";
        return emit(g, list, fb);
    }
    PassReq a;
    a.kind = job.unit_lines ? B2_KIND_COLS : B2_KIND_ROWS;
    if (job.unit_lines) a.kind = B2_KIND_ROWS_TOUT, a.kind = B2_KIND_COLS;
    a.n = (int)M; a.inv = job.inv; a.ops = B2_OP_MUL_IN | B2_OP_MUL_OUT; a.force_generic = true;
    a.in_es = job.es_in; a.out_es = 1;
    mk(in_lines, a);
    a.in_role = job.in_role; a.out_role = ROLE_TEMP;
    a.in_len = (uint32_t)N;
    a.aux0 = chirp; a.aux1 = filt;
    a.what = "bluestein 1/2 chirp+fft+filter";
    // load side may be strided (qfast) but the packed scratch store is contiguous per line
    int rc = emit(g, list, a);
    if (rc != R_SUCCESS) return rc;
    list.back().P.store_qfast = 0;
    list.back().P.load_qfast = job.unit_lines ? 1 : 0;
    PassReq b;
    b.kind = job.unit_lines ? B2_KIND_COLS : B2_KIND_ROWS;
    b.n = (int)M; b.inv = job.inv; b.inner_inverse = 1; b.ops = B2_OP_MUL_OUT | (job.scale != 1.0 ? B2_OP_SCALE : 0);
    b.force_generic = true;
    b.in_es = 1; b.out_es = job.es_out;
    mk(out_lines, b);
    b.in_role = ROLE_TEMP; b.out_role = job.out_role;
    b.out_len = (uint32_t)N;
    b.aux1 = chirp;
    b.scale = job.scale;
    b.what = "bluestein 2/2 ifft+chirp";
    rc = emit(g, list, b);
    if (rc != R_SUCCESS) return rc;
    list.back().P.load_qfast = 0;
    list.back().P.store_qfast = job.unit_lines ? 1 : 0;
    return R_SUCCESS;
}

// Two-factor Four-Step just emitted as list[ia] (strided + phase, -> temp) and list[ia + 1] (contiguous + transpose,
// temp ->): run both as ONE persistent launch with the intermediate in an L2-resident ring (fused4.cuh) when a fused
// kernel exists for (n1, n2).  B200FFT_NO_FUSED4=1 keeps the two launches; B200FFT_FUSED_UNIT_KB / B200FFT_FUSED_RING /
// B200FFT_FUSED_RING_MB tune the ring (unit size, slots, total size).
void try_fuse(PlanGraph& g, std::vector<PassPlan>& list, size_t ia) {
    if (!fused4_enabled() || ia + 2 != list.size() || half_plan(g)) return;
    PassPlan& a = list[ia];
    PassPlan& b = list[ia + 1];
    if (a.out_role != ROLE_TEMP || b.in_role != ROLE_TEMP || a.sync_before || b.sync_before) return;
    if (!a.k || !b.k || a.k->kind != B2_KIND_COLS || b.k->kind != B2_KIND_ROWS_TOUT) return;
    const b2_fused_info* fk = b2_find_fused(g.prec, (int)a.P.n, (int)b.P.n, a.k->inv);
    if (!fk) return;
    uint64_t nseq = 1, nseq_b = 1;
    for (int d = 0; d < B2_MAX_OUTER; ++d) { nseq *= a.P.nb[d]; nseq_b *= b.P.nb[d]; }
    if (nseq != nseq_b || nseq > 0x7fffffffull) return;
    // the tiles are copied in by TMA: whole tiles only, and pass A's input must be ONE dense [sequence][n1][n2] array
    if (a.P.G % fk->qa || b.P.G % fk->qb || a.in_scalar || b.out_scalar) return;
    if (a.P.nb[1] != 1 || a.P.nb[2] != 1 || (a.P.nb[0] > 1 && a.P.in_bs[0] != (int64_t)((uint64_t)a.P.n * b.P.n)) || a.P.in_gs != 1) return;
    const uint64_t N = (uint64_t)a.P.n * b.P.n, esz = esize(g), seq_bytes = N * esz;
    // K = CTAs per group: every CTA of a group takes tiles r, r+K, ... of both passes of one sequence per phase.  One or two
    // tiles of each pass per CTA and phase keep the groups small enough to fill the device evenly and large enough that the
    // scratch of all groups (2 sequences each) stays well inside L2:  K = max(TA, TB) / 2, at least 8, at most 132 (the
    // H100's SMs: the CTAs of a group wait for each other, so one group must be resident at once even at one CTA per SM).
    const uint64_t ga = (a.P.G + fk->qa - 1) / fk->qa, gb = (b.P.G + fk->qb - 1) / fk->qb;
    uint64_t K = std::max<uint64_t>(std::max(ga, gb) / 2, 8);
    if (seq_bytes >= (4ull << 20)) K = std::max(ga, gb);              // long sequences: one tile per CTA and phase, fewer groups
    K = std::min<uint64_t>(K, 132);
    if (const char* e = getenv("B200FFT_FUSED_GROUP")) K = std::max<uint64_t>(1, strtoull(e, nullptr, 10));
    const uint64_t U = K, NU = 0, R = 2, L = 0;
    if (nseq * (ga + gb) > 0x7fffffffull) return;
    a.fused = fk;
    a.fz_nseq = (uint32_t)nseq; a.fz_U = (uint32_t)U; a.fz_NU = (uint32_t)NU; a.fz_R = (uint32_t)R;
    a.fz_TA = (uint32_t)ga; a.fz_TB = (uint32_t)gb; a.fz_L = (uint32_t)L;
    a.lut_id_plain = a.lut_id; b.lut_id_plain = b.lut_id;
    a.lut_id = lut_for(g, std::vector<int>(fk->radices_a, fk->radices_a + fk->ns_a));
    b.lut_id = lut_for(g, std::vector<int>(fk->radices_b, fk->radices_b + fk->ns_b));
    g.ctl_words = std::max<uint64_t>(g.ctl_words, B2_FCTL_WORDS);
    char buf[256];
    snprintf(buf, sizeof buf, " [fused with the next launch: %s, groups of %llu CTAs, %llu + %llu tiles per sequence]", fk->name,
             (unsigned long long)K, (unsigned long long)ga, (unsigned long long)gb);
    a.note += buf;
    b.note += " [runs inside the previous launch]";
}

// Two-factor Four-Step just emitted as list[ia] (COLS n1 + phase, -> temp) and list[ia + 1] (ROWS_TOUT n2, temp ->): run both
// as ONE launch of thread-block clusters (cluster4.cuh), one cluster per sequence with the intermediate in distributed shared
// memory, when a cluster kernel is registered for (n1, n2) with the very CTA shapes and radix schedules of the two kernels
// (the results stay bit-identical to the two launches), both sides are dense FP32 complex, and the device can schedule
// that cluster.  The opt-in L2 fusion (B200FFT_FUSED4) keeps priority.  B200FFT_NO_CLUSTER4=1 (read per plan) keeps the two
// launches: a test hook for the bit-for-bit comparison and for A/B timing.
void try_cluster(PlanGraph& g, std::vector<PassPlan>& list, size_t ia) {
    const char* off = getenv("B200FFT_NO_CLUSTER4");
    if ((off && *off && *off != '0') || ia + 2 != list.size() || half_plan(g) || g.prec != B2_PREC_F32) return;
    PassPlan& a = list[ia];
    PassPlan& b = list[ia + 1];
    if (a.fused || a.sync_before || b.sync_before || a.in_scalar || b.out_scalar) return;
    if (!a.k || !b.k || a.k->jit || b.k->jit || a.k->pipelined || b.k->pipelined || a.k->kind != B2_KIND_COLS || b.k->kind != B2_KIND_ROWS_TOUT) return;
    if (a.k->ops != B2_OP_TWIDDLE_OUT || b.k->ops != 0 || a.k->inv != b.k->inv || a.k->v != 1 || b.k->v != 1) return;
    const b2_cluster_info* ck = b2_find_cluster(g.prec, (int)a.P.n, (int)b.P.n, a.k->inv);
    if (!ck) return;
    // the stage code of exactly these two kernels
    if (ck->tpl_a != a.k->tpl || ck->q_a != a.k->q || ck->tpl_b != b.k->tpl || ck->q_b != b.k->q || ck->ns_a != a.k->ns ||
        ck->ns_b != b.k->ns)
        return;
    for (int s = 0; s < ck->ns_a; ++s) if (ck->radices_a[s] != a.k->radices[s]) return;
    for (int s = 0; s < ck->ns_b; ++s) if (ck->radices_b[s] != b.k->radices[s]) return;
    // one dense n1 x n2 sequence per outer coordinate: columns with unit pitch and element stride n2 in, rows transposed out
    const int64_t n1 = a.P.n, n2 = b.P.n;
    if (a.P.G != (uint32_t)n2 || b.P.G != (uint32_t)n1 || a.P.in_gs != 1 || a.P.in_es != n2 || b.P.out_gs != 1 || b.P.out_es != n1) return;
    if (a.P.tw_sel != 0 || b.P.tw_sel != 0 || a.P.tw_line0 != 0) return;
    uint64_t nseq = 1, nseq_b = 1;
    for (int d = 0; d < B2_MAX_OUTER; ++d) { nseq *= a.P.nb[d]; nseq_b *= b.P.nb[d]; }
    if (nseq != nseq_b || nseq * (uint64_t)ck->cluster > 0x7fffffffull) return;
    // in place: a cluster reads its whole sequence before it writes any of it, so input and output may be the same memory
    // only with the same layout (each sequence then overwrites exactly its own points)
    if (a.in_role == b.out_role) {
        if (a.in_off != b.out_off) return;
        for (int d = 0; d < B2_MAX_OUTER; ++d)
            if (a.P.nb[d] != b.P.nb[d] || (a.P.nb[d] > 1 && a.P.in_bs[d] != b.P.out_bs[d])) return;
    }
    if (ck->max_active(g.desc.device) <= 0) return;      // the device cannot hold such a cluster (or there is none)
    a.cluster = ck;
    a.cl_nseq = (uint32_t)nseq;
    char buf[256];
    snprintf(buf, sizeof buf, " [one cluster launch with the next pass: %s, clusters of %d CTAs]", ck->name, ck->cluster);
    const size_t at = a.note.find(" n=");         // "<what> n=...": name the launch after both passes
    if (at != std::string::npos) a.note = "four-step 1/2+2/2 in one cluster launch" + a.note.substr(at);
    a.note += buf;
    b.note += " [runs inside the previous launch]";
}

int plan_c2c(PlanGraph& g, std::vector<PassPlan>& list, const C2CJob& job) {
    const uint64_t N = job.N;
    const int sc_ops = (job.scale != 1.0) ? B2_OP_SCALE : 0;
    std::vector<Dim> sliced = job.lines;
    int64_t slice_in = 0, slice_out = 0;
    if (job.line_world > 1) {
        const int rs = share_lines(sliced, job.line_world, job.line_rank, job.line_ragged, slice_in, slice_out);
        if (rs != R_SUCCESS) return rs;
    }
    std::vector<Dim> m = merge_dims(sliced);
    const bool contiguous = (job.es_in == 1 && job.es_out == 1);
    const int kind = job.unit_lines ? B2_KIND_COLS : B2_KIND_ROWS;
    const size_t first_launch = list.size();
    struct SyncMark {     // marks the first launch this job emits (whatever branch emits it)
        std::vector<PassPlan>& l; size_t at; bool on;
        ~SyncMark() { if (on && l.size() > at) l[at].sync_before = true; }
    } sync_mark{list, first_launch, job.sync_first};

    if (N == 1) return R_SUCCESS;   // length-1 transform is the identity
    const bool dist = job.world > 1;
    if (dist && (!contiguous || job.unit_lines || count_lines(job.lines) != 1 || !is_smooth(N))) return R_UNSUPPORTED_FFT_LENGTH;
    if (!is_smooth(N)) return plan_bluestein(g, list, job);
    // The Rader stage of the runtime-scheduled kernel is a direct O(p^2) product and measured slower than the two fused
    // Bluestein launches wherever those exist (padded length M <= 4096, i.e. N <= 2048); above that Bluestein needs 5-7
    // launches and the two are comparable.  So a contiguous 1-D length up to 2048
    // with a prime factor of 17 or more runs as Bluestein unless a curated kernel with a direct prime butterfly exists for it
    // (the {17..31} * 2^k lengths).  Factors of a Four-Step split and strided axes keep the Rader stages.
    // Round 2, later: the whole Bluestein transform in ONE launch (blue1_length: padded lengths up to 8192 in FP32, 4096 in FP64)
    // extends the rule to N <= 4096 / 2048.  B200FFT_FORCE_BLUESTEIN=1 sends every contiguous length that way
    // (tests, and A/B timing against the runtime-scheduled kernel on smooth lengths).
    // ... and to every length whose padded transform still has the two specialised launches (FP32: padded length 8192, N <= 4096),
    // where it also measured faster than the Rader stages of the runtime-scheduled kernel
    if (contiguous && !job.unit_lines && !dist && (N <= 2048 || blue1_length(g, N) || blue2_available(g, N)) && !(job.extra_ops & B2_OP_CONV) && !getenv("B200FFT_RADER_MAX_PRIME") &&
        !b2_find_kernel(kind, g.prec, (int)N, 0, 0)) {
        uint64_t mm = N;
        for (int f : {2, 3, 5, 7, 11, 13}) while (mm % f == 0) mm /= f;
        if (mm > 1) return plan_bluestein(g, list, job);
    }
    if (contiguous && !job.unit_lines && !dist && !(job.extra_ops & B2_OP_CONV) && N > 1 && getenv("B200FFT_FORCE_BLUESTEIN") && blue1_length(g, N))
        return plan_bluestein(g, list, job);

    // a strided axis served only by the runtime-scheduled kernel with fewer than 8 neighbouring lines per CTA would
    // read 8..56-byte row fragments: split it instead (falls through to the strided Four-Step below)
    bool poor_strided = false;
    if (job.unit_lines && !b2_find_kernel(kind, g.prec, (int)std::min<uint64_t>(N, 0x7fffffff), 0, 0) && generic_fits(g, N)) {
        const uint64_t per_line = 2ull * (uint64_t)(pad_of(g, N) | 1) * esize(g);
        poor_strided = (GENERIC_SMEM_LIMIT / per_line) < 8 && N >= 64;
    }
    // specialised strided kernels with fewer than 8 neighbouring lines per CTA (N >= 4096) are slower than two
    // launches of well-shaped ones (measured per 2 GiB pass)
    if (job.unit_lines) {
        const b2_kernel_info* kk = b2_find_kernel(kind, g.prec, (int)std::min<uint64_t>(N, 0x7fffffff), 0, 0);
        if (kk && kk->q < 8 && N >= 2048) poor_strided = true;
    }
    bool try_single = !dist && N <= max_single_env() && single_ok(g, kind, N, 0) && (!half_plan(g) || N <= (job.unit_lines ? 2048u : 8192u));
    if (job.extra_ops & B2_OP_CONV) {
        if (!b2_find_kernel(kind, g.prec, (int)std::min<uint64_t>(N, 0x7fffffff), 0, B2_OP_CONV)) return R_UNSUPPORTED_FFT_LENGTH;
        try_single = true; poor_strided = false;
    }
    if (try_single && poor_strided) {
        // only if a split exists
        bool can_split = false;
        for (uint64_t n2 = 2; n2 * 2 <= N && !can_split; ++n2)
            if (N % n2 == 0 && single_ok(g, B2_KIND_COLS, N / n2, B2_OP_TWIDDLE_OUT) && single_ok(g, B2_KIND_COLS, n2, 0) &&
                b2_find_kernel(B2_KIND_COLS, g.prec, (int)(N / n2), 0, B2_OP_TWIDDLE_OUT) && b2_find_kernel(B2_KIND_COLS, g.prec, (int)n2, 0, 0))
                can_split = true;
        if (can_split) try_single = false;
    }
    if (try_single) {
        PassReq rq;
        rq.kind = kind; rq.n = (int)N; rq.inv = job.inv; rq.ops = sc_ops | job.extra_ops;
        rq.aux_u0 = job.aux_u0; rq.aux_u1 = job.aux_u1;
        rq.in_es = job.es_in; rq.out_es = job.es_out;
        if (job.unit_lines) {
            // keep the unit-stride dimension as the grouped one
            if (!m.empty() && m[0].is == 1 && m[0].os == 1) { rq.group = m[0]; m.erase(m.begin()); }
            else rq.group = Dim{1, 1, 1};
        } else {
            if (m.empty()) rq.group = Dim{1, (int64_t)N, (int64_t)N};
            else { rq.group = m[0]; m.erase(m.begin()); }
        }
        rq.outer = m;
        rq.in_role = job.in_role; rq.out_role = job.out_role;
        rq.in_base = job.in_base + slice_in; rq.out_base = job.out_base + slice_out;
        rq.scale = job.scale;
        rq.what = job.unit_lines ? "strided axis" : "single-pass";
        return emit(g, list, rq);
    }
    if (job.unit_lines) {
        // long strided axis: two-launch Four-Step along the stride; neighbouring lanes still walk the unit-stride
        // dimension, the sub-sequence index n2 / k1 becomes an outer dimension (and the phase "line" coordinate)
        if (m.empty() || m[0].is != 1 || m[0].os != 1) return R_UNSUPPORTED_FFT_LENGTH;
        uint64_t best1 = 0, best2 = 0, bestc = ~0ull;
        for (uint64_t n2 = 2; n2 * 2 <= N; ++n2) {
            if (N % n2) continue;
            const uint64_t n1 = N / n2;
            if (!single_ok(g, B2_KIND_COLS, n1, B2_OP_TWIDDLE_OUT) || !single_ok(g, B2_KIND_COLS, n2, 0)) continue;
            uint64_t c = std::max(n1, n2) * 4 + (n2 < n1 ? 1 : 0);
            if (!b2_find_kernel(B2_KIND_COLS, g.prec, (int)n1, 0, B2_OP_TWIDDLE_OUT)) c += 1u << 20;
            if (!b2_find_kernel(B2_KIND_COLS, g.prec, (int)n2, 0, 0)) c += 1u << 20;
            if (c < bestc) { bestc = c; best1 = n1; best2 = n2; }
        }
        if (!best1) return R_UNSUPPORTED_FFT_LENGTH;
        const uint64_t N1 = best1, N2 = best2;
        uint64_t extent = (uint64_t)job.es_out * N;
        for (const Dim& d : job.lines) extent = std::max<uint64_t>(extent, (uint64_t)d.n * (uint64_t)d.os);
        g.temp_elems = std::max<uint64_t>(g.temp_elems, (uint64_t)job.tmp_base + extent);
        const Dim unit = m[0];
        std::vector<Dim> rest(m.begin() + 1, m.end());
        PassReq a;
        a.kind = B2_KIND_COLS; a.n = (int)N1; a.inv = job.inv; a.ops = B2_OP_TWIDDLE_OUT;
        a.in_es = job.es_in * (int64_t)N2; a.out_es = job.es_out * (int64_t)N2;
        a.group = unit;
        a.outer.push_back(Dim{N2, job.es_in, job.es_out});
        a.tw_outer = 0;
        for (const Dim& d : rest) a.outer.push_back(Dim{d.n, d.is, d.os});
        a.in_role = job.in_role; a.out_role = ROLE_TEMP;
        a.in_base = job.in_base + slice_in; a.out_base = job.tmp_base + slice_out;
        a.twM = N;
        a.what = "strided four-step 1/2";
        int rc2 = emit(g, list, a);
        if (rc2 != R_SUCCESS) return rc2;
        PassReq b;
        b.kind = B2_KIND_COLS; b.n = (int)N2; b.inv = job.inv; b.ops = sc_ops;
        b.in_es = job.es_out; b.out_es = job.es_out * (int64_t)N1;
        b.group = Dim{unit.n, 1, 1};
        b.outer.push_back(Dim{N1, job.es_out * (int64_t)N2, job.es_out});
        for (const Dim& d : rest) b.outer.push_back(Dim{d.n, d.os, d.os});
        b.in_role = ROLE_TEMP; b.out_role = job.out_role;
        b.in_base = job.tmp_base + slice_out; b.out_base = job.out_base + slice_out;
        b.scale = job.scale;
        b.what = "strided four-step 2/2";
        return emit(g, list, b);
    }
    if (!contiguous) return R_UNSUPPORTED_FFT_LENGTH;

    std::vector<uint64_t> f = split_four_step(g, N, dist);
    if (f.empty()) return R_UNSUPPORTED_FFT_LENGTH;
    // scratch: sequences keep the output-side layout of the main buffer
    uint64_t extent = N;
    for (const Dim& d : job.lines) extent = std::max<uint64_t>(extent, (uint64_t)d.n * (uint64_t)std::max(d.is, d.os));
    g.temp_elems = std::max<uint64_t>(g.temp_elems, (uint64_t)job.tmp_base + extent);
    std::vector<Dim> s_in_tmp, s_tmp_tmp, s_tmp_out, s_in_in;
    for (const Dim& d : job.lines) {
        // scratch uses the OUTPUT layout (both sides of a temp->temp pass)
        s_in_tmp.push_back(Dim{d.n, d.is, d.os});
        s_tmp_tmp.push_back(Dim{d.n, d.os, d.os});
        s_tmp_out.push_back(Dim{d.n, d.os, d.os});
        s_in_in.push_back(Dim{d.n, d.is, d.is});
    }
    int rc;
    if (f.size() == 2) {
        const uint64_t N1 = f[0], N2 = f[1];
        PassReq a;
        a.kind = B2_KIND_COLS; a.n = (int)N1; a.inv = job.inv; a.ops = B2_OP_TWIDDLE_OUT;
        a.in_es = (int64_t)N2; a.out_es = (int64_t)N2;
        a.group = Dim{N2, 1, 1};
        a.outer = s_in_tmp;
        a.in_role = job.in_role; a.out_role = ROLE_TEMP;
        a.in_base = job.in_base; a.out_base = job.tmp_base;
        a.twM = N;
        a.what = "four-step 1/2 strided+phase";
        if (dist) {
            // columns [rank*N2/R, ...): every column crosses all slabs of the input window (peer loads) and of the
            // temp window (peer stores); the phase line coordinate keeps counting global columns
            uint64_t first;
            if (!slice_dim(a.group, job.world, job.rank, a.in_base, a.out_base, first)) return R_UNSUPPORTED_FFT_LENGTH;
            a.tw_line0 = (uint32_t)first;
            a.sync_before = true;
            a.what = "distributed four-step 1/2 strided+phase (peer loads and stores)";
        }
        if ((rc = emit(g, list, a)) != R_SUCCESS) return rc;
        PassReq b;
        b.kind = B2_KIND_ROWS_TOUT; b.n = (int)N2; b.inv = job.inv; b.ops = sc_ops;
        b.in_es = 1; b.out_es = (int64_t)N1;
        b.group = Dim{N1, (int64_t)N2, 1};
        b.outer = s_tmp_out;
        b.in_role = ROLE_TEMP; b.out_role = job.out_role;
        b.in_base = job.tmp_base; b.out_base = job.out_base;
        b.scale = job.scale;
        b.what = "four-step 2/2 contiguous+transpose";
        if (dist) {
            // rows k1 of this rank's own temp slab (local loads); the transposed store lands in every output slab
            uint64_t first;
            if (!slice_dim(b.group, job.world, job.rank, b.in_base, b.out_base, first)) return R_UNSUPPORTED_FFT_LENGTH;
            b.sync_before = true;
            b.what = "distributed four-step 2/2 contiguous+transpose (peer stores)";
        }
        const size_t ia = list.size() - 1;
        if ((rc = emit(g, list, b)) != R_SUCCESS) return rc;
        if (!dist && job.tmp_base % 16 == 0) try_fuse(g, list, ia);
        if (!dist) try_cluster(g, list, ia);
        return R_SUCCESS;
    }
    const uint64_t N1 = f[0], N2 = f[1], N3 = f[2], M = N2 * N3;
    PassReq a;
    a.kind = B2_KIND_COLS; a.n = (int)N1; a.inv = job.inv; a.ops = B2_OP_TWIDDLE_OUT;
    a.in_es = (int64_t)M; a.out_es = (int64_t)M;
    a.group = Dim{M, 1, 1};
    // first pass runs in place on its input when that is the main buffer, otherwise it moves to temp
    const bool a_inplace = (job.in_role == ROLE_BUFFER) && !dist;
    a.outer = a_inplace ? s_in_in : s_in_tmp;
    a.in_role = job.in_role; a.out_role = a_inplace ? job.in_role : ROLE_TEMP;
    a.in_base = job.in_base; a.out_base = a_inplace ? job.in_base : job.tmp_base;
    a.twM = N;
    a.what = "four-step 1/3 strided+phase";
    if (dist) {
        uint64_t first;
        if (!slice_dim(a.group, job.world, job.rank, a.in_base, a.out_base, first)) return R_UNSUPPORTED_FFT_LENGTH;
        a.tw_line0 = (uint32_t)first;
        a.sync_before = true;
        a.what = "distributed four-step 1/3 strided+phase (peer loads and stores)";
    }
    if ((rc = emit(g, list, a)) != R_SUCCESS) return rc;
    PassReq b;
    b.kind = B2_KIND_COLS; b.n = (int)N2; b.inv = job.inv; b.ops = B2_OP_TWIDDLE_OUT;
    b.in_es = (int64_t)N3; b.out_es = (int64_t)N3;
    b.group = Dim{N3, 1, 1};
    b.outer.push_back(Dim{N1, (int64_t)M, (int64_t)M});
    {
        const std::vector<Dim>& s = a_inplace ? s_in_tmp : s_tmp_tmp;
        b.outer.insert(b.outer.end(), s.begin(), s.end());
    }
    b.in_role = a.out_role; b.out_role = ROLE_TEMP;
    b.in_base = a_inplace ? job.in_base : job.tmp_base; b.out_base = job.tmp_base;
    b.twM = M;
    b.what = "four-step 2/3 strided+phase";
    if (dist) {
        // k1 rows of this rank's own temp slab: local loads, local stores
        uint64_t first;
        if (!slice_dim(b.outer[0], job.world, job.rank, b.in_base, b.out_base, first)) return R_UNSUPPORTED_FFT_LENGTH;
        b.sync_before = true;
        b.what = "distributed four-step 2/3 strided+phase (local)";
    }
    if ((rc = emit(g, list, b)) != R_SUCCESS) return rc;
    PassReq c;
    c.kind = B2_KIND_ROWS_TOUT; c.n = (int)N3; c.inv = job.inv; c.ops = sc_ops;
    c.in_es = 1; c.out_es = (int64_t)(N1 * N2);
    c.group = Dim{N1, (int64_t)M, 1};
    c.outer.push_back(Dim{N2, (int64_t)N3, (int64_t)N1});
    c.outer.insert(c.outer.end(), s_tmp_out.begin(), s_tmp_out.end());
    c.in_role = ROLE_TEMP; c.out_role = job.out_role;
    c.in_base = job.tmp_base; c.out_base = job.out_base;
    c.scale = job.scale;
    c.what = "four-step 3/3 contiguous+transpose";
    if (dist) {
        uint64_t first;
        if (!slice_dim(c.group, job.world, job.rank, c.in_base, c.out_base, first)) return R_UNSUPPORTED_FFT_LENGTH;
        c.what = "distributed four-step 3/3 contiguous+transpose (peer stores)";
    }
    return emit(g, list, c);
}

// ----------------------------------------------------------------------------------------------------------------
struct Layout {            // one side (input or output) of an axis pass
    int role;
    uint64_t stride[B200FFT_MAX_DIMS];   // stride[a] = distance between consecutive indices of dim a+1
    uint64_t batch_stride;
};

// all dims except `axis`, x first when axis != 0; strides taken from the two layouts
std::vector<Dim> other_dims(const PlanGraph& g, const uint64_t* size, uint32_t axis, const Layout& in, const Layout& out) {
    const b200fft_desc& d = g.desc;
    std::vector<Dim> lines;
    for (uint32_t a = 0; a < d.fft_dim; ++a) {
        if (a == axis) continue;
        const int64_t is = a == 0 ? 1 : (int64_t)in.stride[a - 1], os = a == 0 ? 1 : (int64_t)out.stride[a - 1];
        lines.push_back(Dim{size[a], is, os});
    }
    lines.push_back(Dim{g.batches, (int64_t)in.batch_stride, (int64_t)out.batch_stride});
    return lines;
}

// distributed N-D plan: first element of this rank's slab in `buffer` and in scratch (both windows have the same slabs).
// Rank g owns indices [g*n/R, (g+1)*n/R) of the last dimension, so its slab starts g*n/R outermost pitches in -- for R2C
// the pitches of the complex rows, for DCT / DST those of the real rows (real elements); either may be padded so that a slab
// fills whole mapping granules
int64_t slab_base(const PlanGraph& g) {
    const b200fft_desc& d = g.desc;
    const uint32_t la = d.fft_dim - 1;
    return (int64_t)((uint64_t)d.dist_rank * (d.size[la] / d.dist_world) * d.buffer_stride[la - 1]);
}

// distributed N-D plan: one axis of the segment that stays inside this rank's slab, planned by `plan_axis`.  Its scratch must end
// at or before `slab_end` (temp elements), the end of the rank's temp slab: a route that needs more is refused.  `barrier`:
// the segment's first launch waits for every rank.
template <class F>
int plan_in_slab(PlanGraph& g, std::vector<PassPlan>& list, uint64_t slab_end, bool barrier, F&& plan_axis) {
    const uint64_t t0 = g.temp_elems;
    const size_t at = list.size();
    g.temp_elems = 0;
    int r = plan_axis();
    if (r == R_SUCCESS && g.temp_elems > slab_end) r = R_UNSUPPORTED_FFT_LENGTH;
    g.temp_elems = std::max(t0, g.temp_elems);
    if (r == R_SUCCESS && barrier && list.size() > at) list[at].sync_before = true;
    return r;
}

// slab: < 0 ordinary plan;  0: local axis of a distributed N-D plan (this rank's slab only: `size` already holds the slab's
// extent of the last dimension, every base moves to the slab);  1: the axis that crosses the slabs (lines shared out over the ranks)
int plan_c2c_axis(PlanGraph& g, std::vector<PassPlan>& list, const uint64_t* size, uint32_t axis, int inv,
                  const Layout& in, const Layout& out, double scale, int slab = -1, bool sync_first = false) {
    C2CJob job;
    job.N = size[axis]; job.inv = inv;
    job.es_in = axis == 0 ? 1 : (int64_t)in.stride[axis - 1];
    job.es_out = axis == 0 ? 1 : (int64_t)out.stride[axis - 1];
    job.lines = other_dims(g, size, axis, in, out);
    job.unit_lines = (axis != 0);
    job.in_role = in.role; job.out_role = out.role;
    job.scale = scale;
    job.sync_first = sync_first;
    if (slab < 0) {
        if (g.distributed) { job.world = g.desc.dist_world; job.rank = g.desc.dist_rank; }
    } else if (slab == 0) {
        job.in_base = job.out_base = job.tmp_base = slab_base(g);
    } else {
        job.line_world = g.desc.dist_world; job.line_rank = g.desc.dist_rank;
        job.line_ragged = g.desc.perform_r2c != 0;
    }
    return plan_c2c(g, list, job);
}

Layout layout_of(int role, const uint64_t* stride, uint32_t fft_dim) {
    Layout l;
    l.role = role;
    for (int a = 0; a < B200FFT_MAX_DIMS; ++a) l.stride[a] = stride[a];
    l.batch_stride = stride[fft_dim - 1];
    return l;
}

// ---- C2C (any dimensionality) ------------------------------------------------------------------------------------
int plan_direction_c2c(PlanGraph& g, std::vector<PassPlan>& list, int inv) {
    const b200fft_desc& d = g.desc;
    // order of axes: forward 0,1,2..; inverse ..2,1,0 (vkFFT_RunApp.h:111-321 / :466-651)
    std::vector<uint32_t> axes;
    for (uint32_t a = 0; a < d.fft_dim; ++a)
        if (!d.omit_dimension[a] && d.size[a] > 1) axes.push_back(a);
    if (inv) std::reverse(axes.begin(), axes.end());
    double norm = 1.0;
    if (inv && d.normalize)
        for (uint32_t a : axes) norm /= (double)d.size[a];
    axes.erase(std::remove_if(axes.begin(), axes.end(), [&](uint32_t a) { return (int)a == g.skip_axis; }), axes.end());
    // out-of-place plumbing (API guide :365-376): the first launch reads the formatted input, the last launch
    // writes the formatted output, everything in between lives in `buffer`.  The inverse mirrors the forward
    // data flow (outputBuffer -> ... -> buffer, or -> inputBuffer with inverseReturnToInputBuffer).
    const Layout buf = layout_of(ROLE_BUFFER, d.buffer_stride, d.fft_dim);
    const Layout inl = layout_of(ROLE_INPUT, d.input_stride, d.fft_dim);
    const Layout outl = layout_of(ROLE_OUTPUT, d.output_stride, d.fft_dim);
    for (size_t i = 0; i < axes.size(); ++i) {
        const bool first = (i == 0), last = (i + 1 == axes.size());
        Layout in = buf, out = buf;
        if (!inv) {
            if (first && d.is_input_formatted) in = inl;
            if (last && d.is_output_formatted) out = outl;
        } else {
            if (first && d.is_output_formatted) in = outl;
            if (last && d.is_input_formatted && d.inverse_return_to_input) out = inl;
        }
        const size_t before = list.size();
        int rc;
        if (g.distributed && d.fft_dim > 1) {
            // slab decomposition along the last dimension (SURVEY section 8 f4): the lower axes are transformed inside this rank's
            // slab; the last axis is a strided pass over the whole window whose lines are shared out over the ranks -- its loads
            // and stores are the exchange (NVLink reads / writes from inside the FFT launch, as in the 1-D distributed plan).
            // Barriers: before the first launch that reads other ranks' slabs and before the first one that follows it.
            const uint32_t la = d.fft_dim - 1;
            if (axes[i] == la) {
                rc = plan_c2c_axis(g, list, d.size, la, inv, in, out, last ? norm : 1.0, 1, true);
            } else {
                uint64_t lsize[B200FFT_MAX_DIMS];
                for (int a = 0; a < B200FFT_MAX_DIMS; ++a) lsize[a] = d.size[a];
                lsize[la] = d.size[la] / d.dist_world;
                const bool after_cross = inv && i > 0 && axes[i - 1] == la;
                rc = plan_c2c_axis(g, list, lsize, axes[i], inv, in, out, last ? norm : 1.0, 0, after_cross);
            }
        } else {
            // Zero padding at the END of a dimension b (an open system: fft_zeropad_right[b] == size[b], sample_4 / sample_51)
            // makes whole lines of the LOWER axes trivial: forward, every line of axis a < b whose b-coordinate lies in the padded
            // range is all zero (the ranges were cleared above) and stays zero; inverse, it only carries values of the padded
            // range nobody reads.  Those lines are not transformed (the reference skips them the same way,
            // vkFFT_KernelsLevel0/vkFFT_Zeropad.h).  Half-padded 3-D: 1/4 + 1/2 + 1 passes instead of 3.
            uint64_t lsize[B200FFT_MAX_DIMS];
            for (int a = 0; a < B200FFT_MAX_DIMS; ++a) lsize[a] = d.size[a];
            if (!d.frequency_zeropadding && !d.perform_convolution && !d.is_input_formatted && !d.is_output_formatted)
                for (uint32_t b = axes[i] + 1; b < d.fft_dim; ++b)
                    if (d.perform_zeropadding[b] && d.zeropad_right[b] == d.size[b] && d.zeropad_left[b] > 0 && d.zeropad_left[b] < d.size[b] &&
                        !d.omit_dimension[b])
                        lsize[b] = d.zeropad_left[b];
            rc = plan_c2c_axis(g, list, lsize, axes[i], inv, in, out, last ? norm : 1.0);
        }
        if (rc != R_SUCCESS) return rc;
        g.axis_uploads[inv ? 1 : 0][axes[i]] += (uint32_t)(list.size() - before);
    }
    return R_SUCCESS;
}

// ---- R2C / C2R ---------------------------------------------------------------------------------------------------
// Layout facts (vkFFT_InitializeApp.h:994-1040, API guide :305-329): `buffer` holds size[0]/2+1 complex per row
// (bufferStride[0] complex); in place the real rows live in the same rows (2*bufferStride[0] reals apart);
// with isInputFormatted the reals come from inputBuffer with inputBufferStride in REAL elements.
int plan_direction_r2c(PlanGraph& g, std::vector<PassPlan>& list, int inv) {
    const b200fft_desc& d = g.desc;
    const uint64_t N0 = d.size[0], H = N0 / 2 + 1;
    if (d.omit_dimension[0]) return R_UNSUPPORTED_FFT_OMIT;
    if (d.is_output_formatted) return R_UNSUPPORTED_FFT_LENGTH_R2C;
    uint64_t csize[B200FFT_MAX_DIMS];
    for (int a = 0; a < B200FFT_MAX_DIMS; ++a) csize[a] = d.size[a];
    csize[0] = H;                       // the other axes transform H columns (vkFFT_Scheduler.h:2281-2283)
    // distributed (slabs along the last dimension): the x axis and, in 3-D, the y axis run on this rank's slab only
    uint64_t rsize[B200FFT_MAX_DIMS], lcsize[B200FFT_MAX_DIMS];
    for (int a = 0; a < B200FFT_MAX_DIMS; ++a) { rsize[a] = d.size[a]; lcsize[a] = csize[a]; }
    const uint32_t la = d.fft_dim - 1;
    const int64_t base = g.distributed ? slab_base(g) : 0;
    if (g.distributed) { rsize[la] /= d.dist_world; lcsize[la] /= d.dist_world; }
    Layout buf = layout_of(ROLE_BUFFER, d.buffer_stride, d.fft_dim);
    // one batch: its pitch addresses nothing, but sizes the scratch of a Four-Step -- a slab's worth, not the whole window
    if (g.distributed) buf.batch_stride = rsize[la] * d.buffer_stride[la - 1];
    double norm = 1.0;
    if (inv && d.normalize)
        for (uint32_t a = 0; a < d.fft_dim; ++a)
            if (!d.omit_dimension[a]) norm /= (double)d.size[a];
    const bool even = (N0 % 2 == 0) && N0 > 2;   // N0 = 2 has no half-length transform: it takes the zero-imaginary path of the odd lengths
    const uint64_t n = even ? N0 / 2 : N0;
    // half-precision storage: only the even lengths, whose real samples are addressed in pairs (one 32-bit element), and only
    // where the half-length C2C has a half plan.  The runtime-scheduled kernel has no half variant, so a length without a fused
    // half kernel runs as the half-length C2C + the half Hermitian launch, and fails where that C2C does (Bluestein lengths,
    // among them the bare primes 17...31, which a C2C plan sends to Bluestein although a one-radix kernel exists)
    const bool half = half_plan(g);
    if (half && (!even || n == 17 || n == 19 || n == 23 || n == 29 || n == 31)) return R_UNSUPPORTED_FFT_LENGTH_R2C;
    const int hops = half ? (B2_OP_HALF_IN | B2_OP_HALF_OUT) : 0;
    const bool fused = n >= 2 && ((!half && is_smooth(n) && generic_fits(g, n)) ||
                                  (even && b2_find_kernel(B2_KIND_ROWS, g.prec, (int)n, 0, B2_OP_REAL_EVEN | hops) != nullptr));
    const bool odd_composed = !fused && !even && n >= 3;   // long / non-smooth odd lengths: C2C plan on scratch + copy launches
    if (!fused && !even && !odd_composed) return R_UNSUPPORTED_FFT_LENGTH_R2C;

    // real side of the axis-0 launch, in units of the pointer type the operator uses
    const bool real_ext = d.is_input_formatted && (!inv || d.inverse_return_to_input);
    const int real_role = real_ext ? ROLE_INPUT : ROLE_BUFFER;
    // strides of the real rows in REAL elements
    uint64_t rstride[B200FFT_MAX_DIMS];
    for (int a = 0; a < B200FFT_MAX_DIMS; ++a) rstride[a] = real_ext ? d.input_stride[a] : 2 * d.buffer_stride[a];
    const uint64_t rbatch = g.distributed ? 2 * buf.batch_stride : rstride[d.fft_dim - 1];
    if (even)
        for (uint32_t a = 0; a < d.fft_dim; ++a)
            if (rstride[a] % 2) return R_UNSUPPORTED_FFT_LENGTH_R2C;
    const uint64_t unit = even ? 2 : 1;    // even trick addresses the reals as complex pairs

    auto axis0 = [&](bool forward, double scale) -> int {
        PassReq rq;
        rq.kind = B2_KIND_ROWS; rq.n = (int)n; rq.force_generic = true;
        std::vector<Dim> lines;
        for (uint32_t a = 1; a < d.fft_dim; ++a) {
            const int64_t rs = (int64_t)(rstride[a - 1] / unit), cs = (int64_t)d.buffer_stride[a - 1];
            lines.push_back(forward ? Dim{rsize[a], rs, cs} : Dim{rsize[a], cs, rs});
        }
        lines.push_back(forward ? Dim{g.batches, (int64_t)(rbatch / unit), (int64_t)buf.batch_stride}
                                : Dim{g.batches, (int64_t)buf.batch_stride, (int64_t)(rbatch / unit)});
        std::vector<Dim> m = merge_dims(lines);
        if (m.empty()) rq.group = Dim{1, 0, 0};
        else { rq.group = m[0]; m.erase(m.begin()); }
        rq.outer = m;
        rq.in_es = 1; rq.out_es = 1;
        rq.in_base = rq.out_base = base;   // in place: the real pairs and the spectrum start at the same element
        // specialised kernel with the Hermitian pass fused in (one HBM round trip, registers + shared memory)
        if (even && b2_find_kernel(B2_KIND_ROWS, g.prec, (int)n, forward ? 0 : 1, B2_OP_REAL_EVEN | hops)) {
            rq.force_generic = false;
            rq.inv = forward ? 0 : 1;
            rq.ops = B2_OP_REAL_EVEN | ((!forward && scale != 1.0) ? B2_OP_SCALE : 0);
            rq.scale = forward ? 1.0 : scale;
            rq.aux0 = aux_for(g, AUX_R2C, N0);
            rq.in_role = forward ? real_role : ROLE_BUFFER;
            rq.out_role = forward ? ROLE_BUFFER : real_role;
            rq.what = forward ? "r2c axis0 (fused)" : "c2r axis0 (fused)";
            return emit(g, list, rq);
        }
        if (forward) {
            rq.in_role = real_role; rq.out_role = ROLE_BUFFER;
            if (even) { rq.store_io = B2_IO_R2C_EVEN; rq.aux0 = aux_for(g, AUX_R2C, N0); rq.out_len = (uint32_t)(n + 1); }
            else { rq.load_io = B2_IO_REAL; rq.out_len = (uint32_t)H; }
            rq.what = "r2c axis0";
        } else {
            rq.in_role = ROLE_BUFFER; rq.out_role = real_role;
            rq.inner_inverse = 1;
            if (even) { rq.load_io = B2_IO_C2R_EVEN; rq.aux0 = aux_for(g, AUX_R2C, N0); }
            else { rq.load_io = B2_IO_HERM; rq.store_io = B2_IO_REAL; rq.aux_u1 = (uint32_t)N0; }
            rq.ops = (scale != 1.0) ? B2_OP_SCALE : 0;
            rq.scale = scale;
            rq.what = "c2r axis0";
        }
        return emit(g, list, rq);
    };
    // long or non-smooth even lengths: half-length C2C (Four-Step / Bluestein as needed) + separate Hermitian pass
    // (the reference's bigSequenceEvenR2C path, vkFFT_Scheduler.h:2261-2270)
    auto axis0_composed = [&](bool forward, double scale) -> int {
        std::vector<Dim> rc_lines, cc_lines;   // real(complex view)->complex and complex->complex line dims
        for (uint32_t a = 1; a < d.fft_dim; ++a) {
            const int64_t rs = (int64_t)(rstride[a - 1] / 2), cs = (int64_t)d.buffer_stride[a - 1];
            rc_lines.push_back(forward ? Dim{rsize[a], rs, cs} : Dim{rsize[a], cs, rs});
            cc_lines.push_back(Dim{rsize[a], cs, cs});
        }
        rc_lines.push_back(forward ? Dim{g.batches, (int64_t)(rbatch / 2), (int64_t)buf.batch_stride}
                                   : Dim{g.batches, (int64_t)buf.batch_stride, (int64_t)(rbatch / 2)});
        cc_lines.push_back(Dim{g.batches, (int64_t)buf.batch_stride, (int64_t)buf.batch_stride});
        PassReq ew;
        ew.elementwise = true; ew.ew_items = (uint32_t)(n / 2 + 1); ew.n = (int)n;
        ew.in_es = ew.out_es = 1; ew.in_role = ew.out_role = ROLE_BUFFER;
        ew.aux0 = aux_for(g, AUX_R2C, N0);
        ew.in_base = ew.out_base = base;
        C2CJob job;
        job.N = n; job.es_in = job.es_out = 1; job.lines = rc_lines; job.unit_lines = false;
        job.in_base = job.out_base = job.tmp_base = base;
        int r;
        if (forward) {
            job.inv = 0; job.in_role = real_role; job.out_role = ROLE_BUFFER; job.scale = 1.0;
            if ((r = plan_c2c(g, list, job)) != R_SUCCESS) return half ? R_UNSUPPORTED_FFT_LENGTH_R2C : r;
            ew.ew_op = 1; ew.what = "r2c hermitian pass";
            return emit_ew(g, list, ew, cc_lines);
        }
        ew.ew_op = 2; ew.what = "c2r hermitian pass";
        if ((r = emit_ew(g, list, ew, cc_lines)) != R_SUCCESS) return r;
        job.inv = 1; job.in_role = ROLE_BUFFER; job.out_role = real_role; job.scale = scale;
        r = plan_c2c(g, list, job);
        return (r != R_SUCCESS && half) ? R_UNSUPPORTED_FFT_LENGTH_R2C : r;
    };
    // odd lengths the single-launch kernel cannot take (prime factors above 127, or too long for shared memory): the real
    // lines are widened to complex lines in scratch, transformed by an ordinary C2C plan (Bluestein / Four-Step as needed)
    // and the first n/2+1 points copied out; the inverse rebuilds the full Hermitian spectrum first.  Three extra streaming
    // launches -- the reference's generated kernels read the real data directly (vkFFT_ReadWrite.h:411).
    auto axis0_odd = [&](bool forward, double scale) -> int {
        std::vector<Dim> r2t, t2t, t2c;   // real<->scratch, scratch<->scratch, scratch<->complex buffer line dims
        uint64_t ts = N0, nlines = 1;
        for (uint32_t a = 1; a <= d.fft_dim; ++a) {
            const bool isb = (a == d.fft_dim);
            const uint64_t cnt = isb ? g.batches : d.size[a];
            const int64_t rs = (int64_t)(isb ? rbatch : rstride[a - 1]), cs = (int64_t)(isb ? buf.batch_stride : d.buffer_stride[a - 1]);
            r2t.push_back(forward ? Dim{cnt, rs, (int64_t)ts} : Dim{cnt, (int64_t)ts, rs});
            t2t.push_back(Dim{cnt, (int64_t)ts, (int64_t)ts});
            t2c.push_back(forward ? Dim{cnt, (int64_t)ts, cs} : Dim{cnt, cs, (int64_t)ts});
            ts *= cnt; nlines *= cnt;
        }
        const uint64_t region = nlines * N0;
        g.temp_elems = std::max<uint64_t>(g.temp_elems, region);
        PassReq ew;
        ew.elementwise = true; ew.in_es = ew.out_es = 1;
        C2CJob job;
        job.N = N0; job.es_in = job.es_out = 1; job.lines = t2t; job.unit_lines = false;
        job.in_role = job.out_role = ROLE_TEMP; job.tmp_base = (int64_t)region;
        int r;
        if (forward) {
            ew.ew_op = 6; ew.n = (int)N0; ew.ew_items = (uint32_t)N0; ew.in_role = real_role; ew.out_role = ROLE_TEMP;
            ew.what = "odd r2c: real -> complex scratch";
            if ((r = emit_ew(g, list, ew, r2t)) != R_SUCCESS) return r;
            list.back().in_scalar = true;
            job.inv = 0; job.scale = 1.0;
            if ((r = plan_c2c(g, list, job)) != R_SUCCESS) return r;
            ew.ew_op = 0; ew.n = (int)H; ew.ew_items = (uint32_t)H; ew.in_len = ew.out_len = (uint32_t)H;
            ew.in_role = ROLE_TEMP; ew.out_role = ROLE_BUFFER; ew.what = "odd r2c: first n/2+1 points";
            return emit_ew(g, list, ew, t2c);
        }
        ew.ew_op = 7; ew.n = (int)H; ew.ew_items = (uint32_t)H; ew.aux_u0 = (uint32_t)N0; ew.in_role = ROLE_BUFFER; ew.out_role = ROLE_TEMP;
        ew.what = "odd c2r: hermitian expansion";
        if ((r = emit_ew(g, list, ew, t2c)) != R_SUCCESS) return r;
        job.inv = 1; job.scale = 1.0;
        if ((r = plan_c2c(g, list, job)) != R_SUCCESS) return r;
        ew.ew_op = 8; ew.n = (int)N0; ew.ew_items = (uint32_t)N0; ew.aux_u0 = 0; ew.in_role = ROLE_TEMP; ew.out_role = real_role;
        ew.ops = (scale != 1.0) ? B2_OP_SCALE : 0; ew.scale = scale;
        ew.what = "odd c2r: real part";
        if ((r = emit_ew(g, list, ew, r2t)) != R_SUCCESS) return r;
        list.back().out_scalar = true;
        return R_SUCCESS;
    };
    auto axis0_any = [&](bool forward, double scale) -> int {
        return fused ? axis0(forward, scale) : (odd_composed ? axis0_odd(forward, scale) : axis0_composed(forward, scale));
    };
    int rc;
    size_t mark = list.size();
    auto count = [&](uint32_t a) { g.axis_uploads[inv ? 1 : 0][a] += (uint32_t)(list.size() - mark); mark = list.size(); };
    if (g.distributed) {
        // Slabs along the last dimension (DESIGN section 7): x (and y) inside this rank's slab, then -- after a barrier -- the
        // last axis as strided launches over the whole window on this rank's share of the H*ny spectrum columns; the inverse
        // runs the other way round.  Whatever scratch the local launches use must stay inside this rank's temp slab.
        const uint64_t slab_end = (uint64_t)base + rsize[la] * d.buffer_stride[la - 1];
        auto local = [&](uint32_t a, bool barrier) -> int {
            const int r = plan_in_slab(g, list, slab_end, barrier, [&] {
                return a == 0 ? (fused ? axis0(!inv, inv ? norm : 1.0) : axis0_composed(!inv, inv ? norm : 1.0))
                              : plan_c2c_axis(g, list, lcsize, a, inv, buf, buf, 1.0, 0);
            });
            count(a);
            return r;
        };
        if (!inv) {
            for (uint32_t a = 0; a < la; ++a)
                if ((a == 0 || d.size[a] > 1) && (rc = local(a, false)) != R_SUCCESS) return rc;
            if ((rc = plan_c2c_axis(g, list, csize, la, 0, buf, buf, 1.0, 1, true)) != R_SUCCESS) return rc;
            count(la);
        } else {
            if ((rc = plan_c2c_axis(g, list, csize, la, 1, buf, buf, 1.0, 1, true)) != R_SUCCESS) return rc;
            count(la);
            bool barrier = true;
            for (uint32_t a = la; a-- > 0;) {
                if (a > 0 && d.size[a] == 1) continue;
                if ((rc = local(a, barrier)) != R_SUCCESS) return rc;
                barrier = false;
            }
        }
        return R_SUCCESS;
    }
    if (!inv) {
        if ((rc = axis0_any(true, 1.0)) != R_SUCCESS) return rc;
        count(0);
        for (uint32_t a = 1; a < d.fft_dim; ++a) {
            if (d.omit_dimension[a] || d.size[a] == 1 || (int)a == g.skip_axis) continue;
            if ((rc = plan_c2c_axis(g, list, csize, a, 0, buf, buf, 1.0)) != R_SUCCESS) return rc;
            count(a);
        }
    } else {
        for (uint32_t a = d.fft_dim; a-- > 1;) {
            if (d.omit_dimension[a] || d.size[a] == 1 || (int)a == g.skip_axis) continue;
            if ((rc = plan_c2c_axis(g, list, csize, a, 1, buf, buf, 1.0)) != R_SUCCESS) return rc;
            count(a);
        }
        if ((rc = axis0_any(false, norm)) != R_SUCCESS) return rc;
        count(0);
    }
    return R_SUCCESS;
}

// ---- DCT-I..IV ---------------------------------------------------------------------------------------------------
// Real buffer, every non-omitted axis is transformed (API guide :330-339, :581-591).  kind 2/3 swap roles under
// inversion, 1 and 4 are self-inverse.  Lines are paired (two real lines as re/im of one complex line) except
// for DCT-IV which maps one real line of length N to one complex line of length N/2.
int plan_direction_dct(PlanGraph& g, std::vector<PassPlan>& list, int inv) {
    const b200fft_desc& d = g.desc;
    const bool is_dst = d.perform_dst != 0;
    int type = (int)(is_dst ? d.perform_dst : d.perform_dct);
    if (inv && (type == 2 || type == 3)) type = 5 - type;
    const bool conv = g.conv_axis >= 0;   // type-2 forward, kernel product and type-3 inverse of this axis in one launch
    std::vector<uint32_t> axes;
    for (uint32_t a = 0; a < d.fft_dim; ++a)
        if (!d.omit_dimension[a] && d.size[a] > 1 && (int)a != g.skip_axis && (!conv || (int)a == g.conv_axis)) axes.push_back(a);
    if (inv) std::reverse(axes.begin(), axes.end());
    // out of place: the same data flow as plan_direction_c2c -- the first axis reads the formatted source, the last axis
    // writes the formatted destination, everything in between lives in `buffer`.  No launch writes the source.
    const Layout buf = layout_of(ROLE_BUFFER, d.buffer_stride, d.fft_dim);
    const Layout inl = layout_of(ROLE_INPUT, d.input_stride, d.fft_dim);
    const Layout outl = layout_of(ROLE_OUTPUT, d.output_stride, d.fft_dim);
    // One axis.  `size`: the extents its lines are counted over.  Distributed plans (slabs along the last dimension): a local
    // axis gets the slab's extents and `base`, the slab's first real element; the axis that crosses the slabs (`share`) runs on
    // this rank's share of its lines (share_lines over column pairs: the complex view and the paired real lines of the
    // runtime-scheduled kernel both read two neighbouring columns as one line, so a pair is never cut).
    auto plan_axis = [&](uint32_t axis, const uint64_t* size, const Layout& in, const Layout& out, int64_t base, bool share) -> int {
        const uint64_t N = size[axis];
        const int64_t cbase = (base + 1) / 2;   // first element of the slab in complex units (scratch, complex view)
        double scale = 1.0;
        if ((inv || conv) && d.normalize) scale = 1.0 / (type == 1 ? (is_dst ? 2.0 * (double)(N + 1) : 2.0 * (double)(N - 1)) : 2.0 * (double)N);
        uint64_t n;
        PassReq rq;
        rq.force_generic = true;
        switch (type) {
            case 1:
                if (is_dst) { n = 2 * N + 2; rq.load_io = rq.store_io = B2_IO_DST1; }
                else { n = 2 * N - 2; rq.load_io = rq.store_io = B2_IO_DCT1; }
                rq.aux_u1 = (uint32_t)N; rq.real_pairs = true; break;
            case 2: n = N; rq.load_io = rq.store_io = B2_IO_DCT2; rq.aux0 = aux_for(g, AUX_DCT23, N); rq.real_pairs = true; break;
            case 3: n = N; rq.load_io = rq.store_io = B2_IO_DCT3; rq.aux0 = aux_for(g, AUX_DCT23, N); rq.real_pairs = true;
                    rq.inner_inverse = 1; break;
            case 4:
                if (N % 2 || N == 2) {   // odd length (or N = 2): no half-length trick; phases around a zero-padded 2N-point transform
                    n = 2 * N; rq.load_io = rq.store_io = B2_IO_DCT4_ODD; rq.aux_u1 = (uint32_t)N;
                    rq.aux0 = aux_for(g, AUX_DCT4ODD_PRE, N); rq.aux1 = aux_for(g, AUX_DCT4ODD_POST, N); break;
                }
                n = N / 2; rq.load_io = rq.store_io = B2_IO_DCT4;
                rq.aux0 = aux_for(g, AUX_DCT4_PRE, N); rq.aux1 = aux_for(g, AUX_DCT4_POST, N); break;
            default: return R_UNSUPPORTED_FFT_LENGTH_R2R;
        }
        // DCT-II/III on the specialised kernels: contiguous real lines (axis 0) or pairs of neighbouring real columns
        // viewed as one complex column (other axes)
        if (conv || (!is_dst && (type == 2 || type == 3))) {
            const int kkind = axis == 0 ? B2_KIND_ROWS : B2_KIND_COLS;
            const int kinv = type == 3 ? 1 : 0;
            std::vector<Dim> lines = other_dims(g, size, axis, in, out);
            const int cop = conv ? B2_OP_CONV : 0;
            bool ok = b2_find_kernel(kkind, g.prec, (int)N, kinv, B2_OP_DCT23 | cop) != nullptr;
            PassReq fr;
            fr.kind = kkind; fr.n = (int)N; fr.inv = kinv; fr.ops = B2_OP_DCT23 | cop | ((scale != 1.0) ? B2_OP_SCALE : 0);
            fr.scale = scale; fr.aux0 = aux_for(g, AUX_DCT23, N);
            fr.in_role = in.role; fr.out_role = out.role;
            fr.what = "dct axis (fused)";
            if (conv) {
                // the kernel operand takes aux0 (ROLE_KERNEL), the phase table aux1; DST-II -> DST-III through the flags
                fr.aux1 = fr.aux0; fr.aux0 = -1;
                fr.dst_flags = is_dst ? (B2_DST_NEG_ODD_IN | B2_DST_REV_OUT | B2_DST_ALT_OUT) : 0;
                fr.what = "fused r2r convolution (dct-ii, kernel product, dct-iii)";
            }
            // complex view of the real data (pairs of neighbouring columns): size[0] and every stride of both sides even
            auto even_view = [&](const Layout& l) {
                bool e = l.batch_stride % 2 == 0;
                for (uint32_t a = 1; a < d.fft_dim; ++a) e = e && (l.stride[a - 1] % 2 == 0);
                return e;
            };
            const bool view_ok = axis != 0 && d.size[0] % 2 == 0 && even_view(in) && even_view(out);
            std::vector<Dim> cl, vl;              // complex-view line dims (columns first); vl: this rank's share of them
            int64_t vin = cbase, vout = cbase;    // first complex element of vl on the load / store side
            if (view_ok) {
                cl.push_back(Dim{size[0] / 2, 1, 1});
                for (size_t li = 1; li < lines.size(); ++li) cl.push_back(Dim{lines[li].n, lines[li].is / 2, lines[li].os / 2});
                vl = cl;
                if (share && share_lines(vl, d.dist_world, d.dist_rank, true, vin, vout) != R_SUCCESS) return R_UNSUPPORTED_FFT_LENGTH;
            }
            if (ok && axis == 0) {
                // the kernel pairs real lines 2j and 2j+1 of the group: aux_u1 / aux_u2 = their distance on the load / store side
                std::vector<Dim> m = merge_dims(lines);
                Dim grp = m.empty() ? Dim{1, 0, 0} : m[0];
                if (!m.empty()) m.erase(m.begin());
                fr.real_pairs = true; fr.scalar_units = true;
                fr.aux_u0 = (uint32_t)grp.n; fr.aux_u1 = (uint32_t)grp.is; fr.aux_u2 = (uint32_t)grp.os;
                fr.group = Dim{grp.n, 2 * grp.is, 2 * grp.os};
                fr.outer = m;
                fr.in_es = fr.out_es = 1;
                fr.in_base = fr.out_base = base;
            } else if (ok) {
                ok = view_ok;
                if (ok) {
                    std::vector<Dim> m = merge_dims(vl);
                    if (!m.empty() && m[0].is == 1) { fr.group = m[0]; m.erase(m.begin()); }
                    else fr.group = Dim{1, 1, 1};
                    fr.outer = m;
                    fr.in_es = (int64_t)in.stride[axis - 1] / 2;
                    fr.out_es = (int64_t)out.stride[axis - 1] / 2;
                    fr.in_base = vin; fr.out_base = vout;
                }
            }
            // long strided axis (no well-shaped single-launch kernel): Four-Step along the stride with the Makhoul
            // permutation folded into the first gather (DCT-II) / the last scatter (DCT-III) and a separate split/merge launch
            bool long_strided = false;
            uint64_t L1 = 0, L2 = 0;
            if (!conv && view_ok && N % 2 == 0) {
                const b2_kernel_info* single = b2_find_kernel(B2_KIND_COLS, g.prec, (int)N, kinv, B2_OP_DCT23);
                if (!single || single->q < 8) {
                    uint64_t bestc = ~0ull;
                    for (uint64_t n2 = 2; n2 * 2 <= N; ++n2) {
                        if (N % n2) continue;
                        const uint64_t n1 = N / n2;
                        const bool have = kinv == 0
                            ? (b2_find_kernel(B2_KIND_COLS, g.prec, (int)n1, 0, B2_OP_TWIDDLE_OUT | B2_OP_PERM_IN) && b2_find_kernel(B2_KIND_COLS, g.prec, (int)n2, 0, 0))
                            : (b2_find_kernel(B2_KIND_COLS, g.prec, (int)n1, 1, B2_OP_TWIDDLE_OUT) && b2_find_kernel(B2_KIND_COLS, g.prec, (int)n2, 1, B2_OP_PERM_OUT));
                        if (!have) continue;
                        const uint64_t c = std::max(n1, n2);
                        if (c < bestc) { bestc = c; L1 = n1; L2 = n2; }
                    }
                    long_strided = L1 != 0;
                }
            }
            if (long_strided) {
                // scratch and every launch after the first one use the destination's complex view (esc, rest[].os):
                // DCT-II   source -> temp (gather+phase), temp -> destination, split+phase in place on the destination;
                // DCT-III  source -> destination (phase+merge), destination -> temp, temp -> destination (scatter)
                // A rank's share of a distributed axis is whole columns (rows k and N-k of a column stay together): its three
                // launches touch only its own columns in both windows and need no barrier between them.
                const int64_t esc_in = (int64_t)in.stride[axis - 1] / 2, esc = (int64_t)out.stride[axis - 1] / 2;
                std::vector<Dim> m = merge_dims(vl);
                if (m.empty() || m[0].is != 1) return R_UNSUPPORTED_FFT_LENGTH_R2R;
                const Dim unit = m[0];
                std::vector<Dim> rest(m.begin() + 1, m.end()), rest_out;
                for (const Dim& dd : rest) rest_out.push_back(Dim{dd.n, dd.os, dd.os});
                uint64_t extent = (uint64_t)esc * N;
                for (const Dim& dd : cl) extent = std::max<uint64_t>(extent, (uint64_t)dd.n * (uint64_t)dd.os);
                g.temp_elems = std::max<uint64_t>(g.temp_elems, (uint64_t)cbase + extent);
                const int aux = aux_for(g, AUX_DCT23, N);
                PassReq ew;
                ew.elementwise = true; ew.n = (int)unit.n; ew.ew_items = (uint32_t)unit.n;
                ew.in_es = ew.out_es = 1; ew.out_role = out.role;
                ew.aux0 = aux; ew.aux_u0 = (uint32_t)N;
                ew.in_base = kinv == 0 ? vout : vin; ew.out_base = vout;
                std::vector<Dim> ewl;
                int rcl;
                PassReq a, b;
                a.kind = b.kind = B2_KIND_COLS; a.n = (int)L1; b.n = (int)L2; a.inv = b.inv = kinv;
                a.group = unit; b.group = Dim{unit.n, 1, 1};
                const int64_t esa = kinv == 0 ? esc_in : esc;   // DCT-II: pass A reads the source, DCT-III: the destination
                a.in_es = esa * (int64_t)L2; a.out_es = esc * (int64_t)L2;
                a.outer.push_back(Dim{L2, kinv == 0 ? 0 : esc, esc});
                a.tw_outer = 0; a.twM = N;
                for (const Dim& dd : (kinv == 0 ? rest : rest_out)) a.outer.push_back(dd);
                a.in_role = kinv == 0 ? in.role : out.role; a.out_role = ROLE_TEMP;
                a.in_base = kinv == 0 ? vin : vout; a.out_base = b.in_base = b.out_base = vout;   // scratch at the data's positions
                b.in_es = esc; b.out_es = esc * (int64_t)L1;
                b.outer.push_back(Dim{L1, esc * (int64_t)L2, kinv == 0 ? esc : 0});
                for (const Dim& dd : rest_out) b.outer.push_back(dd);
                b.in_role = ROLE_TEMP; b.out_role = out.role;
                if (kinv == 0) {   // DCT-II
                    a.ops = B2_OP_TWIDDLE_OUT | B2_OP_PERM_IN; a.aux_u0 = (uint32_t)N; a.aux_u1 = (uint32_t)L2;
                    a.what = "long dct-ii 1/3 gather+phase";
                    if ((rcl = emit(g, list, a)) != R_SUCCESS) return rcl;
                    b.ops = 0; b.what = "long dct-ii 2/3";
                    if ((rcl = emit(g, list, b)) != R_SUCCESS) return rcl;
                    ew.ew_op = 3; ew.ops = (scale != 1.0) ? B2_OP_SCALE : 0; ew.scale = scale; ew.what = "long dct-ii 3/3 split+phase";
                    ew.in_role = out.role;
                    ewl.push_back(Dim{N / 2 + 1, esc, esc});
                    ewl.insert(ewl.end(), rest_out.begin(), rest_out.end());
                    if ((rcl = emit_ew(g, list, ew, ewl)) != R_SUCCESS) return rcl;
                } else {           // DCT-III
                    ew.ew_op = 4; ew.what = "long dct-iii 1/3 phase+merge";
                    ew.in_role = in.role;
                    ewl.push_back(Dim{N / 2 + 1, esc_in, esc});
                    ewl.insert(ewl.end(), rest.begin(), rest.end());
                    if ((rcl = emit_ew(g, list, ew, ewl)) != R_SUCCESS) return rcl;
                    a.ops = B2_OP_TWIDDLE_OUT; a.what = "long dct-iii 2/3";
                    if ((rcl = emit(g, list, a)) != R_SUCCESS) return rcl;
                    b.ops = B2_OP_PERM_OUT | ((scale != 1.0) ? B2_OP_SCALE : 0); b.scale = scale;
                    b.tw_outer = 0; b.aux_u0 = (uint32_t)N; b.aux_u1 = (uint32_t)L1;
                    b.what = "long dct-iii 3/3 scatter";
                    if ((rcl = emit(g, list, b)) != R_SUCCESS) return rcl;
                }
                return R_SUCCESS;
            }
            if (ok) return emit(g, list, fr);
            if (conv) return R_UNSUPPORTED_FFT_LENGTH;
        }
        if (n < 2) return R_UNSUPPORTED_FFT_LENGTH_R2R;
        if (!is_smooth(n) || !generic_fits(g, n)) {
            // transform length with a prime factor above 127, or too long for one shared-memory pass: the operator's load
            // and store sides become launches of their own around an ordinary C2C plan on scratch (one real line per
            // complex line; DCT-IV always in its zero-padded 2N form here).  A local axis of a distributed plan keeps the
            // scratch in its temp slab (which it does not fit in practice); across the slabs the route is not planned.
            if (share) return R_UNSUPPORTED_FFT_LENGTH;
            uint32_t dflags = 0;
            if (is_dst) dflags = type == 2 ? (B2_DST_NEG_ODD_IN | B2_DST_REV_OUT) : ((type == 3 || type == 4) ? (B2_DST_REV_IN | B2_DST_ALT_OUT) : 0);
            int io; uint64_t nc; int a0 = -1, a1 = -1;
            switch (type) {
                case 1: io = is_dst ? B2_IO_DST1 : B2_IO_DCT1; nc = is_dst ? 2 * N + 2 : 2 * N - 2; break;
                case 2: io = B2_IO_DCT2; nc = N; a0 = aux_for(g, AUX_DCT23, N); break;
                case 3: io = B2_IO_DCT3; nc = N; a0 = aux_for(g, AUX_DCT23, N); break;
                default: io = B2_IO_DCT4_ODD; nc = 2 * N; a0 = aux_for(g, AUX_DCT4ODD_PRE, N); a1 = aux_for(g, AUX_DCT4ODD_POST, N); break;
            }
            if (nc > 0x7fffffffull) return R_UNSUPPORTED_FFT_LENGTH_R2R;
            const int64_t es_in = axis == 0 ? 1 : (int64_t)in.stride[axis - 1], es_out = axis == 0 ? 1 : (int64_t)out.stride[axis - 1];
            std::vector<Dim> real_lines = other_dims(g, size, axis, in, out), r2t, t2t, t2r;
            uint64_t ts = nc, nlines = 1;
            for (const Dim& rl : real_lines) {
                r2t.push_back(Dim{rl.n, rl.is, (int64_t)ts});
                t2t.push_back(Dim{rl.n, (int64_t)ts, (int64_t)ts});
                t2r.push_back(Dim{rl.n, (int64_t)ts, rl.os});
                ts *= rl.n; nlines *= rl.n;
            }
            const uint64_t region = nlines * nc;
            g.temp_elems = std::max<uint64_t>(g.temp_elems, (uint64_t)cbase + region);
            PassReq ew;
            ew.elementwise = true; ew.store_io = io; ew.dst_flags = dflags; ew.aux0 = a0; ew.aux1 = a1;
            ew.aux_u0 = (uint32_t)N; ew.aux_u1 = (uint32_t)nc;
            ew.ew_op = 9; ew.n = (int)nc; ew.ew_items = (uint32_t)nc; ew.in_es = es_in; ew.out_es = 1;
            ew.in_role = in.role; ew.out_role = ROLE_TEMP; ew.what = "r2r (composed): operator load side";
            ew.in_base = base; ew.out_base = cbase;
            int rc2;
            if ((rc2 = emit_ew(g, list, ew, r2t)) != R_SUCCESS) return rc2;
            list.back().in_scalar = true;
            C2CJob job;
            job.N = nc; job.inv = (type == 3) ? 1 : 0; job.es_in = job.es_out = 1; job.lines = t2t; job.unit_lines = false;
            job.in_role = job.out_role = ROLE_TEMP; job.in_base = job.out_base = cbase; job.tmp_base = cbase + (int64_t)region;
            job.scale = 1.0;
            if ((rc2 = plan_c2c(g, list, job)) != R_SUCCESS) return rc2 == R_UNSUPPORTED_FFT_LENGTH ? R_UNSUPPORTED_FFT_LENGTH_R2R : rc2;
            const uint64_t items = (type == 3) ? nc : N;
            ew.ew_op = 10; ew.n = (int)items; ew.ew_items = (uint32_t)items; ew.in_es = 1; ew.out_es = es_out;
            ew.in_role = ROLE_TEMP; ew.out_role = out.role; ew.what = "r2r (composed): operator store side";
            ew.in_base = cbase; ew.out_base = base;
            ew.ops = (scale != 1.0) ? B2_OP_SCALE : 0; ew.scale = scale;
            if ((rc2 = emit_ew(g, list, ew, t2r)) != R_SUCCESS) return rc2;
            list.back().out_scalar = true;
            return R_SUCCESS;
        }
        if (is_dst) {   // sign / reversal wrappers (API guide :581-583)
            if (type == 2) rq.dst_flags = B2_DST_NEG_ODD_IN | B2_DST_REV_OUT;
            if (type == 3) rq.dst_flags = B2_DST_REV_IN | B2_DST_ALT_OUT;
            if (type == 4) rq.dst_flags = B2_DST_REV_IN | B2_DST_ALT_OUT;
        }
        rq.n = (int)n;
        rq.kind = axis == 0 ? B2_KIND_ROWS : B2_KIND_COLS;
        rq.in_es = axis == 0 ? 1 : (int64_t)in.stride[axis - 1];
        rq.out_es = axis == 0 ? 1 : (int64_t)out.stride[axis - 1];
        rq.in_role = in.role; rq.out_role = out.role;
        std::vector<Dim> lines = other_dims(g, size, axis, in, out);
        rq.in_base = rq.out_base = base;
        if (share) {
            // lines[0] is the x columns: share them out as pairs, then count the share's real columns again (an odd nx leaves
            // the last pair with one column: the kernel runs it unpaired)
            const uint64_t nx = lines[0].n, pairs = (nx + 1) / 2;
            lines[0] = Dim{pairs, 2, 2};
            if (share_lines(lines, d.dist_world, d.dist_rank, true, rq.in_base, rq.out_base) != R_SUCCESS) return R_UNSUPPORTED_FFT_LENGTH;
            const bool last = lines[0].n == pairs || d.dist_rank + 1 == d.dist_world;   // the share ends with column nx-1
            lines[0] = Dim{2 * lines[0].n - (last && nx % 2 ? 1 : 0), 1, 1};
        }
        std::vector<Dim> m = merge_dims(lines);
        if (axis != 0) {
            if (!m.empty() && m[0].is == 1) { rq.group = m[0]; m.erase(m.begin()); }
            else rq.group = Dim{1, 1, 1};
        } else {
            if (m.empty()) rq.group = Dim{1, 0, 0};
            else { rq.group = m[0]; m.erase(m.begin()); }
        }
        rq.aux_u0 = (uint32_t)rq.group.n;
        rq.outer = m;
        rq.ops = (scale != 1.0) ? B2_OP_SCALE : 0;
        rq.scale = scale;
        rq.what = "dct axis";
        return emit(g, list, rq);
    };

    if (g.distributed) {
        // Slabs along the last dimension (DESIGN section 7), in the order of the R2C slab plans: forward, the lower axes inside
        // this rank's slab, a barrier, then the last axis over the whole window on this rank's share of its lines; the inverse
        // runs the other way round.  The local axes keep their scratch inside the rank's temp slab: the same bytes as its data
        // slab, in complex (temp) elements.
        const uint32_t la = d.fft_dim - 1;
        uint64_t lsize[B200FFT_MAX_DIMS];
        for (int a = 0; a < B200FFT_MAX_DIMS; ++a) lsize[a] = d.size[a];
        lsize[la] /= d.dist_world;
        Layout slab = buf;
        // one batch: its pitch addresses nothing, but sizes the scratch of a long strided axis -- a slab's worth, not the window
        slab.batch_stride = lsize[la] * d.buffer_stride[la - 1];
        const int64_t base = slab_base(g);
        const uint64_t slab_end = ((uint64_t)base + slab.batch_stride) / 2;
        for (size_t i = 0; i < axes.size(); ++i) {
            const size_t before = list.size();
            int rc;
            if (axes[i] == la) {
                rc = plan_axis(la, d.size, buf, buf, 0, true);
                if (rc == R_SUCCESS && list.size() > before) list[before].sync_before = true;
            } else {
                const bool after_cross = inv && i > 0 && axes[i - 1] == la;
                rc = plan_in_slab(g, list, slab_end, after_cross, [&] { return plan_axis(axes[i], lsize, slab, slab, base, false); });
            }
            if (rc != R_SUCCESS) return rc;
            g.axis_uploads[inv ? 1 : 0][axes[i]] += (uint32_t)(list.size() - before);
        }
        return R_SUCCESS;
    }
    for (size_t i = 0; i < axes.size(); ++i) {
        Layout in = buf, out = buf;
        if (!inv) {
            if (i == 0 && d.is_input_formatted && !conv) in = inl;   // the fused launch reads what the other axes wrote to `buffer`
            if (i + 1 == axes.size() && d.is_output_formatted) out = outl;
        } else {
            if (i == 0 && d.is_output_formatted) in = outl;
            if (i + 1 == axes.size() && d.is_input_formatted && d.inverse_return_to_input) out = inl;
        }
        const size_t before = list.size();
        const int rc = plan_axis(axes[i], d.size, in, out, 0, false);
        if (rc != R_SUCCESS) return rc;
        g.axis_uploads[inv ? 1 : 0][axes[i]] += (uint32_t)(list.size() - before);
    }
    return R_SUCCESS;
}

}  // namespace

static int build_plan_impl(const b200fft_desc& din, PlanGraph& g) {
    g = PlanGraph{};
    b200fft_desc d = din;
    if (d.fft_dim == 0) return R_EMPTY_FFTDIM;
    if (d.fft_dim > B200FFT_MAX_DIMS) return R_FFTDIM_GT_MAX;
    if (d.size[0] == 0) return R_EMPTY_SIZE;
    for (uint32_t a = 1; a < B200FFT_MAX_DIMS; ++a)
        if (d.size[a] == 0 || a >= d.fft_dim) d.size[a] = 1;
    if (d.number_batches == 0) d.number_batches = 1;
    if (d.coordinate_features == 0) d.coordinate_features = 1;
    if (d.precision > B200FFT_F16_IO) return R_UNSUPPORTED_FFT_LENGTH;
    // B200FFT_F16_IO (the reference's halfPrecisionMemoryOnly, vkFFT_InitAPIParameters.h:153-172: half only where the forward
    // transform first reads and where the inverse transform last writes): the caller's inputBuffer is half, buffer / tempBuffer /
    // outputBuffer are FP32 -- forward inputBuffer -> buffer, inverse (inverseReturnToInputBuffer) buffer -> inputBuffer
    if (d.precision == B200FFT_F16_IO && !d.is_input_formatted) return R_UNSUPPORTED_FFT_LENGTH;
    // half-precision storage: complex transforms and (halfPrecision only) even-length R2C / C2R -- the conversion is fused into the
    // first-stage load / last-stage store of the specialised kernels; DCT / DST, convolution and zero padding have no half variant
    if ((d.precision == B200FFT_F16 || d.precision == B200FFT_F16_IO) && (d.perform_dct || d.perform_dst || d.perform_convolution || d.dist_world > 1))
        return R_UNSUPPORTED_FFT_LENGTH;
    if (d.precision == B200FFT_F16_IO && d.perform_r2c) return R_UNSUPPORTED_FFT_LENGTH;
    if (d.perform_dct > 4 || d.perform_dst > 4) return R_UNSUPPORTED_FFT_LENGTH_R2R;
    if ((d.perform_r2c && (d.perform_dct || d.perform_dst)) || (d.perform_dct && d.perform_dst)) return R_UNSUPPORTED_FFT_LENGTH_R2R;
    if (d.omit_dimension[0] && d.perform_r2c) return R_UNSUPPORTED_FFT_OMIT;
    // default strides (vkFFT_InitializeApp.h:994-1040)
    auto fill = [&](uint64_t* s, uint64_t s0) {
        if (s[0] == 0) s[0] = s0;
        for (int a = 1; a < B200FFT_MAX_DIMS; ++a)
            if (s[a] == 0) s[a] = s[a - 1] * d.size[a];
    };
    if (d.perform_r2c) {
        fill(d.buffer_stride, d.size[0] / 2 + 1);
        fill(d.input_stride, d.is_input_formatted ? d.size[0] : d.size[0] + 2);
        fill(d.output_stride, d.is_output_formatted ? d.size[0] : d.size[0] + 2);
    } else {
        fill(d.buffer_stride, d.size[0]); fill(d.input_stride, d.size[0]); fill(d.output_stride, d.size[0]);
    }
    if (d.dist_world > 1) {
        // in-place transforms over peer windows, one batch: nothing else is defined for a distributed plan
        if (d.dist_rank >= d.dist_world) return R_INVALID_DEVICE;
        // 1-D: one long sequence (Four-Step over the window).  2-D / 3-D: slabs along the last dimension, default strides.
        // 2-D / 3-D R2C: slabs of the in-place layout (H = nx/2+1 complex per row), pitches that may be padded; even nx > 2
        // only, whose x axis needs no scratch beyond the rank's own slab (the odd lengths' composed path does).
        // 2-D / 3-D DCT / DST: slabs of the real array (bufferStride in real elements), pitches that may be padded
        const bool real_tf = d.perform_r2c || d.perform_dct || d.perform_dst;
        const bool real_slab = real_tf && (d.fft_dim == 2 || d.fft_dim == 3);
        if (d.fft_dim > 3 || d.number_batches * d.coordinate_features != 1 || (real_tf && !real_slab) ||
            d.is_input_formatted || d.is_output_formatted || d.omit_dimension[0] ||
            (!real_slab && d.buffer_stride[0] != d.size[0]))
            return R_UNSUPPORTED_FFT_LENGTH;
        if (real_slab) {
            for (uint32_t a = 0; a < d.fft_dim; ++a)
                if (d.omit_dimension[a]) return R_UNSUPPORTED_FFT_LENGTH;
            const uint64_t row = d.perform_r2c ? d.size[0] / 2 + 1 : d.size[0];
            if ((d.perform_r2c && (d.size[0] % 2 || d.size[0] <= 2)) || d.size[d.fft_dim - 1] % d.dist_world || d.buffer_stride[0] < row ||
                (d.fft_dim == 3 && d.buffer_stride[1] < d.size[1] * d.buffer_stride[0]))
                return R_UNSUPPORTED_FFT_LENGTH;
        } else if (d.fft_dim > 1) {
            uint64_t st = 1;
            for (uint32_t a = 0; a < d.fft_dim; ++a) {
                st *= d.size[a];
                if (d.buffer_stride[a] != st || d.omit_dimension[a]) return R_UNSUPPORTED_FFT_LENGTH;
            }
            if (d.size[d.fft_dim - 1] % d.dist_world) return R_UNSUPPORTED_FFT_LENGTH;
        }
        if (!d.user_temp_buffer) return R_EMPTY_TEMPBUFFER;
    } else {
        d.dist_world = 1; d.dist_rank = 0;
    }
    g.desc = d;
    g.distributed = d.dist_world > 1;
    g.prec = (d.precision == B200FFT_F16 || d.precision == B200FFT_F16_IO) ? B2_PREC_F32 : (int)d.precision;
    if (d.precision == B200FFT_F16_IO) g.role_half[ROLE_INPUT] = true;
    if (d.precision == B200FFT_F16)
        for (int r : {ROLE_BUFFER, ROLE_TEMP, ROLE_INPUT, ROLE_OUTPUT}) g.role_half[r] = true;
    for (int a = 0; a < B200FFT_MAX_DIMS; ++a) g.stride[a] = d.buffer_stride[a];
    g.batches = d.number_batches * d.coordinate_features;
    g.batch_stride = d.buffer_stride[d.fft_dim - 1];
    g.total_elems = g.batches;
    for (uint32_t a = 0; a < d.fft_dim; ++a) g.total_elems *= d.size[a];

    uint32_t naxes = 0;
    g.flops = 0;
    const bool real_tf = d.perform_r2c || d.perform_dct || d.perform_dst;
    for (uint32_t a = 0; a < d.fft_dim; ++a) {
        if (d.omit_dimension[a]) continue;
        ++naxes;
        const double n = (double)d.size[a];
        g.flops += (real_tf ? 2.5 : 5.0) * (double)g.total_elems * std::log2(n);
    }
    const uint64_t esz = role_esize(g, ROLE_BUFFER);
    // algorithmic bytes: one read + one write of every point per transformed axis (real data: half the bytes)
    g.algorithmic_bytes = 2 * (real_tf ? esz / 2 : esz) * g.total_elems * naxes;

    g.has_fwd = !d.make_inverse_plan_only;
    g.has_inv = !d.make_forward_plan_only;
    // zero padding: clear the flagged ranges before the first read of the direction they apply to
    bool any_zp = false;
    for (uint32_t a = 0; a < d.fft_dim; ++a) any_zp = any_zp || (d.perform_zeropadding[a] && d.zeropad_right[a] > d.zeropad_left[a]);
    auto zero_fill = [&](std::vector<PassPlan>& list, int inv) -> int {
        if (!any_zp || (inv != 0) != (d.frequency_zeropadding != 0)) return R_SUCCESS;
        if (d.dist_world > 1) return R_UNSUPPORTED_FFT_LENGTH;
        // the data being read lives in `buffer` (a formatted input / output buffer of the caller is never modified)
        if ((!inv && d.is_input_formatted) || (inv && d.is_output_formatted)) return R_UNSUPPORTED_FFT_LENGTH;
        const bool real_buf = (d.perform_dct || d.perform_dst) || (d.perform_r2c && !inv);   // R2C: real rows before the forward transform
        const uint64_t unit = (d.perform_r2c && !inv) ? 2 : 1;                                // real rows of R2C: 2 * complex stride
        for (uint32_t a = 0; a < d.fft_dim; ++a) {
            if (!d.perform_zeropadding[a] || d.zeropad_right[a] <= d.zeropad_left[a]) continue;
            const uint64_t extent = (d.perform_r2c && inv && a == 0) ? d.size[0] / 2 + 1 : d.size[a];
            const uint64_t L = d.zeropad_left[a], R = std::min<uint64_t>(d.zeropad_right[a], extent);
            if (L >= R) continue;
            auto stride_of = [&](uint32_t ax) -> int64_t { return ax == 0 ? 1 : (int64_t)(d.buffer_stride[ax - 1] * unit); };
            PassReq z;
            z.elementwise = true; z.ew_op = 11; z.in_es = z.out_es = 1;
            z.in_role = z.out_role = ROLE_BUFFER;
            z.aux_u0 = real_buf ? 1 : 0;
            std::vector<Dim> lines;
            uint64_t items;
            if (a == 0) { items = R - L; z.out_base = (int64_t)L; }
            else {
                items = (d.perform_r2c && inv) ? d.size[0] / 2 + 1 : d.size[0];
                z.out_base = (int64_t)L * stride_of(a);
                lines.push_back(Dim{R - L, stride_of(a), stride_of(a)});
            }
            // where a higher dimension b is padded at its end, its own clearing pass covers every point with a b-coordinate in
            // the padded range: this pass only needs the rest (half-padded 3-D: 1/8 + 1/4 + 1/2 of the buffer instead of 3 x 1/2)
            for (uint32_t b = 1; b < d.fft_dim; ++b)
                if (b != a) {
                    uint64_t nb_ = d.size[b];
                    if (b > a && d.perform_zeropadding[b] && d.zeropad_right[b] == d.size[b] && d.zeropad_left[b] > 0 && d.zeropad_left[b] < d.size[b])
                        nb_ = d.zeropad_left[b];
                    lines.push_back(Dim{nb_, stride_of(b), stride_of(b)});
                }
            const int64_t bstride = (int64_t)(d.buffer_stride[d.fft_dim - 1] * unit);
            lines.push_back(Dim{g.batches, bstride, bstride});
            z.in_base = z.out_base;
            z.n = (int)std::min<uint64_t>(items, 0x7fffffff); z.ew_items = (uint32_t)items;
            z.what = "zero padding: clear the padded range";
            int zr = emit_ew(g, list, z, lines);
            if (zr != R_SUCCESS) return zr;
            list.back().in_scalar = list.back().out_scalar = real_buf;
        }
        return R_SUCCESS;
    };
    auto plan = [&](std::vector<PassPlan>& list, int inv) {
        if (int zr = zero_fill(list, inv)) return zr;
        if (d.perform_r2c) return plan_direction_r2c(g, list, inv);
        if (d.perform_dct || d.perform_dst) return plan_direction_dct(g, list, inv);
        return plan_direction_c2c(g, list, inv);
    };
    int rc;
    if (d.perform_convolution) {
        // forward transform -> product with the kernel spectrum -> inverse transform, all behind VkFFTAppend(app, -1)
        // (vkFFT_RunApp.h:111-321 runs the same chain; the reference fuses the product into the last-axis kernel,
        // vkFFT_Convolution.h:125 -- here it is its own streaming launch)
        const uint64_t C = d.coordinate_features, B = d.number_batches, NK = d.number_kernels ? d.number_kernels : 1;
        const uint32_t M = d.matrix_convolution >= 2 ? d.matrix_convolution : 0;
        // DCT / DST: forward type-k transform, product with a real kernel in the buffer's layout, inverse transform (the
        // inverse pairs and normalisation of plan_direction_dct).  Conjugation and cross-power normalisation have no meaning
        // for real spectra.
        const bool r2r = d.perform_dct || d.perform_dst;
        if (d.is_output_formatted || d.dist_world > 1) return R_UNSUPPORTED_FFT_LENGTH;
        if (r2r && (d.conjugate_convolution || d.cross_power_spectrum_normalization)) return R_UNSUPPORTED_FFT_LENGTH;
        for (uint32_t a = 0; a < d.fft_dim; ++a) if (d.omit_dimension[a]) return r2r ? R_UNSUPPORTED_FFT_LENGTH : R_UNSUPPORTED_FFT_OMIT;
        if (M > 3 || (M && C != M) || C > 255 || (NK > 1 && B > 1)) return R_UNSUPPORTED_FFT_LENGTH;
        g.has_fwd = true; g.has_inv = false;
        // Fused last axis: per-feature product, one kernel set, packed layout, and a fused kernel for the length of the
        // last transformed axis (contiguous lines in 1-D, strided axis otherwise).  That launch runs the axis forward,
        // multiplies and runs it inverse; the remaining axes keep their ordinary forward / inverse passes around it.
        if (!r2r) {
            const uint32_t la = d.fft_dim - 1;
            bool packed = !d.is_output_formatted && (la > 0 || (!d.perform_r2c && !d.is_input_formatted));
            uint64_t want = d.perform_r2c ? d.size[0] / 2 + 1 : d.size[0];
            for (uint32_t a = 0; a < d.fft_dim && packed; ++a) { packed = d.buffer_stride[a] == want; want *= (a + 1 < d.fft_dim ? d.size[a + 1] : 1); }
            const uint64_t plane = d.buffer_stride[la], KS = C * plane;
            const int ckind = la == 0 ? B2_KIND_ROWS : B2_KIND_COLS;
            if (packed && !M && NK == 1 && d.size[la] > 1 && d.size[la] <= 0x7fffffff && KS < (1ull << 32) && !getenv("B200FFT_NO_FUSED_CONV") &&
                b2_find_kernel(ckind, g.prec, (int)d.size[la], 0, B2_OP_CONV)) {
                g.batches = B * C;
                g.skip_axis = (int)la;
                if ((rc = plan(g.fwd, 0)) != R_SUCCESS) return rc;
                uint64_t csize[B200FFT_MAX_DIMS];
                for (int a = 0; a < B200FFT_MAX_DIMS; ++a) csize[a] = d.size[a];
                if (d.perform_r2c) csize[0] = d.size[0] / 2 + 1;
                const Layout bl = layout_of(ROLE_BUFFER, d.buffer_stride, d.fft_dim);
                C2CJob job;
                job.N = d.size[la]; job.inv = 0;
                job.es_in = job.es_out = la == 0 ? 1 : (int64_t)bl.stride[la - 1];
                job.lines = other_dims(g, csize, la, bl, bl);
                job.unit_lines = (la != 0);
                job.in_role = job.out_role = ROLE_BUFFER;
                job.scale = 1.0;         // the inverse passes of the other axes (or this one, below) carry the normalisation
                job.extra_ops = B2_OP_CONV;
                job.aux_u0 = (uint32_t)KS;
                job.aux_u1 = (d.conjugate_convolution == 1 ? (1u << 13) : 0) | (d.conjugate_convolution == 2 ? (1u << 14) : 0) |
                             (d.cross_power_spectrum_normalization ? (1u << 15) : 0);
                std::vector<PassPlan> tail;
                b200fft_desc back = g.desc;
                g.desc.is_input_formatted = 0; g.desc.inverse_return_to_input = 0;
                rc = plan(tail, 1);
                g.desc = back;
                if (rc != R_SUCCESS) return rc;
                // the direction planners put the whole 1/N on their last pass; with nothing left for them (1-D) the fused
                // launch scales itself
                if (tail.empty() && d.normalize) job.scale = 1.0 / (double)d.size[la];
                if ((rc = plan_c2c(g, g.fwd, job)) != R_SUCCESS) return rc;
                g.fwd.back().aux0_role = ROLE_KERNEL;
                g.fwd.back().note = "fused convolution (fft, kernel product, ifft)  " + g.fwd.back().note;
                g.fwd.insert(g.fwd.end(), tail.begin(), tail.end());
                g.skip_axis = -1;
                return R_SUCCESS;
            }
        }
        if (r2r) {
            // Fused last axis of a DCT-II / DST-II convolution under the C2C conditions (packed layout, one kernel set, no
            // matrix, a kernel for the length): DCT-II forward, pair pass with the kernel product, DCT-III inverse in one
            // launch (stockham.cuh RMODE 12), the other axes keep their R2R passes around it: 2*nd-1 launches.
            const uint32_t la = d.fft_dim - 1;
            const int kind = (int)(d.perform_dst ? d.perform_dst : d.perform_dct);
            bool packed = la > 0 || !d.is_input_formatted;
            uint64_t want = d.size[0];
            for (uint32_t a = 0; a < d.fft_dim && packed; ++a) { packed = d.buffer_stride[a] == want; want *= (a + 1 < d.fft_dim ? d.size[a + 1] : 1); }
            const uint64_t KS = C * d.buffer_stride[la];
            const int ckind = la == 0 ? B2_KIND_ROWS : B2_KIND_COLS;
            if (kind == 2 && packed && !M && NK == 1 && d.size[la] > 1 && d.size[la] <= 0x7fffffff && KS < (1ull << 32) &&
                (la == 0 || d.size[0] % 2 == 0) && !getenv("B200FFT_NO_FUSED_CONV") &&
                b2_find_kernel(ckind, g.prec, (int)d.size[la], 0, B2_OP_DCT23 | B2_OP_CONV)) {
                g.batches = B * C;
                g.skip_axis = (int)la;
                rc = plan(g.fwd, 0);
                g.skip_axis = -1;
                if (rc != R_SUCCESS) return rc;
                const size_t before = g.fwd.size();
                g.conv_axis = (int)la;
                rc = plan_direction_dct(g, g.fwd, 0);
                g.conv_axis = -1;
                if (rc != R_SUCCESS) return rc;
                for (size_t i = before; i < g.fwd.size(); ++i) {
                    g.fwd[i].aux0_role = ROLE_KERNEL;
                    g.fwd[i].P.in_len = (uint32_t)KS;          // the kernel's features x plane block, in real elements
                }
                std::vector<PassPlan> tail;
                b200fft_desc back = g.desc;
                g.desc.is_input_formatted = 0; g.desc.inverse_return_to_input = 0;
                g.skip_axis = (int)la;
                rc = plan(tail, 1);
                g.skip_axis = -1;
                g.desc = back;
                if (rc != R_SUCCESS) return rc;
                g.fwd.insert(g.fwd.end(), tail.begin(), tail.end());
                return R_SUCCESS;
            }
        }
        g.batches = B * C;
        if ((rc = plan(g.fwd, 0)) != R_SUCCESS) return rc;
        const uint64_t plane = d.buffer_stride[d.fft_dim - 1];
        PassReq cv;
        cv.elementwise = true; cv.ew_op = r2r ? 12 /* B2_EW_CONV_REAL */ : 5 /* B2_EW_CONV */;
        cv.n = (int)std::min<uint64_t>(plane, 0x7fffffff); cv.ew_items = (uint32_t)plane;
        if (plane > 0x7fffffffull) return R_UNSUPPORTED_FFT_LENGTH;
        cv.in_es = cv.out_es = (int64_t)plane;
        cv.aux_u0 = (uint32_t)C | (M << 8) | (d.symmetric_kernel ? (1u << 12) : 0) | (d.conjugate_convolution == 1 ? (1u << 13) : 0) |
                    (d.conjugate_convolution == 2 ? (1u << 14) : 0) | (d.cross_power_spectrum_normalization ? (1u << 15) : 0);
        cv.aux_u1 = (uint32_t)NK;
        cv.in_role = cv.out_role = ROLE_BUFFER;
        cv.what = r2r ? "convolution: real spectrum x kernel" : "convolution: spectrum x kernel";
        std::vector<Dim> cvl;
        {
            // packed layout: one line = one plane.  Padded pitches: one line = one row, so that the gaps between rows and planes
            // (a bigger array of the caller's, for a sub-volume) are neither read nor written
            uint64_t csize0 = d.perform_r2c ? d.size[0] / 2 + 1 : d.size[0], want = csize0;
            bool dense = true;
            for (uint32_t a = 0; a < d.fft_dim && dense; ++a) { dense = d.buffer_stride[a] == want; want *= (a + 1 < d.fft_dim ? d.size[a + 1] : 1); }
            if (!dense) {
                cv.n = (int)std::min<uint64_t>(csize0, 0x7fffffff); cv.ew_items = (uint32_t)csize0;
                for (uint32_t a = 1; a < d.fft_dim; ++a) cvl.push_back(Dim{d.size[a], (int64_t)d.buffer_stride[a - 1], (int64_t)d.buffer_stride[a - 1]});
            }
        }
        cvl.push_back(Dim{B, (int64_t)(C * plane), (int64_t)(C * plane)});      // kernel k writes output batch k (one input, NK outputs)
        if ((rc = emit_ew(g, g.fwd, cv, cvl)) != R_SUCCESS) return rc;
        g.fwd.back().aux0_role = ROLE_KERNEL;
        g.fwd.back().in_scalar = g.fwd.back().out_scalar = r2r;
        // the inverse runs in `buffer` on every output batch
        b200fft_desc back = g.desc;
        g.desc.is_input_formatted = 0; g.desc.inverse_return_to_input = 0;
        g.batches = std::max(B, NK) * C;
        std::vector<PassPlan> tail;
        rc = plan(tail, 1);
        g.desc = back;
        if (rc != R_SUCCESS) return rc;
        g.fwd.insert(g.fwd.end(), tail.begin(), tail.end());
        g.total_elems = g.total_elems / B * std::max(B, NK);
        return R_SUCCESS;
    }
    if (g.has_fwd && (rc = plan(g.fwd, 0)) != R_SUCCESS) return rc;
    if (g.has_inv && (rc = plan(g.inv, 1)) != R_SUCCESS) return rc;
    return R_SUCCESS;
}

int build_plan(const b200fft_desc& din, PlanGraph& g) {
    const int rc = build_plan_impl(din, g);
    if (rc != R_SUCCESS) return rc;
    // Caller-owned scratch (userTempBuffer = 1): this engine's plans can need MORE scratch than `buffer` holds (Bluestein,
    // odd-length R2C, composed DCT/DST), so the size is checked on every path, convolution plans included.  Without a
    // tempBufferSize the reference's contract applies ("same size as buffer"): the buffer size stands in.  The required
    // size is published through b200fft_plan_get_info().temp_bytes either way.
    if (g.desc.user_temp_buffer && g.temp_elems) {
        const uint64_t need = g.temp_elems * role_esize(g, ROLE_TEMP);
        const uint64_t have = din.temp_buffer_size ? din.temp_buffer_size : din.buffer_size;
        if (have != 0 && need > have) return R_USER_TEMP_TOO_SMALL;
    }
    return R_SUCCESS;
}

}  // namespace b200fft
