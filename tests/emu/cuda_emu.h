// TEST INFRASTRUCTURE ONLY -- never linked into the product library.
//
// A tiny CPU emulation of the CUDA execution model, good enough to run the engine's kernel *bodies*
// (the same templates nvcc compiles for sm_90a) inside the CPU test-suite: one OS thread per CUDA
// thread of a block, a std::barrier for __syncthreads(), blocks executed one after another.
// It exists because the development container has no GPU: index maps, twiddle tables and the autosort
// scatter are checked here against the double-precision oracle before GPU minutes are spent, and the
// shared-memory access log lets the tests assert "bank-conflict free" per configuration.
#pragma once
#include <algorithm>
#include <atomic>
#include <barrier>
#include <cstdlib>
#include <memory>
#include <cstdint>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

struct float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(16) double2 { double x, y; };

namespace b2emu {
struct idx3 { unsigned x, y, z; };
struct SmemRec { uint32_t addr; uint16_t bytes; uint16_t store; };
struct State {
    idx3 blockDim{1, 1, 1}, gridDim{1, 1, 1};
    std::barrier<>* bar = nullptr;
    unsigned char* smem = nullptr;
    bool log = false;
    bool launch_refused = false;             // set by launch() when the configuration exceeds the device limits
    size_t smem_bytes = 0;
    bool smem_oob = false;                   // a shared-memory access outside the CTA's allocation (reported as a failed launch)
    std::vector<std::vector<SmemRec>> recs;  // per thread (block 0 only)
    // race check (what compute-sanitizer racecheck reports on the device): per 4-byte word of shared memory the last
    // writer and the last reader(s) with the barrier interval ("epoch") they acted in; two different threads touching a
    // word in the same interval, at least one of them writing, is a hazard
    struct WordMeta { std::atomic<uint64_t> w{0}, r{0}; };
    std::unique_ptr<WordMeta[]> meta;
    size_t meta_words = 0;
    bool racecheck = true;
    std::atomic<int> hazards{0};
    uint32_t hazard_addr = 0, hazard_kind = 0;   // first hazard: byte offset, 1 = write-write, 2 = write-after-read, 3 = read-after-write
};
inline State& st() { static State s; return s; }
inline thread_local idx3 t_threadIdx{0, 0, 0};
inline thread_local idx3 t_blockIdx{0, 0, 0};
inline thread_local uint64_t t_epoch = 1;

inline void syncthreads() { st().bar->arrive_and_wait(); ++t_epoch; }
inline void log_access(const void* base, size_t index, size_t elem_bytes, bool store) {
    State& s = st();
    {   // bounds of the dynamic shared-memory allocation (what compute-sanitizer memcheck would flag on the device)
        const unsigned char* a = (const unsigned char*)base + index * elem_bytes;
        if (a < s.smem || a + elem_bytes > s.smem + s.smem_bytes) s.smem_oob = true;
    }
    if (s.racecheck && s.meta && !s.smem_oob) {
        const size_t off = (size_t)((const unsigned char*)base - s.smem) + index * elem_bytes;
        const uint64_t tid = t_threadIdx.x, key = (t_epoch << 20) | tid;
        for (size_t wd = off / 4; wd < (off + elem_bytes + 3) / 4 && wd < s.meta_words; ++wd) {
            State::WordMeta& m = s.meta[wd];
            int kind = 0;
            if (store) {
                const uint64_t ow = m.w.exchange(key);
                if ((ow >> 20) == t_epoch && (ow & 0x7ffff) != tid) kind = 1;
                const uint64_t rd = m.r.load();
                if ((rd >> 20) == t_epoch && ((rd & 0x7ffff) != tid || (rd & 0x80000))) kind = kind ? kind : 2;
            } else {
                uint64_t old = m.r.load(), want;
                do {
                    want = key;
                    if ((old >> 20) == t_epoch && ((old & 0x7ffff) != tid || (old & 0x80000))) want |= 0x80000;   // several readers
                } while (!m.r.compare_exchange_weak(old, want));
                const uint64_t wv = m.w.load();
                if ((wv >> 20) == t_epoch && (wv & 0x7ffff) != tid) kind = 3;
            }
            if (kind && s.hazards.fetch_add(1) == 0) { s.hazard_addr = (uint32_t)(wd * 4); s.hazard_kind = (uint32_t)kind; }
        }
    }
    if (!s.log || t_blockIdx.x != 0) return;
    s.recs[t_threadIdx.x].push_back(SmemRec{(uint32_t)(index * elem_bytes), (uint16_t)elem_bytes, (uint16_t)store});
}

struct ConflictReport {
    double worst = 1.0;     // worst wavefronts/ideal over all warp-wide accesses
    double mean = 1.0;      // traffic-weighted mean
    size_t accesses = 0;
};

// Analyse the log of block 0: for every warp and every k-th shared access, count the wavefronts the
// 32-bank x 4-byte crossbar needs (64-bit accesses are served per half-warp, 128-bit per quarter-warp).
inline ConflictReport analyse(unsigned nthreads) {
    State& s = st();
    ConflictReport rep;
    double tot_act = 0, tot_ideal = 0;
    for (unsigned w0 = 0; w0 < nthreads; w0 += 32) {
        unsigned lanes = std::min(32u, nthreads - w0);
        size_t nacc = s.recs[w0].size();
        bool uniform = true;
        for (unsigned l = 0; l < lanes; ++l) uniform &= (s.recs[w0 + l].size() == nacc);
        if (!uniform) continue;  // divergent (guarded) access sequence: skip this warp
        for (size_t i = 0; i < nacc; ++i) {
            unsigned bytes = s.recs[w0][i].bytes;
            unsigned per_phase = bytes == 4 ? 32 : (bytes == 8 ? 16 : 8);
            unsigned wave = 0, ideal = 0;
            for (unsigned p0 = 0; p0 < lanes; p0 += per_phase) {
                // distinct 4-byte words per bank
                std::vector<std::vector<uint32_t>> bank(32);
                for (unsigned l = p0; l < std::min(lanes, p0 + per_phase); ++l) {
                    const SmemRec& r = s.recs[w0 + l][i];
                    for (unsigned b = 0; b < r.bytes; b += 4) {
                        uint32_t word = (r.addr + b) / 4;
                        auto& v = bank[word % 32];
                        if (std::find(v.begin(), v.end(), word) == v.end()) v.push_back(word);
                    }
                }
                unsigned deg = 0;
                for (auto& v : bank) deg = std::max<unsigned>(deg, (unsigned)v.size());
                wave += deg;
                ideal += 1;
            }
            double ratio = (double)wave / ideal;
            rep.worst = std::max(rep.worst, ratio);
            tot_act += wave;
            tot_ideal += ideal;
            rep.accesses++;
        }
    }
    rep.mean = tot_ideal > 0 ? tot_act / tot_ideal : 1.0;
    return rep;
}

// run f(smem) for every thread of every block
template <class F>
inline void launch(unsigned grid, unsigned block, size_t smem_bytes, F&& f, bool log = false) {
    State& s = st();
    // what cudaLaunchKernel would refuse on sm_90 (1024 threads, 227 KiB opt-in shared memory, 2^31-1 CTAs)
    if (block == 0 || block > 1024 || smem_bytes > 232448 || grid == 0 || grid > 0x7fffffffu) { s.launch_refused = true; return; }
    s.blockDim = {block, 1, 1};
    s.gridDim = {grid, 1, 1};
    std::vector<unsigned char> smem(smem_bytes + 65536);   // slack: an out-of-bounds access is reported, not a host crash
    s.smem = smem.data();
    s.smem_bytes = smem_bytes;
    s.racecheck = !getenv("B2EMU_NO_RACECHECK");
    s.meta_words = smem_bytes / 4 + 16;
    s.meta.reset(s.racecheck && smem_bytes ? new State::WordMeta[s.meta_words] : nullptr);
    std::barrier<> bar((std::ptrdiff_t)block);
    s.bar = &bar;
    s.log = log;
    s.recs.assign(block, {});
    std::vector<std::thread> th;
    th.reserve(block);
    for (unsigned t = 0; t < block; ++t) {
        th.emplace_back([&, t]() {
            t_threadIdx = {t, 0, 0};
            for (unsigned b = 0; b < grid; ++b) {
                t_blockIdx = {b, 0, 0};
                f(s.smem);
                s.bar->arrive_and_wait();
                ++t_epoch;
            }
        });
    }
    for (auto& x : th) x.join();
    s.bar = nullptr;
}
}  // namespace b2emu

#define threadIdx (::b2emu::t_threadIdx)
#define blockIdx (::b2emu::t_blockIdx)
#define blockDim (::b2emu::st().blockDim)
#define gridDim (::b2emu::st().gridDim)
#define __syncthreads() ::b2emu::syncthreads()
#define B2_SMEM_LD(sm, i) (::b2emu::log_access((sm), (size_t)(i), sizeof((sm)[0]), false), (sm)[(i)])
#define B2_SMEM_ST(sm, i, v) (::b2emu::log_access((sm), (size_t)(i), sizeof((sm)[0]), true), (void)((sm)[(i)] = (v)))
