// TEST INFRASTRUCTURE ONLY -- never linked into the product library.
//
// The CPU emulation of the CUDA execution model (cuda_emu.h) extended by thread-block clusters.  Selected instead of
// cuda_emu.h by -DB2_EMU_CLUSTER (tests/emu/build_cluster.sh); same interface, so every kernel body runs on it unchanged.
// One OS thread per CUDA thread of a block, a std::barrier for __syncthreads(), blocks executed one after another -- or, for
// a launch with thread-block clusters (launch_cluster), the CTAs of one cluster at the same time, each with its own shared
// memory and __syncthreads barrier, plus a cluster-wide barrier (cluster_sync) and distributed shared memory (dsmem_st /
// dsmem_ld: byte offset in the shared memory of CTA `rank`).  Every shared-memory access, local or distributed, is checked
// for bounds and for races: threads of one CTA are ordered by __syncthreads and cluster barriers, threads of different CTAs
// by cluster barriers only.
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

// Its own namespace: a test process may load both emulation libraries, and the process-wide unique symbols of inline
// functions and variables (the emulation state, the thread-local indices) must not be shared between the two layouts.
// The kernel bodies and drivers keep writing b2emu::.
namespace b2emu_cluster {
struct idx3 { unsigned x, y, z; };
struct SmemRec { uint32_t addr; uint16_t bytes; uint16_t store; };
struct State {
    idx3 blockDim{1, 1, 1}, gridDim{1, 1, 1};
    bool log = false;
    bool launch_refused = false;             // set by launch() when the configuration exceeds the device limits
    size_t smem_bytes = 0;
    bool smem_oob = false;                   // a shared-memory access outside the CTA's allocation (reported as a failed launch)
    std::vector<std::vector<SmemRec>> recs;  // per thread (block 0 only)
    // race check (what compute-sanitizer racecheck reports on the device): per 4-byte word of shared memory the last
    // writer and the last reader(s) with the barrier interval ("epoch") they acted in; two different threads touching a
    // word in the same interval, at least one of them writing, is a hazard
    struct WordMeta { std::atomic<uint64_t> w{0}, r{0}; };
    size_t meta_words = 0;
    bool racecheck = true;
    std::atomic<int> hazards{0};
    uint32_t hazard_addr = 0, hazard_kind = 0;   // first hazard: byte offset, 1 = write-write, 2 = write-after-read, 3 = read-after-write
    // thread-block clusters (launch_cluster): the `cluster` CTAs of one cluster run concurrently, each with its own shared
    // memory, __syncthreads barrier and race metadata; a plain launch is a cluster of one CTA, blocks run one after another
    unsigned cluster = 1;
    std::vector<unsigned char*> smem;        // per CTA of the running cluster
    std::vector<std::unique_ptr<std::barrier<>>> bars;
    std::unique_ptr<std::barrier<>> cluster_bar;
    std::vector<std::unique_ptr<WordMeta[]>> meta;
    bool cluster_capable = false;            // what the emulated device reports to the planner (emu.set_cluster_capable)
};
inline State& st() { static State s; return s; }
inline thread_local idx3 t_threadIdx{0, 0, 0};
inline thread_local idx3 t_blockIdx{0, 0, 0};
inline thread_local unsigned t_rank = 0;     // CTA rank within the cluster
inline thread_local uint64_t t_epoch = 1;    // __syncthreads intervals (cluster barriers end one as well)
inline thread_local uint64_t t_cepoch = 1;   // cluster-barrier intervals

// race-check record: [cluster epoch:16][epoch:28][several readers:1][thread of the cluster:19]
constexpr uint64_t TID_MASK = 0x7ffff, MULTI = 0x80000;
inline uint64_t rec_key(uint64_t gtid) { return ((t_cepoch & 0xffff) << 48) | ((t_epoch & 0xfffffff) << 20) | gtid; }
// may the access recorded as `old` race with this thread's current one?  Threads of one CTA are ordered by __syncthreads and
// cluster barriers, threads of different CTAs by cluster barriers only
inline bool same_interval(uint64_t old, uint64_t gtid) {
    if (old == 0 || (old >> 48) != (t_cepoch & 0xffff)) return false;
    const uint64_t block = st().blockDim.x;
    if ((old & TID_MASK) / block != gtid / block) return true;
    return ((old >> 20) & 0xfffffff) == (t_epoch & 0xfffffff);
}
inline void check_word(State::WordMeta& m, bool store, uint32_t byte_addr) {
    State& s = st();
    const uint64_t gtid = (uint64_t)t_rank * s.blockDim.x + t_threadIdx.x, key = rec_key(gtid);
    int kind = 0;
    if (store) {
        const uint64_t ow = m.w.exchange(key);
        if (same_interval(ow, gtid) && (ow & TID_MASK) != gtid) kind = 1;
        const uint64_t rd = m.r.load();
        if (same_interval(rd, gtid) && ((rd & TID_MASK) != gtid || (rd & MULTI))) kind = kind ? kind : 2;
    } else {
        uint64_t old = m.r.load(), want;
        do {
            want = key;
            if (same_interval(old, gtid) && ((old & TID_MASK) != gtid || (old & MULTI))) want |= MULTI;   // several readers
        } while (!m.r.compare_exchange_weak(old, want));
        const uint64_t wv = m.w.load();
        if (same_interval(wv, gtid) && (wv & TID_MASK) != gtid) kind = 3;
    }
    if (kind && s.hazards.fetch_add(1) == 0) { s.hazard_addr = byte_addr; s.hazard_kind = (uint32_t)kind; }
}
// one access of `bytes` bytes at byte offset `off` of CTA `rank`'s shared memory
inline void check_access(unsigned rank, size_t off, size_t bytes, bool store) {
    State& s = st();
    if (rank >= s.cluster || off + bytes > s.smem_bytes) { s.smem_oob = true; return; }
    if (!s.racecheck || !s.meta[rank]) return;
    for (size_t wd = off / 4; wd < (off + bytes + 3) / 4 && wd < s.meta_words; ++wd) check_word(s.meta[rank][wd], store, (uint32_t)(wd * 4));
}

inline void syncthreads() { st().bars[t_rank]->arrive_and_wait(); ++t_epoch; }
// barrier.cluster.arrive.release + barrier.cluster.wait.acquire
inline void cluster_sync() { st().cluster_bar->arrive_and_wait(); ++t_epoch; ++t_cepoch; }
inline void log_access(const void* base, size_t index, size_t elem_bytes, bool store) {
    State& s = st();
    // bounds of the CTA's own dynamic shared-memory allocation (what compute-sanitizer memcheck would flag on the device)
    const unsigned char* a = (const unsigned char*)base + index * elem_bytes;
    const unsigned char* own = s.smem[t_rank];
    if (a < own || a + elem_bytes > own + s.smem_bytes) { s.smem_oob = true; return; }
    check_access(t_rank, (size_t)(a - own), elem_bytes, store);
    if (!s.log || t_blockIdx.x != 0) return;
    s.recs[t_threadIdx.x].push_back(SmemRec{(uint32_t)(index * elem_bytes), (uint16_t)elem_bytes, (uint16_t)store});
}
// distributed shared memory: byte offset `off` of CTA `rank` of this cluster (mapa + st.shared::cluster / ld.shared::cluster)
template <class T> inline void dsmem_st(unsigned rank, size_t off, const T& v) {
    State& s = st();
    check_access(rank, off, sizeof(T), true);
    if (rank < s.cluster && off + sizeof(T) <= s.smem_bytes) std::memcpy(s.smem[rank] + off, &v, sizeof(T));
}
template <class T> inline T dsmem_ld(unsigned rank, size_t off) {
    State& s = st();
    check_access(rank, off, sizeof(T), false);
    T v{};
    if (rank < s.cluster && off + sizeof(T) <= s.smem_bytes) std::memcpy(&v, s.smem[rank] + off, sizeof(T));
    return v;
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

// run f(smem) for every thread of every block; cluster > 1: the blocks come in clusters of that many consecutive blocks, the
// blocks of one cluster run concurrently (one OS thread per CUDA thread of the cluster), clusters one after another
template <class F>
inline void launch_cluster(unsigned grid, unsigned cluster, unsigned block, size_t smem_bytes, F&& f, bool log = false) {
    State& s = st();
    // what cudaLaunchKernelEx would refuse on sm_90 (1024 threads, 227 KiB opt-in shared memory, 2^31-1 CTAs, clusters of at
    // most 16 CTAs -- more than 8 only as a non-portable size -- that divide the grid)
    if (block == 0 || block > 1024 || smem_bytes > 232448 || grid == 0 || grid > 0x7fffffffu || cluster == 0 || cluster > 16 ||
        grid % cluster) { s.launch_refused = true; return; }
    s.blockDim = {block, 1, 1};
    s.gridDim = {grid, 1, 1};
    s.cluster = cluster;
    std::vector<std::vector<unsigned char>> mem(cluster);
    s.smem.assign(cluster, nullptr);
    s.racecheck = !getenv("B2EMU_NO_RACECHECK");
    s.meta_words = smem_bytes / 4 + 16;
    s.meta.clear();
    s.bars.clear();
    for (unsigned r = 0; r < cluster; ++r) {
        mem[r].assign(smem_bytes + 65536, 0);   // slack: an out-of-bounds access is reported, not a host crash
        s.smem[r] = mem[r].data();
        s.meta.emplace_back(s.racecheck && smem_bytes ? new State::WordMeta[s.meta_words] : nullptr);
        s.bars.emplace_back(new std::barrier<>((std::ptrdiff_t)block));
    }
    s.cluster_bar.reset(new std::barrier<>((std::ptrdiff_t)(block * cluster)));
    s.smem_bytes = smem_bytes;
    s.log = log;
    s.recs.assign(block, {});
    std::vector<std::thread> th;
    th.reserve((size_t)block * cluster);
    for (unsigned r = 0; r < cluster; ++r)
        for (unsigned t = 0; t < block; ++t) {
            th.emplace_back([&, r, t]() {
                t_threadIdx = {t, 0, 0};
                t_rank = r;
                for (unsigned c = 0; c < grid / cluster; ++c) {
                    t_blockIdx = {c * cluster + r, 0, 0};
                    f(s.smem[r]);
                    s.cluster_bar->arrive_and_wait();    // every CTA of the cluster is done before the next one reuses the memory
                    ++t_epoch;
                    ++t_cepoch;
                }
            });
        }
    for (auto& x : th) x.join();
    s.cluster = 1;
}
template <class F>
inline void launch(unsigned grid, unsigned block, size_t smem_bytes, F&& f, bool log = false) {
    launch_cluster(grid, 1, block, smem_bytes, f, log);
}
}  // namespace b2emu_cluster
namespace b2emu = b2emu_cluster;

#define threadIdx (::b2emu::t_threadIdx)
#define blockIdx (::b2emu::t_blockIdx)
#define blockDim (::b2emu::st().blockDim)
#define gridDim (::b2emu::st().gridDim)
#define __syncthreads() ::b2emu::syncthreads()
#define B2_SMEM_LD(sm, i) (::b2emu::log_access((sm), (size_t)(i), sizeof((sm)[0]), false), (sm)[(i)])
#define B2_SMEM_ST(sm, i, v) (::b2emu::log_access((sm), (size_t)(i), sizeof((sm)[0]), true), (void)((sm)[(i)] = (v)))
