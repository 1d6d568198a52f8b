// cuda_emu.h — just enough of the CUDA execution model to run polypolish_b200/csrc/polish_dev.cuh on the CPU (g++), so that
// the kernels' logic can be checked against the oracle without a GPU (tests/test_emu_polish.py).  TEST INFRASTRUCTURE: one OS
// thread per CUDA thread of a block, blocks one after another, __syncthreads = a block barrier, warp shuffles / votes through a
// per-warp exchange buffer + warp barrier.  Slow and simple; not part of the product.
#pragma once
#include <algorithm>
#include <atomic>
#include <barrier>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#define PP_EMULATE 1
#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __noinline__
#define __grid_constant__
#define __restrict__
#define __launch_bounds__(...)
#define __align__(n) alignas(n)
#define __constant__ static

struct dim3 { unsigned x = 1, y = 1, z = 1; };
struct uint2 { uint32_t x, y; };
struct alignas(16) uint4 { uint32_t x, y, z, w; };
struct alignas(16) ulonglong2 { unsigned long long x, y; };
struct alignas(16) double2 { double x, y; };
struct alignas(32) double4 { double x, y, z, w; };
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return {x, y}; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return {x, y, z, w}; }
static inline ulonglong2 make_ulonglong2(unsigned long long x, unsigned long long y) { return {x, y}; }
static inline double4 make_double4(double x, double y, double z, double w) { return {x, y, z, w}; }

namespace emu {
struct Warp {
    std::barrier<> bar;
    unsigned long long xchg[32];
    explicit Warp(int n) : bar(n) {}
};

// ---- The chunk ring's bulk copies and mbarriers (stage_* in polish_dev.cuh), modelled strictly, so that a protocol error fails
// on the CPU instead of hanging k_tile on the device.  One RingBar per mbarrier, keyed by its address in the block's shared memory.
//   init:      arrival count 1; re-initialising a barrier with a phase armed is an error.
//   expect:    the phase's one arrival, tx += bytes.  A second arrival in an unfinished phase is an error (it would complete early).
//              A phase whose arrival is in and whose copies add up to tx completes first: the device finishes it on its own.
//              A barrier belongs to the warp whose thread initialised it: before phase q is armed, every lane of that warp must
//              have waited for phase q - 1 (a refill of a stage the warp may still be reading is an error).
//   copy:      dst inside the block's shared memory, dst and src 16-byte aligned, bytes a non-zero multiple of 16, no overlap with a
//              copy still in flight, the phase armed, at most tx bytes per phase.  At issue dst is filled with POISON; the bytes,
//              recorded at issue, land when the phase completes.
//   wait:      each lane counts its own waits per barrier: its next phase is that count, and the parity it passes must be that
//              phase's.  The phase completes (and its bytes land) when its arrival is in and its copies add up to tx.  A barrier two
//              or more phases ahead of the lane is an error (parity aliasing); a phase that does not complete within a generous
//              wall-clock bound (EMU_RING_HANG_MS, default 10 s) is reported as "would hang" with the barrier's state.
//   block end: every barrier idle: no phase armed, no copy in flight.
// Not modelled: the ordering fence.proxy.async gives between generic and async-proxy accesses (stage_fence is a no-op here).
// An error prints one line starting "ring model:" and ends the process.
struct RingCopy { unsigned char* dst; std::vector<unsigned char> bytes; };
struct RingBar {
    unsigned init_tid = 0, n_lanes = 0;   // the initialising thread's warp: its first thread and lane count
    uint64_t phase = 0;                   // phases completed
    uint32_t arrivals = 0;                // arrivals in the current phase (0 or 1)
    uint64_t tx = 0, copied = 0;          // bytes the current phase expects / bytes issued to it
    std::vector<RingCopy> inflight;
    uint64_t waits[32] = {};              // per lane: waits returned (= the phase the lane waits for next)
    bool idle() const { return arrivals == 0 && tx == 0 && copied == 0 && inflight.empty(); }
    bool done() const { return arrivals == 1 && copied == tx; }
};
inline constexpr unsigned char RING_POISON = 0xA6;

struct Block {
    std::barrier<> bar;
    std::vector<std::unique_ptr<Warp>> warps;
    std::vector<unsigned char> shared;
    size_t shared_used = 0;
    std::mutex ring_mu;
    std::map<uintptr_t, RingBar> ring;
    explicit Block(int n) : bar(n) {}
};
struct ThreadState { dim3 tid, bid, bdim, gdim; Block* block = nullptr; Warp* warp = nullptr; };
inline thread_local ThreadState T;

inline void* shared_base() { return (void*)(((uintptr_t)T.block->shared.data() + 63) & ~(uintptr_t)63); }

[[noreturn]] inline void ring_fail(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
inline void ring_fail(const char* fmt, ...) {
    char msg[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(msg, sizeof msg, fmt, ap);
    va_end(ap);
    fprintf(stderr, "ring model: block %u thread %u: %s\n", T.bid.x, T.tid.x, msg);
    fflush(stderr);
    std::_Exit(86);
}
inline uintptr_t ring_off(const void* p) { return (uintptr_t)p - (uintptr_t)shared_base(); }
inline RingBar& ring_bar(unsigned long long* bar, const char* what) {
    auto it = T.block->ring.find((uintptr_t)bar);
    if (it == T.block->ring.end()) ring_fail("%s on barrier +%zu, which was never initialised", what, (size_t)ring_off(bar));
    return it->second;
}
inline void ring_state(const RingBar& b, char* out, size_t n) {
    snprintf(out, n, "phase %llu, arrivals %u of 1, tx expected %llu, copied %llu, %zu copies in flight", (unsigned long long)b.phase,
             b.arrivals, (unsigned long long)b.tx, (unsigned long long)b.copied, b.inflight.size());
}
inline void ring_complete(RingBar& b) {                 // (caller holds ring_mu and has checked done())
    for (const RingCopy& c : b.inflight) memcpy(c.dst, c.bytes.data(), c.bytes.size());
    b.inflight.clear();
    b.arrivals = 0; b.tx = b.copied = 0;
    b.phase++;
}

inline void ring_init(unsigned long long* bar) {
    std::lock_guard<std::mutex> g(T.block->ring_mu);
    RingBar& b = T.block->ring[(uintptr_t)bar];
    if (!b.idle()) {
        char st[160];
        ring_state(b, st, sizeof st);
        ring_fail("barrier +%zu initialised again with a phase armed (%s)", (size_t)ring_off(bar), st);
    }
    b = RingBar{};
    b.init_tid = T.tid.x & ~31u;
    b.n_lanes = std::min(32u, T.bdim.x - b.init_tid);
}
inline void ring_expect(unsigned long long* bar, uint32_t bytes) {
    std::lock_guard<std::mutex> g(T.block->ring_mu);
    RingBar& b = ring_bar(bar, "expect_tx");
    if (b.done()) ring_complete(b);
    if (b.arrivals) {
        char st[160];
        ring_state(b, st, sizeof st);
        ring_fail("second arrival (expect_tx %u) in an unfinished phase of barrier +%zu: it would complete early (%s)", bytes,
                  (size_t)ring_off(bar), st);
    }
    for (unsigned l = 0; l < b.n_lanes; ++l)
        if (b.waits[l] < b.phase)
            ring_fail("barrier +%zu armed for phase %llu while lane %u of its warp has waited for %llu phases: a refill of a stage the warp "
                      "may still be reading", (size_t)ring_off(bar), (unsigned long long)b.phase, l, (unsigned long long)b.waits[l]);
    b.arrivals = 1;
    b.tx += bytes;
}
inline void ring_copy(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
    std::lock_guard<std::mutex> g(T.block->ring_mu);
    RingBar& b = ring_bar(bar, "copy");
    const uintptr_t base = (uintptr_t)shared_base(), d = (uintptr_t)dst;
    if (d < base || d + bytes > base + T.block->shared.size() - 64)
        ring_fail("copy of %u bytes to %p: outside the block's shared memory", bytes, dst);
    if ((d | (uintptr_t)src) & 15) ring_fail("copy of %u bytes to +%zu from %p: not 16-byte aligned", bytes, (size_t)(d - base), src);
    if (bytes == 0 || bytes % 16) ring_fail("copy of %u bytes to +%zu: not a non-zero multiple of 16", bytes, (size_t)(d - base));
    for (const auto& [key, o] : T.block->ring)
        for (const RingCopy& c : o.inflight)
            if (d < (uintptr_t)c.dst + c.bytes.size() && (uintptr_t)c.dst < d + bytes)
                ring_fail("copy to [+%zu, +%zu) overlaps a copy still in flight to [+%zu, +%zu) (barrier +%zu)", (size_t)(d - base),
                          (size_t)(d - base + bytes), (size_t)((uintptr_t)c.dst - base), (size_t)((uintptr_t)c.dst - base + c.bytes.size()),
                          (size_t)(key - base));
    if (!b.arrivals) ring_fail("copy of %u bytes on barrier +%zu before its phase was armed by expect_tx", bytes, (size_t)ring_off(bar));
    if (b.copied + bytes > b.tx)
        ring_fail("copies of %llu bytes on barrier +%zu exceed the %llu bytes its phase expects", (unsigned long long)(b.copied + bytes),
                  (size_t)ring_off(bar), (unsigned long long)b.tx);
    b.inflight.push_back(RingCopy{(unsigned char*)dst, std::vector<unsigned char>((const unsigned char*)src, (const unsigned char*)src + bytes)});
    b.copied += bytes;
    memset(dst, RING_POISON, bytes);
}
inline void ring_wait(unsigned long long* bar, uint32_t parity) {
    static const long hang_ms = [] { const char* e = getenv("EMU_RING_HANG_MS"); return e ? atol(e) : 10000L; }();
    const auto t0 = std::chrono::steady_clock::now();
    for (;;) {
        {
            std::lock_guard<std::mutex> g(T.block->ring_mu);
            RingBar& b = ring_bar(bar, "wait");
            const unsigned lane = T.tid.x - b.init_tid;
            if (T.tid.x < b.init_tid || lane >= b.n_lanes) ring_fail("wait on barrier +%zu from outside the warp that owns it", (size_t)ring_off(bar));
            const uint64_t w = b.waits[lane];
            if ((w & 1) != parity)
                ring_fail("wait(parity %u) on barrier +%zu, but lane %u's next phase is %llu: a parity that was not flipped (the device "
                          "returns on a stale phase or waits forever)", parity, (size_t)ring_off(bar), lane, (unsigned long long)w);
            if (b.phase == w && b.done()) ring_complete(b);
            if (b.phase >= w + 2)
                ring_fail("lane %u waits for phase %llu of barrier +%zu, which has completed %llu phases: parity aliasing", lane,
                          (unsigned long long)w, (size_t)ring_off(bar), (unsigned long long)b.phase);
            if (b.phase == w + 1) { b.waits[lane]++; return; }
            if (std::chrono::steady_clock::now() - t0 > std::chrono::milliseconds(hang_ms)) {
                char st[160];
                ring_state(b, st, sizeof st);
                ring_fail("would hang: lane %u waits for phase %llu of barrier +%zu (%s)", lane, (unsigned long long)w, (size_t)ring_off(bar), st);
            }
        }
        std::this_thread::sleep_for(std::chrono::microseconds(20));
    }
}
inline void ring_block_end(Block& blk, unsigned b) {
    const uintptr_t base = ((uintptr_t)blk.shared.data() + 63) & ~(uintptr_t)63;
    for (const auto& [key, o] : blk.ring)
        if (!o.idle()) {
            char st[160];
            ring_state(o, st, sizeof st);
            T.bid = {b, 0, 0}; T.tid = {o.init_tid, 0, 0};
            ring_fail("the block exits with barrier +%zu busy (%s)", (size_t)(key - base), st);
        }
}

// Runs `body` as a grid of `grid` blocks of `threads` threads (1-D), with `shared_bytes` of block-shared memory.
inline void launch(unsigned grid, unsigned threads, size_t shared_bytes, const std::function<void()>& body) {
    for (unsigned b = 0; b < grid; ++b) {
        Block blk((int)threads);
        blk.shared.assign(shared_bytes + 64, 0xCD);          // uninitialised shared memory is garbage, like on the device
        for (unsigned w = 0; w < (threads + 31) / 32; ++w) blk.warps.emplace_back(new Warp((int)std::min(32u, threads - 32 * w)));
        std::vector<std::thread> th;
        for (unsigned t = 0; t < threads; ++t)
            th.emplace_back([&, t] {
                T.tid = {t, 0, 0}; T.bid = {b, 0, 0}; T.bdim = {threads, 1, 1}; T.gdim = {grid, 1, 1};
                T.block = &blk; T.warp = blk.warps[t / 32].get();
                body();
            });
        for (auto& x : th) x.join();
        ring_block_end(blk, b);
    }
}
}  // namespace emu

#define threadIdx (emu::T.tid)
#define blockIdx (emu::T.bid)
#define blockDim (emu::T.bdim)
#define gridDim (emu::T.gdim)

static inline void __syncthreads() { emu::T.block->bar.arrive_and_wait(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { emu::T.warp->bar.arrive_and_wait(); }
static inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }

template <class V> static inline V emu_exchange(V v, int src_lane) {   // every thread of the warp calls it
    static_assert(sizeof(V) <= 8, "shuffle of <= 8 bytes");
    emu::Warp* w = emu::T.warp;
    unsigned long long raw = 0;
    memcpy(&raw, &v, sizeof v);
    w->xchg[threadIdx.x & 31] = raw;
    w->bar.arrive_and_wait();
    const unsigned long long got = w->xchg[src_lane & 31];
    w->bar.arrive_and_wait();
    V out;
    memcpy(&out, &got, sizeof out);
    return out;
}
template <class V> static inline V __shfl_sync(unsigned, V v, int src) { return emu_exchange(v, src); }
template <class V> static inline V __shfl_up_sync(unsigned, V v, unsigned d) {
    const int lane = threadIdx.x & 31;
    V got = emu_exchange(v, lane >= (int)d ? lane - (int)d : lane);
    return lane >= (int)d ? got : v;
}
template <class V> static inline V __shfl_down_sync(unsigned, V v, unsigned d) {
    const int lane = threadIdx.x & 31;
    const int n = std::min(32u, blockDim.x - (threadIdx.x & ~31u));
    V got = emu_exchange(v, lane + (int)d < n ? lane + (int)d : lane);
    return lane + (int)d < n ? got : v;
}
static inline unsigned __ballot_sync(unsigned, int pred) {
    emu::Warp* w = emu::T.warp;
    w->xchg[threadIdx.x & 31] = pred ? 1 : 0;
    w->bar.arrive_and_wait();
    unsigned m = 0;
    const int n = std::min(32u, blockDim.x - (threadIdx.x & ~31u));
    for (int i = 0; i < n; ++i) m |= (unsigned)w->xchg[i] << i;
    w->bar.arrive_and_wait();
    return m;
}
static inline unsigned __reduce_max_sync(unsigned, unsigned v) {
    unsigned m = v;
    for (int o = 16; o > 0; o >>= 1) m = std::max(m, __shfl_down_sync(0xffffffffu, m, o));
    return __shfl_sync(0xffffffffu, m, 0);
}

// ---- atomics (relaxed is what the device gives; the barriers order everything else)
template <class V> static inline V atomicAdd(V* p, V v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline double atomicAdd(double* p, double v) {
    unsigned long long* q = (unsigned long long*)p;
    unsigned long long old = __atomic_load_n(q, __ATOMIC_RELAXED), want;
    double od;
    do { memcpy(&od, &old, 8); const double nd = od + v; memcpy(&want, &nd, 8); } while (!__atomic_compare_exchange_n(q, &old, want, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED));
    return od;
}
template <class V> static inline V atomicOr(V* p, V v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
template <class V> static inline V atomicMin(V* p, V v) {
    V old = __atomic_load_n(p, __ATOMIC_RELAXED);
    while (v < old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    return old;
}
template <class V> static inline V atomicMax(V* p, V v) {
    V old = __atomic_load_n(p, __ATOMIC_RELAXED);
    while (v > old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    return old;
}
template <class V> static inline V atomicCAS(V* p, V cmp, V val) {
    __atomic_compare_exchange_n(p, &cmp, val, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
    return cmp;
}
template <class V> static inline V __ldg(const V* p) { return *p; }
template <class V> static inline V __ldcg(const V* p) { return __atomic_load_n(p, __ATOMIC_SEQ_CST); }

// ---- intrinsics
static inline unsigned __brev(unsigned x) {
    x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
    x = ((x >> 2) & 0x33333333u) | ((x & 0x33333333u) << 2);
    x = ((x >> 4) & 0x0F0F0F0Fu) | ((x & 0x0F0F0F0Fu) << 4);
    return __builtin_bswap32(x);
}
static inline unsigned long long __brevll(unsigned long long x) { return ((unsigned long long)__brev((unsigned)x) << 32) | __brev((unsigned)(x >> 32)); }
static inline int __ffsll(long long x) { return __builtin_ffsll(x); }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned shift) { return (unsigned)((((unsigned long long)hi << 32) | lo) >> (shift & 31)); }
static inline long long __double_as_longlong(double x) { long long r; memcpy(&r, &x, 8); return r; }
static inline double __longlong_as_double(long long x) { double r; memcpy(&r, &x, 8); return r; }
static inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
static inline double __dsub_rn(double a, double b) { volatile double r = a - b; return r; }
static inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
static inline double __ddiv_rn(double a, double b) { volatile double r = a / b; return r; }
using std::max;
using std::min;
static inline unsigned min(unsigned a, int b) { return a < (unsigned)b ? a : (unsigned)b; }
static inline unsigned long long min(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
