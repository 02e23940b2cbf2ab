// TEST INFRASTRUCTURE ONLY -- a tiny CUDA-on-CPU emulator.
//
// The build container has nvcc but no GPU, and a GPU run costs minutes of a small budget, so the
// `not gpu` tests compile the SAME kernel sources (matchering_b200/csrc/*.cu) for the host with
// this header force-included (-DMGB_EMULATE) and run them block by block: every CUDA thread of a
// block is a fiber on one OS thread, __syncthreads()/__shfl_*_sync() are cooperative barriers,
// `__shared__` is a thread_local static.  Blocks run in blockIdx order, so decoupled look-back
// kernels always find their predecessors finished.  It checks kernel LOGIC (indexing, barriers,
// scan carries) against the oracle; it proves nothing about performance and is never loaded by
// the product package (matchering_b200/_native.py only ever loads the nvcc-built library).
//
// Memory a block has not written is not trusted to be benign:
// - Dynamic shared memory is a fresh allocation at every block start, filled with 0xFF (NaN as a
//   float or double, -1 as an int), so a read of a word the block never wrote shows up in the result.
// - Static `__shared__` arrays are thread_local statics: they keep the previous block's values.
//
// Schedule: between two synchronisation points a fiber runs alone, and each round resumes the
// block's ready fibers in the order MGB_EMUL_ORDER names: `forward` (ascending thread index, the
// default), `reverse`, or `seeded` (a fresh permutation every round from MGB_EMUL_SEED, default 1).
// A missing barrier whose reader runs after its writer in one order runs before it in another.
//
// Race checking (-DMGB_EMUL_RACECHECK, with the kernel sources built -fsanitize=thread): every
// emulated thread is a ThreadSanitizer fiber, created for its block and destroyed at the block's end,
// and switches between fibers carry no happens-before edge.  Edges exist only where CUDA gives them:
// - __syncthreads: release on arrival, acquire on departure (an exited thread counts as arrived);
// - __syncwarp and the warp shuffles / votes: the same among the warp's participating lanes;
// - atomics are relaxed __atomic operations: concurrent ones are not races, and they order nothing;
// - TMA completion: release by the copying thread, acquire by each waiter;
// - a launch is ordered after the host code before it, and the host code after it after the whole
//   launch.  Blocks of one launch are also ordered one after another: races BETWEEN blocks are not
//   looked for, since static `__shared__` arrays cannot be given fresh shadow memory per block.
// - ThreadSanitizer tells at most 256 live threads apart.  A block of more than 224 threads therefore shares
//   fibers among lanes of one warp, in one of two groupings that alternate by block and launch (cuda_emul.cpp);
//   every pair of lanes has fibers of its own in one of them.  A kernel launched once with a single block is
//   seen in one grouping only: there, races between the few lanes of a warp that share a fiber go unreported.
// - A warp keeps one barrier counter, and a warp barrier completes when as many lanes as its mask names
//   have arrived.  Two disjoint lane groups of one warp that synchronise under partial masks at the same time
//   would be ordered with each other, which CUDA does not do.  (Every warp intrinsic in the kernels names the
//   full warp.)
// The scheduler and its bookkeeping live in cuda_emul.cpp, which is never instrumented.
#pragma once
#ifndef MGB_EMULATE
#error "cuda_emul.h is only for -DMGB_EMULATE host builds"
#endif

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

// ----------------------------------------------------------------------------- keywords
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __shared__ static thread_local
#define __constant__ static
#define __align__(n) alignas(n)
#define __grid_constant__

struct uint3 { unsigned x, y, z; };
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct alignas(8) float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(16) double2 { double x, y; };
struct alignas(8) int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(4) short2 { short x, y; };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline double2 make_double2(double x, double y) { return double2{x, y}; }
static inline int2 make_int2(int x, int y) { return int2{x, y}; }

typedef void* cudaStream_t;
typedef int cudaError_t;
enum { cudaSuccess = 0 };

namespace emul {

struct Fiber {
    void* sp = nullptr;
    char* stack = nullptr;
    bool done = false;
    unsigned tid = 0;
    void* tsan = nullptr;  // the fiber's ThreadSanitizer context (race-checking build)
};

struct WarpState {
    uint64_t vals[32];
    unsigned arrived = 0, gen = 0;
    unsigned ballot_acc = 0;
    char sync[2];  // release/acquire objects of the warp barrier, by generation parity
};

struct BlockState {
    unsigned nthreads = 0, alive = 0;
    unsigned arrived = 0, gen = 0;
    std::vector<Fiber> fibers;
    std::vector<WarpState> warps;
    std::function<void()> body;
    void* sched_sp = nullptr;
    void* sched_tsan = nullptr;
    unsigned current = 0;
    unsigned char* dyn_smem = nullptr;
    char sync[2];         // release/acquire objects of __syncthreads, by generation parity
    char exit_sync;       // threads that have exited -> the arrival that completes a barrier
    char start_sync, end_sync;  // host -> every fiber at its start; every fiber at its end -> host
};

BlockState& block();
void yield();
void launch(dim3 grid, dim3 blockdim, size_t smem_bytes, const std::function<void()>& body);
unsigned char* dyn_smem();
// The synchronisation points, in cuda_emul.cpp so that the race-checking build never instruments the
// scheduler's bookkeeping: the block barrier, a barrier of `expected` lanes of the caller's warp, and a
// shuffle of a raw 8-byte payload from `src_lane`.
void syncthreads();
void warp_barrier(unsigned expected);
uint64_t shfl_raw(unsigned expected, uint64_t raw, unsigned src_lane);

}  // namespace emul

extern thread_local uint3 threadIdx;
extern thread_local uint3 blockIdx;
extern thread_local dim3 blockDim;
extern thread_local dim3 gridDim;

// ----------------------------------------------------------------------------- barriers
static inline void __syncthreads() { emul::syncthreads(); }

namespace emul {
static inline unsigned lane_id() { return threadIdx.x & 31u; }
static inline unsigned warp_width() {
    // number of live lanes in this warp (last warp of a block may be partial)
    unsigned base = threadIdx.x & ~31u;
    unsigned n = block().nthreads - base;
    return n > 32 ? 32 : n;
}
template <typename T>
static inline T shfl_generic(unsigned mask, T v, int src_lane) {
    static_assert(sizeof(T) <= 8, "shuffle payload");
    unsigned expected = std::min<unsigned>(__builtin_popcount(mask), warp_width());
    uint64_t raw = 0;
    std::memcpy(&raw, &v, sizeof(T));
    uint64_t got = shfl_raw(expected, raw, (unsigned)src_lane & 31u);
    T out;
    std::memcpy(&out, &got, sizeof(T));
    return out;
}
}  // namespace emul

static inline void __syncwarp(unsigned mask = 0xffffffffu) {
    emul::warp_barrier(std::min<unsigned>(__builtin_popcount(mask), emul::warp_width()));
}
template <typename T>
static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
    int lane = (int)emul::lane_id();
    int base = lane & ~(width - 1);
    return emul::shfl_generic(mask, v, base + (src & (width - 1)));
}
template <typename T>
static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    int lane = (int)emul::lane_id();
    int base = lane & ~(width - 1);
    int src = lane - (int)delta;
    if (src < base) src = lane;
    return emul::shfl_generic(mask, v, src);
}
template <typename T>
static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    int lane = (int)emul::lane_id();
    int base = lane & ~(width - 1);
    int src = lane + (int)delta;
    if (src >= base + width) src = lane;
    return emul::shfl_generic(mask, v, src);
}
template <typename T>
static inline T __shfl_xor_sync(unsigned mask, T v, int lanemask, int width = 32) {
    int lane = (int)emul::lane_id();
    (void)width;
    return emul::shfl_generic(mask, v, lane ^ lanemask);
}
static inline unsigned __ballot_sync(unsigned mask, int pred) {
    unsigned bit = pred ? (1u << emul::lane_id()) : 0u;
    unsigned acc = 0;
    for (int l = 0; l < 32; ++l) {
        unsigned b = __shfl_sync(mask, bit, l);
        if ((mask >> l) & 1u) acc |= (b & (1u << l));
    }
    return acc;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __all_sync(unsigned mask, int pred) {
    unsigned live = mask;
    unsigned w = emul::warp_width();
    if (w < 32) live &= ((1u << w) - 1u);
    return (__ballot_sync(mask, pred) & live) == live;
}

// ----------------------------------------------------------------------------- memory / atomics
static inline void __threadfence() { __sync_synchronize(); }
static inline void __threadfence_block() { __sync_synchronize(); }
static inline void __nanosleep(unsigned) { emul::yield(); }
template <typename T>
static inline T __ldg(const T* p) { return *p; }
template <typename T>
static inline T __ldcg(const T* p) { return *(const volatile T*)p; }

// Relaxed, like CUDA's atomics: concurrent ones are not a race, and none of them orders other accesses.
namespace emul {
template <typename T, typename F>
static inline T atomic_rmw(T* p, F f) {
    T o, n;
    __atomic_load(p, &o, __ATOMIC_RELAXED);
    do n = f(o);
    while (!__atomic_compare_exchange(p, &o, &n, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED));
    return o;
}
}  // namespace emul
static inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline float atomicAdd(float* p, float v) { return emul::atomic_rmw(p, [v](float o) { return o + v; }); }
static inline double atomicAdd(double* p, double v) { return emul::atomic_rmw(p, [v](double o) { return o + v; }); }
static inline int atomicMax(int* p, int v) { return emul::atomic_rmw(p, [v](int o) { return v > o ? v : o; }); }
static inline unsigned atomicMax(unsigned* p, unsigned v) { return emul::atomic_rmw(p, [v](unsigned o) { return v > o ? v : o; }); }
static inline int atomicExch(int* p, int v) { return __atomic_exchange_n(p, v, __ATOMIC_RELAXED); }
static inline unsigned atomicExch(unsigned* p, unsigned v) { return __atomic_exchange_n(p, v, __ATOMIC_RELAXED); }
static inline int atomicCAS(int* p, int c, int v) {
    __atomic_compare_exchange_n(p, &c, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED);
    return c;
}
static inline unsigned atomicOr(unsigned* p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }

// ----------------------------------------------------------------------------- math intrinsics
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
static inline unsigned __float_as_uint(float f) { unsigned i; std::memcpy(&i, &f, 4); return i; }
static inline float __uint_as_float(unsigned i) { float f; std::memcpy(&f, &i, 4); return f; }
static inline long long __double_as_longlong(double d) { long long i; std::memcpy(&i, &d, 8); return i; }
static inline double __longlong_as_double(long long i) { double d; std::memcpy(&d, &i, 8); return d; }
static inline float __fmaf_rn(float a, float b, float c) { return std::fmaf(a, b, c); }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline double __fma_rn(double a, double b, double c) { return std::fma(a, b, c); }
static inline float __double2float_rn(double d) { return (float)d; }
static inline double rsqrt(double x) { return 1.0 / std::sqrt(x); }
static inline float rsqrtf(float x) { return 1.0f / std::sqrt(x); }
static inline void sincospi(double x, double* s, double* c) {
    // exact quadrant reduction so that multiples of 1/2 give exact 0/+-1 like CUDA's sincospi
    double r = std::fmod(x, 2.0);
    if (r < 0) r += 2.0;
    int q = (int)std::floor(r * 2.0 + 0.5);  // nearest multiple of 1/2
    double t = r - 0.5 * q;
    double st = std::sin(M_PI * t), ct = std::cos(M_PI * t);
    switch (q & 3) {
        case 0: *s = st; *c = ct; break;
        case 1: *s = ct; *c = -st; break;
        case 2: *s = -st; *c = -ct; break;
        default: *s = -ct; *c = st; break;
    }
}
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __clz(int v) { return v == 0 ? 32 : __builtin_clz((unsigned)v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
using std::fabs;
using std::fmax;
using std::fmin;
using std::sqrt;
using std::max;
using std::min;
static inline float fabsf_(float x) { return std::fabs(x); }
