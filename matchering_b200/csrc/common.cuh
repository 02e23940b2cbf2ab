// Shared device helpers for the matchering_b200 kernels (sm_90a).
//
// The same sources are also compiled for the host by the test-only emulator
// (tests/emul/cuda_emul.h, -DMGB_EMULATE); everything PTX-specific therefore lives behind the
// small wrappers in this file.
#pragma once

#ifndef MGB_EMULATE
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "../../include/matchering_b200.h"

namespace mgb {

// ------------------------------------------------------------------------------------------------
// error plumbing (no exceptions cross the C ABI)
// ------------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_status(const char* what);  // 0 or MGB_ERR_CUDA, recording cudaGetLastError()

#define MGB_REQUIRE(cond, code, ...)     \
    do {                                 \
        if (!(cond)) {                   \
            ::mgb::set_error(__VA_ARGS__); \
            return (code);               \
        }                                \
    } while (0)

#define MGB_TRY(expr)                 \
    do {                              \
        int mgb_rc_ = (expr);         \
        if (mgb_rc_ != MGB_OK) return mgb_rc_; \
    } while (0)

// ------------------------------------------------------------------------------------------------
// launch helper
// ------------------------------------------------------------------------------------------------
#ifdef MGB_EMULATE
#define MGB_DYN_SMEM(name) unsigned char* name = ::emul::dyn_smem()
template <typename... KA, typename... A>
inline int launch(const char* what, void (*kernel)(KA...), dim3 grid, dim3 block, size_t smem, cudaStream_t,
                  A... args) {
    (void)what;
    if (grid.x == 0 || grid.y == 0 || grid.z == 0) return MGB_OK;
    ::emul::launch(grid, block, smem, [&]() { kernel(static_cast<KA>(args)...); });
    return MGB_OK;
}
#else
#define MGB_DYN_SMEM(name) extern __shared__ __align__(128) unsigned char name[]
// launch bookkeeping (api.cu): a counter of kernel launches and, when profiling is switched on,
// a CUDA-event pair around every launch on the launching stream
extern long long g_launch_count;
extern int g_profile;
void profile_mark(const char* what, cudaStream_t stream, bool begin);

template <typename... KA, typename... A>
inline int launch(const char* what, void (*kernel)(KA...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                  A... args) {
    if (grid.x == 0 || grid.y == 0 || grid.z == 0) return MGB_OK;
    g_launch_count++;
    if (smem > 48 * 1024) {
        // opt in to large dynamic shared memory once per kernel and size (a driver call per launch
        // would sit on the critical path of an 11-launch, sub-millisecond pipeline)
        static thread_local const void* done_kernel = nullptr;
        static thread_local size_t done_smem = 0;
        if (done_kernel != (const void*)kernel || done_smem < smem) {
            cudaError_t e = cudaFuncSetAttribute((const void*)kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) {
                set_error("%s: cudaFuncSetAttribute(%zu B smem): %s", what, smem, cudaGetErrorString(e));
                return MGB_ERR_CUDA;
            }
            done_kernel = (const void*)kernel;
            done_smem = smem;
        }
    }
    if (g_profile) profile_mark(what, stream, true);
    kernel<<<grid, block, smem, stream>>>(static_cast<KA>(args)...);
    if (g_profile) profile_mark(what, stream, false);
    return cuda_status(what);
}
#endif

int num_sms();

// ------------------------------------------------------------------------------------------------
// small numeric helpers
// ------------------------------------------------------------------------------------------------
template <typename T>
struct cpx {
    T x, y;
};
template <typename T>
__device__ __forceinline__ cpx<T> cmul(cpx<T> a, cpx<T> b) {
    return cpx<T>{a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x};
}
template <typename T>
__device__ __forceinline__ cpx<T> cadd(cpx<T> a, cpx<T> b) { return cpx<T>{a.x + b.x, a.y + b.y}; }
template <typename T>
__device__ __forceinline__ cpx<T> csub(cpx<T> a, cpx<T> b) { return cpx<T>{a.x - b.x, a.y - b.y}; }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide sum of a double; result valid in thread 0 (and broadcast through `scratch[0]`
// after the trailing barrier).  `scratch` holds >= 32 doubles.  All threads must call.
__device__ __forceinline__ double block_sum(double v, double* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();  // scratch may still be read from a previous call
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    if (warp == 0) {
        double t = (lane < nwarps) ? scratch[lane] : 0.0;
        t = warp_sum(t);
        if (lane == 0) scratch[0] = t;
    }
    __syncthreads();
    return scratch[0];
}
__device__ __forceinline__ float block_max(float v, float* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    if (warp == 0) {
        float t = (lane < nwarps) ? scratch[lane] : 0.0f;
        t = warp_max(t);
        if (lane == 0) scratch[0] = t;
    }
    __syncthreads();
    return scratch[0];
}

// Block-wide maxima of two non-negative floats at once; both results valid in every thread.
// Non-negative floats order like their bit patterns, so each warp reduces with one integer
// redux.sync per value and its lane 0 folds the result into shared memory with an atomic max: one
// barrier in all.  `slot` (2 unsigned words in shared memory) must be zero on entry; callers that
// loop alternate between two slots and clear the idle one.  All threads must call.
__device__ __forceinline__ unsigned warp_max_bits(unsigned v) {
#ifdef MGB_EMULATE
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned other = __shfl_xor_sync(0xffffffffu, v, o);
        v = other > v ? other : v;
    }
    return v;
#else
    return __reduce_max_sync(0xffffffffu, v);
#endif
}
__device__ __forceinline__ void block_max2(float& a, float& b, unsigned* slot) {
    const unsigned ua = warp_max_bits(__float_as_uint(a)), ub = warp_max_bits(__float_as_uint(b));
    if ((threadIdx.x & 31) == 0) {
        atomicMax(&slot[0], ua);
        atomicMax(&slot[1], ub);
    }
    __syncthreads();
    a = __uint_as_float(slot[0]);
    b = __uint_as_float(slot[1]);
}

// Power-of-two factor that brings `small` up to the scale of `large` (exact in floating point).
// mid and side ride one complex FFT as z = mid + i*g*side: the transform's rounding noise is
// relative to the LARGER part, so without the factor a quiet channel would inherit the loud one's
// noise (and a matching FIR with a huge gain on the quiet channel would amplify it).
__device__ __forceinline__ float balance_factor(float large, float small) {
    if (!(small > 0.0f) || !(large > 0.0f)) return 1.0f;
    // the difference of the two binary exponents is within one of floor(log2(large / small)), which is
    // all the balancing needs; integer work on the bit patterns instead of log2f, a division and exp2f
    int e = (int)((__float_as_uint(large) >> 23) & 0xffu) - (int)((__float_as_uint(small) >> 23) & 0xffu);
    e = e < -60 ? -60 : (e > 60 ? 60 : e);
    return __uint_as_float((unsigned)(127 + e) << 23);
}

// sqrt with the special-function unit alone (sqrt.approx: one MUFU, relative error <= 2^-23) instead of
// sqrtf's correctly rounded sequence (nine instructions and a branch).  For magnitudes that are summed
// over hundreds of frames the half ulp does not matter; the issue slots do.
__device__ __forceinline__ float sqrt_approx(float x) {
#ifdef MGB_EMULATE
    return sqrtf(x);
#else
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#endif
}

// Non-negative floats order like their bit patterns: atomic max through the integer unit.
__device__ __forceinline__ void atomic_max_nonneg(float* addr, float v) {
    atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
}

// ------------------------------------------------------------------------------------------------
// TMA 1-D bulk copy (cp.async.bulk, SASS UBLKCP) completing on an mbarrier.
// One thread arms the barrier with the byte count and issues the copy; every consumer waits on
// the barrier's phase parity.  Sizes and both addresses must be multiples of 16 bytes.
// ------------------------------------------------------------------------------------------------
#ifdef MGB_EMULATE
// the completed phase is a release by the copying thread and an acquire by each waiter, as the mbarrier's is
struct TmaBarrier {
    unsigned phase_done;  // number of completed phases
};
__device__ __forceinline__ void tma_barrier_init(TmaBarrier* b) { __atomic_store_n(&b->phase_done, 0u, __ATOMIC_RELAXED); }
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, TmaBarrier* b) {
    if (bytes) memcpy(smem_dst, gmem_src, bytes);
    __atomic_fetch_add(&b->phase_done, 1u, __ATOMIC_RELEASE);
}
__device__ __forceinline__ void tma_barrier_wait(TmaBarrier* b, uint32_t phase_index) {
    while (__atomic_load_n(&b->phase_done, __ATOMIC_ACQUIRE) <= phase_index) ::emul::yield();
}
__device__ __forceinline__ void fence_proxy_async() {}
#else
struct __align__(8) TmaBarrier {
    unsigned long long bar;
};
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void tma_barrier_init(TmaBarrier* b) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&b->bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, TmaBarrier* b) {
    // bytes == 0 still has to complete the phase: a plain arrive does that.
    if (bytes == 0) {
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&b->bar)) : "memory");
        return;
    }
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&b->bar)), "r"(bytes) : "memory");
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(&b->bar))
        : "memory");
}
__device__ __forceinline__ void tma_barrier_wait(TmaBarrier* b, uint32_t phase_index) {
    const uint32_t parity = phase_index & 1u;
    const uint32_t addr = smem_u32(&b->bar);
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
    } while (!done);
}
#endif

}  // namespace mgb
