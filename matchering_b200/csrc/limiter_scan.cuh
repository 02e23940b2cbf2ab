// Block scans and decoupled look-back shared by the limiter's kernels (limiter.cu, limiter_wide.cuh): the
// recursive sections' blocked scan over their state vector, and the 16-byte publish / poll of a chunk's state.
#pragma once
#include "kernels.cuh"

namespace mgb {

namespace {

constexpr int NT = kLimiterThreads;
constexpr int CORE_EPT = kLimiterCoreEpt;
constexpr int LC = kLimiterCore;

// ------------------------------------------------------------------------------------------------
// Recursive sections of order N (hold and release low-passes).  lfilter(b, a, x) is
//     y[n] = sum_{i=0..N} b[i] x[n-i] - sum_{i=1..N} a[i] y[n-i]          (a[0] = 1, zero initial state)
// The feed-forward sum is formed per sample from the thread's own inputs; the recursion is a linear
// recurrence over the STATE s = (y[n-1], ..., y[n-N]) with the companion matrix C (row 0 = -a[1..N], row i =
// e_{i-1}): a segment maps s -> C^len s + (its zero-state end state), which is what the blocked scan and the
// look-back combine.  N = 1 is the scalar scan of a single pole; every loop below unrolls away there.
// ------------------------------------------------------------------------------------------------
template <int N>
struct StVec {
    double v[N];
};
template <int N>
__device__ __forceinline__ StVec<N> st_zero() {
    StVec<N> z;
#pragma unroll
    for (int i = 0; i < N; ++i) z.v[i] = 0.0;
    return z;
}
template <int N>
__device__ __forceinline__ StVec<N> st_shfl_up(StVec<N> a, int d) {
#pragma unroll
    for (int i = 0; i < N; ++i) a.v[i] = __shfl_up_sync(0xffffffffu, a.v[i], d);
    return a;
}
template <int N>
__device__ __forceinline__ StVec<N> st_shfl(StVec<N> a, int src) {
#pragma unroll
    for (int i = 0; i < N; ++i) a.v[i] = __shfl_sync(0xffffffffu, a.v[i], src);
    return a;
}
// y += M x
template <int N>
__device__ __forceinline__ void st_addmul(StVec<N>& y, const double (*M)[N], const StVec<N>& x) {
#pragma unroll
    for (int r = 0; r < N; ++r)
#pragma unroll
        for (int c = 0; c < N; ++c) y.v[r] += M[r][c] * x.v[c];
}
template <int N>
__device__ __forceinline__ StVec<N> st_mul(const double (*M)[N], const StVec<N>& x) {
    StVec<N> y = st_zero<N>();
    st_addmul<N>(y, M, x);
    return y;
}

// Exclusive carry of the section's state across the block: given each thread's zero-state end state B, returns
// the state just before the thread's first element when the state before the block's first element is zero
// (the chunk's carry-in is added later, section_lead).  Same structure and the same single barrier as
// scan_carry; scratch: >= 32*N doubles, alternate between two buffers.  Every thread of the block must call.
template <int N>
__device__ __forceinline__ StVec<N> section_scan(StVec<N> B, const SectionTab<N>* t, double* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    StVec<N> v = B;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const StVec<N> up = st_shfl_up<N>(v, d);
        if (lane >= d) st_addmul<N>(v, t->ql[d], up);
    }
    if (lane == 31) {
#pragma unroll
        for (int i = 0; i < N; ++i) scratch[warp * N + i] = v.v[i];
    }
    __syncthreads();
    StVec<N> w = st_zero<N>();
    if (lane < NT / 32) {
#pragma unroll
        for (int i = 0; i < N; ++i) w.v[i] = scratch[lane * N + i];
    }
#pragma unroll
    for (int d = 1; d < NT / 32; d <<= 1) {
        const StVec<N> up = st_shfl_up<N>(w, d);
        if (lane >= d) st_addmul<N>(w, t->qw[d], up);
    }
    // state at the end of the previous warp: inclusive total of warps 0..warp-1
    StVec<N> warp_carry = st_shfl<N>(w, (warp + 31) & 31);
    if (warp == 0) warp_carry = st_zero<N>();
    StVec<N> prev = st_shfl_up<N>(v, 1);
    if (lane == 0) prev = st_zero<N>();
    st_addmul<N>(prev, t->ql[lane], warp_carry);
    return prev;
}

// C^(tid * CORE_EPT) applied to the chunk's carry-in: what the carry-in contributes to the state just before
// the thread's first element.
template <int N>
__device__ __forceinline__ StVec<N> section_lead(const SectionTab<N>* t, const StVec<N>& cin) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    return st_mul<N>(t->ql[lane], st_mul<N>(t->qw[warp], cin));
}

// 16-byte publish / poll of a LookbackWord through L2 (st.cg / ld.cg: coherent device-wide).
__device__ __forceinline__ void publish(LookbackWord* w, double v, int status) {
#ifdef MGB_EMULATE
    // value and status travel together in one 16-byte store: two 8-byte atomics are as close as the host gets
    __atomic_store_n((long long*)&w->value, __double_as_longlong(v), __ATOMIC_RELAXED);
    __atomic_store_n(&w->status, (long long)status, __ATOMIC_RELAXED);
#else
    asm volatile("st.global.cg.v2.u64 [%0], {%1, %2};" ::"l"(w), "l"(__double_as_longlong(v)), "l"((long long)status) : "memory");
#endif
}
__device__ __forceinline__ int poll(const LookbackWord* w, double* v) {
#ifdef MGB_EMULATE
    *v = __longlong_as_double(__atomic_load_n((const long long*)&w->value, __ATOMIC_RELAXED));
    return (int)__atomic_load_n(&w->status, __ATOMIC_RELAXED);
#else
    long long a, b;
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(w) : "memory");
    *v = __longlong_as_double(a);
    return (int)b;
#endif
}

// Carry into chunk `chunk` of a section whose per-chunk transition is P = pc[1] (decoupled look-back).  One warp
// inspects 32 predecessors at a time: every lane polls one predecessor's words, the window is cut at the nearest
// predecessor whose INCLUSIVE state is known, each lane weighs its state by P^distance, and one warp reduction
// at the very end adds them up.  The walk stops when whatever lies further back weighs less than 1e-9 (all
// states are gains in [0, 1], so that bounds the absolute error of the carry).  A state of N doubles travels as
// N words that each carry the status: a reader that catches the writer between two words sees different
// statuses and polls again.  Called by all 32 lanes of one warp.
template <int N>
__device__ __forceinline__ StVec<N> lookback(const LookbackWord* words /* this section's words of chunk 0 */, int chunk,
                                             const SectionTab<N>* t) {
    constexpr int STRIDE = 2 * N;  // words per chunk: hold[N] then release[N]
    const int lane = threadIdx.x & 31;
    if constexpr (N == 1) {
        // a single pole: scalar weights, the running product P^32, P^64, ... is exact enough (no table)
        double acc1 = 0.0, m1 = 1.0;
        for (int base = chunk - 1; base >= 0 && m1 > 1e-9; base -= 32) {
            const int j = base - lane;
            int st = 2;  // before the first chunk: inclusive state 0 (lfilter starts from rest)
            double val = 0.0;
            if (j >= 0) {
                const LookbackWord* w = words + (long long)j * STRIDE;
                while ((st = poll(w, &val)) == 0) __nanosleep(20);
            }
            const unsigned inclusive = __ballot_sync(0xffffffffu, st == 2);
            const int first = inclusive ? __ffs((int)inclusive) - 1 : 32;
            if (lane <= first) acc1 += m1 * t->pc[lane][0][0] * val;
            if (inclusive) break;
            m1 *= t->pc[32][0][0];
        }
        StVec<N> out;
        out.v[0] = warp_sum(acc1);
        return out;
    }
    StVec<N> acc = st_zero<N>();
    double mult[N][N];  // C^(LC*32*jump): weight of this window's nearest chunk
    int jump = 0;       // windows of 32 chunks already behind us
    for (int base = chunk - 1; base >= 0; base -= 32, ++jump) {
        // From the table (a running product would cost a digit per multiplication for a pole pair); beyond
        // the table -- 2048 chunks back, where the weights of any ordinary release are long below the cut-off
        // -- the product of what is left is good enough.
        if (N > 1 && jump < kLookbackJumps) {
#pragma unroll
            for (int r = 0; r < N; ++r)
#pragma unroll
                for (int c = 0; c < N; ++c) mult[r][c] = t->pj[jump][r][c];
        } else if (jump == 0) {
#pragma unroll
            for (int r = 0; r < N; ++r)
#pragma unroll
                for (int c = 0; c < N; ++c) mult[r][c] = r == c ? 1.0 : 0.0;
        } else {  // (a single pole: the running product is exact enough, no table)
            double next[N][N];
#pragma unroll
            for (int r = 0; r < N; ++r)
#pragma unroll
                for (int c = 0; c < N; ++c) {
                    double sum = 0.0;
#pragma unroll
                    for (int k = 0; k < N; ++k) sum += mult[r][k] * t->pc[32][k][c];
                    next[r][c] = sum;
                }
#pragma unroll
            for (int r = 0; r < N; ++r)
#pragma unroll
                for (int c = 0; c < N; ++c) mult[r][c] = next[r][c];
        }
        // (past its peak at 1/(1-|p|) samples the norm of C^m only falls: once this window's nearest chunk
        // weighs less than 1e-9, so does everything behind it)
        double bound = 0.0;
#pragma unroll
        for (int r = 0; r < N; ++r) {
            double rowsum = 0.0;
#pragma unroll
            for (int c = 0; c < N; ++c) rowsum += fabs(mult[r][c]);
            bound = fmax(bound, rowsum);
        }
        if (bound <= 1e-9) break;
        const int j = base - lane;
        int st = 2;  // before the first chunk: inclusive state 0 (lfilter starts from rest)
        StVec<N> val = st_zero<N>();
        if (j >= 0) {
            const LookbackWord* w = words + (long long)j * STRIDE;
            for (;;) {
                st = poll(w, &val.v[0]);
                bool same = st != 0;
#pragma unroll
                for (int i = 1; i < N; ++i) same = same && poll(w + i, &val.v[i]) == st;
                if (same) break;
                __nanosleep(20);
            }
        }
        const unsigned inclusive = __ballot_sync(0xffffffffu, st == 2);
        const int first = inclusive ? __ffs((int)inclusive) - 1 : 32;
        if (lane <= first) st_addmul<N>(acc, mult, st_mul<N>(t->pc[lane], val));
        if (inclusive) break;
    }
#pragma unroll
    for (int i = 0; i < N; ++i) acc.v[i] = warp_sum(acc.v[i]);
    return acc;
}
template <int N>
__device__ __forceinline__ void publish_state(LookbackWord* words, const StVec<N>& s, int status) {
#pragma unroll
    for (int i = 0; i < N; ++i) publish(words + i, s.v[i], status);
}

}  // namespace

}  // namespace mgb
