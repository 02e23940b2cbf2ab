// Block-wide selection shared by the LOWESS robustness weights (design.cu) and the loudness range (loudness.cuh).
#pragma once
#include "common.cuh"

namespace mgb {

namespace {

// k-th smallest (0-based) of n NON-NEGATIVE doubles: radix select on the bit patterns, one byte per pass.
// Every thread of the block calls and gets the value; barriers inside.
__device__ double block_kth_smallest(const double* __restrict__ v, int n, int k) {
    __shared__ unsigned hist[256];
    __shared__ unsigned long long sel_prefix;
    __shared__ int sel_rank;
    const int tid = threadIdx.x, nthr = blockDim.x;
    // The first pass starts from prefix 0 and rank k without reading sel_prefix / sel_rank: other threads may
    // still be reading the previous call's result there.  Thread 0 first writes them after this call's
    // second barrier, which every thread reaches only after that read.
    unsigned long long mask = 0ull;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int b = tid; b < 256; b += nthr) hist[b] = 0u;
        __syncthreads();
        const unsigned long long prefix = shift == 56 ? 0ull : sel_prefix;
        for (int j = tid; j < n; j += nthr) {
            const unsigned long long bits = (unsigned long long)__double_as_longlong(v[j]);
            if ((bits & mask) == prefix) atomicAdd(&hist[(unsigned)(bits >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            int rank = shift == 56 ? k : sel_rank, b = 0;
            while (b < 255 && rank >= (int)hist[b]) {
                rank -= (int)hist[b];
                ++b;
            }
            sel_rank = rank;
            sel_prefix = prefix | ((unsigned long long)b << shift);
        }
        mask |= 0xffull << shift;
        __syncthreads();
    }
    return __longlong_as_double((long long)sel_prefix);
}

}  // namespace

}  // namespace mgb
