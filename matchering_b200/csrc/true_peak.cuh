// K6t -- the true-peak detector of the limiter's true-peak mode (mgb_limiter_params.true_peak = L, Config(true_peak=True)).
//
// The meter's interpolator (loudness.cuh, tp_centre): 12 L + 1 Kaiser-windowed sinc taps, beta = 8, L = 4 / 2 / 1.
//   y_c[n, ph] = upfirdn(h, x_c, up=L)[(n + 6) L + ph]   the interpolated value at n + ph/L (phase 0 is x_c[n] itself)
//   u[n]       = max over both channels and all phases of |y_c[n, ph]|
//   d[n]       = max(u[n], u[n - 1]), u[-1] = 0          every interpolated point within one sample of frame n
// The limiter then takes d where the reference's rectifier takes max(|L|, |R|) (limiter.cu P1, limiter_wide.cuh's gain
// kernel), and its early-out and the normalised output take max(d) where they take the sample peak.
//
//   true_peak_detect_kernel<L>   one read of the track (8 B/frame plus a 6-frame halo per side), the plane d
//                                (4 B/frame) and max(d) by a float-bits atomicMax: exact and order-free
//   true_peak_final_kernel       one thread: normalize_coef and limiter_engaged of a track from gain * max(d)
// (included by limiter.cu)
#pragma once
#include <math.h>

namespace mgb {

namespace {

constexpr int kTpThreads = 256;
constexpr int kTpTile = kTpThreads * 8;  // frames per CTA
constexpr int kTpHalo = 6;               // u[n - 1] reads x[n - 6 .. n + 5], u[n] reads x[n - 5 .. n + 6]

// Phases 1..L-1 of the interpolator: w[ph - 1][t + 5] = h[(6 - t) L + ph] weighs x[n + t], t = -5 .. 6 (t = -6 falls
// beyond the last tap for every phase but 0).  Passed by value: the taps follow from L alone.
struct TruePeakTaps {
    float w[3][12];
};

template <int OS>
__global__ void __launch_bounds__(kTpThreads) true_peak_detect_kernel(TruePeakTaps taps, const float2* __restrict__ x,
                                                                      long long frames, float* __restrict__ d,
                                                                      float* __restrict__ d_max) {
    __shared__ float2 xs[kTpTile + 2 * kTpHalo];  // frames s0 - 6 .. s0 + kTpTile + 5, zero outside the signal
    __shared__ float us[kTpTile + 1];             // u at frames s0 - 1 .. s0 + kTpTile - 1
    __shared__ float red[32];
    const int tid = threadIdx.x;
    const long long s0 = (long long)blockIdx.x * kTpTile;
    for (int i = tid; i < kTpTile + 2 * kTpHalo; i += kTpThreads) {
        const long long n = s0 - kTpHalo + i;
        xs[i] = (n >= 0 && n < frames) ? __ldg(x + n) : make_float2(0.0f, 0.0f);
    }
    __syncthreads();
    for (int i = tid; i <= kTpTile; i += kTpThreads) {
        const long long n = s0 - 1 + i;  // frame n sits at xs[i + 5]
        float m = 0.0f;
        if (n >= 0 && n < frames) {
            const float2 c = xs[i + 5];
            m = fmaxf(fabsf(c.x), fabsf(c.y));
#pragma unroll
            for (int ph = 1; ph < OS; ++ph) {
                float aL = 0.0f, aR = 0.0f;
#pragma unroll
                for (int t = -5; t <= 6; ++t) {
                    const float2 v = xs[i + 5 + t];
                    aL = fmaf(taps.w[ph - 1][t + 5], v.x, aL);
                    aR = fmaf(taps.w[ph - 1][t + 5], v.y, aR);
                }
                m = fmaxf(m, fmaxf(fabsf(aL), fabsf(aR)));
            }
        }
        us[i] = m;
    }
    __syncthreads();
    float pk = 0.0f;
    for (int j = tid; j < kTpTile; j += kTpThreads) {
        const long long n = s0 + j;
        if (n < frames) {
            const float v = fmaxf(us[j + 1], us[j]);
            d[n] = v;
            pk = fmaxf(pk, v);
        }
    }
    pk = block_max(pk, red);
    if (tid == 0) atomic_max_nonneg(d_max, pk);
}

// true_peak_detect_kernel for a version of the main (linked versions): d[n] = max(d[n], its detector at n).  A copy of
// that kernel rather than a flag on it, which changed its register allocation.
template <int OS>
__global__ void __launch_bounds__(kTpThreads) true_peak_accumulate_kernel(TruePeakTaps taps, const float2* __restrict__ x,
                                                                          long long frames, float* __restrict__ d,
                                                                          float* __restrict__ d_max) {
    __shared__ float2 xs[kTpTile + 2 * kTpHalo];  // frames s0 - 6 .. s0 + kTpTile + 5, zero outside the signal
    __shared__ float us[kTpTile + 1];             // u at frames s0 - 1 .. s0 + kTpTile - 1
    __shared__ float red[32];
    const int tid = threadIdx.x;
    const long long s0 = (long long)blockIdx.x * kTpTile;
    for (int i = tid; i < kTpTile + 2 * kTpHalo; i += kTpThreads) {
        const long long n = s0 - kTpHalo + i;
        xs[i] = (n >= 0 && n < frames) ? __ldg(x + n) : make_float2(0.0f, 0.0f);
    }
    __syncthreads();
    for (int i = tid; i <= kTpTile; i += kTpThreads) {
        const long long n = s0 - 1 + i;  // frame n sits at xs[i + 5]
        float m = 0.0f;
        if (n >= 0 && n < frames) {
            const float2 c = xs[i + 5];
            m = fmaxf(fabsf(c.x), fabsf(c.y));
#pragma unroll
            for (int ph = 1; ph < OS; ++ph) {
                float aL = 0.0f, aR = 0.0f;
#pragma unroll
                for (int t = -5; t <= 6; ++t) {
                    const float2 v = xs[i + 5 + t];
                    aL = fmaf(taps.w[ph - 1][t + 5], v.x, aL);
                    aR = fmaf(taps.w[ph - 1][t + 5], v.y, aR);
                }
                m = fmaxf(m, fmaxf(fabsf(aL), fabsf(aR)));
            }
        }
        us[i] = m;
    }
    __syncthreads();
    float pk = 0.0f;
    for (int j = tid; j < kTpTile; j += kTpThreads) {
        const long long n = s0 + j;
        if (n < frames) {
            const float v = fmaxf(d[n], fmaxf(us[j + 1], us[j]));
            d[n] = v;
            pk = fmaxf(pk, v);
        }
    }
    pk = block_max(pk, red);
    if (tid == 0) atomic_max_nonneg(d_max, pk);
}

// sample-peak mode's linked detector: d[n] = max over the entries of max(|L|, |R|), one read of every entry per frame
__global__ void __launch_bounds__(256) versions_detect_kernel(const __grid_constant__ VersionPlanes vp, long long frames,
                                                              float* __restrict__ d, float* __restrict__ d_max) {
    __shared__ float red[32];
    float pk = 0.0f;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < frames; n += stride) {
        float m = 0.0f;
        for (int j = 0; j < vp.count; ++j) {
            const float2 v = __ldg(vp.in[j] + n);
            m = fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.y)));
        }
        d[n] = m;
        pk = fmaxf(pk, m);
    }
    pk = block_max(pk, red);
    if (threadIdx.x == 0) atomic_max_nonneg(d_max, pk);
}

// correction_final_kernel's normalisation coefficient and early-out flag (correct.cu), from the true peak instead of
// the sample peak: peak = gain * max(d)
__global__ void true_peak_final_kernel(const float* __restrict__ d_max, double eps, double threshold,
                                       mgb_track_state* __restrict__ state) {
    const double peak = (double)(*d_max) * state->gain;
    state->normalize_coef = fmax(eps, peak / threshold);
    const double r = fmax(peak, threshold) / threshold;
    state->limiter_engaged = (fabs(r - 1.0) <= 1e-8 + 1e-5) ? 0 : 1;
}

// I0 by its power series, in long double (terms fall below the sum's last bit long before k = 60 at beta = 8)
long double bessel_i0(long double z) {
    long double sum = 1.0L, term = 1.0L;
    const long double q = 0.25L * z * z;
    for (int k = 1; k < 60; ++k) {
        term *= q / ((long double)k * (long double)k);
        sum += term;
    }
    return sum;
}

}  // namespace

// h[m] = sinc((m - 6L)/L) * I0(8 sqrt(1 - ((m - 6L)/(6L))^2)) / I0(8), m = 0 .. 12L: numpy's
// sinc(...) * kaiser(12L + 1, 8), the meter's interpolator
void true_peak_filter(int os, double* h) {
    const long double pi = 3.14159265358979323846264338327950288L, beta = 8.0L;
    const long double i0b = bessel_i0(beta);
    for (int m = 0; m <= 12 * os; ++m) {
        const long double x = (long double)(m - 6 * os) / (long double)os;
        const long double s = m == 6 * os ? 1.0L : sinl(pi * x) / (pi * x);
        const long double r = (long double)(m - 6 * os) / (long double)(6 * os);
        h[m] = (double)(s * bessel_i0(beta * sqrtl(1.0L - r * r)) / i0b);
    }
}

int64_t true_peak_plane_bytes(const mgb_limiter_params& lp, int64_t frames) {
    return lp.true_peak ? (frames * 4 + 255) / 256 * 256 : 0;
}

static TruePeakTaps true_peak_taps(int os) {
    double h[49];
    true_peak_filter(os, h);
    TruePeakTaps taps;
    memset(&taps, 0, sizeof(taps));
    for (int ph = 1; ph < os; ++ph)
        for (int t = -5; t <= 6; ++t) taps.w[ph - 1][t + 5] = (float)h[(6 - t) * os + ph];
    return taps;
}

// d_max must hold 0 (or a smaller true peak) before the launch
int launch_true_peak_detect(int os, const float2* x, int64_t frames, float* d, float* d_max, cudaStream_t stream) {
    const TruePeakTaps taps = true_peak_taps(os);
    const dim3 grid((unsigned)((frames + kTpTile - 1) / kTpTile));
    if (os == 4)
        return launch("true_peak_detect_kernel", true_peak_detect_kernel<4>, grid, dim3(kTpThreads), 0, stream, taps, x,
                      (long long)frames, d, d_max);
    if (os == 2)
        return launch("true_peak_detect_kernel", true_peak_detect_kernel<2>, grid, dim3(kTpThreads), 0, stream, taps, x,
                      (long long)frames, d, d_max);
    return launch("true_peak_detect_kernel", true_peak_detect_kernel<1>, grid, dim3(kTpThreads), 0, stream, taps, x,
                  (long long)frames, d, d_max);
}

int launch_true_peak_accumulate(int os, const float2* x, int64_t frames, float* d, float* d_max, cudaStream_t stream) {
    const TruePeakTaps taps = true_peak_taps(os);
    const dim3 grid((unsigned)((frames + kTpTile - 1) / kTpTile));
    if (os == 4)
        return launch("true_peak_accumulate_kernel", true_peak_accumulate_kernel<4>, grid, dim3(kTpThreads), 0, stream, taps, x,
                      (long long)frames, d, d_max);
    if (os == 2)
        return launch("true_peak_accumulate_kernel", true_peak_accumulate_kernel<2>, grid, dim3(kTpThreads), 0, stream, taps, x,
                      (long long)frames, d, d_max);
    return launch("true_peak_accumulate_kernel", true_peak_accumulate_kernel<1>, grid, dim3(kTpThreads), 0, stream, taps, x,
                  (long long)frames, d, d_max);
}

// d_max must hold 0 before the launch
int launch_versions_detect(const VersionPlanes& vp, int64_t frames, float* d, float* d_max, cudaStream_t stream) {
    const long long blocks = (frames + 1023) / 1024;  // four frames per thread
    const unsigned grid = (unsigned)(blocks < 4LL * num_sms() ? (blocks > 0 ? blocks : 1) : 4LL * num_sms());
    return launch("versions_detect_kernel", versions_detect_kernel, dim3(grid), dim3(256), 0, stream, vp, (long long)frames, d,
                  d_max);
}

int launch_true_peak_final(const float* d_max, double eps, double threshold, mgb_track_state* state, cudaStream_t stream) {
    return launch("true_peak_final_kernel", true_peak_final_kernel, dim3(1), dim3(1), 0, stream, d_max, eps, threshold, state);
}

}  // namespace mgb

extern "C" int mgb_true_peak_taps(int32_t oversample, double* out) {
    using namespace mgb;
    MGB_REQUIRE(oversample == 1 || oversample == 2 || oversample == 4, MGB_ERR_INVALID,
                "true_peak_taps: oversampling %d (1, 2 or 4)", oversample);
    MGB_REQUIRE(out != nullptr, MGB_ERR_INVALID, "true_peak_taps: out is NULL");
    true_peak_filter(oversample, out);
    return MGB_OK;
}
