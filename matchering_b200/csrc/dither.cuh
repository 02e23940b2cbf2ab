// K5d -- dithered PCM encode: TPDF and noise-shaped dither for 16- and 24-bit results (mgb_pcm_encode_dithered).
//
// The definition (DESIGN.md §4 "Dither"), per channel c of a stereo float32 buffer of N frames, in float64,
// top = 2^(bits-1) - 1:
//   d[n, c] = (a - b) / 2^24, a = z >> 40, b = (z >> 16) & 0xFFFFFF,
//             z = splitmix64_finalizer(seed + (2n + c + 1) * 0x9E3779B97F4A7C15)      TPDF in (-1, 1) LSB
//   u = x * top (exact), fb = 0 then fb += h_k * e[n - k] for k = K .. 1 (oldest first, no FMA contraction)
//   v = u - fb, w = v + d, q = rint(w), e[n] = q - v, out = clip(q, -top - 1, top)
//   a non-finite q: e[n] = 0 and the plain encoder's sample (quantize)
// Each channel is cut into segments of kDitherSegment frames; segment s starts with a zero error history at frame
// max(0, s S - kDitherWarmup), runs the loop through the warm-up and writes its own frames only.  So every output bit
// follows from the definition, whatever the grid, and each segment is an independent error-feedback loop.
//
//   pcm_dither_encode_kernel<BITS, K>   one thread per (segment, channel), 32 segments per CTA; the error history is
//                                       an unrolled shift register of K doubles, the taps are kernel parameters
//                                       (constant bank).  Frames go through shared memory in tiles of 32 frames
//                                       per segment, so global loads and stores are 256 / 128 / 192 contiguous bytes
//                                       per segment instead of one sample per thread 8 KB apart.
// (included by correct.cu)
#pragma once
#include <math.h>

namespace mgb {

namespace {

constexpr int kDitherSegment = 1024;  // S: frames a segment writes
constexpr int kDitherWarmup = 32;     // W: frames it runs before them (>= every K)
constexpr int kDitherTile = 32;       // frames per segment staged at a time (the warm-up is one tile)
constexpr int kDitherSegs = 32;       // segments per CTA: lane = segment, warp = channel
constexpr int kDitherThreads = 2 * kDitherSegs;
static_assert(kDitherWarmup == kDitherTile && kDitherSegment % kDitherTile == 0, "the warm-up is one tile");
static_assert(kDitherWarmup >= MGB_MAX_DITHER_TAPS, "the warm-up covers the longest history");

// the kernel's view of mgb_dither_params: h zero-padded to the instance's K (zero taps change no bit)
struct DitherArgs {
    unsigned long long seed;
    double h[MGB_MAX_DITHER_TAPS];
};

// float64 product, sum and difference, each rounded on its own: the device never contracts them into an FMA.  (The
// emulator's host build rounds plain double arithmetic the same way: C++17 mode does not contract, and x86-64 SSE2
// has no FMA.)
#ifdef MGB_EMULATE
__device__ __forceinline__ double dmul(double a, double b) { return a * b; }
__device__ __forceinline__ double dadd(double a, double b) { return a + b; }
__device__ __forceinline__ double dsub(double a, double b) { return a - b; }
#else
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
#endif

__device__ __forceinline__ unsigned long long splitmix64_finalize(unsigned long long z) {
    z ^= z >> 30;
    z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27;
    z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    return z;
}

template <int BITS, int K>
__global__ void __launch_bounds__(kDitherThreads)
pcm_dither_encode_kernel(DitherArgs args, const float2* __restrict__ in, long long frames, unsigned char* __restrict__ out) {
    constexpr int kBytes = BITS / 8 * 2;              // bytes per output frame
    constexpr int kRowWords = kDitherTile * kBytes / 4 + 1;  // a segment's output tile in 32-bit words, padded
    constexpr double top = BITS == 16 ? 32767.0 : 8388607.0;
    __shared__ float xs[2][kDitherSegs * (kDitherTile + 1)];  // [channel][segment][frame], rows padded
    __shared__ unsigned int os[kDitherSegs * kRowWords];      // [segment][the tile's output bytes]
    const int tid = threadIdx.x;
    const int seg = tid & 31, c = tid >> 5;  // this thread's loop
    const long long s_first = (long long)blockIdx.x * kDitherSegs;

    // tile t (-1 = the warm-up) of every segment of the CTA into registers: warp w loads segments w, w + 2, ...,
    // 32 consecutive frames (256 bytes) per load; frames outside [0, frames) read as 0
    float2 pre[kDitherSegs / 2];
    auto load_tile = [&](int t) {
#pragma unroll
        for (int m = 0; m < kDitherSegs / 2; ++m) {
            const int r = (tid >> 5) + 2 * m;
            const long long f = (s_first + r) * kDitherSegment + (long long)t * kDitherTile + (tid & 31);
            pre[m] = (f >= 0 && f < frames) ? in[f] : make_float2(0.0f, 0.0f);
        }
    };
    auto stage_tile = [&]() {
#pragma unroll
        for (int m = 0; m < kDitherSegs / 2; ++m) {
            const int r = (tid >> 5) + 2 * m;
            xs[0][r * (kDitherTile + 1) + (tid & 31)] = pre[m].x;
            xs[1][r * (kDitherTile + 1) + (tid & 31)] = pre[m].y;
        }
    };

    double e[K > 0 ? K : 1];  // e[k] = e[n - 1 - k]
#pragma unroll
    for (int k = 0; k < K; ++k) e[k] = 0.0;
    // z of this thread's first warm-up frame; the counter steps by two samples per frame
    const unsigned long long golden = 0x9E3779B97F4A7C15ull;
    const long long n_first = (s_first + seg) * kDitherSegment - kDitherWarmup;
    unsigned long long zc = args.seed + (unsigned long long)(2 * n_first + c + 1) * golden;

    load_tile(-1);
    for (int t = -1; t < kDitherSegment / kDitherTile; ++t) {
        __syncthreads();  // the previous tile's xs reads and os reads are done
        stage_tile();
        if (t + 1 < kDitherSegment / kDitherTile) load_tile(t + 1);  // in flight while this tile is quantised
        __syncthreads();
        const float* xr = &xs[c][seg * (kDitherTile + 1)];
        unsigned char* orow = reinterpret_cast<unsigned char*>(&os[seg * kRowWords]);
#pragma unroll(K > 16 ? 8 : kDitherTile)  // (the longest history would otherwise not fit in registers)
        for (int j = 0; j < kDitherTile; ++j) {
            const float x = xr[j];
            const unsigned long long z = splitmix64_finalize(zc);
            zc += 2 * golden;
            const double d = (double)((int)(z >> 40) - (int)((z >> 16) & 0xFFFFFFull)) * (1.0 / 16777216.0);
            const double u = dmul((double)x, top);
            double fb = 0.0;
#pragma unroll
            for (int k = K - 1; k >= 0; --k) fb = dadd(fb, dmul(args.h[k], e[k]));
            const double v = dsub(u, fb);
            const double q = rint(dadd(v, d));
            const bool finite = isfinite(q);
            const double err = finite ? dsub(q, v) : 0.0;
#pragma unroll
            for (int k = K - 1; k > 0; --k) e[k] = e[k - 1];
            if (K > 0) e[0] = err;
            const int y = finite ? (int)fmin(top, fmax(-top - 1.0, q)) : quantize(x, top);
            if (BITS == 16) {
                reinterpret_cast<short*>(orow)[2 * j + c] = (short)y;
            } else {
                unsigned char* p = orow + 6 * j + 3 * c;
                p[0] = (unsigned char)(y & 0xff);
                p[1] = (unsigned char)((y >> 8) & 0xff);
                p[2] = (unsigned char)((y >> 16) & 0xff);
            }
        }
        if (t < 0) {
            // segment 0 has no frames before its own: its history starts at zero at frame 0
            if (s_first + seg == 0) {
#pragma unroll
                for (int k = 0; k < K; ++k) e[k] = 0.0;
            }
            continue;  // the warm-up writes nothing
        }
        __syncthreads();
        // the tile's output, warp by warp along each segment's contiguous bytes
        constexpr int kWords = kDitherTile * kBytes / 4;
        for (int i = tid; i < kDitherSegs * kWords; i += kDitherThreads) {
            const int r = i / kWords, w = i - r * kWords;
            const long long f0 = (s_first + r) * kDitherSegment + (long long)t * kDitherTile;  // first frame of the row
            const long long valid = (frames - f0) * kBytes;  // bytes of the row inside the track
            if (valid <= 4LL * w) continue;
            const unsigned int word = os[r * kRowWords + w];
            unsigned char* dst = out + f0 * kBytes + 4LL * w;
            if (valid >= 4LL * w + 4) {
                *reinterpret_cast<unsigned int*>(dst) = word;
            } else {
                for (int b = 0; b < valid - 4LL * w; ++b) dst[b] = (unsigned char)(word >> (8 * b));
            }
        }
    }
}

}  // namespace

}  // namespace mgb
