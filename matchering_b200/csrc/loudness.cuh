// Loudness meter (ITU-R BS.1770-4, EBU Tech 3342): integrated loudness, loudness range, momentary and short-term
// maxima, sample and true peak of a stereo float32 track (include/matchering_b200.h, mgb_loudness).
//
// Included once, at the end of limiter.cu: the K-weighting sections are order-2 recursive filters like the
// limiter's hold and release sections, so they run on the same float64 blocked scans and look-back words
// (limiter_scan.cuh) over the same chunks of kLimiterCore frames, with the tables fill_section_tables builds.  Only the
// look-back's walk is the meter's own (lookback_fixed): it combines the predecessors in a fixed way, so that two runs
// give the same bits.
//
//   loudness_kernel<OS>     one CTA per chunk, one read of every frame (8 B/frame plus a 6-frame halo per side):
//                           shelf then high-pass per channel, the chunk's share of every sub-block energy it
//                           touches, its sample peak and the true peak of the interpolated centres it owns
//   loudness_fold_kernel    sub-block energies e_b from the chunk shares, in chunk order
//   loudness_windows_kernel momentary (4 sub-blocks) and short-term (30) mean squares as direct window sums
//   loudness_finish_kernel  one CTA: gates, the two loudness-range percentiles, peak folds, the result
// No float atomics anywhere: every sum has a fixed order, so the result is deterministic.
#pragma once
#include "limiter_scan.cuh"
#include "select.cuh"

namespace mgb {

namespace {

constexpr int kMeterSlots = 8;  // sub-blocks one chunk can touch: (kLimiterCore - 1) / 800 + 2 = 7 at 8 kHz
constexpr int kMeterHalo = 6;   // the interpolator reads 6 frames on each side of a centre
constexpr int kMeterSpan = LC + 2 * kMeterHalo;
constexpr int kMeterFinishThreads = 1024;
constexpr int kMeterWords = 8;  // look-back words per chunk and channel: shelf aggregate[2], inclusive[2], high-pass the same

struct MeterTables {
    SectionTab<2> shelf, highpass;
};

// Workspace of one meter call (all 256-byte aligned).  Only the look-back words need clearing before a launch:
// every other region is written in full before it is read.
struct MeterWorkspace {
    LookbackWord* words;  // [2 channels][chunks][kMeterWords] (lookback_fixed)
    double* part;         // [chunks][kMeterSlots]: the chunk's share of sub-blocks first_sub .. first_sub + 7
    double* peak;         // [chunks][4]: sample peak L, R, true peak L, R
    double* energy;       // [nb]
    double* mom;          // [nm] momentary mean squares
    double* st;           // [ns] short-term mean squares, then the loudness-range candidates
    int64_t chunks, nb, nm, ns, words_bytes, total;
};

// (align256: limiter_wide.cuh)
MeterWorkspace carve_meter(const mgb_loudness_params& lp, int64_t frames, void* base) {
    MeterWorkspace w;
    w.chunks = (frames + LC - 1) / LC;
    w.nb = frames / lp.block;
    w.nm = w.nb >= 4 ? w.nb - 3 : 0;
    w.ns = w.nb >= 30 ? w.nb - 29 : 0;
    unsigned char* p = (unsigned char*)base;
    int64_t off = 0;
    auto take = [&](int64_t bytes) {
        unsigned char* r = p ? p + off : nullptr;
        off += align256(bytes);
        return r;
    };
    w.words_bytes = align256(2 * w.chunks * kMeterWords * (int64_t)sizeof(LookbackWord));
    w.words = (LookbackWord*)take(w.words_bytes);
    w.part = (double*)take(w.chunks * kMeterSlots * 8);
    w.peak = (double*)take(w.chunks * 4 * 8);
    w.energy = (double*)take(w.nb * 8);
    w.mom = (double*)take(w.nm * 8);
    w.st = (double*)take(w.ns * 8);
    w.total = off;
    return w;
}

// The meter workspaces of an album's tracks carved from one block (mgb_album_loudness, the album loudness search):
// every track's look-back words in one range (one clear), its own chunk shares and energies, and its momentary,
// short-term and per-chunk peak arrays as consecutive slices of three pooled arrays.  A finish or integrated kernel
// run once over a pooled array then meters the union of the tracks' windows, and no window straddles two tracks.
// `all` describes the pooled arrays (chunks, nm and ns the sums; words and words_bytes the whole range); st_copy is
// room for a copy of the pooled short-term array, which the finish kernel rewrites in place.
struct AlbumMeter {
    MeterWorkspace all;
    double* st_copy;
    int64_t total;
};

AlbumMeter carve_album_meter(const mgb_loudness_params& lp, int tracks, const int64_t* frames, void* base,
                             MeterWorkspace* per_track) {
    AlbumMeter a;
    MeterWorkspace& all = a.all;
    all.chunks = all.nb = all.nm = all.ns = 0;
    int64_t words_bytes = 0;
    for (int t = 0; t < tracks; ++t) {
        const MeterWorkspace c = carve_meter(lp, frames[t], nullptr);
        per_track[t] = c;
        words_bytes += c.words_bytes;
        all.chunks += c.chunks;
        all.nb += c.nb;
        all.nm += c.nm;
        all.ns += c.ns;
    }
    unsigned char* p = (unsigned char*)base;
    int64_t off = 0;
    auto take = [&](int64_t bytes) {
        unsigned char* r = p ? p + off : nullptr;
        off += align256(bytes);
        return r;
    };
    all.words_bytes = words_bytes;
    all.words = (LookbackWord*)take(words_bytes);
    all.part = nullptr;
    all.energy = nullptr;
    all.peak = (double*)take(all.chunks * 4 * 8);
    all.mom = (double*)take(all.nm * 8);
    all.st = (double*)take(all.ns * 8);
    a.st_copy = (double*)take(all.ns * 8);
    int64_t words = 0, chunks = 0, nm = 0, ns = 0;
    for (int t = 0; t < tracks; ++t) {
        MeterWorkspace& w = per_track[t];
        w.part = (double*)take(w.chunks * kMeterSlots * 8);
        w.energy = (double*)take(w.nb * 8);
        if (p) {
            w.words = (LookbackWord*)((unsigned char*)all.words + words);
            w.peak = all.peak + chunks * 4;
            w.mom = all.mom + nm;
            w.st = all.st + ns;
        }
        words += w.words_bytes;
        chunks += w.chunks;
        nm += w.nm;
        ns += w.ns;
    }
    all.total = a.total = off;
    return a;
}

__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide maximum of non-negative doubles, valid in every thread (the shape of block_sum).
__device__ __forceinline__ double block_max_d(double v, double* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
    v = warp_max_d(v);
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    if (warp == 0) {
        double t = lane < nwarps ? scratch[lane] : 0.0;
        t = warp_max_d(t);
        if (lane == 0) scratch[0] = t;
    }
    __syncthreads();
    return scratch[0];
}

// One order-2 section over the thread's CORE_EPT samples from zero state: y = lfilter(b, a, u) with u[-1], u[-2]
// the section's inputs just before the thread's first sample.
__device__ __forceinline__ void section_local(const double* b, const double* a, const double* u, double um1, double um2,
                                              double* y) {
#pragma unroll
    for (int e = 0; e < CORE_EPT; ++e) {
        double acc = b[0] * u[e] + b[1] * (e >= 1 ? u[e - 1] : um1) + b[2] * (e >= 2 ? u[e - 2] : (e == 1 ? um1 : um2));
        if (e >= 1) acc -= a[1] * y[e - 1];
        if (e >= 2) acc -= a[2] * y[e - 2];
        y[e] = acc;
    }
}

// Carry into chunk `chunk` in a FIXED combination, so that the meter repeats bit for bit: the limiter's `lookback`
// stops at whichever predecessor happens to have published its inclusive state, and sums of the same carry taken
// over different predecessors differ in the last bits.  Here chunks form groups of 32; the carry into chunk g + p
// (g = its group's first chunk) is always C^(p LC) I(g-1) + sum over j = g .. g+p-1 of C^((g+p-1-j) LC) A(j): the
// inclusive state of the previous group's last chunk and the aggregates of the chunks between, lane l weighing
// chunk - 1 - l, one warp reduction in a fixed order.  Only a group's last chunk publishes its inclusive state, in
// words of its own (an aggregate is never overwritten).  `words` = this section's 4 words of chunk 0: aggregate[2],
// inclusive[2], every kMeterWords words per chunk.  Called by all 32 lanes of one warp.
__device__ __forceinline__ StVec<2> lookback_fixed(const LookbackWord* words, int chunk, const SectionTab<2>* t) {
    const int lane = threadIdx.x & 31;
    const int g = chunk & ~31, j = chunk - 1 - lane;
    StVec<2> val = st_zero<2>();
    if (j >= g - 1 && j >= 0) {
        const LookbackWord* w = words + (long long)j * kMeterWords + (j >= g ? 0 : 2);
        const int want = j >= g ? 1 : 2;
        for (;;) {
            const bool ok = poll(w, &val.v[0]) == want && poll(w + 1, &val.v[1]) == want;
            if (ok) break;
            __nanosleep(20);
        }
    }
    StVec<2> acc = st_mul<2>(t->pc[lane], val);
#pragma unroll
    for (int i = 0; i < 2; ++i) acc.v[i] = warp_sum(acc.v[i]);
    return acc;
}

// The zero-carry results of one section in both channels -> final outputs: block scan, publish the chunk's aggregate,
// look-back (warp c for channel c), add the carries, publish the inclusive state at a group's end.  Returns each
// channel's state just before the thread's first sample.  `words` = this section's words of chunk 0 in channel 0's
// array; channel 1's array follows `chan_stride` words later.
__device__ __forceinline__ void section_finish(double (*y)[CORE_EPT], const SectionTab<2>* tab, LookbackWord* words,
                                               long long chan_stride, int chunk, double* scratch0, double* scratch1,
                                               double* bcast, StVec<2>* prev) {
    const int tid = threadIdx.x;
    StVec<2> carry[2];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        StVec<2> end;
        end.v[0] = y[c][CORE_EPT - 1];
        end.v[1] = y[c][CORE_EPT - 2];
        carry[c] = section_scan<2>(end, tab, c == 0 ? scratch0 : scratch1);
        if (tid == NT - 1) {
            st_addmul<2>(end, tab->ql[1], carry[c]);
            publish_state<2>(words + c * chan_stride + (long long)chunk * kMeterWords, end, 1);
        }
    }
    if (tid < 64) {
        const int c = tid >> 5;
        const StVec<2> cin = lookback_fixed(words + c * chan_stride, chunk, tab);
        if ((tid & 31) == 0) {
            bcast[2 * c] = cin.v[0];
            bcast[2 * c + 1] = cin.v[1];
        }
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        StVec<2> cin;
        cin.v[0] = bcast[2 * c];
        cin.v[1] = bcast[2 * c + 1];
        prev[c] = section_lead<2>(tab, cin);
        prev[c].v[0] += carry[c].v[0];
        prev[c].v[1] += carry[c].v[1];
#pragma unroll
        for (int e = 0; e < CORE_EPT; ++e) y[c][e] += tab->pe[e][0] * prev[c].v[0] + tab->pe[e][1] * prev[c].v[1];
        if (tid == NT - 1 && (chunk & 31) == 31) {
            StVec<2> end;
            end.v[0] = y[c][CORE_EPT - 1];
            end.v[1] = y[c][CORE_EPT - 2];
            publish_state<2>(words + c * chan_stride + (long long)chunk * kMeterWords + 2, end, 2);
        }
    }
}

// |interpolated x| at output (n + 6) * OS + phase of upfirdn(h, x, up=OS), maximised over the phases: the taps
// h[(6 - t) OS + phase] weigh x[n + t], t = -6 .. 6.  w[i] = x[n - 6 + i].
template <int OS>
__device__ __forceinline__ double tp_centre(const mgb_loudness_params& lp, const double* w) {
    double m = 0.0;
#pragma unroll
    for (int ph = 0; ph < OS; ++ph) {
        double acc = 0.0;
#pragma unroll
        for (int t = -6; t <= 6; ++t) {
            const int k = (6 - t) * OS + ph;
            if (k <= 12 * OS) acc += w[t + 6] * lp.tp_taps[k];
        }
        m = fmax(m, fabs(acc));
    }
    return m;
}

// GATED (every kernel of the meter, loudness_target.cuh): the grid returns at once while *skip is set -- a pass of a
// loudness-target search that the search did not need
template <int OS, bool GATED = false>
__global__ void __launch_bounds__(NT) loudness_kernel(mgb_loudness_params lp, const float2* __restrict__ x, long long frames,
                                                      LookbackWord* __restrict__ words, double* __restrict__ part,
                                                      double* __restrict__ peak, const MeterTables* __restrict__ tabs,
                                                      const int* __restrict__ skip) {
    __shared__ float2 xs[kMeterSpan];  // frames s0 - 6 .. s0 + LC + 5, zero outside the signal
    __shared__ double scratch[4][32 * 2];
    __shared__ double bcast[4];
    __shared__ double wsum[NT / 32][2];
    __shared__ int wsub[NT / 32];
    __shared__ double wmax[NT / 32][4];
    if constexpr (GATED) {
        if (*skip) return;
    }
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int chunk = blockIdx.x;  // (the look-back waits on lower chunks only: blocks start in index order)
    const long long s0 = (long long)chunk * LC;
    const long long chan_stride = (long long)gridDim.x * kMeterWords;
    for (int i = tid; i < kMeterSpan; i += NT) {
        const long long n = s0 - kMeterHalo + i;
        xs[i] = (n >= 0 && n < frames) ? __ldg(x + n) : make_float2(0.0f, 0.0f);
    }
    __syncthreads();
    const int base = tid * CORE_EPT;  // the thread's first core frame, at xs[base + 6]
    const long long n0 = s0 + base;

    // ---- shelf, zero-state per thread
    double y[2][CORE_EPT];
    {
        double u[2][CORE_EPT];
#pragma unroll
        for (int e = 0; e < CORE_EPT; ++e) {
            const float2 v = xs[base + kMeterHalo + e];
            u[0][e] = (double)v.x;
            u[1][e] = (double)v.y;
        }
        const float2 m1 = xs[base + kMeterHalo - 1], m2 = xs[base + kMeterHalo - 2];
        section_local(lp.shelf_b, lp.shelf_a, u[0], (double)m1.x, (double)m2.x, y[0]);
        section_local(lp.shelf_b, lp.shelf_a, u[1], (double)m1.y, (double)m2.y, y[1]);
    }

    // ---- peaks, while the predecessors publish: the thread's centres are its core frames; chunk 0 also owns
    // the centres -6 .. -1 and the last chunk frames .. frames + 5 (upfirdn's full output)
    double pk[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        double w[CORE_EPT + 2 * kMeterHalo];  // frames n0 - 6 .. n0 + CORE_EPT + 5
#pragma unroll
        for (int i = 0; i < CORE_EPT + 2 * kMeterHalo; ++i) {
            const float2 v = xs[base + i];
            w[i] = (double)(c == 0 ? v.x : v.y);
        }
#pragma unroll
        for (int e = 0; e < CORE_EPT; ++e) {
            if (n0 + e < frames) {
                pk[c] = fmax(pk[c], fabs(w[e + kMeterHalo]));
                pk[2 + c] = fmax(pk[2 + c], tp_centre<OS>(lp, &w[e]));
            }
        }
    }
    // the centres outside the signal: six from c0 on, their frames read from xs (every frame of the signal they
    // reach is staged; the rest are zeros)
    auto edge = [&](long long c0) {
        for (int q = 0; q < kMeterHalo; ++q) {
            double v[2][2 * kMeterHalo + 1];
            for (int t = 0; t <= 2 * kMeterHalo; ++t) {
                const long long i = c0 + q + t - s0;  // xs index of frame c0 + q - 6 + t
                const float2 f = (i >= 0 && i < kMeterSpan) ? xs[i] : make_float2(0.0f, 0.0f);
                v[0][t] = (double)f.x;
                v[1][t] = (double)f.y;
            }
            pk[2] = fmax(pk[2], tp_centre<OS>(lp, v[0]));
            pk[3] = fmax(pk[3], tp_centre<OS>(lp, v[1]));
        }
    };
    if (chunk == 0 && tid == 0) edge(-kMeterHalo);
    if (chunk == (int)gridDim.x - 1 && tid == NT - 1) edge(frames);

    // ---- shelf carries, then the high-pass on the shelf's output
    StVec<2> prev[2];
    section_finish(y, &tabs->shelf, words, chan_stride, chunk, scratch[0], scratch[1], bcast, prev);
    double z[2][CORE_EPT];
    section_local(lp.highpass_b, lp.highpass_a, y[0], prev[0].v[0], prev[0].v[1], z[0]);
    section_local(lp.highpass_b, lp.highpass_a, y[1], prev[1].v[0], prev[1].v[1], z[1]);
    __syncthreads();  // bcast is written again below
    section_finish(z, &tabs->highpass, words + 4, chan_stride, chunk, scratch[2], scratch[3], bcast, prev);

    // ---- the chunk's share of each sub-block's energy.  A warp spans 32 * CORE_EPT = 288 frames, less than a
    // sub-block (>= 800 frames), so its frames fall into the sub-blocks jw and jw + 1.
    const long long B = lp.block;
    const long long first_sub = s0 / B;
    const long long jw = (s0 + (long long)warp * 32 * CORE_EPT) / B;
    double acc0 = 0.0, acc1 = 0.0;
#pragma unroll
    for (int e = 0; e < CORE_EPT; ++e) {
        const long long n = n0 + e;
        if (n < frames) {
            const double en = z[0][e] * z[0][e] + z[1][e] * z[1][e];
            if (n / B == jw) acc0 += en;
            else acc1 += en;
        }
    }
    acc0 = warp_sum(acc0);
    acc1 = warp_sum(acc1);
#pragma unroll
    for (int k = 0; k < 4; ++k) pk[k] = warp_max_d(pk[k]);
    if (lane == 0) {
        wsum[warp][0] = acc0;
        wsum[warp][1] = acc1;
        wsub[warp] = (int)(jw - first_sub);
#pragma unroll
        for (int k = 0; k < 4; ++k) wmax[warp][k] = pk[k];
    }
    __syncthreads();
    if (tid < kMeterSlots) {
        double s = 0.0;
        for (int w = 0; w < NT / 32; ++w) {
            if (wsub[w] == tid) s += wsum[w][0];
            if (wsub[w] + 1 == tid) s += wsum[w][1];
        }
        part[(long long)chunk * kMeterSlots + tid] = s;
    } else if (tid >= 32 && tid < 36) {
        const int k = tid - 32;
        double m = 0.0;
        for (int w = 0; w < NT / 32; ++w) m = fmax(m, wmax[w][k]);
        peak[(long long)chunk * 4 + k] = m;
    }
}

// e_b = the shares of the chunks that touch sub-block b, in chunk order
template <bool GATED = false>
__global__ void loudness_fold_kernel(long long block, long long nb, const double* __restrict__ part, double* __restrict__ energy,
                                     const int* __restrict__ skip) {
    if constexpr (GATED) {
        if (*skip) return;
    }
    const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const long long lo = b * block, c0 = lo / LC, c1 = (lo + block - 1) / LC;
    double e = 0.0;
    for (long long c = c0; c <= c1; ++c) e += part[c * kMeterSlots + (b - c * LC / block)];
    energy[b] = e;
}

// (GATED: momentary windows only -- a search's pass meters integrated loudness alone)
template <bool GATED = false>
__global__ void loudness_windows_kernel(long long block, long long nb, const double* __restrict__ energy,
                                        double* __restrict__ mom, double* __restrict__ st, const int* __restrict__ skip) {
    if constexpr (GATED) {
        if (*skip) return;
    }
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j + 4 <= nb) {
        double s = 0.0;
        for (int i = 0; i < 4; ++i) s += energy[j + i];
        mom[j] = s / (4.0 * (double)block);
    }
    if (!GATED && j + 30 <= nb) {
        double s = 0.0;
        for (int i = 0; i < 30; ++i) s += energy[j + i];
        st[j] = s / (30.0 * (double)block);
    }
}

__device__ __forceinline__ double lufs(double mean_square) { return -0.691 + 10.0 * log10(mean_square); }

__global__ void __launch_bounds__(kMeterFinishThreads) loudness_finish_kernel(long long chunks, long long nm, long long ns,
                                                                              const double* __restrict__ peak,
                                                                              const double* __restrict__ mom, double* st,
                                                                              mgb_loudness_result* out) {
    __shared__ double red[32];
    const int tid = threadIdx.x, nt = blockDim.x;
    const double neg_inf = -INFINITY;

    // integrated loudness: absolute gate at -70 LUFS, relative gate 10 LU below the mean of what passed (repeated by
    // loudness_integrated_kernel below: change both together; the loudness-target tests compare the two to the bit)
    double sa = 0.0, ca = 0.0, mmax = 0.0;
    for (long long j = tid; j < nm; j += nt) {
        const double z = mom[j];
        if (lufs(z) > -70.0) {
            sa += z;
            ca += 1.0;
        }
        mmax = fmax(mmax, z);
    }
    sa = block_sum(sa, red);
    ca = block_sum(ca, red);
    mmax = block_max_d(mmax, red);
    double integrated = neg_inf;
    if (ca > 0.0) {
        const double gate = lufs(sa / ca) - 10.0;
        double sr = 0.0, cr = 0.0;
        for (long long j = tid; j < nm; j += nt) {
            const double z = mom[j], l = lufs(z);
            if (l > -70.0 && l > gate) {
                sr += z;
                cr += 1.0;
            }
        }
        sr = block_sum(sr, red);
        cr = block_sum(cr, red);
        if (cr > 0.0) integrated = lufs(sr / cr);
    }

    // loudness range: absolute gate, relative gate 20 LU below, then the 10th and 95th percentiles of what is
    // left.  Gated-out windows become 0 in place, below every survivor (> -70 LUFS), so the percentiles are
    // ranks (ns - n) + p (n - 1) of all ns values.
    double ss = 0.0, cs = 0.0, smax = 0.0;
    for (long long k = tid; k < ns; k += nt) {
        const double s = st[k];
        if (lufs(s) > -70.0) {
            ss += s;
            cs += 1.0;
        }
        smax = fmax(smax, s);
    }
    ss = block_sum(ss, red);
    cs = block_sum(cs, red);
    smax = block_max_d(smax, red);
    double lra = 0.0;
    if (cs > 0.0) {
        const double gate = lufs(ss / cs) - 20.0;
        double n = 0.0;
        for (long long k = tid; k < ns; k += nt) {
            const double l = lufs(st[k]);
            if (l > -70.0 && l > gate) n += 1.0;
            else st[k] = 0.0;
        }
        n = block_sum(n, red);  // (its barriers also publish the zeros)
        if (n > 0.0) {
            const long long zeros = ns - (long long)n;
            const long long lo = zeros + (long long)floor(0.10 * (n - 1.0) + 0.5);
            const long long hi = zeros + (long long)floor(0.95 * (n - 1.0) + 0.5);
            const double vlo = block_kth_smallest(st, (int)ns, (int)lo);
            const double vhi = block_kth_smallest(st, (int)ns, (int)hi);
            lra = lufs(vhi) - lufs(vlo);
        }
    }

    double pk[4] = {0.0, 0.0, 0.0, 0.0};
    for (long long c = tid; c < chunks; c += nt)
        for (int k = 0; k < 4; ++k) pk[k] = fmax(pk[k], peak[c * 4 + k]);
    for (int k = 0; k < 4; ++k) pk[k] = block_max_d(pk[k], red);

    if (tid == 0) {
        out->integrated = integrated;
        out->loudness_range = lra;
        out->momentary_max = nm > 0 ? lufs(mmax) : neg_inf;
        out->short_term_max = ns > 0 ? lufs(smax) : neg_inf;
        out->sample_peak[0] = pk[0];
        out->sample_peak[1] = pk[1];
        out->true_peak[0] = pk[2];
        out->true_peak[1] = pk[3];
        out->momentary_count = nm;
        out->short_term_count = ns;
    }
}

// loudness_finish_kernel's integrated loudness alone, into *integrated_out (a loudness-target search's pass meter, gated
// like the GATED kernels above).  Its own kernel rather than a flag on, or a helper shared with, the finish kernel: a
// template flag there reordered two of the finish kernel's instructions, and the finish kernel stays unchanged to the
// instruction.  The gate below is the finish kernel's, in the same order (change both together).
__global__ void __launch_bounds__(kMeterFinishThreads) loudness_integrated_kernel(long long nm, const double* __restrict__ mom,
                                                                                  const int* __restrict__ skip,
                                                                                  double* __restrict__ integrated_out) {
    __shared__ double red[32];
    if (*skip) return;
    const int tid = threadIdx.x, nt = blockDim.x;
    double sa = 0.0, ca = 0.0;
    for (long long j = tid; j < nm; j += nt) {
        const double z = mom[j];
        if (lufs(z) > -70.0) {
            sa += z;
            ca += 1.0;
        }
    }
    sa = block_sum(sa, red);
    ca = block_sum(ca, red);
    double integrated = -INFINITY;
    if (ca > 0.0) {
        const double gate = lufs(sa / ca) - 10.0;
        double sr = 0.0, cr = 0.0;
        for (long long j = tid; j < nm; j += nt) {
            const double z = mom[j], l = lufs(z);
            if (l > -70.0 && l > gate) {
                sr += z;
                cr += 1.0;
            }
        }
        sr = block_sum(sr, red);
        cr = block_sum(cr, red);
        if (cr > 0.0) integrated = lufs(sr / cr);
    }
    if (tid == 0) *integrated_out = integrated;
}

int loudness_validate(const mgb_loudness_params* lp) {
    MGB_REQUIRE(lp != nullptr, MGB_ERR_INVALID, "loudness: params is NULL");
    MGB_REQUIRE(lp->sample_rate >= 8000 && lp->sample_rate <= 384000, MGB_ERR_INVALID,
                "loudness: sample rate %d outside [8000, 384000]", lp->sample_rate);
    const int os = lp->sample_rate < 96000 ? 4 : (lp->sample_rate < 192000 ? 2 : 1);
    MGB_REQUIRE(lp->block == (lp->sample_rate + 5) / 10 && lp->oversample == os && lp->taps == 12 * os + 1, MGB_ERR_INVALID,
                "loudness: block %d, oversample %d, taps %d do not follow from the rate %d", lp->block, lp->oversample,
                lp->taps, lp->sample_rate);
    return MGB_OK;
}

// The meter's kernels up to the finish for one track (its look-back words cleared by the caller)
int launch_meter_windows(const mgb_loudness_params& lp, const float2* x, int64_t frames, const MeterWorkspace& w,
                         cudaStream_t st) {
    const MeterTables* tabs = (const MeterTables*)lp.d_tables;
    const dim3 grid((unsigned)w.chunks);
    const int* no_skip = nullptr;
    if (lp.oversample == 4)
        MGB_TRY(launch("loudness_kernel", loudness_kernel<4>, grid, dim3(NT), 0, st, lp, x, (long long)frames, w.words,
                       w.part, w.peak, tabs, no_skip));
    else if (lp.oversample == 2)
        MGB_TRY(launch("loudness_kernel", loudness_kernel<2>, grid, dim3(NT), 0, st, lp, x, (long long)frames, w.words,
                       w.part, w.peak, tabs, no_skip));
    else
        MGB_TRY(launch("loudness_kernel", loudness_kernel<1>, grid, dim3(NT), 0, st, lp, x, (long long)frames, w.words,
                       w.part, w.peak, tabs, no_skip));
    const long long B = lp.block;
    MGB_TRY(launch("loudness_fold_kernel", loudness_fold_kernel<>, dim3((unsigned)((w.nb + 255) / 256)), dim3(256), 0, st, B,
                   (long long)w.nb, (const double*)w.part, w.energy, no_skip));
    return launch("loudness_windows_kernel", loudness_windows_kernel<>, dim3((unsigned)((w.nm + 255) / 256)), dim3(256), 0,
                  st, B, (long long)w.nb, (const double*)w.energy, w.mom, w.st, no_skip);
}

int launch_meter_finish(const MeterWorkspace& w, double* st_values, mgb_loudness_result* out, cudaStream_t st) {
    return launch("loudness_finish_kernel", loudness_finish_kernel, dim3(1), dim3(kMeterFinishThreads), 0, st,
                  (long long)w.chunks, (long long)w.nm, (long long)w.ns, (const double*)w.peak, (const double*)w.mom,
                  st_values, out);
}

}  // namespace

}  // namespace mgb

extern "C" {

int64_t mgb_loudness_tables_bytes(void) { return mgb::align256((int64_t)sizeof(mgb::MeterTables)); }

int mgb_loudness_fill_tables(const mgb_loudness_params* params, void* d_tables, void* stream) {
    using namespace mgb;
    MGB_TRY(loudness_validate(params));
    MGB_REQUIRE(d_tables != nullptr && ((uintptr_t)d_tables & 15) == 0, MGB_ERR_INVALID, "loudness: tables NULL or misaligned");
    MeterTables t;
    fill_section_tables(params->shelf_a, &t.shelf);
    fill_section_tables(params->highpass_a, &t.highpass);
#ifdef MGB_EMULATE
    (void)stream;
    memcpy(d_tables, &t, sizeof(t));
#else
    // (from pageable memory: staged before the call returns, so `t` may go out of scope)
    if (cudaMemcpyAsync(d_tables, &t, sizeof(t), cudaMemcpyHostToDevice, (cudaStream_t)stream) != cudaSuccess)
        return cuda_status("loudness tables");
#endif
    return MGB_OK;
}

int64_t mgb_loudness_workspace_bytes(const mgb_loudness_params* params, int64_t frames) {
    if (mgb::loudness_validate(params) != MGB_OK || frames <= 0) return -1;
    return mgb::carve_meter(*params, frames, nullptr).total;
}

int mgb_loudness(const mgb_loudness_params* params, const float* d_lr, int64_t frames, void* d_workspace,
                 int64_t workspace_bytes, mgb_loudness_result* d_result, void* stream) {
    using namespace mgb;
    MGB_TRY(loudness_validate(params));
    MGB_REQUIRE(frames > 0, MGB_ERR_INVALID, "loudness: no frames");
    MGB_REQUIRE(frames <= (int64_t)INT32_MAX * LC, MGB_ERR_INVALID, "loudness: too many frames");
    auto aligned = [](const void* p) { return p != nullptr && ((uintptr_t)p & 15) == 0; };
    MGB_REQUIRE(aligned(d_lr) && aligned(d_workspace) && aligned(d_result) && aligned(params->d_tables), MGB_ERR_INVALID,
                "loudness: NULL or misaligned pointer (16 bytes needed)");
    const MeterWorkspace w = carve_meter(*params, frames, d_workspace);
    MGB_REQUIRE(workspace_bytes >= w.total, MGB_ERR_INVALID, "loudness: workspace of %lld bytes, need %lld",
                (long long)workspace_bytes, (long long)w.total);
    cudaStream_t st = (cudaStream_t)stream;
#ifdef MGB_EMULATE
    memset(w.words, 0, w.words_bytes);
#else
    if (cudaMemsetAsync(w.words, 0, w.words_bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
    MGB_TRY(launch_meter_windows(*params, (const float2*)d_lr, frames, w, st));
    return launch_meter_finish(w, w.st, d_result, st);
}

int64_t mgb_album_loudness_workspace_bytes(const mgb_loudness_params* params, int32_t tracks, const int64_t* frames) {
    if (mgb::loudness_validate(params) != MGB_OK || tracks < 1 || tracks > MGB_MAX_ALBUM_TRACKS || frames == nullptr) return -1;
    for (int t = 0; t < tracks; ++t)
        if (frames[t] <= 0) return -1;
    mgb::MeterWorkspace per_track[MGB_MAX_ALBUM_TRACKS];
    return mgb::carve_album_meter(*params, tracks, frames, nullptr, per_track).total;
}

int mgb_album_loudness(const mgb_loudness_params* params, int32_t tracks, const float* const* d_lr, const int64_t* frames,
                       void* d_workspace, int64_t workspace_bytes, mgb_loudness_result* d_album_result,
                       mgb_loudness_result* d_track_results, void* stream) {
    using namespace mgb;
    MGB_TRY(loudness_validate(params));
    MGB_REQUIRE(tracks >= 1 && tracks <= MGB_MAX_ALBUM_TRACKS, MGB_ERR_INVALID, "album loudness: %d tracks (1 .. %d)",
                (int)tracks, MGB_MAX_ALBUM_TRACKS);
    MGB_REQUIRE(d_lr != nullptr && frames != nullptr, MGB_ERR_INVALID, "album loudness: the track arrays are NULL");
    auto aligned = [](const void* p) { return p != nullptr && ((uintptr_t)p & 15) == 0; };
    for (int t = 0; t < tracks; ++t) {
        MGB_REQUIRE(frames[t] > 0, MGB_ERR_INVALID, "album loudness: track %d has no frames", t);
        MGB_REQUIRE(frames[t] <= (int64_t)INT32_MAX * LC, MGB_ERR_INVALID, "album loudness: track %d has too many frames", t);
        MGB_REQUIRE(aligned(d_lr[t]), MGB_ERR_INVALID, "album loudness: track %d: NULL or misaligned samples", t);
    }
    MGB_REQUIRE(aligned(d_workspace) && aligned(d_album_result) && aligned(params->d_tables) &&
                    (d_track_results == nullptr || aligned(d_track_results)),
                MGB_ERR_INVALID, "album loudness: NULL or misaligned pointer (16 bytes needed)");
    MeterWorkspace w[MGB_MAX_ALBUM_TRACKS];
    const AlbumMeter a = carve_album_meter(*params, tracks, frames, d_workspace, w);
    MGB_REQUIRE(workspace_bytes >= a.total, MGB_ERR_WORKSPACE, "album loudness: workspace of %lld bytes, need %lld",
                (long long)workspace_bytes, (long long)a.total);
    MGB_REQUIRE(a.all.ns <= INT32_MAX, MGB_ERR_INVALID, "album loudness: too many short-term windows");
    cudaStream_t st = (cudaStream_t)stream;
#ifdef MGB_EMULATE
    memset(a.all.words, 0, a.all.words_bytes);
#else
    if (cudaMemsetAsync(a.all.words, 0, a.all.words_bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
    for (int t = 0; t < tracks; ++t) MGB_TRY(launch_meter_windows(*params, (const float2*)d_lr[t], frames[t], w[t], st));
    if (d_track_results == nullptr) return launch_meter_finish(a.all, a.all.st, d_album_result, st);
    // each track's finish gates its own slice of the short-term values in place: the album's reads a copy
#ifdef MGB_EMULATE
    memcpy(a.st_copy, a.all.st, a.all.ns * 8);
#else
    if (a.all.ns > 0 && cudaMemcpyAsync(a.st_copy, a.all.st, a.all.ns * 8, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        return cuda_status("album loudness: short-term copy");
#endif
    for (int t = 0; t < tracks; ++t) MGB_TRY(launch_meter_finish(w[t], w[t].st, d_track_results + t, st));
    return launch_meter_finish(a.all, a.st_copy, d_album_result, st);
}

}  // extern "C"
