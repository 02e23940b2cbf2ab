// K4 -- overlap-save FFT convolution of the target's mid/side with the two matching FIRs.
//
// Replaces (reference file:line):
//   match_frequencies.convolve        stage_helpers/match_frequencies.py:104-119
//     = scipy.signal.fftconvolve(x, fir, "same") per channel: full linear convolution sliced at
//       (F-1)//2 = F/2-1, edges zero-padded (scipy/signal/_signaltools.py fftconvolve/_centered)
//   dsp.lr_to_ms / dsp.ms_to_lr       dsp.py:57-68   (fused into the load and the store)
//   dsp.amplify by the RMS coefficient match_levels.py:114-131 (folded into the FIR spectra)
//   the first RMS-correction step's clip + per-piece sum of squares   stages.py:151-159
//   the peak that dsp.normalize / the limiter's early-out need        dsp.py:97, hyrax.py:83
//
// Framing: the FIR has F taps with fir[0] == 0 (symmetric Hann is zero at index 0), so taps
// 1..F-1 matter and output sample n needs inputs n-F/2 .. n+F/2-2.  A frame of N = 2F inputs
// starting at n0 - F/2 therefore yields the F outputs n0 .. n0+F-1 (circular index i = F-1 ..
// 2F-2), with n0 a multiple of F: every frame start is 16-byte aligned for the TMA bulk copy.
// mid and side ride one complex transform: z = mid + i*side, Y[k] = Hm[k] M[k] + i Hs[k] S[k]
// with M, S recovered from Z[k], Z[N-k]; real part of the inverse is the mid output, imaginary
// part the side output.  The 64 KB landing buffer of the bulk copy is reused in place as the two
// FFT planes.
#include "fft.cuh"
#include "kernels.cuh"

namespace mgb {

namespace {

template <int N>
struct ConvSmem {
    static constexpr int kPlaneBytes = (int)((PackedPlanes::bytes(N) + 15) / 16 * 16);
    static constexpr int kBytes = kPlaneBytes + 16 + 32 * 8 + 32 * 8 + 64 * 4 + 32;
};

struct ConvFirst {
    const float2* raw;  // landing buffer, index 0 = sample `origin`
    int lo, hi;         // indices of the buffer that lie inside the signal: [lo, hi)
    const float2* fixup;
    int fix_index;
    __device__ __forceinline__ float2 sample(int i) const {
        float2 v = make_float2(0.0f, 0.0f);
        if (i >= lo && i < hi) {
            v = raw[i];
            if (i == fix_index) v = *fixup;
        }
        return v;
    }
};

// ---- float32 or float64 transforms -----------------------------------------------------------------
// A float32 transform's rounding noise is spread over all N bins, relative to the frame's norm.  The FIR spectrum
// scales every bin by its gain, also the bins where the target has no content, and the inverse transform spreads
// the product over the frame's outputs, before a transient as much as after it.  An output sample's error is then
// about u sqrt(log2 N) (a random walk over the passes) times max|c0 H| (the largest gain of the FIR as applied)
// times the frame's level, which max|target| bounds; on band-limited and transient material the ratio of the
// measured error to that estimate stayed below 0.9.  Broadband material has gains near 20 (the benchmark's
// 3-minute tracks: 23, an estimate of 2.6e-6, measured errors below 1e-6).  A dull or band-limited target matched to a
// bright reference has gains of 300 to 10^4 in its empty band, and the float32 result misses the 1e-5 parity
// bound by up to 10x.  Where the estimate exceeds kConvPreciseError, half that bound, the track is convolved with
// float64 transforms (convolve_precise_kernel, rounding noise 2^-53 instead of 2^-24).  The choice comes from the
// track state the design kernel leaves (both FIR peaks) and the target's peak (Workspace::target_peak, from
// spectrum_mean_kernel): every convolution kernel evaluates the same products, the float32 kernels return at once
// where it says float64, and the float64 kernel, launched after them for every track, returns at once otherwise;
// the float64 kernel records the choice in mgb_track_state::conv_precise.
constexpr double kConvPreciseError = 5e-6;
template <int N>
__device__ __forceinline__ bool conv_precise(const mgb_track_state* __restrict__ state, const float* __restrict__ target_peak) {
    constexpr int kLog2N = N == 1024 ? 10 : N == 2048 ? 11 : N == 4096 ? 12 : N == 8192 ? 13 : N == 16384 ? 14 : 15;
    static_assert((1 << kLog2N) == N, "frame length");
    // (products only, the same in every kernel: no contraction can make two kernels disagree)
    const double e = 0x1p-24 * (double)N * (double)fmaxf(state->fir_peak_mid_bits, state->fir_peak_side_bits) *
                     (double)*target_peak;
    return e * e * (double)kLog2N > kConvPreciseError * kConvPreciseError;
}

// ---- shared by both kernels: frame load + channel balance, FIR spectra on a pair, the epilogue -----
struct ConvBalance {
    float inv_g;
    bool mid_silent, side_silent, any_silent;
};

// The part of a frame's N input samples that lies inside the signal, and how the bulk copy brings it in.
struct ConvSpan {
    long long lo, hi;   // [lo, hi) absolute sample indices
    long long count;    // samples the bulk copy moves (even: 16-byte granules)
    int fix_index;      // buffer index of the odd last sample that comes through a plain load, or -1
};
template <int N>
__device__ __forceinline__ ConvSpan conv_span(long long frames, long long origin) {
    ConvSpan sp;
    sp.lo = origin < 0 ? 0 : origin;
    sp.hi = (origin + N < frames) ? origin + N : frames;  // exclusive
    // lo - origin is 0 or F/2 (multiple of 2): source and destination stay 16-byte aligned
    sp.count = sp.hi - sp.lo;
    sp.fix_index = -1;
    if (sp.count & 1) {  // odd tail: the last sample comes through a plain load
        sp.fix_index = (int)(sp.hi - 1 - origin);
        sp.count -= 1;
    }
    return sp;
}
// (one thread) start the bulk copy of the frame at `origin` into the landing buffer
template <int N>
__device__ __forceinline__ void conv_issue_frame(const float2* __restrict__ x, long long frames, long long origin, float2* raw,
                                                 TmaBarrier* bar) {
    const ConvSpan sp = conv_span<N>(frames, origin);
    tma_load_1d(raw + (sp.lo - origin), x + sp.lo, (uint32_t)(sp.count * 8), bar);
}

// Loads the frame's N input samples (clipped to the signal) into the landing buffer, hands every thread
// its 16 points z[r] = mid + i*g*side of index tid + r*THREADS.  On return every thread is past a
// barrier that follows its last read of the landing buffer.
// `prefetched_phase` >= 0: the bulk copy was issued earlier (conv_issue_frame) on a barrier that is in that
// phase, and red_u is already zero; the function only waits.
template <int N, int PTS = 16>
__device__ __forceinline__ ConvBalance conv_load_frame(const float2* __restrict__ x, long long frames, long long origin,
                                                       float2* raw, TmaBarrier* bar, unsigned* red_u, int use_tma,
                                                       cpx<float>* z, int prefetched_phase = -1) {
    constexpr int THREADS = N / PTS;
    const int tid = threadIdx.x;
    const ConvSpan span = conv_span<N>(frames, origin);
    const long long lo = span.lo, hi = span.hi;
    ConvFirst first;
    first.raw = raw;
    first.lo = (int)(lo - origin);
    first.hi = (int)(hi - origin);
    first.fixup = span.fix_index >= 0 ? x + (hi - 1) : nullptr;
    first.fix_index = span.fix_index;
    if (prefetched_phase >= 0) {
        tma_barrier_wait(bar, (uint32_t)prefetched_phase);
    } else {
        if (tid == 0) red_u[0] = red_u[1] = 0u;
        if (use_tma) {
            if (tid == 0) tma_barrier_init(bar);
            __syncthreads();
            if (tid == 0) tma_load_1d(raw + (lo - origin), x + lo, (uint32_t)(span.count * 8), bar);
            tma_barrier_wait(bar, 0);
        } else {
            first.fixup = nullptr;
            first.fix_index = -1;
            for (long long n = lo + tid; n < hi; n += THREADS) raw[n - origin] = x[n];
            __syncthreads();
        }
    }
    float max_mid = 0.0f, max_side = 0.0f;
    // each channel from L and R directly, one rounding each: (L-R)/2 is the reference's mid - R, and
    // forming it from the already rounded mid would put mid's rounding error into a quiet side
    auto take = [&](int r, float2 v) {
        z[r].x = (v.x + v.y) * 0.5f;
        z[r].y = (v.x - v.y) * 0.5f;
        max_mid = fmaxf(max_mid, fabsf(z[r].x));
        max_side = fmaxf(max_side, fabsf(z[r].y));
    };
    if (lo == origin && hi == origin + N) {  // a frame inside the signal (all but the first and the last few):
#pragma unroll                               // no bounds, no fix-up, nothing per sample but the load
        for (int r = 0; r < N / THREADS; ++r) take(r, raw[tid + r * THREADS]);
    } else {
#pragma unroll
        for (int r = 0; r < N / THREADS; ++r) take(r, first.sample(tid + r * THREADS));
    }
    block_max2(max_mid, max_side, red_u);  // its barrier also ends everybody's reads of the landing buffer
    const float g_side = balance_factor(max_mid, max_side);  // >= 1 when the side is the quiet one, < 1 otherwise
#pragma unroll
    for (int r = 0; r < N / THREADS; ++r) z[r].y *= g_side;
    ConvBalance b;
    b.inv_g = 1.0f / g_side;  // exact: a power of two
    b.mid_silent = max_mid == 0.0f;
    b.side_silent = max_side == 0.0f;
    b.any_silent = b.mid_silent || b.side_silent;
    return b;
}

// Z[k], Z[N-k] of z = mid + i*g*side  ->  Y[k], Y[N-k] of the filtered pair (k <= F indexes the FIR spectra).
__device__ __forceinline__ void conv_apply_pair(cpx<float>& zk, cpx<float>& zn, int k, const float2* __restrict__ h_mid,
                                                const float2* __restrict__ h_side, const ConvBalance& bal) {
    const float zr = zk.x, zi = zk.y, nr = zn.x, ni = zn.y;
    // M = (Z[k] + conj Z[N-k])/2 ; g S = (Z[k] - conj Z[N-k])/(2i)
    const float mr = 0.5f * (zr + nr), mi = 0.5f * (zi - ni);
    const float sr = 0.5f * (zi + ni) * bal.inv_g, si = 0.5f * (nr - zr) * bal.inv_g;
    const float2 hm = h_mid[k], hs = h_side[k];
    float pmr = hm.x * mr - hm.y * mi, pmi = hm.x * mi + hm.y * mr;
    float psr = hs.x * sr - hs.y * si, psi = hs.x * si + hs.y * sr;
    if (bal.any_silent) {  // (uniform over the CTA) a channel that is exactly silent in this frame stays exactly
        if (bal.mid_silent) pmr = pmi = 0.0f;   // silent, as in the reference
        if (bal.side_silent) psr = psi = 0.0f;
    }
    // Y[k] = Pm + i Ps ; Y[N-k] = conj(Pm) + i conj(Ps)
    zk = cpx<float>{pmr - psi, pmi + psr};
    zn = cpx<float>{pmr + psi, psr - pmi};
}

// Output side of a frame of OUT outputs: circular index F-1+o of the inverse transform is output sample n0+o.
// mid/side -> L/R (dsp.ms_to_lr), the first RMS-correction step's sum of clip(mid)^2 per piece, the peak,
// and the loud lists of the later correction steps (kernels.cuh: kLoudMid).
template <int OUT>
struct ConvEpilogue {
    float2* res;
    LoudList loud;
    int valid, boundary, count_to;
    long long pa;
    int divisions;
    bool mid_silent, side_silent, any_silent;
    bool full;  // every output of the frame exists, is counted, belongs to piece pa, no channel is silent: nothing to test per sample
    double sq_a = 0.0, sq_b = 0.0;
    float peak = 0.0f;
    __device__ __forceinline__ ConvEpilogue(float2* result, const LoudList& loud_, long long n0, long long frames,
                                            long long piece, int divisions_, const ConvBalance& bal) {
        res = result + n0;
        loud = loud_;
        if (n0 == 0 && threadIdx.x == 0) *loud.result_slot = result;  // for the correction steps' full passes
        valid = (int)((frames - n0 < OUT) ? frames - n0 : OUT);
        const long long counted = piece * divisions_;  // samples that enter the piece RMS (dsp.unfold)
        pa = n0 / piece;
        const long long brel = (pa + 1) * piece - n0;  // first output of the next piece
        boundary = (int)(brel < OUT ? brel : OUT);
        count_to = (int)((counted - n0 < 0) ? 0 : (counted - n0 < OUT ? counted - n0 : OUT));
        divisions = divisions_;
        mid_silent = bal.mid_silent;
        side_silent = bal.side_silent;
        any_silent = bal.any_silent;
        full = valid == OUT && boundary == OUT && count_to == OUT && !any_silent;
    }
    __device__ __forceinline__ void emit_full(int o, cpx<float> y) {  // emit() when `full` (which implies: no silent channel)
        const float m = y.x, sd = y.y;
        const float l = m + sd, r = m - sd;
        res[o] = make_float2(l, r);
        peak = fmaxf(peak, fmaxf(fabsf(l), fabsf(r)));
        const float cf = fminf(1.0f, fmaxf(-1.0f, m));  // dsp.clip
        sq_a += (double)cf * (double)cf;
    }
    __device__ __forceinline__ void emit(int o, cpx<float> y) {
        if (o < valid) {
            // (the inverse transform leaves rounding dust in a channel whose spectrum was exactly zero)
            const float m = mid_silent ? 0.0f : y.x, sd = side_silent ? 0.0f : y.y;
            const float l = m + sd, r = m - sd;
            res[o] = make_float2(l, r);
            peak = fmaxf(peak, fmaxf(fabsf(l), fabsf(r)));
            if (o < count_to) {
                const float cf = fminf(1.0f, fmaxf(-1.0f, m));  // dsp.clip
                const double c2 = (double)cf * (double)cf;
                if (o < boundary) sq_a += c2; else sq_b += c2;
            }
        }
    }
    // emit() from a float64 transform (convolve_precise_kernel): L and R rounded once each, from mid +- side
    __device__ __forceinline__ void emit_wide(int o, cpx<double> y) {
        if (o < valid) {
            const double md = mid_silent ? 0.0 : y.x, sd = side_silent ? 0.0 : y.y;
            const float m = (float)md, l = (float)(md + sd), r = (float)(md - sd);
            res[o] = make_float2(l, r);
            peak = fmaxf(peak, fmaxf(fabsf(l), fabsf(r)));
            if (o < count_to) {
                const float cf = fminf(1.0f, fmaxf(-1.0f, m));  // dsp.clip
                const double c2 = (double)cf * (double)cf;
                if (o < boundary) sq_a += c2; else sq_b += c2;
            }
        }
    }
    // Appends the loud ones among K outputs per thread to the loud lists: outputs(k) is the k-th output's
    // index o (< 0: none), mids(k) its transform value's real part.  Every lane of the warp calls, with
    // the same K; per warp and piece one atomicAdd reserves the room for all K.  Entries past a list's
    // capacity are dropped, but still counted: the correction steps see the overflow and do not use it.
    template <int K, typename O, typename M>
    __device__ __forceinline__ void append_loud(O outputs, M mids) {
        const unsigned lane = threadIdx.x & 31u, below = (1u << lane) - 1u;
        auto loud_in = [&](int k, bool second) {  // counted, loud, and in piece pa (second: pa + 1)
            const int o = outputs(k);
            if (o < 0 || o >= count_to || mid_silent) return false;
            return fabsf(mids(k)) >= kLoudMid && (o >= boundary) == second;
        };
        unsigned na = 0, nb = 0;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            na += __popc(__ballot_sync(0xffffffffu, loud_in(k, false)));
            if (!full) nb += __popc(__ballot_sync(0xffffffffu, loud_in(k, true)));
        }
        unsigned base_a = 0, base_b = 0;
        if (lane == 0) {
            if (na) base_a = atomicAdd(&loud.count[pa], na);
            if (nb) base_b = atomicAdd(&loud.count[pa + 1], nb);
        }
        if (na == 0 && nb == 0) return;
        base_a = __shfl_sync(0xffffffffu, base_a, 0);
        base_b = __shfl_sync(0xffffffffu, base_b, 0);
        float* row_a = loud.values + pa * loud.capacity;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const bool a = loud_in(k, false);
            const unsigned ba = __ballot_sync(0xffffffffu, a);
            const unsigned ia = base_a + __popc(ba & below);
            if (a && ia < loud.capacity) row_a[ia] = mids(k);
            base_a += __popc(ba);
            if (!full) {
                const bool b = loud_in(k, true);
                const unsigned bb = __ballot_sync(0xffffffffu, b);
                const unsigned ib = base_b + __popc(bb & below);
                if (b && ib < loud.capacity) row_a[loud.capacity + ib] = mids(k);
                base_b += __popc(bb);
            }
        }
    }
    // one barrier: every warp leaves its three partial results in shared memory, warp 0 folds them
    __device__ __forceinline__ void finish(double* red_a, double* red_b, float* red_f, double* piece_sums,
                                           mgb_track_state* state) {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
        const double wa = warp_sum(sq_a);
        const double wb = full ? 0.0 : warp_sum(sq_b);
        const float wp = warp_max(peak);
        if (lane == 0) {
            red_a[warp] = wa;
            red_b[warp] = wb;
            red_f[warp] = wp;
        }
        __syncthreads();
        if (warp == 0) {
            const double ta = warp_sum(lane < nwarps ? red_a[lane] : 0.0);
            const double tb = full ? 0.0 : warp_sum(lane < nwarps ? red_b[lane] : 0.0);
            const float pk = warp_max(lane < nwarps ? red_f[lane] : 0.0f);
            if (lane == 0) {
                if (pa < divisions && ta != 0.0) atomicAdd(&piece_sums[pa], ta);
                if (pa + 1 < divisions && tb != 0.0) atomicAdd(&piece_sums[pa + 1], tb);
                atomic_max_nonneg(&state->conv_peak_bits, pk);
            }
        }
    }
};

template <int N>
struct ConvPointers {
    PackedPlanes planes;
    float2* raw;
    TmaBarrier* bar;
    double *red_a, *red_b;
    float* red_f;
    unsigned* red_u;
    __device__ __forceinline__ explicit ConvPointers(unsigned char* smem) {
        planes = PackedPlanes{reinterpret_cast<float2*>(smem)};
        raw = reinterpret_cast<float2*>(smem);  // the landing buffer IS the frame's storage: unpadded
                                                // until the first pass has gathered it, padded after
        unsigned char* tail = smem + ConvSmem<N>::kPlaneBytes;
        tail += (16 - (reinterpret_cast<uintptr_t>(tail) & 15)) & 15;
        bar = reinterpret_cast<TmaBarrier*>(tail);
        red_a = reinterpret_cast<double*>(tail + 16);
        red_b = red_a + 32;
        red_f = reinterpret_cast<float*>(red_b + 32);
        red_u = reinterpret_cast<unsigned*>(red_f + 32);  // [2] slot of block_max2
    }
};

// ---- generic kernel: every pass through shared memory (any radix schedule) -------------------------
template <int F, bool CHAIN>
__global__ void __launch_bounds__(F / 8, (F <= 4096 ? 2 : 1))
convolve_kernel(const float2* __restrict__ x, long long frames, long long piece, int divisions,
                const cpx<float>* __restrict__ tw, const float2* __restrict__ h_mid,
                const float2* __restrict__ h_side, float2* __restrict__ result, LoudList loud,
                double* __restrict__ piece_sums, mgb_track_state* __restrict__ state, const float* __restrict__ target_peak, int use_tma) {
    constexpr int N = 2 * F;
    constexpr int THREADS = N / 16;
    if (conv_precise<N>(state, target_peak)) return;  // convolve_precise_kernel's track
    MGB_DYN_SMEM(smem);
    const ConvPointers<N> sp(smem);
    const PackedPlanes planes = sp.planes;
    const int tid = threadIdx.x;
    const long long n0 = (long long)blockIdx.x * F;

    cpx<float> z[N / THREADS];
    const ConvBalance bal = conv_load_frame<N>(x, frames, n0 - F / 2, sp.raw, sp.bar, sp.red_u, use_tma, z);

    // ---- forward transform of z = mid + i*g*side ---------------------------------------------------
    fft_first_pass_regs<N, +1, THREADS, float>(planes, z, /*barrier_before_store=*/false);
    __syncthreads();
    fft_remaining<N, +1, THREADS, float, CHAIN>(planes, tw, PlaneStore<PackedPlanes>{planes}, true);
    __syncthreads();

    // ---- apply both FIR spectra on the pair (k, N-k) ---------------------------------------------
    for (int k = tid; k <= F; k += THREADS) {
        const int kn = (N - k) & (N - 1);
        cpx<float> zk = planes.load(k), zn = planes.load(kn);
        conv_apply_pair(zk, zn, k, h_mid, h_side, bal);
        planes.store(k, zk);
        if (kn != k) planes.store(kn, zn);
    }
    __syncthreads();

    // ---- inverse transform, in place ------------------------------------------------------------------
    fft_first_pass<N, -1, THREADS, float>(planes, tw, PlaneLoad<PackedPlanes>{planes}, /*in_place=*/true);
    __syncthreads();
    fft_remaining<N, -1, THREADS, float, CHAIN>(planes, tw, PlaneStore<PackedPlanes>{planes}, /*last_in_place=*/true);
    __syncthreads();

    // ---- epilogue: coalesced stores -------------------------------------------------------------------
    ConvEpilogue<F> ep(result, loud, n0, frames, piece, divisions, bal);
#pragma unroll
    for (int k = 0; k < F / THREADS; ++k) {
        const int o = tid + k * THREADS;
        if (o < ep.valid) ep.emit(o, planes.load(F - 1 + o));
    }
    ep.template append_loud<F / THREADS>([&](int k) { return tid + k * THREADS; },
                                         [&](int k) { return planes.load(F - 1 + tid + k * THREADS).x; });
    ep.finish(sp.red_a, sp.red_b, sp.red_f, piece_sums, state);
}

// ---- fused kernel: the frame makes 6 trips through shared memory instead of 9.5 ---------------------
// The forward schedule ends and the inverse schedule (InverseRadices) starts with a radix-8 pass of
// N/8 = 2*THREADS butterflies, butterfly j touching the points j + r*N/8 in both.  A thread takes the
// butterflies j and N/8 - j: between them they hold every pair Z[k], Z[N-k] the FIR spectra need, so
// the last forward pass, the spectral product and the first inverse pass happen in registers.  The
// inverse schedule also ends with a radix-8 pass over j + r*N/8: its outputs q >= Q0 = 8F/N are the
// circular indices >= F, i.e. output samples j + 1 + (q-Q0)*N/8 -- contiguous across the block, so the
// epilogue runs straight from registers (outputs q < Q0 are never formed, except index F-1 = output 0).
//
// OVS = N/F is the overlap-save frame length in FIR lengths.  OVS = 2 spends a 2F-point transform pair
// on F outputs; OVS = 4 spends a 4F-point pair on 3F outputs: 5*4F*log2(4F)*2 / 3F = 187 flop per output
// frame for F = 4096 against 260 (-28 %), at one 139 KB CTA of 1024 threads per SM instead of two
// 70 KB CTAs of 512.
//
// PERSIST (option "conv_persistent"): one CTA per SM walks the frames blockIdx.x, blockIdx.x + gridDim.x, ...; as
// soon as every thread has gathered its inputs of the last inverse pass the frame buffer is free, and the bulk copy
// of the CTA's NEXT frame is issued into it -- it lands while the last butterflies, the epilogue's stores and the
// block reduction run, instead of being waited for with the whole SM idle at the top of the frame.
template <int F, int OVS, bool CHAIN, bool PERSIST>
__global__ void __launch_bounds__(OVS * F / 16, (OVS * F <= 8192 ? 2 : 1))
convolve_fused_kernel(const float2* __restrict__ x, long long frames, long long piece, int divisions,
                      const cpx<float>* __restrict__ tw, const float2* __restrict__ h_mid,
                      const float2* __restrict__ h_side, float2* __restrict__ result, LoudList loud,
                      double* __restrict__ piece_sums, mgb_track_state* __restrict__ state, const float* __restrict__ target_peak, int use_tma, int nframes) {
    constexpr int N = OVS * F;
    constexpr int OUT = N - F;  // outputs per frame
    constexpr int THREADS = N / 16;
    constexpr int NB8 = N / 8;
    constexpr int Q0 = F / NB8;  // first output q of the last inverse pass that is an output sample
    using Fwd = Radices<N>;
    using Inv = InverseRadices<N>;
    static_assert(Inv::fused && Fwd::r[Fwd::n - 1] == 8 && Inv::r[0] == 8 && Inv::r[Inv::n - 1] == 8, "schedule");
    static_assert(fft_last_pass_ns<Fwd>() == NB8 && fft_last_pass_ns<Inv>() == NB8 && NB8 == 2 * THREADS, "schedule");
    static_assert(Q0 * NB8 == F && Q0 >= 1 && Q0 < 8, "frame length");
    const cpx<float>* tw_inv = tw + fft_schedule_twiddles<Fwd>();
    if (conv_precise<N>(state, target_peak)) return;  // convolve_precise_kernel's track
    MGB_DYN_SMEM(smem);
    const ConvPointers<N> sp(smem);
    const PackedPlanes planes = sp.planes;
    const PlaneLoad<PackedPlanes> sl{planes};
    const int tid = threadIdx.x;
    if constexpr (PERSIST) {
        if (tid == 0) {
            tma_barrier_init(sp.bar);
            sp.red_u[0] = sp.red_u[1] = 0u;
        }
        __syncthreads();
        if (tid == 0 && (int)blockIdx.x < nframes) conv_issue_frame<N>(x, frames, (long long)blockIdx.x * OUT - F / 2, sp.raw, sp.bar);
    }
    const int frame_end = PERSIST ? nframes : (int)blockIdx.x + 1;
    int phase = 0;
    for (int frame = blockIdx.x; frame < frame_end; frame += gridDim.x, ++phase) {
        const long long n0 = (long long)frame * OUT;

        ConvBalance bal;
        {
            cpx<float> z[N / THREADS];
            bal = conv_load_frame<N>(x, frames, n0 - F / 2, sp.raw, sp.bar, sp.red_u, use_tma, z, PERSIST ? phase : -1);
            fft_first_pass_regs<N, +1, THREADS, float>(planes, z, /*barrier_before_store=*/false);
        }
        __syncthreads();
        fft_middle<N, +1, THREADS, float, CHAIN, Fwd>(planes, tw);

        // ---- last forward pass, FIR spectra, first inverse pass ----------------------------------------
        {
            const int ja = tid, jb = tid == 0 ? NB8 / 2 : NB8 - tid;
            cpx<float> a[8], b[8];
            fft_gather<8, NB8>(sl, ja, a);
            fft_gather<8, NB8>(sl, jb, b);
            __syncthreads();  // in place: everybody has gathered before anybody scatters
            const cpx<float>* tw_last = tw + fft_last_pass_twiddles<Fwd>();
            fft_butterfly<8, NB8, +1, CHAIN>(tw_last, ja, a);  // a[q] = Z[ja + q*NB8]
            fft_butterfly<8, NB8, +1, CHAIN>(tw_last, jb, b);  // b[q] = Z[jb + q*NB8]
            if (tid != 0) {
                // N - (ja + q*NB8) = jb + (7-q)*NB8
    #pragma unroll
                for (int q = 0; q < 4; ++q) {
                    conv_apply_pair(a[q], b[7 - q], ja + q * NB8, h_mid, h_side, bal);
                    conv_apply_pair(b[q], a[7 - q], jb + q * NB8, h_mid, h_side, bal);
                }
            } else {
                // butterflies 0 and N/16 pair with themselves: a[q] <-> a[8-q], b[q] <-> b[7-q]
                cpx<float> t = a[0];
                conv_apply_pair(a[0], t, 0, h_mid, h_side, bal);
                t = a[4];
                conv_apply_pair(a[4], t, N / 2, h_mid, h_side, bal);
    #pragma unroll
                for (int q = 1; q < 4; ++q) conv_apply_pair(a[q], a[8 - q], q * NB8, h_mid, h_side, bal);
    #pragma unroll
                for (int q = 0; q < 4; ++q) conv_apply_pair(b[q], b[7 - q], NB8 / 2 + q * NB8, h_mid, h_side, bal);
            }
            Dft<8, -1, float>::run(a);
            Dft<8, -1, float>::run(b);
    #pragma unroll
            for (int q = 0; q < 8; ++q) planes.store(ja * 8 + q, a[q]);
    #pragma unroll
            for (int q = 0; q < 8; ++q) planes.store(jb * 8 + q, b[q]);
        }
        __syncthreads();
        fft_middle<N, -1, THREADS, float, CHAIN, Inv>(planes, tw_inv);

        // ---- last inverse pass straight into the epilogue ------------------------------------------------
        ConvEpilogue<OUT> ep(result, loud, n0, frames, piece, divisions, bal);
        const cpx<float>* tw_last = tw_inv + fft_last_pass_twiddles<Inv>();
    #pragma unroll
        for (int p = 0; p < 2; ++p) {
            const int j = tid + p * THREADS;
            cpx<float> v[8];
            fft_gather<8, NB8>(sl, j, v);
            if constexpr (PERSIST) {
                if (p == 1) {  // the frame buffer has been read for the last time: the next frame may land in it
                    if (tid == 0) sp.red_u[0] = sp.red_u[1] = 0u;
                    __syncthreads();
                    if (tid == 0 && frame + (int)gridDim.x < nframes) {
                        fence_proxy_async();
                        conv_issue_frame<N>(x, frames, (long long)(frame + gridDim.x) * OUT - F / 2, sp.raw, sp.bar);
                    }
                }
            }
            fft_butterfly<8, NB8, -1, CHAIN>(tw_last, j, v);  // v[q] = y[j + q*NB8]
            if (ep.full) {
    #pragma unroll
                for (int q = Q0; q < 7; ++q) ep.emit_full(j + 1 + (q - Q0) * NB8, v[q]);
                if (j != NB8 - 1) ep.emit_full(j + 1 + (7 - Q0) * NB8, v[7]);  // (o = OUT for j = NB8-1: not an output)
                else ep.emit_full(0, v[Q0 - 1]);
            } else {
    #pragma unroll
                for (int q = Q0; q < 8; ++q) ep.emit(j + 1 + (q - Q0) * NB8, v[q]);  // (o = OUT for j = NB8-1, q = 7: not valid)
                if (j == NB8 - 1) ep.emit(0, v[Q0 - 1]);
            }
            ep.template append_loud<8>(
                [&](int q) { return q >= Q0 ? j + 1 + (q - Q0) * NB8 : (q == Q0 - 1 && j == NB8 - 1 ? 0 : -1); },
                [&](int q) { return v[q].x; });
        }
        ep.finish(sp.red_a, sp.red_b, sp.red_f, piece_sums, state);
    }  // frames of this CTA
}

// ---- fft_size 16384: the frame lives in global memory ------------------------------------------------
// A 2F = 32768-point float frame is 262 KB, more than one SM's shared memory.  This kernel keeps each CTA's frame
// in a scratch region of the workspace (L2-resident) and runs the same passes on it through generic pointers:
// every pass costs a trip through L2 instead of shared memory -- a rare Config, correct first.  A CTA walks the
// frames blockIdx.x, blockIdx.x + gridDim.x, ...; the input is read twice from global memory (once for the
// channel balance, once while it is gathered for the first pass).
constexpr int kConvGlobalThreads = 512;
template <int F, bool CHAIN>
__global__ void __launch_bounds__(kConvGlobalThreads)
convolve_global_kernel(const float2* __restrict__ x, long long frames, long long piece, int divisions,
                       const cpx<float>* __restrict__ tw, const float2* __restrict__ h_mid,
                       const float2* __restrict__ h_side, float2* __restrict__ result, LoudList loud,
                       double* __restrict__ piece_sums, mgb_track_state* __restrict__ state, const float* __restrict__ target_peak, float2* scratch, int nframes) {
    constexpr int N = 2 * F;
    constexpr int THREADS = kConvGlobalThreads;
    __shared__ double red_a[32], red_b[32];
    __shared__ float red_f[32];
    __shared__ unsigned red_u[2];
    if (conv_precise<N>(state, target_peak)) return;  // convolve_precise_kernel's track
    const PackedPlanes planes{scratch + (long long)blockIdx.x * PackedPlanes::elems(N)};
    const int tid = threadIdx.x;
    for (int frame = blockIdx.x; frame < nframes; frame += gridDim.x) {
        const long long n0 = (long long)frame * F;
        const long long origin = n0 - F / 2;
        const ConvSpan span = conv_span<N>(frames, origin);
        ConvFirst first;
        first.raw = x + origin;  // (only indices inside [lo, hi) are dereferenced)
        first.lo = (int)(span.lo - origin);
        first.hi = (int)(span.hi - origin);
        first.fixup = nullptr;
        first.fix_index = -1;
        float max_mid = 0.0f, max_side = 0.0f;
        for (int i = tid; i < N; i += THREADS) {
            const float2 v = first.sample(i);
            max_mid = fmaxf(max_mid, fabsf((v.x + v.y) * 0.5f));
            max_side = fmaxf(max_side, fabsf((v.x - v.y) * 0.5f));
        }
        if (tid == 0) red_u[0] = red_u[1] = 0u;
        __syncthreads();
        block_max2(max_mid, max_side, red_u);
        const float g_side = balance_factor(max_mid, max_side);
        ConvBalance bal;
        bal.inv_g = 1.0f / g_side;
        bal.mid_silent = max_mid == 0.0f;
        bal.side_silent = max_side == 0.0f;
        bal.any_silent = bal.mid_silent || bal.side_silent;
        // forward transform of z = mid + i*g*side, formed while the first pass gathers its inputs
        auto z_of = [&](int i) {
            const float2 v = first.sample(i);
            return cpx<float>{(v.x + v.y) * 0.5f, (v.x - v.y) * 0.5f * g_side};
        };
        fft_run<N, +1, THREADS, float, CHAIN>(planes, tw, z_of, PlaneStore<PackedPlanes>{planes}, /*first_in_place=*/false,
                                              /*last_in_place=*/true);
        __syncthreads();
        for (int k = tid; k <= F; k += THREADS) {
            const int kn = (N - k) & (N - 1);
            cpx<float> zk = planes.load(k), zn = planes.load(kn);
            conv_apply_pair(zk, zn, k, h_mid, h_side, bal);
            planes.store(k, zk);
            if (kn != k) planes.store(kn, zn);
        }
        __syncthreads();
        fft_run<N, -1, THREADS, float, CHAIN>(planes, tw, PlaneLoad<PackedPlanes>{planes}, PlaneStore<PackedPlanes>{planes},
                                              /*first_in_place=*/true, /*last_in_place=*/true);
        __syncthreads();
        ConvEpilogue<F> ep(result, loud, n0, frames, piece, divisions, bal);
        for (int o0 = 0; o0 < ep.valid; o0 += THREADS) {  // (whole warps to the end: append_loud votes per warp)
            const int o = o0 + tid;
            if (o < ep.valid) ep.emit(o, planes.load(F - 1 + o));
            ep.template append_loud<1>([&](int) { return o; }, [&](int) { return planes.load(F - 1 + o).x; });
        }
        ep.finish(red_a, red_b, red_f, piece_sums, state);
        __syncthreads();  // the frame buffer and the reduction slots serve the CTA's next frame
    }
}

// ---- float64 transforms, for the tracks conv_precise picks ----------------------------------------------
// The same overlap-save frames as the float32 kernel of the track (N = OVS*F points, OUT = N - F outputs, the FIR
// spectra on the same grid), transformed in float64: mid and side formed exactly from L and R, one complex
// transform for both (no balancing: float64 noise is 2^-29 of float32's), the product with the float32 FIR
// spectra in float64, and L, R = mid +- side rounded once each.  Each CTA keeps its frame as two padded float64
// planes in a workspace region (L2-resident) and walks the frames blockIdx.x, blockIdx.x + gridDim.x, ...;
// the epilogue (per-piece sums, loud lists, peak) is the float32 kernels' own.  Not tuned: correct first.
constexpr int kConvPreciseThreads = 512;
template <int F, int OVS>
__global__ void __launch_bounds__(kConvPreciseThreads, 1)
convolve_precise_kernel(const float2* __restrict__ x, long long frames, long long piece, int divisions,
                        const cpx<double>* __restrict__ tw, const float2* __restrict__ h_mid,
                        const float2* __restrict__ h_side, float2* __restrict__ result, LoudList loud,
                        double* __restrict__ piece_sums, mgb_track_state* __restrict__ state, const float* __restrict__ target_peak, double* scratch, int nframes) {
    constexpr int N = OVS * F;
    constexpr int OUT = N - F;
    constexpr int THREADS = kConvPreciseThreads;
    using Planes = SplitPlanes<double>;
    __shared__ double red_a[32], red_b[32];
    __shared__ float red_f[32];
    __shared__ unsigned red_u[2];
    if (!conv_precise<N>(state, target_peak)) return;  // the float32 kernel's track
    if (blockIdx.x == 0 && threadIdx.x == 0) state->conv_precise = 1;
    double* re = scratch + (long long)blockIdx.x * 2 * Planes::elems(N);
    const Planes planes{re, re + Planes::elems(N)};
    const int tid = threadIdx.x;
    for (int frame = blockIdx.x; frame < nframes; frame += gridDim.x) {
        const long long n0 = (long long)frame * OUT;
        const long long origin = n0 - F / 2;
        const ConvSpan span = conv_span<N>(frames, origin);
        ConvFirst first;
        first.raw = x + origin;  // (only indices inside [lo, hi) are dereferenced)
        first.lo = (int)(span.lo - origin);
        first.hi = (int)(span.hi - origin);
        first.fixup = nullptr;
        first.fix_index = -1;
        // which channels are exactly silent in this frame (they stay so, as in the reference)
        float max_mid = 0.0f, max_side = 0.0f;
        for (int i = tid; i < N; i += THREADS) {
            const float2 v = first.sample(i);
            max_mid = fmaxf(max_mid, fabsf(v.x + v.y));
            max_side = fmaxf(max_side, fabsf(v.x - v.y));
        }
        if (tid == 0) red_u[0] = red_u[1] = 0u;
        __syncthreads();
        block_max2(max_mid, max_side, red_u);
        ConvBalance bal;
        bal.inv_g = 1.0f;
        bal.mid_silent = max_mid == 0.0f;
        bal.side_silent = max_side == 0.0f;
        bal.any_silent = bal.mid_silent || bal.side_silent;
        auto z_of = [&](int i) {  // (L +- R)/2 of two floats is exact in float64
            const float2 v = first.sample(i);
            return cpx<double>{0.5 * ((double)v.x + (double)v.y), 0.5 * ((double)v.x - (double)v.y)};
        };
        fft_run<N, +1, THREADS, double>(planes, tw, z_of, PlaneStore<Planes>{planes}, /*first_in_place=*/false,
                                        /*last_in_place=*/true);
        __syncthreads();
        for (int k = tid; k <= N / 2; k += THREADS) {
            const int kn = (N - k) & (N - 1);
            const cpx<double> zk = planes.load(k), zn = planes.load(kn);
            // M = (Z[k] + conj Z[N-k])/2 ; S = (Z[k] - conj Z[N-k])/(2i)
            const double mr = 0.5 * (zk.x + zn.x), mi = 0.5 * (zk.y - zn.y);
            const double sr = 0.5 * (zk.y + zn.y), si = 0.5 * (zn.x - zk.x);
            const float2 hm = h_mid[k], hs = h_side[k];
            double pmr = hm.x * mr - hm.y * mi, pmi = hm.x * mi + hm.y * mr;
            double psr = hs.x * sr - hs.y * si, psi = hs.x * si + hs.y * sr;
            if (bal.mid_silent) pmr = pmi = 0.0;
            if (bal.side_silent) psr = psi = 0.0;
            planes.store(k, cpx<double>{pmr - psi, pmi + psr});
            if (kn != k) planes.store(kn, cpx<double>{pmr + psi, psr - pmi});
        }
        __syncthreads();
        fft_run<N, -1, THREADS, double>(planes, tw, PlaneLoad<Planes>{planes}, PlaneStore<Planes>{planes},
                                        /*first_in_place=*/true, /*last_in_place=*/true);
        __syncthreads();
        ConvEpilogue<OUT> ep(result, loud, n0, frames, piece, divisions, bal);
        for (int o0 = 0; o0 < ep.valid; o0 += THREADS) {  // (whole warps to the end: append_loud votes per warp)
            const int o = o0 + tid;
            if (o < ep.valid) ep.emit_wide(o, planes.load(F - 1 + o));
            ep.template append_loud<1>([&](int) { return o; }, [&](int) { return (float)planes.load(F - 1 + o).x; });
        }
        ep.finish(red_a, red_b, red_f, piece_sums, state);
        __syncthreads();  // the frame's planes and the reduction slots serve the CTA's next frame
    }
}

// frame length (points) and CTAs of the float64 convolution, whose planes share the workspace region of
// convolve_global_kernel's frames (the two never run on the same track)
static int conv_precise_points(int fft_size) { return (fft_size == 2048 || fft_size == 4096) ? 4 * fft_size : 2 * fft_size; }
static int conv_precise_ctas(int fft_size, long long target_frames) {
    const long long nframes = (target_frames + fft_size - 1) / fft_size;  // (at least as many as any OVS needs)
    return (int)(nframes < num_sms() ? nframes : num_sms());
}

template <int F, int OVS>
int launch_convolve_precise(const mgb_plan& plan, const mgb_track_layout& layout, const float2* target, float2* result,
                            const Workspace& ws, mgb_track_state* state, cudaStream_t stream) {
    MGB_REQUIRE(plan.d_tw_f64_2F != nullptr, MGB_ERR_INVALID, "convolve: d_tw_f64_2F is NULL");
    const long long T = layout.target_frames;
    const LoudList loud{ws.loud_values, ws.loud_count, (long long)ws.loud_capacity, ws.result_slot};
    const int nframes = (int)((T + (OVS - 1) * F - 1) / ((OVS - 1) * F));
    const int ctas = conv_precise_ctas(F, T);
    // the 4F-point table lives behind the 2F-point one (mgb_plan_twiddle_bytes)
    const cpx<double>* tw = (const cpx<double>*)plan.d_tw_f64_2F + (OVS == 4 ? twiddle_count(2 * F) : 0);
    return launch("convolve_precise_kernel", convolve_precise_kernel<F, OVS>, dim3(nframes < ctas ? nframes : ctas),
                  dim3(kConvPreciseThreads), 0, stream, target, T, (long long)layout.target_piece, layout.target_divisions,
                  tw, (const float2*)ws.h_mid, (const float2*)ws.h_side, result, loud, ws.piece_sums, state, ws.target_peak,
                  (double*)ws.conv_scratch, nframes);
}

template <int F>
int launch_convolve_f32(const mgb_plan& plan, const mgb_track_layout& layout, const float2* target, float2* result,
                        const Workspace& ws, mgb_track_state* state, cudaStream_t stream);

// the float32 kernel, then the float64 one: on every track one of the two returns at once (conv_precise)
template <int F>
int launch_convolve_t(const mgb_plan& plan, const mgb_track_layout& layout, const float2* target, float2* result,
                      const Workspace& ws, mgb_track_state* state, cudaStream_t stream) {
    MGB_TRY(launch_convolve_f32<F>(plan, layout, target, result, ws, state, stream));
    if constexpr (F == 2048 || F == 4096) {
        if (conv_frame_ovs(plan.fft_size, layout.target_piece) == 4)
            return launch_convolve_precise<F, 4>(plan, layout, target, result, ws, state, stream);
    }
    return launch_convolve_precise<F, 2>(plan, layout, target, result, ws, state, stream);
}

template <int F>
int launch_convolve_f32(const mgb_plan& plan, const mgb_track_layout& layout, const float2* target, float2* result,
                        const Workspace& ws, mgb_track_state* state, cudaStream_t stream) {
    const long long T = layout.target_frames;
    const LoudList loud{ws.loud_values, ws.loud_count, (long long)ws.loud_capacity, ws.result_slot};
    if constexpr (F > 8192) {
        const int nframes = (int)((T + F - 1) / F);
        auto kernel = g_twiddle_chain ? convolve_global_kernel<F, true> : convolve_global_kernel<F, false>;
        return launch("convolve_kernel", kernel, dim3(conv_global_ctas(F, T)), dim3(kConvGlobalThreads), 0, stream, target, T,
                      (long long)layout.target_piece, layout.target_divisions, (const cpx<float>*)plan.d_tw_f32_2F,
                      (const float2*)ws.h_mid, (const float2*)ws.h_side, result, loud, ws.piece_sums, state, ws.target_peak,
                      ws.conv_scratch, nframes);
    } else {
        const int ovs = conv_frame_ovs(plan.fft_size, layout.target_piece);
        auto args = [&](auto kernel, int out, int threads, size_t smem) {
            const unsigned nframes = (unsigned)((T + out - 1) / out);
            return launch("convolve_kernel", kernel, dim3(nframes), dim3(threads), smem, stream, target, T,
                          (long long)layout.target_piece, layout.target_divisions, (const cpx<float>*)plan.d_tw_f32_2F,
                          (const float2*)ws.h_mid, (const float2*)ws.h_side, result, loud, ws.piece_sums, state, ws.target_peak,
                          g_use_tma);
        };
        auto args2 = [&](auto kernel, int out, int threads, size_t smem) {  // (the fused kernel also takes the frame count)
            const unsigned nframes = (unsigned)((T + out - 1) / out);
            return launch("convolve_kernel", kernel, dim3(nframes), dim3(threads), smem, stream, target, T,
                          (long long)layout.target_piece, layout.target_divisions, (const cpx<float>*)plan.d_tw_f32_2F,
                          (const float2*)ws.h_mid, (const float2*)ws.h_side, result, loud, ws.piece_sums, state, ws.target_peak,
                          g_use_tma, (int)nframes);
        };
        if constexpr (InverseRadices<4 * F>::fused) {
            if (ovs == 4) {
                // twiddles of the 4F transform live behind the 2F tables (mgb_plan_twiddle_bytes)
                const cpx<float>* tw4 = (const cpx<float>*)plan.d_tw_f32_2F + twiddle_count(2 * F) + inverse_twiddle_count(2 * F);
                const unsigned nframes = (unsigned)((T + 3 * F - 1) / (3 * F));
                if (g_conv_persistent && g_use_tma && 4 * F > 8192) {  // (one CTA per SM: the 16384-point frames)
                    const unsigned grid = nframes < (unsigned)num_sms() ? nframes : (unsigned)num_sms();
                    auto kernel = g_twiddle_chain ? convolve_fused_kernel<F, 4, true, true> : convolve_fused_kernel<F, 4, false, true>;
                    return launch("convolve_kernel", kernel, dim3(grid), dim3(4 * F / 16), ConvSmem<4 * F>::kBytes, stream, target, T,
                                  (long long)layout.target_piece, layout.target_divisions, tw4, (const float2*)ws.h_mid,
                                  (const float2*)ws.h_side, result, loud, ws.piece_sums, state, ws.target_peak, g_use_tma, (int)nframes);
                }
                auto kernel = g_twiddle_chain ? convolve_fused_kernel<F, 4, true, false> : convolve_fused_kernel<F, 4, false, false>;
                return launch("convolve_kernel", kernel, dim3(nframes), dim3(4 * F / 16), ConvSmem<4 * F>::kBytes, stream, target, T,
                              (long long)layout.target_piece, layout.target_divisions, tw4, (const float2*)ws.h_mid,
                              (const float2*)ws.h_side, result, loud, ws.piece_sums, state, ws.target_peak, g_use_tma, (int)nframes);
            }
        }
        if constexpr (InverseRadices<2 * F>::fused) {
            if (g_conv_fused) {
                if (g_conv_persistent && g_use_tma && 2 * F > 8192) {  // (fft_size 8192: 16384-point frames, one CTA per SM)
                    const unsigned nframes = (unsigned)((T + F - 1) / F);
                    const unsigned grid = nframes < (unsigned)num_sms() ? nframes : (unsigned)num_sms();
                    auto kernel = g_twiddle_chain ? convolve_fused_kernel<F, 2, true, true> : convolve_fused_kernel<F, 2, false, true>;
                    return launch("convolve_kernel", kernel, dim3(grid), dim3(F / 8), ConvSmem<2 * F>::kBytes, stream, target, T,
                                  (long long)layout.target_piece, layout.target_divisions, (const cpx<float>*)plan.d_tw_f32_2F,
                                  (const float2*)ws.h_mid, (const float2*)ws.h_side, result, loud, ws.piece_sums, state, ws.target_peak,
                                  g_use_tma, (int)nframes);
                }
                return args2(g_twiddle_chain ? convolve_fused_kernel<F, 2, true, false> : convolve_fused_kernel<F, 2, false, false>, F, F / 8,
                             ConvSmem<2 * F>::kBytes);
            }
        }
        return args(g_twiddle_chain ? convolve_kernel<F, true> : convolve_kernel<F, false>, F, F / 8, ConvSmem<2 * F>::kBytes);
    }
}

}  // namespace

// scratch of convolve_global_kernel: one padded 2F-point frame per CTA (carve_workspace)
int conv_global_ctas(int fft_size, long long target_frames) {
    if (fft_size <= 8192) return 0;
    const long long nframes = (target_frames + fft_size - 1) / fft_size;
    const long long cap = 2LL * num_sms();
    return (int)(nframes < cap ? nframes : cap);
}
int64_t conv_global_scratch_bytes(int fft_size, long long target_frames) {
    const int64_t global = (int64_t)conv_global_ctas(fft_size, target_frames) * (int64_t)PackedPlanes::bytes(2 * fft_size);
    const int64_t precise = (int64_t)conv_precise_ctas(fft_size, target_frames) *
                            (int64_t)SplitPlanes<double>::bytes(conv_precise_points(fft_size));
    return global > precise ? global : precise;
}

// Overlap-save frame length, in FIR lengths, of the convolution (and therefore the grid the design kernel
// must put the FIR spectra on): 4 where the 4F-point fused kernel exists, is switched on and every output
// frame of 3F samples touches at most two pieces; 2 otherwise.
int conv_frame_ovs(int fft_size, long long target_piece) {
    if (g_conv_ovs == 4 && g_conv_fused && (fft_size == 4096 || fft_size == 2048) && target_piece >= 3LL * fft_size) return 4;
    return 2;
}

int launch_convolve(const mgb_plan& plan, const mgb_track_layout& layout, const float2* target, float2* result,
                    const Workspace& ws, mgb_track_state* state, cudaStream_t stream) {
    if (layout.target_piece < plan.fft_size) {
        set_error("convolve: piece (%lld) shorter than fft_size", (long long)layout.target_piece);
        return MGB_ERR_UNSUPPORTED;
    }
    switch (plan.fft_size) {
        case 512: return launch_convolve_t<512>(plan, layout, target, result, ws, state, stream);
        case 1024: return launch_convolve_t<1024>(plan, layout, target, result, ws, state, stream);
        case 2048: return launch_convolve_t<2048>(plan, layout, target, result, ws, state, stream);
        case 4096: return launch_convolve_t<4096>(plan, layout, target, result, ws, state, stream);
        case 8192: return launch_convolve_t<8192>(plan, layout, target, result, ws, state, stream);
        case 16384: return launch_convolve_t<16384>(plan, layout, target, result, ws, state, stream);
        default: break;
    }
    set_error("convolve: fft_size %d has no kernel", plan.fft_size);
    return MGB_ERR_UNSUPPORTED;
}

}  // namespace mgb
