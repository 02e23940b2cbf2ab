// K3 -- level statistics and matching-FIR design: tiny, latency-bound, all float64.
//
// (the level statistics -- normalize_reference, loudest-piece masks, match RMS, c0 -- live in
//  tail.cuh and run in the last CTA of the reference's analysis pass)
// These kernels replace
//   __average_fft's mean over the loudest pieces   stage_helpers/match_frequencies.py:42
//   get_fir                                        stage_helpers/match_frequencies.py:78-101
//   __smooth_exponentially                         stage_helpers/match_frequencies.py:45-75
//   dsp.smooth_lowess (statsmodels lowess, it=0)   dsp.py:103-106
// and additionally emits the FIR's spectrum on the 2F-point grid of the overlap-save
// convolution (convolve.cu), with the level-matching gain c0 and the 1/(2F) of the inverse
// transform folded in.
//
// One CTA per channel (mid, side).  The Config-only parts (spline LU factors, evaluation weights,
// LOWESS neighbourhoods) come from the plan; the substitution sweeps run block-parallel with a
// warm-up of kWarm rows (the factors decay like 0.27^n, so 48 rows are exact to < 1e-27).
#include "fft.cuh"
#include "kernels.cuh"
#include "select.cuh"
#include "tail.cuh"

namespace mgb {

namespace {

constexpr int kDesignThreads = 512;
constexpr int kWarm = 48;
constexpr int kBatch = 16;  // rows fetched together in the substitution sweeps
constexpr int kDesignBlocks = 4;  // scratch blocks per channel: one per design CTA (up to 4 residue classes)

// ------------------------------------------------------------------------------------------------
struct SplineTables {
    const double* hinv;  // [n-1]
    const double* lu;    // [3][n-2]
    const double* end;   // [4]
};

// Second derivatives of the not-a-knot cubic through (knots, y): M[0..n).  z is scratch [n].
// The two substitution sweeps are first-order recurrences; each thread runs a block of rows after
// a kWarm-row warm-up.  Operands are fetched kBatch rows at a time so that the L2 latency of the
// factor tables overlaps instead of adding up along the dependent chain.
__device__ void spline_moments(const double* __restrict__ y, int n, SplineTables t, double* __restrict__ z,
                               double* __restrict__ M) {
    const int m = n - 2;
    const double* fa = t.lu;
    const double* invden = t.lu + m;
    const double* cp = t.lu + 2 * m;
    const int tid = threadIdx.x, nthr = blockDim.x;
    // right-hand side scaled by the pivot, all rows in parallel (row i = interior knot i+1)
    for (int i = tid; i < m; i += nthr)
        z[i] = 6.0 * ((y[i + 2] - y[i + 1]) * t.hinv[i + 1] - (y[i + 1] - y[i]) * t.hinv[i]) * invden[i];
    __syncthreads();
    const int block = (m + nthr - 1) / nthr;
    const int lo = tid * block;
    const int hi = min(m, lo + block);
    // forward sweep: z (scaled right-hand side) -> M (used as scratch for the swept values)
    if (lo < m) {
        double acc = 0.0;
        int i = max(0, lo - kWarm);
        while (i < hi) {
            double dv[kBatch], fv[kBatch];
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {
                const int r = min(i + u, m - 1);
                dv[u] = z[r];
                fv[u] = fa[r];
            }
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {
                if (i + u < hi) {
                    acc = dv[u] - fv[u] * acc;
                    if (i + u >= lo) M[i + u] = acc;
                }
            }
            i += kBatch;
        }
    }
    __syncthreads();
    // backward sweep: M (swept) -> z[i+1] (moment of interior knot i+1)
    if (lo < m) {
        double acc = 0.0;
        int i = min(m - 1, hi - 1 + kWarm);
        while (i >= lo) {
            double zv[kBatch], cv[kBatch];
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {
                const int r = max(i - u, 0);
                zv[u] = M[r];
                cv[u] = cp[r];
            }
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {
                if (i - u >= lo) {
                    acc = zv[u] - cv[u] * acc;
                    if (i - u < hi) z[i - u + 1] = acc;
                }
            }
            i -= kBatch;
        }
    }
    __syncthreads();
    for (int i = 1 + tid; i <= m; i += nthr) M[i] = z[i];
    __syncthreads();
    if (tid == 0) {
        M[0] = t.end[0] * M[1] + t.end[1] * M[2];
        M[n - 1] = t.end[2] * M[n - 2] + t.end[3] * M[n - 3];
    }
    __syncthreads();
}

__device__ __forceinline__ double spline_eval(const double* __restrict__ y, const double* __restrict__ M, int idx,
                                              const double* __restrict__ w) {
    return w[0] * y[idx] + w[1] * y[idx + 1] + w[2] * M[idx] + w[3] * M[idx + 1];
}

// ---- LOWESS pieces (statsmodels nonparametric/_smoothers_lowess.pyx semantics, dsp.py:103-106) --------
// abscissa j of numpy.linspace(0, 1, n)
__device__ __forceinline__ double lowess_x(int j, int n) { return j == n - 1 ? 1.0 : (double)j * (1.0 / (double)(n - 1)); }

// fitted values at the regression points (fit[f]) -> all n abscissae by the `delta` interpolation
// (update_indices / interpolate_skipped_fits).  Ends with a barrier.
__device__ __forceinline__ void lowess_interpolate(const mgb_plan& plan, const double* __restrict__ fit, double* __restrict__ out) {
    const int last = plan.lowess_nfit - 1;
    for (int j = threadIdx.x; j < plan.n_log; j += blockDim.x) {
        const int sg = plan.d_lw_seg[j];
        const double al = plan.d_lw_alpha[j];  // 0 at a regression point
        out[j] = al * fit[min(sg + 1, last)] + (1.0 - al) * fit[sg];
    }
    __syncthreads();
}

// One local regression per warp with weights tricube(distance / radius) * resid_w (calculate_weights,
// calculate_y_fit): fit = sum_j w_j (1 + (x_i - xbar)(x_j - xbar)/sqdev) y_j with w normalised; "not ok"
// (sum w <= 0 or a single non-zero weight) -> fit = y_i.  No trailing barrier.
__device__ void lowess_weighted_fits(const mgb_plan& plan, const double* __restrict__ y, const double* __restrict__ resid_w,
                                     double* __restrict__ fit) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int k = plan.lowess_k, n = plan.n_log;
    for (int f = warp; f < plan.lowess_nfit; f += nwarps) {
        const int i = plan.d_lw_fit_idx[f], left = plan.d_lw_fit_left[f];
        const double xi = lowess_x(i, n);
        const double radius = fmax(xi - lowess_x(left, n), lowess_x(left + k - 1, n) - xi);
        double sw = 0.0, swx = 0.0, nz = 0.0;
        for (int j = lane; j < k; j += 32) {
            const double xj = lowess_x(left + j, n);
            const double d = fabs(xj - xi);
            double w = d / radius;
            w = 1.0 - w * w * w;
            w = w * w * w;
            if (d >= radius) w = 0.0;
            w *= resid_w[left + j];
            sw += w;
            swx += w * xj;
            nz += w != 0.0 ? 1.0 : 0.0;
        }
        sw = warp_sum(sw);
        swx = warp_sum(swx);
        nz = warp_sum(nz);
        double value = y[i];
        if (sw > 0.0 && nz != 1.0) {
            const double xbar = swx / sw;
            double sqdev = 0.0, swy = 0.0, swdy = 0.0;
            for (int j = lane; j < k; j += 32) {
                const double xj = lowess_x(left + j, n);
                const double d = fabs(xj - xi);
                double w = d / radius;
                w = 1.0 - w * w * w;
                w = w * w * w;
                if (d >= radius) w = 0.0;
                w = w * resid_w[left + j] / sw;
                const double dx = xj - xbar;
                sqdev += w * dx * dx;
                swy += w * y[left + j];
                swdy += w * dx * y[left + j];
            }
            sqdev = warp_sum(sqdev);
            swy = warp_sum(swy);
            swdy = warp_sum(swdy);
            value = swy + (xi - xbar) / sqdev * swdy;
        }
        if (lane == 0) fit[f] = value;
    }
}

// (block_kth_smallest: select.cuh)

// bisquare weights of the residuals (calculate_residual_weights): scale 6 * median|y - fit|; a zero median
// leaves weight 1 on the exact fits and 0 elsewhere.  `absres` is scratch [n].  Ends with a barrier.
__device__ void lowess_residual_weights(const double* __restrict__ y, const double* __restrict__ fitted, int n,
                                        double* __restrict__ absres, double* __restrict__ resid_w) {
    for (int j = threadIdx.x; j < n; j += blockDim.x) absres[j] = fabs(y[j] - fitted[j]);
    __syncthreads();
    double median = block_kth_smallest(absres, n, n / 2);
    if (!(n & 1)) median = 0.5 * (median + block_kth_smallest(absres, n, n / 2 - 1));
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        double u = absres[j];
        if (median == 0.0) u = u > 0.0 ? 1.0 : 0.0;
        else u /= 6.0 * median;
        if (u >= 1.0) u = 1.0;
        const double t = 1.0 - u * u;
        resid_w[j] = t * t;
    }
    __syncthreads();
}

// Scratch layout of one channel's design vectors (doubles): m, M1, s [n_lin each], then
// mlog, slog, zz, M2 [n_log each], then fir [F].
// smooth_curve: m -> s, match_frequencies.__smooth_exponentially (:45-75): cubic spline to the
// log grid, LOWESS, cubic spline back, then out[0] = 0 and out[1] = m[1].  Every step is linear in
// m (lowess_it == 0), which is what operator_columns_kernel exploits.  Contains barriers.
__device__ void smooth_curve(const mgb_plan& plan, double* __restrict__ base) {
    const int tid = threadIdx.x, nthr = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarps = nthr >> 5;
    const int HB = plan.n_lin, NL = plan.n_log;
    double* m = base;
    double* M1 = m + HB;
    double* s = M1 + HB;
    double* mlog = s + HB;
    double* slog = mlog + NL;
    double* zz = slog + NL;
    double* M2 = zz + NL;

    // ---- B/C: cubic spline linear grid -> log grid (match_frequencies.py:60-61) --------------
    spline_moments(m, HB, SplineTables{plan.d_sa_hinv, plan.d_sa_lu, plan.d_sa_end}, zz, M1);
    for (int j = tid; j < NL; j += nthr) mlog[j] = spline_eval(m, M1, plan.d_sa_eval_idx[j], plan.d_sa_eval_w + 4LL * j);
    __syncthreads();

    // ---- D: LOWESS (dsp.py:103-106) -----------------------------------------------------------
    if (plan.lowess_it == 0) {
        // no robustness iterations: each regression is a Config-only row of k coefficients
        const int k = plan.lowess_k;
        const int nfit = plan.lowess_nfit;
        for (int f = warp; f < nfit; f += 2 * nwarps) {  // two regressions per pass: twice the loads in flight
            const int f2 = min(f + nwarps, nfit - 1);
            const double* row_a = plan.d_lw_rows + (long long)plan.d_lw_row_idx[f] * k;
            const double* row_b = plan.d_lw_rows + (long long)plan.d_lw_row_idx[f2] * k;
            const double* ya = mlog + plan.d_lw_fit_left[f];
            const double* yb = mlog + plan.d_lw_fit_left[f2];
            double acc_a = 0.0, acc_b = 0.0;
            for (int j = lane; j < k; j += 32) {
                acc_a += row_a[j] * ya[j];
                acc_b += row_b[j] * yb[j];
            }
            acc_a = warp_sum(acc_a);
            acc_b = warp_sum(acc_b);
            if (lane == 0) {
                zz[f] = acc_a;
                if (f + nwarps < nfit) zz[f2] = acc_b;  // else f2 is clamped: nfit - 1 is another warp's
            }
        }
        __syncthreads();
        lowess_interpolate(plan, zz, slog);
    } else {
        // lowess_it > 0: every pass after the first multiplies the tricube weights by the bisquare weights of
        // the previous pass's residuals, so the regressions depend on the data.  M2 (free until step E) holds
        // the residual weights.
        double* resid_w = M2;
        for (int j = tid; j < NL; j += nthr) resid_w[j] = 1.0;
        __syncthreads();
        for (int pass = 0; pass <= plan.lowess_it; ++pass) {
            lowess_weighted_fits(plan, mlog, resid_w, zz);
            __syncthreads();
            lowess_interpolate(plan, zz, slog);
            if (pass < plan.lowess_it) lowess_residual_weights(mlog, slog, NL, zz, resid_w);
        }
    }

    // ---- E: cubic spline log grid -> linear grid, then the two overrides (:67-73) -------------
    spline_moments(slog, NL, SplineTables{plan.d_sb_hinv, plan.d_sb_lu, plan.d_sb_end}, zz, M2);
    for (int k = tid; k < HB; k += nthr) {
        double v = spline_eval(slog, M2, plan.d_sb_eval_idx[k], plan.d_sb_eval_w + 4LL * k);
        if (k == 0) v = 0.0;
        if (k == 1) v = m[1];
        s[k] = v;
    }
    __syncthreads();

}

struct DesignArgs {
    // average-spectrum inputs
    const float* spec_part_t;
    const float* spec_part_r;
    unsigned char* mask_t;  // global copies of the loudest-piece masks (written for inspection)
    unsigned char* mask_r;
    const float* absmax_t;       // [div_t*slots_t + 1] the target's peaks per (piece, slot) and of its tail
    float* target_peak;          // out: their maximum (Workspace::target_peak)
    LevelsArgs levels;
    int div_t, slots_t, div_r, slots_r;
    long long frames_per_piece_t, frames_per_piece_r;
    const double* avg_override;  // [4][n_lin] or null
    // outputs
    double* scratch;             // [2][stride]
    long long stride;
    double* fir_out;             // [2][F] or null
    float2* h_mid;
    float2* h_side;
    mgb_track_state* state;        // null with avg_override: c0 = 1, coef = 1
    int s_ready;                   // the smoothed curve is already in the scratch (operator path)
    int ovs;                       // FIR spectra on the ovs*F-point grid of the convolution (2 or 4): ovs CTAs per channel
};

// Matching curve m[k] = mean|rfft(reference)| / max(eps, mean|rfft(target)|) from the per-(piece,
// slot) partial sums of analyze.cu, over the loudest pieces only (match_frequencies.py:42,93-94).
// grid = (ceil(n_lin/32), 2 channels); block = 32 bins x 32 slices of the (piece, slot) items, four loads of a
// slice in flight at a time (the partial spectra sit in L2: the sums are bound by load latency, not bandwidth).
struct PrefetchList {
    const void* ptr[14];
    long long bytes[14];
    int count;
};

__device__ __forceinline__ void prefetch_l2(const void* p) {
#ifndef MGB_EMULATE
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
#else
    (void)p;
#endif
}

constexpr int kMeanBins = 32, kMeanSlices = 32;

// What one spectrum-mean launch folds.  kPaired: target and reference partials into the matching curve.
// kProfiled: the target's partials, the reference half from a profile (mgb_match_levels_profiled).  kProfile: the
// reference's partials alone into a profile (mgb_analyze_reference; div_t = 0).  The halves that exist run the
// same code in every mode, so a profile holds exactly the reference terms a paired job computes, bit for bit.
enum class MeanMode { kPaired, kProfiled, kProfile };

struct ProfileIO {
    const mgb_reference_profile* in;  // kProfiled: the profile (header, then spectra [2][n_lin])
    mgb_reference_profile* out;       // kProfile: where the profile goes
    mgb_reference_profile header;     // kProfile: its fingerprint and geometry, filled by the host
};

template <MeanMode MODE>
__global__ void __launch_bounds__(kMeanBins * kMeanSlices)
spectrum_mean_kernel(DesignArgs a, int n_lin, int fft_size, double eps, PrefetchList pf, ProfileIO io) {
    constexpr int BINS = kMeanBins, SLICES = kMeanSlices;
    constexpr bool kHasT = MODE != MeanMode::kProfile, kHasR = MODE != MeanMode::kProfiled;
    __shared__ double part_t[SLICES][BINS + 1], part_r[SLICES][BINS + 1];
    MGB_DYN_SMEM(smem);  // loudest-piece masks: [div_t] then [div_r] bytes
    unsigned char* mask_t = smem;
    unsigned char* mask_r = smem + a.div_t;
    // The design kernels that follow walk Config-only tables that the streaming kernels in between
    // have pushed out of L2: pull them back in from here, where there are CTAs to spare.
    {
        const long long gtid = ((long long)blockIdx.y * gridDim.x + blockIdx.x) * blockDim.x + threadIdx.x;
        const long long gsize = (long long)gridDim.x * gridDim.y * blockDim.x;
        for (int t = 0; t < pf.count; ++t)
            for (long long off = gtid * 128; off < pf.bytes[t]; off += gsize * 128)
                prefetch_l2(reinterpret_cast<const char*>(pf.ptr[t]) + off);
    }
    // Level statistics (match_levels.py:29-131), recomputed identically by every CTA from the analysis pass's
    // partial sums.  The partial sums are folded per piece by the whole block first -- one warp per piece, lanes
    // over its slots, so every load is in flight at once (a lane walking a piece's 34 slots alone was 25 us of
    // serial L2 latency) -- then warp 0 derives the statistics from the per-piece sums with shuffles and leaves
    // the masks and the scalars in shared memory; CTA (0,0) records them in the track state.
    __shared__ LevelsResult lv_s;
    __shared__ unsigned peak_bits_s, target_peak_bits_s;
    double* piece_sum = reinterpret_cast<double*>(smem + ((a.div_t + a.div_r + 15) / 16) * 16);  // [div_t + div_r]
    {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
        if (threadIdx.x == 0) peak_bits_s = target_peak_bits_s = 0u;
        __syncthreads();
        if constexpr (kHasR) {
            float pk = 0.0f;
            for (int i = threadIdx.x; i < a.div_r * a.slots_r + 1; i += blockDim.x) pk = fmaxf(pk, a.levels.absmax_r[i]);
            pk = warp_max_f(pk);
            if (lane == 0 && pk > 0.0f) atomicMax(&peak_bits_s, __float_as_uint(pk));  // non-negative floats order like their bits
        }
        if (kHasT && blockIdx.x == 0 && blockIdx.y == 0) {  // the target's peak: the convolution's choice of precision needs it
            float tpk = 0.0f;
            for (int i = threadIdx.x; i < a.div_t * a.slots_t + 1; i += blockDim.x) tpk = fmaxf(tpk, a.absmax_t[i]);
            tpk = warp_max_f(tpk);
            if (lane == 0 && tpk > 0.0f) atomicMax(&target_peak_bits_s, __float_as_uint(tpk));
        }
        for (int p = warp; p < a.div_t + a.div_r; p += nwarps) {
            const bool is_t = p < a.div_t;
            const double* part = is_t ? a.levels.sumsq_t + (long long)p * a.slots_t
                                      : a.levels.sumsq_r + (long long)(p - a.div_t) * a.slots_r;
            const int slots = is_t ? a.slots_t : a.slots_r;
            double sum = 0.0;
            for (int k = lane; k < slots; k += 32) sum += part[k];
            sum = warp_sum(sum);
            if (lane == 0) piece_sum[p] = sum;
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            LevelsResult mine;
            if constexpr (MODE == MeanMode::kPaired) {
                LevelsArgs folded = a.levels;
                folded.sumsq_t = piece_sum;
                folded.sumsq_r = piece_sum + a.div_t;
                folded.slots_t = folded.slots_r = 1;
                const float peak = __uint_as_float(peak_bits_s);
                folded.absmax_r = &peak;
                folded.div_r_items_override = 1;
                mine = levels_compute_warp(folded, mask_t, mask_r);
            } else if constexpr (MODE == MeanMode::kProfiled) {  // levels_compute_warp's target half, the rest recorded
                const SignalLevels t = signal_levels_warp(piece_sum, a.div_t, 1, (double)a.levels.piece_t, mask_t);
                mine.peak = io.in->reference_peak;
                mine.coef = io.in->final_amplitude_coef;
                mine.match_t = t.match;
                mine.match_r = io.in->reference_match_rms;
                mine.c0 = mine.match_r / fmax(a.levels.eps, mine.match_t);
                mine.loud_t = t.loud;
                mine.loud_r = io.in->reference_loud_pieces;
            } else {  // levels_compute_warp's reference half
                const float peak = __uint_as_float(peak_bits_s);
                mine.peak = (double)warp_max_f(lane == 0 ? fmaxf(0.0f, peak) : 0.0f);
                mine.coef = reference_coef(mine.peak, a.levels.threshold, a.levels.eps);
                const SignalLevels r = signal_levels_warp(piece_sum, a.div_r, 1, (double)a.levels.piece_r, mask_r);
                mine.match_t = 0.0;
                mine.match_r = r.match / mine.coef;
                mine.c0 = 0.0;
                mine.loud_t = 0;
                mine.loud_r = r.loud;
            }
            if (threadIdx.x == 0) lv_s = mine;
        }
    }
    __syncthreads();
    const LevelsResult lv = lv_s;
    if (blockIdx.x == 0 && blockIdx.y == 0) {
        if (threadIdx.x == 0) {
            if constexpr (kHasT) {
                levels_store(lv, a.state);
                a.state->conv_peak_bits = 0.0f;
                a.state->fir_peak_mid_bits = 0.0f;
                a.state->fir_peak_side_bits = 0.0f;
                a.state->conv_precise = 0;
                *a.target_peak = __uint_as_float(target_peak_bits_s);
            } else {
                mgb_reference_profile h = io.header;
                h.reference_loud_pieces = lv.loud_r;
                h.reference_peak = lv.peak;
                h.final_amplitude_coef = lv.coef;
                h.reference_match_rms = lv.match_r;
                *io.out = h;
            }
        }
        for (int p = threadIdx.x; p < a.div_t; p += blockDim.x) a.mask_t[p] = mask_t[p];
        for (int p = threadIdx.x; p < a.div_r; p += blockDim.x) a.mask_r[p] = mask_r[p];
    }
    // The loudest pieces' (piece, slot) items as two compact lists (piece ranks by warp 0 with a ballot prefix, the
    // lists filled by the whole block; the same order in every CTA): the sums below then touch selected items only -- no mask test, no division per element, and 40 % fewer
    // loads when 8 of 13 pieces count.
    unsigned short* sel = reinterpret_cast<unsigned short*>(piece_sum + a.div_t + a.div_r);  // [items_t + items_r]
    __shared__ int n_sel_s[2];
    // (piece_sum is free now: it becomes each piece's offset into its signal's list, in units of pieces)
    int* piece_rank = reinterpret_cast<int*>(piece_sum);  // [div_t + div_r]: number of selected pieces before this one
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        for (int sig = 0; sig < 2; ++sig) {
            const unsigned char* mask = sig == 0 ? mask_t : mask_r;
            const int div = sig == 0 ? a.div_t : a.div_r;
            int* rank = piece_rank + (sig == 0 ? 0 : a.div_t);
            int count = 0;
            for (int base_p = 0; base_p < div; base_p += 32) {
                const int p = base_p + lane;
                const bool keep = p < div && mask[p];
                const unsigned votes = __ballot_sync(0xffffffffu, keep);
                if (p < div) rank[p] = count + __popc(votes & ((1u << lane) - 1u));
                count += __popc(votes);
            }
            if (lane == 0) n_sel_s[sig] = count * (sig == 0 ? a.slots_t : a.slots_r);
        }
    }
    __syncthreads();
    for (int sig = 0; sig < 2; ++sig) {  // every thread files its share of the items: piece by piece, slot by slot
        const unsigned char* mask = sig == 0 ? mask_t : mask_r;
        const int slots = sig == 0 ? a.slots_t : a.slots_r;
        const int items = (sig == 0 ? a.div_t : a.div_r) * slots;
        const int* rank = piece_rank + (sig == 0 ? 0 : a.div_t);
        unsigned short* out = sel + (sig == 0 ? 0 : a.div_t * a.slots_t);
        for (int it = threadIdx.x; it < items; it += blockDim.x) {
            const int p = it / slots;
            if (mask[p]) out[rank[p] * slots + (it - p * slots)] = (unsigned short)it;
        }
    }
    __syncthreads();
    const int bx = threadIdx.x % BINS, sy = threadIdx.x / BINS;
    const int k = blockIdx.x * BINS + bx;
    const int ch = blockIdx.y;
    double st = 0.0, sr = 0.0;
    if (k < n_lin) {
        auto selected_sum = [&](const float* part, const unsigned short* list, int count) {
            double total = 0.0;
            for (int i = sy; i < count; i += 8 * SLICES) {
                float v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int iu = i + u * SLICES;
                    v[u] = iu < count ? part[((long long)list[iu] * 2 + ch) * n_lin + k] : 0.0f;
                }
                total += (((double)v[0] + (double)v[1]) + ((double)v[2] + (double)v[3])) +
                         (((double)v[4] + (double)v[5]) + ((double)v[6] + (double)v[7]));
            }
            return total;
        };
        if constexpr (kHasT) st = selected_sum(a.spec_part_t, sel, n_sel_s[0]);
        if constexpr (kHasR) sr = selected_sum(a.spec_part_r, sel + a.div_t * a.slots_t, n_sel_s[1]);
    }
    part_t[sy][bx] = st;
    part_r[sy][bx] = sr;
    __syncthreads();
    if (sy == 0 && k < n_lin) {
        for (int q = 1; q < SLICES; ++q) {
            st += part_t[q][bx];
            sr += part_r[q][bx];
        }
        // |rfft| is positively homogeneous: the level-matching gain c0 (target) and the reference
        // normalisation 1/coef are applied to the means instead of to the samples
        const double norm_t = lv.c0 / ((double)lv.loud_t * (double)a.frames_per_piece_t * (double)fft_size);
        const double norm_r = 1.0 / (lv.coef * (double)lv.loud_r * (double)a.frames_per_piece_r * (double)fft_size);
        if constexpr (MODE == MeanMode::kPaired) {
            a.scratch[(long long)(kDesignBlocks * ch) * a.stride + k] = (sr * norm_r) / fmax(eps, st * norm_t);
        } else if constexpr (MODE == MeanMode::kProfiled) {
            const double* spectra = reinterpret_cast<const double*>(io.in + 1);
            a.scratch[(long long)(kDesignBlocks * ch) * a.stride + k] = spectra[(long long)ch * n_lin + k] / fmax(eps, st * norm_t);
        } else {
            reinterpret_cast<double*>(io.out + 1)[(long long)ch * n_lin + k] = sr * norm_r;
        }
    }
}

// fft_size 16384: the float64 planes (2 x 132 KB) do not fit one SM; they live in the CTA's scratch block in
// global memory instead (L2-resident; the passes and their barriers are the same code on generic pointers).
template <int F>
struct DesignSmem {
    static constexpr bool kGlobalPlanes = F > 8192;
    static constexpr int kPlane = fft_padded_size(F);
    static constexpr int kBytes = kGlobalPlanes ? 64 : 2 * kPlane * 8 + 64;
};

// The one float64 transform of the design kernel: forward, in place on the planes (barriers inside and between
// its gathers and scatters; the caller puts one before and one after).
template <int F>
__device__ __noinline__ void design_fft(SplitPlanes<double> planes, const cpx<double>* __restrict__ tw) {
    fft_run<F, +1, kDesignThreads, double>(planes, tw, PlaneLoad<SplitPlanes<double>>{planes},
                                           PlaneStore<SplitPlanes<double>>{planes}, true, true);
}

// Steps F-G of a design CTA: fir = ifftshift(irfft(s)) * hann from the curve s(k), k = 0 .. F/2, then the FIR's
// spectrum bins of residue `parity` on the ovs*F grid of the convolution with c0/(ovs*F) folded in, and its peak
// into the track state.  design_kernel passes the curve it smoothed; design_native_kernel passes the analysis job's
// curve carried over to its own grid.  Contains barriers.
template <int F, typename Curve>
__device__ __forceinline__ void design_fir_spectrum(SplitPlanes<double> planes, const cpx<double>* __restrict__ tw,
                                                    const double* __restrict__ hann, Curve s, int ch, int parity, int ovs,
                                                    double c0, double* __restrict__ fir_out, float2* __restrict__ H,
                                                    mgb_track_state* state) {
    const int tid = threadIdx.x, nthr = blockDim.x;
    double* re = planes.re;
    double* im = planes.im;
    // ---- F: fir = ifftshift(irfft(s)) * hann (match_frequencies.py:98-99) ---------------------
    // s is real, so its Hermitian extension X[k] = X[F-k] = s[k] is real and even and the inverse transform
    // equals the forward one: all transforms of this kernel are ONE in-place forward FFT (design_fft, not
    // inlined) -- the kernel runs once per CTA on cold instruction caches, and three unrolled copies of a
    // float64 radix-16 FFT cost a third of its time in instruction fetches.
    constexpr int PER = F / kDesignThreads;
    static_assert(PER >= 1 && F % kDesignThreads == 0, "design: fft_size is a multiple of the block size");
    double taps[PER];  // the thread's FIR taps tid + q*nthr
    {
#pragma unroll
        for (int q = 0; q < PER; ++q) {
            const int i = tid + q * kDesignThreads;
            planes.store(i, cpx<double>{s(i <= F / 2 ? i : F - i), 0.0});
        }
        __syncthreads();
        design_fft<F>(planes, tw);
        __syncthreads();
        const double inv = 1.0 / (double)F;
#pragma unroll
        for (int q = 0; q < PER; ++q) {
            const int i = tid + q * kDesignThreads;
            const int src = (i + F / 2) & (F - 1);
            taps[q] = re[fft_pad(src)] * inv * hann[i];
            if (fir_out && parity == 0) fir_out[(long long)ch * F + i] = taps[q];
        }
        __syncthreads();  // every tap has been read out of the planes
    }

    // ---- G: spectrum of the FIR on the ovs*F grid, bins 0..ovs*F/2 --------------------------------
    // bin ovs*j + r = FFT_F(fir[n] * exp(-2*pi*i*r*n/(ovs*F)))[j].  ovs CTAs per channel: all have just designed
    // the same FIR (steps A-F are cheap and deterministic), CTA r transforms it for the bins of residue r.
    {
        const double scale = c0 / ((double)ovs * (double)F);
        float hpeak = 0.0f;  // max |H| of this CTA's bins: the convolution compares the two channels' peaks
        const double step = -2.0 * (double)parity / ((double)ovs * (double)F);
#pragma unroll
        for (int q = 0; q < PER; ++q) {
            const int i = tid + q * kDesignThreads;
            double sn = 0.0, cs = 1.0;
            if (parity != 0) sincospi(step * (double)i, &sn, &cs);
            planes.store(i, cpx<double>{taps[q] * cs, taps[q] * sn});
        }
        __syncthreads();
        design_fft<F>(planes, tw);
        __syncthreads();
        // bins ovs*j + parity <= ovs*F/2  (j = F/2 only for parity 0, where it wraps to the real bin F/2 of FFT_F)
        const int jmax = (ovs * F / 2 - parity) / ovs;
        for (int j = tid; j <= jmax; j += nthr) {
            const int jj = j & (F - 1);
            const float2 h = make_float2((float)(re[fft_pad(jj)] * scale), (float)(im[fft_pad(jj)] * scale));
            H[ovs * j + parity] = h;
            hpeak = fmaxf(hpeak, sqrtf(h.x * h.x + h.y * h.y));
        }
        __shared__ float red_peak[32];
        hpeak = block_max(hpeak, red_peak);
        if (tid == 0 && state) atomic_max_nonneg(ch == 0 ? &state->fir_peak_mid_bits : &state->fir_peak_side_bits, hpeak);
    }
}

template <int F>
__global__ void __launch_bounds__(kDesignThreads)
design_kernel(mgb_plan plan, DesignArgs a) {
    constexpr int HB = F / 2 + 1;
    MGB_DYN_SMEM(smem);
    const int tid = threadIdx.x, nthr = blockDim.x;
    const int ch = blockIdx.x / a.ovs;
    const int parity = blockIdx.x % a.ovs;  // which residue class of the FIR spectrum's bins this CTA produces (step G)
    // (global planes: behind the design vectors of this CTA's scratch block, see design_doubles_per_channel)
    double* re = DesignSmem<F>::kGlobalPlanes
                     ? a.scratch + ((long long)(kDesignBlocks * ch) + parity) * a.stride + (a.stride - 2 * DesignSmem<F>::kPlane)
                     : reinterpret_cast<double*>(smem);
    double* im = re + DesignSmem<F>::kPlane;
    const SplitPlanes<double> planes{re, im};
    const int NL = plan.n_log;
    const cpx<double>* tw = (const cpx<double>*)plan.d_tw_f64_F;

    // scratch blocks: [channel][parity]; the matching curve m (and, on the operator path, the smoothed
    // curve s) are produced into the parity-0 block by the kernels that ran before
    double* base0 = a.scratch + (long long)(kDesignBlocks * ch) * a.stride;
    double* base = base0 + (long long)parity * a.stride;
    double* m = base;                       // [HB] matching curve
    double* s = (a.s_ready ? base0 : base) + 2 * HB;  // [HB] smoothed curve on the linear grid

    const double eps = plan.min_value;
    double c0 = 1.0, coef = 1.0;
    if (a.state) {
        c0 = a.state->rms_coefficient;
        coef = a.state->final_amplitude_coef;
    }

    // ---- A: matching curve = reference average / max(eps, target average) ---------------------
    if (a.avg_override) {
        for (int k = tid; k < HB; k += nthr) {
            const double at = a.avg_override[(long long)ch * HB + k];
            const double ar = a.avg_override[(long long)(2 + ch) * HB + k];
            m[k] = ar / fmax(eps, at);
        }
    } else if (parity != 0 && !a.s_ready) {
        for (int k = tid; k < HB; k += nthr) m[k] = base0[k];  // own copy: the direct chain works in place
    }  // otherwise spectrum_mean_kernel / ratio_kernel has already written m into the parity-0 block
    __syncthreads();

    // ---- B-E: smoothing on the log-frequency grid, unless the operator kernel already produced s ---
    if (!a.s_ready) smooth_curve(plan, base);

    // ---- F-G: the FIR and its spectrum on the convolution's grid ----------------------------------
    design_fir_spectrum<F>(planes, tw, plan.d_hann, [&](int k) { return s[k]; }, ch, parity, a.ovs, c0, a.fir_out,
                           ch == 0 ? a.h_mid : a.h_side, a.state);
}

// ---- native-rate jobs: the analysis job's curve on the native rate's FIR grid --------------------------------
// (mgb_match_frequencies_native; DESIGN.md section 4 "Native-rate masters")
struct NativeDesignArgs {
    const double* curve;        // the analysis job's smoothed curve of channel 0 (its parity-0 design block, at 2 n_lin)
    long long curve_stride;     // doubles from channel 0's curve to channel 1's
    const int* idx;             // [F/2 + 2] the native plan's tables (mgb_plan::d_native_idx, d_native_w)
    const double* w;
    double* scratch;            // the native workspace's design blocks (the float64 planes at F = 16384)
    long long stride;
    double* fir_out;            // [2][F] or null
    float2* h_mid;
    float2* h_side;
    mgb_track_state* state;     // the native job's state: c0 from the analysis, the FIR peaks recorded here
    int ovs;
};

// s'[j] = s[i] + w (s[i+1] - s[i]) up to the edge f_e; above it exp((1 - t) ln g_e), g_e = s(f_e) (the tables' last
// entry), which crossfades to g_inf = 1 at R/2 and holds it; g_e <= 1 gives g_inf = g_e, a constant.  Then steps F-G
// at the native length, exactly as design_kernel runs them.
template <int F>
__global__ void __launch_bounds__(kDesignThreads)
design_native_kernel(mgb_plan plan, NativeDesignArgs a) {
    constexpr int HB = F / 2 + 1;
    MGB_DYN_SMEM(smem);
    const int ch = blockIdx.x / a.ovs;
    const int parity = blockIdx.x % a.ovs;
    double* re = DesignSmem<F>::kGlobalPlanes
                     ? a.scratch + ((long long)(kDesignBlocks * ch) + parity) * a.stride + (a.stride - 2 * DesignSmem<F>::kPlane)
                     : reinterpret_cast<double*>(smem);
    const SplitPlanes<double> planes{re, re + DesignSmem<F>::kPlane};
    const double* s = a.curve + (long long)ch * a.curve_stride;
    const double ge = s[a.idx[HB]] + a.w[HB] * (s[a.idx[HB] + 1] - s[a.idx[HB]]);
    const double log_ge = ge > 1.0 ? log(ge) : 0.0;
    auto curve = [&](int j) {
        const int i = a.idx[j];
        if (i >= 0) return s[i] + a.w[j] * (s[i + 1] - s[i]);
        return ge > 1.0 ? exp((1.0 - a.w[j]) * log_ge) : ge;
    };
    design_fir_spectrum<F>(planes, (const cpx<double>*)plan.d_tw_f64_F, plan.d_hann, curve, ch, parity, a.ovs,
                           a.state->rms_coefficient, a.fir_out, ch == 0 ? a.h_mid : a.h_side, a.state);
}

__global__ void ratio_kernel(const double* __restrict__ avg, double* __restrict__ scratch, long long stride, int n_lin,
                             double eps) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x, ch = blockIdx.y;
    if (k < n_lin) scratch[(long long)(kDesignBlocks * ch) * stride + k] = avg[(long long)(2 + ch) * n_lin + k] / fmax(eps, avg[(long long)ch * n_lin + k]);
}

// ---- the smoothing as a Config-only matrix ------------------------------------------------------
// s = S m with S [n_lin][n_lin]: column c of S is smooth_curve applied to the unit vector e_c.
// Built once per plan by running the direct algorithm on every unit vector (persistent CTAs, one
// scratch block each); per track the whole spline/LOWESS/spline chain is then one GEMV spread over
// the GPU instead of two latency-bound CTAs.
__global__ void __launch_bounds__(256)
operator_columns_kernel(mgb_plan plan, double* scratch, long long stride, double* st /*[n_lin][n_lin], column-major S*/) {
    const int HB = plan.n_lin;
    double* base = scratch + (long long)blockIdx.x * stride;
    for (int c = blockIdx.x; c < HB; c += gridDim.x) {
        for (int k = threadIdx.x; k < HB; k += blockDim.x) base[k] = (k == c) ? 1.0 : 0.0;
        __syncthreads();
        smooth_curve(plan, base);
        const double* s = base + 2 * HB;
        for (int k = threadIdx.x; k < HB; k += blockDim.x) st[(long long)c * HB + k] = s[k];
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256)
transpose_kernel(const double* __restrict__ in, double* __restrict__ out, int n) {
    __shared__ double tile[32][33];
    const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
    for (int r = ty; r < 32; r += 8)
        if (by + r < n && bx + tx < n) tile[r][tx] = in[(long long)(by + r) * n + bx + tx];
    __syncthreads();
    for (int r = ty; r < 32; r += 8)
        if (bx + r < n && by + tx < n) out[(long long)(bx + r) * n + by + tx] = tile[tx][r];
}

// s[ch] = S m[ch] for both channels from the row bands of S; one warp per row, four rows per CTA.  A row is
// ~300 doubles (at most ~530) at the default Config: each lane takes pairs with 16-byte loads, all of a
// lane's loads (at most 9 pairs) issued before the first use.
__global__ void __launch_bounds__(128)
smooth_operator_kernel(const double* __restrict__ S, const int4* __restrict__ rows, double* __restrict__ scratch,
                       long long stride, int n_lin) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r = blockIdx.x * 4 + warp;
    if (r >= n_lin) return;
    const int4 row = rows[r];  // offset (even), first column, count
    const double2* vals = reinterpret_cast<const double2*>(S + row.x);
    const double* m0 = scratch + row.y;                           // channel 0, parity-0 block
    const double* m1 = scratch + kDesignBlocks * stride + row.y;  // channel 1, parity-0 block
    const int pairs = row.z >> 1;
    double a0 = 0.0, a1 = 0.0, b0 = 0.0, b1 = 0.0;
    for (int base = 0; base < pairs; base += 32 * 4) {
        double2 w[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int p = base + lane + 32 * u;
            w[u] = p < pairs ? vals[p] : make_double2(0.0, 0.0);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int p = base + lane + 32 * u;
            if (p < pairs) {
                a0 += w[u].x * m0[2 * p];
                a1 += w[u].y * m0[2 * p + 1];
                b0 += w[u].x * m1[2 * p];
                b1 += w[u].y * m1[2 * p + 1];
            }
        }
    }
    if ((row.z & 1) && lane == 0) {
        const double w = S[row.x + row.z - 1];
        a0 += w * m0[row.z - 1];
        b0 += w * m1[row.z - 1];
    }
    const double sa = warp_sum(a0 + a1), sb = warp_sum(b0 + b1);
    if (lane == 0) {
        scratch[2LL * n_lin + r] = sa;
        scratch[kDesignBlocks * stride + 2LL * n_lin + r] = sb;
    }
}

// ---- album mastering: spectrum_mean_kernel's profiled half pooled over the tracks of an album -------------------------
// (mgb_album_match; DESIGN.md section 4 "Album mastering").  The tracks travel as a kernel parameter: no copy on the
// stream, no table in a workspace.
struct AlbumMeanTrack {
    const float* spec_part;    // [D][S][2][n_lin] the track's analysis partials
    const double* sumsq_part;  // [D][S]
    const float* absmax_part;  // [D*S + 1]
    unsigned char* mask;       // [D] out: the track's pieces in the album's loud mask
    float* target_peak;        // out: the track's own peak (its convolution's choice of precision)
    mgb_track_state* state;    // out: the album's level statistics
    long long piece, frames_per_piece;
    int div, slots;
};
struct AlbumMeanTable {
    AlbumMeanTrack t[MGB_MAX_ALBUM_TRACKS];
    int count;
};

// The album's pieces in track order are one list of G = sum D_t pieces; everything the single-track kernel does per
// piece and per (piece, slot) item runs over that list in the same order, so a one-track album is the profiled job
// bit for bit.  grid = (ceil(n_lin/32), 2), as spectrum_mean_kernel.
__global__ void __launch_bounds__(kMeanBins * kMeanSlices)
album_mean_kernel(const __grid_constant__ AlbumMeanTable tab, const mgb_reference_profile* __restrict__ profile,
                  double* __restrict__ scratch, long long stride, int n_lin, int fft_size, double eps, PrefetchList pf) {
    constexpr int BINS = kMeanBins, SLICES = kMeanSlices;
    __shared__ double part_t[SLICES][BINS + 1];
    __shared__ int piece_off[MGB_MAX_ALBUM_TRACKS + 1], sel_off[MGB_MAX_ALBUM_TRACKS + 1];
    __shared__ LevelsResult lv_s;
    __shared__ long long frames_s;  // boxcar frames of the loud pieces of every track
    MGB_DYN_SMEM(smem);
    const int K = tab.count;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    {
        const long long gtid = ((long long)blockIdx.y * gridDim.x + blockIdx.x) * blockDim.x + threadIdx.x;
        const long long gsize = (long long)gridDim.x * gridDim.y * blockDim.x;
        for (int t = 0; t < pf.count; ++t)
            for (long long off = gtid * 128; off < pf.bytes[t]; off += gsize * 128)
                prefetch_l2(reinterpret_cast<const char*>(pf.ptr[t]) + off);
    }
    if (threadIdx.x == 0) {
        piece_off[0] = 0;
        for (int t = 0; t < K; ++t) piece_off[t + 1] = piece_off[t] + tab.t[t].div;
    }
    __syncthreads();
    const int G = piece_off[K];
    auto track_of = [&](int g) {
        int t = 0;
        while (piece_off[t + 1] <= g) ++t;
        return t;
    };
    unsigned char* mask = smem;                                                   // [G]
    double* piece_sum = reinterpret_cast<double*>(smem + (G + 15) / 16 * 16);     // [G]
    int* piece_rank = reinterpret_cast<int*>(piece_sum + G);                      // [G]
    unsigned* sel = reinterpret_cast<unsigned*>(piece_rank + (G + 1) / 2 * 2);    // [sum of items]: track << 16 | item
    if (blockIdx.x == 0 && blockIdx.y == 0) {  // each track's own peak, for its convolution
        for (int t = warp; t < K; t += nwarps) {
            float tpk = 0.0f;
            for (int i = lane; i < tab.t[t].div * tab.t[t].slots + 1; i += 32) tpk = fmaxf(tpk, tab.t[t].absmax_part[i]);
            tpk = warp_max_f(tpk);
            if (lane == 0) *tab.t[t].target_peak = tpk;
        }
    }
    for (int g = warp; g < G; g += nwarps) {
        const int t = track_of(g);
        const int slots = tab.t[t].slots;
        const double* part = tab.t[t].sumsq_part + (long long)(g - piece_off[t]) * slots;
        double sum = 0.0;
        for (int k = lane; k < slots; k += 32) sum += part[k];
        sum = warp_sum(sum);
        if (lane == 0) piece_sum[g] = sum;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        // signal_levels_warp over the album's pieces, each with its own track's piece length
        double acc = 0.0;
        for (int g = lane; g < G; g += 32) {
            const double r = sqrt(piece_sum[g] / (double)tab.t[track_of(g)].piece);
            acc += r * r;
        }
        const double avg = sqrt(warp_sum(acc) / (double)G);
        double accm = 0.0, cnt = 0.0;
        for (int g = lane; g < G; g += 32) {
            const double r = sqrt(piece_sum[g] / (double)tab.t[track_of(g)].piece);
            const bool m = r >= avg;
            mask[g] = m ? 1 : 0;
            if (m) {
                accm += r * r;
                cnt += 1.0;
            }
        }
        const double tm = warp_sum(accm);
        const double tc = warp_sum(cnt);
        LevelsResult mine;
        mine.peak = profile->reference_peak;
        mine.coef = profile->final_amplitude_coef;
        mine.match_t = sqrt(tm / tc);
        mine.match_r = profile->reference_match_rms;
        mine.c0 = mine.match_r / fmax(eps, mine.match_t);
        mine.loud_t = (int)tc;
        mine.loud_r = profile->reference_loud_pieces;
        __syncwarp();
        // each track's loud pieces ranked as spectrum_mean_kernel ranks one signal's; the album's item list is the
        // tracks' lists one after another
        int items = 0;
        long long frames = 0;
        for (int t = 0; t < K; ++t) {
            const int div = tab.t[t].div, off = piece_off[t];
            int count = 0;
            for (int base_p = 0; base_p < div; base_p += 32) {
                const int p = base_p + lane;
                const bool keep = p < div && mask[off + p];
                const unsigned votes = __ballot_sync(0xffffffffu, keep);
                if (p < div) piece_rank[off + p] = count + __popc(votes & ((1u << lane) - 1u));
                count += __popc(votes);
            }
            if (lane == 0) sel_off[t] = items;
            items += count * tab.t[t].slots;
            frames += (long long)count * tab.t[t].frames_per_piece;
        }
        if (lane == 0) {
            sel_off[K] = items;
            frames_s = frames;
            lv_s = mine;
        }
    }
    __syncthreads();
    const LevelsResult lv = lv_s;
    if (blockIdx.x == 0 && blockIdx.y == 0) {
        if (threadIdx.x < K) {
            mgb_track_state* st = tab.t[threadIdx.x].state;
            levels_store(lv, st);
            st->conv_peak_bits = 0.0f;
            st->fir_peak_mid_bits = 0.0f;
            st->fir_peak_side_bits = 0.0f;
            st->conv_precise = 0;
        }
        for (int g = threadIdx.x; g < G; g += blockDim.x) {
            const int t = track_of(g);
            tab.t[t].mask[g - piece_off[t]] = mask[g];
        }
    }
    for (int t = 0; t < K; ++t) {  // every thread files its share of each track's items: piece by piece, slot by slot
        const int slots = tab.t[t].slots, off = piece_off[t];
        const int items = tab.t[t].div * slots;
        unsigned* out = sel + sel_off[t];
        for (int it = threadIdx.x; it < items; it += blockDim.x) {
            const int p = it / slots;
            if (mask[off + p]) out[piece_rank[off + p] * slots + (it - p * slots)] = ((unsigned)t << 16) | (unsigned)it;
        }
    }
    __syncthreads();
    const int bx = threadIdx.x % BINS, sy = threadIdx.x / BINS;
    const int k = blockIdx.x * BINS + bx;
    const int ch = blockIdx.y;
    double st = 0.0;
    if (k < n_lin) {
        const int count = sel_off[K];
        for (int i = sy; i < count; i += 8 * SLICES) {
            float v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int iu = i + u * SLICES;
                float x = 0.0f;
                if (iu < count) {
                    const unsigned e = sel[iu];
                    x = tab.t[e >> 16].spec_part[((long long)(e & 0xffffu) * 2 + ch) * n_lin + k];
                }
                v[u] = x;
            }
            st += (((double)v[0] + (double)v[1]) + ((double)v[2] + (double)v[3])) +
                  (((double)v[4] + (double)v[5]) + ((double)v[6] + (double)v[7]));
        }
    }
    part_t[sy][bx] = st;
    __syncthreads();
    if (sy == 0 && k < n_lin) {
        for (int q = 1; q < SLICES; ++q) st += part_t[q][bx];
        const double norm_t = lv.c0 / ((double)frames_s * (double)fft_size);
        const double* spectra = reinterpret_cast<const double*>(profile + 1);
        scratch[(long long)(kDesignBlocks * ch) * stride + k] = spectra[(long long)ch * n_lin + k] / fmax(eps, st * norm_t);
    }
}

// dynamic shared memory of spectrum_mean_kernel: both masks, the per-piece sums and the two item lists
size_t spectrum_mean_smem(int div_t, int64_t items_t, int div_r, int64_t items_r) {
    return (size_t)((div_t + div_r + 15) / 16 * 16 + (int64_t)(div_t + div_r) * 8 + (items_t + items_r) * 2 + 16);
}

template <int F>
int launch_design_t(const mgb_plan& plan, const DesignArgs& a, cudaStream_t stream) {
    return launch("design_kernel", design_kernel<F>, dim3(2 * a.ovs), dim3(kDesignThreads), DesignSmem<F>::kBytes, stream, plan, a);
}

int launch_design_kernel(const mgb_plan& plan, const DesignArgs& a, cudaStream_t stream) {
    switch (plan.fft_size) {
        case 512: return launch_design_t<512>(plan, a, stream);
        case 1024: return launch_design_t<1024>(plan, a, stream);
        case 2048: return launch_design_t<2048>(plan, a, stream);
        case 4096: return launch_design_t<4096>(plan, a, stream);
        case 8192: return launch_design_t<8192>(plan, a, stream);
        case 16384: return launch_design_t<16384>(plan, a, stream);
        default: break;
    }
    set_error("design: fft_size %d has no kernel", plan.fft_size);
    return MGB_ERR_UNSUPPORTED;
}

}  // namespace

int64_t design_doubles_per_channel(const mgb_plan& plan) {
    int64_t n = 3LL * plan.n_lin + 4LL * plan.n_log + plan.fft_size + 16;
    n = (n + 31) / 32 * 32;
    if (plan.fft_size > 8192) n += 2LL * fft_padded_size(plan.fft_size) + 32;  // the design FFT's planes (DesignSmem::kGlobalPlanes)
    return n;
}

int g_design_direct = 0;

int64_t operator_workspace_bytes(const mgb_plan& plan) {
    const int64_t ctas = plan.n_lin < 2 * num_sms() ? plan.n_lin : 2 * num_sms();
    const int64_t stride = (design_doubles_per_channel(plan) + 31) / 32 * 32;
    return ctas * stride * 8 + (int64_t)plan.n_lin * plan.n_lin * 8 + 512;
}

int build_operator(const mgb_plan& plan, double* op_out, void* workspace, cudaStream_t stream) {
    const int ctas = plan.n_lin < 2 * num_sms() ? plan.n_lin : 2 * num_sms();
    const int64_t stride = (design_doubles_per_channel(plan) + 31) / 32 * 32;
    double* scratch = (double*)workspace;
    double* st = scratch + ctas * stride;
    MGB_TRY(launch("operator_columns_kernel", operator_columns_kernel, dim3(ctas), dim3(256), 0, stream, plan, scratch,
                   (long long)stride, st));
    const unsigned tiles = (plan.n_lin + 31) / 32;
    return launch("transpose_kernel", transpose_kernel, dim3(tiles, tiles), dim3(256), 0, stream, (const double*)st, op_out,
                  plan.n_lin);
}

int launch_design(const mgb_plan& plan, const mgb_track_layout& layout, const Workspace& ws,
                  const double* avg_override, double* fir_out, mgb_track_state* state, cudaStream_t stream) {
    DesignArgs a;
    a.spec_part_t = ws.spec_part_t;
    a.spec_part_r = ws.spec_part_r;
    a.mask_t = ws.mask_t;
    a.mask_r = ws.mask_r;
    a.absmax_t = ws.absmax_part_t;
    a.target_peak = ws.target_peak;
    a.levels.sumsq_t = ws.sumsq_part_t;
    a.levels.sumsq_r = ws.sumsq_part_r;
    a.levels.absmax_r = ws.absmax_part_r;
    a.levels.piece_t = layout.target_piece;
    a.levels.piece_r = layout.reference_piece;
    a.levels.div_t = layout.target_divisions;
    a.levels.slots_t = layout.target_slots;
    a.levels.div_r = layout.reference_divisions;
    a.levels.slots_r = layout.reference_slots;
    a.levels.threshold = plan.threshold;
    a.levels.eps = plan.min_value;
    a.levels.div_r_items_override = 0;
    a.div_t = layout.target_divisions;
    a.slots_t = layout.target_slots;
    a.div_r = layout.reference_divisions;
    a.slots_r = layout.reference_slots;
    a.frames_per_piece_t = layout.target_piece / plan.fft_size;
    a.frames_per_piece_r = layout.reference_piece / plan.fft_size;
    a.avg_override = avg_override;
    a.scratch = ws.design;
    a.stride = ws.design_stride;
    a.fir_out = fir_out;
    a.h_mid = ws.h_mid;
    a.h_side = ws.h_side;
    a.state = avg_override ? nullptr : state;
    a.s_ready = 0;
    a.ovs = conv_frame_ovs(plan.fft_size, layout.target_piece);
    if (!avg_override) {
        PrefetchList pf;
        pf.count = 0;
        auto add = [&](const void* p, long long bytes) {
            if (p && pf.count < 14) {
                pf.ptr[pf.count] = p;
                pf.bytes[pf.count] = bytes;
                pf.count++;
            }
        };
        const long long nl = plan.n_lin, ng = plan.n_log, F = plan.fft_size;
        add(plan.d_sa_hinv, (nl - 1) * 8);
        add(plan.d_sa_lu, 3 * (nl - 2) * 8);
        add(plan.d_sa_eval_idx, ng * 4);
        add(plan.d_sa_eval_w, ng * 32);
        add(plan.d_sb_hinv, (ng - 1) * 8);
        add(plan.d_sb_lu, 3 * (ng - 2) * 8);
        add(plan.d_sb_eval_idx, nl * 4);
        add(plan.d_sb_eval_w, nl * 32);
        add(plan.d_lw_fit_left, (long long)plan.lowess_nfit * 4);
        add(plan.d_lw_row_idx, (long long)plan.lowess_nfit * 4);
        add(plan.d_lw_seg, ng * 4);
        add(plan.d_lw_alpha, ng * 8);
        add(plan.d_lw_rows, (long long)plan.lowess_nrows * plan.lowess_k * 8);
        add(plan.d_hann, F * 8);
        const dim3 grid((plan.n_lin + kMeanBins - 1) / kMeanBins, 2);
        const size_t smem = spectrum_mean_smem(layout.target_divisions, (int64_t)layout.target_divisions * layout.target_slots,
                                               layout.reference_divisions,
                                               (int64_t)layout.reference_divisions * layout.reference_slots);
        ProfileIO io;
        memset(&io, 0, sizeof(io));
        if (ws.profile) {  // a profiled layout: the reference half comes from the workspace's copy of the profile
            io.in = ws.profile;
            MGB_TRY(launch("spectrum_mean_profiled_kernel", spectrum_mean_kernel<MeanMode::kProfiled>, grid,
                           dim3(kMeanBins * kMeanSlices), smem, stream, a, plan.n_lin, plan.fft_size, plan.min_value, pf, io));
        } else {
            MGB_TRY(launch("spectrum_mean_kernel", spectrum_mean_kernel<MeanMode::kPaired>, grid, dim3(kMeanBins * kMeanSlices),
                           smem, stream, a, plan.n_lin, plan.fft_size, plan.min_value, pf, io));
        }
    }
    if (plan.d_smooth_op && plan.d_smooth_op_rows && !(avg_override && g_design_direct)) {
        if (avg_override) {
            // test entry: the matching curve has to exist before the GEMV
            MGB_TRY(launch("ratio_kernel", ratio_kernel, dim3((plan.n_lin + 255) / 256, 2), dim3(256), 0, stream, avg_override,
                           a.scratch, a.stride, plan.n_lin, plan.min_value));
            a.avg_override = nullptr;
        }
        MGB_TRY(launch("smooth_operator_kernel", smooth_operator_kernel, dim3((plan.n_lin + 3) / 4), dim3(128), 0, stream,
                       plan.d_smooth_op, (const int4*)plan.d_smooth_op_rows, a.scratch, a.stride, plan.n_lin));
        a.s_ready = 1;
    }
    return launch_design_kernel(plan, a, stream);
}

int launch_design_native(const mgb_plan& plan, const Workspace& ws, const mgb_plan& nplan, const mgb_track_layout& nlayout,
                         const Workspace& nws, double* fir_out, mgb_track_state* nstate, cudaStream_t stream) {
    NativeDesignArgs a;
    a.curve = ws.design + 2LL * plan.n_lin;
    a.curve_stride = (long long)kDesignBlocks * ws.design_stride;
    a.idx = nplan.d_native_idx;
    a.w = nplan.d_native_w;
    a.scratch = nws.design;
    a.stride = nws.design_stride;
    a.fir_out = fir_out;
    a.h_mid = nws.h_mid;
    a.h_side = nws.h_side;
    a.state = nstate;
    a.ovs = conv_frame_ovs(nplan.fft_size, nlayout.target_piece);
#define MGB_NATIVE_CASE(FF)                                                                                           \
    case FF:                                                                                                          \
        return launch("design_native_kernel<" #FF ">", design_native_kernel<FF>, dim3(2 * a.ovs), dim3(kDesignThreads), \
                      DesignSmem<FF>::kBytes, stream, nplan, a);
    switch (nplan.fft_size) {
        MGB_NATIVE_CASE(512)
        MGB_NATIVE_CASE(1024)
        MGB_NATIVE_CASE(2048)
        MGB_NATIVE_CASE(4096)
        MGB_NATIVE_CASE(8192)
        MGB_NATIVE_CASE(16384)
        default: break;
    }
#undef MGB_NATIVE_CASE
    set_error("design_native: fft_size %d has no kernel", nplan.fft_size);
    return MGB_ERR_UNSUPPORTED;
}

int launch_reference_profile(const mgb_plan& plan, const ReferenceGeometry& g, const ReferenceRegions& r,
                             mgb_reference_profile* out, cudaStream_t stream) {
    DesignArgs a;
    memset(&a, 0, sizeof(a));
    a.spec_part_r = r.spec_part;
    a.mask_r = r.mask;
    a.levels.sumsq_r = r.sumsq_part;
    a.levels.absmax_r = r.absmax_part;
    a.levels.piece_r = g.piece;
    a.levels.div_r = g.divisions;
    a.levels.slots_r = g.slots;
    a.levels.threshold = plan.threshold;
    a.levels.eps = plan.min_value;
    a.div_r = g.divisions;
    a.slots_r = g.slots;
    a.frames_per_piece_r = g.piece / plan.fft_size;
    PrefetchList pf;
    memset(&pf, 0, sizeof(pf));
    ProfileIO io;
    memset(&io, 0, sizeof(io));
    io.out = out;
    mgb_reference_profile& h = io.header;
    h.version = MGB_REFERENCE_PROFILE_VERSION;
    h.sample_rate = plan.sample_rate;
    h.fft_size = plan.fft_size;
    h.n_lin = plan.n_lin;
    h.max_piece_size = plan.max_piece_size;
    h.threshold = plan.threshold;
    h.min_value = plan.min_value;
    h.reference_frames = g.frames;
    h.reference_piece = g.piece;
    h.reference_divisions = g.divisions;
    return launch("reference_profile_kernel", spectrum_mean_kernel<MeanMode::kProfile>,
                  dim3((plan.n_lin + kMeanBins - 1) / kMeanBins, 2), dim3(kMeanBins * kMeanSlices),
                  spectrum_mean_smem(0, 0, g.divisions, (int64_t)g.divisions * g.slots), stream, a, plan.n_lin, plan.fft_size,
                  plan.min_value, pf, io);
}

size_t album_mean_smem(const AlbumTrack* tracks, int count) {
    int64_t pieces = 0, items = 0;
    for (int t = 0; t < count; ++t) {
        pieces += tracks[t].layout.target_divisions;
        items += (int64_t)tracks[t].layout.target_divisions * tracks[t].layout.target_slots;
    }
    return (size_t)((pieces + 15) / 16 * 16 + pieces * 8 + (pieces + 1) / 2 * 8 + items * 4 + 16);
}

int launch_album_mean(const mgb_plan& plan, const AlbumTrack* tracks, int count, const mgb_reference_profile* profile,
                      double* design, int64_t design_stride, cudaStream_t stream) {
    AlbumMeanTable tab;
    memset(&tab, 0, sizeof(tab));
    tab.count = count;
    for (int t = 0; t < count; ++t) {
        const mgb_track_layout& L = tracks[t].layout;
        const Workspace& ws = tracks[t].ws;
        AlbumMeanTrack& d = tab.t[t];
        d.spec_part = ws.spec_part_t;
        d.sumsq_part = ws.sumsq_part_t;
        d.absmax_part = ws.absmax_part_t;
        d.mask = ws.mask_t;
        d.target_peak = ws.target_peak;
        d.state = tracks[t].state;
        d.piece = L.target_piece;
        d.frames_per_piece = L.target_piece / plan.fft_size;
        d.div = L.target_divisions;
        d.slots = L.target_slots;
    }
    // (the design kernels' tables, pulled back into L2 as spectrum_mean_kernel does)
    PrefetchList pf;
    memset(&pf, 0, sizeof(pf));
    auto add = [&](const void* p, long long bytes) {
        if (p && pf.count < 14) {
            pf.ptr[pf.count] = p;
            pf.bytes[pf.count] = bytes;
            pf.count++;
        }
    };
    const long long nl = plan.n_lin, ng = plan.n_log;
    add(plan.d_sa_hinv, (nl - 1) * 8);
    add(plan.d_sa_lu, 3 * (nl - 2) * 8);
    add(plan.d_sa_eval_idx, ng * 4);
    add(plan.d_sa_eval_w, ng * 32);
    add(plan.d_sb_hinv, (ng - 1) * 8);
    add(plan.d_sb_lu, 3 * (ng - 2) * 8);
    add(plan.d_sb_eval_idx, nl * 4);
    add(plan.d_sb_eval_w, nl * 32);
    add(plan.d_lw_fit_left, (long long)plan.lowess_nfit * 4);
    add(plan.d_lw_row_idx, (long long)plan.lowess_nfit * 4);
    add(plan.d_lw_seg, ng * 4);
    add(plan.d_lw_alpha, ng * 8);
    add(plan.d_lw_rows, (long long)plan.lowess_nrows * plan.lowess_k * 8);
    add(plan.d_hann, (long long)plan.fft_size * 8);
    return launch("album_mean_kernel", album_mean_kernel, dim3((plan.n_lin + kMeanBins - 1) / kMeanBins, 2),
                  dim3(kMeanBins * kMeanSlices), album_mean_smem(tracks, count), stream, tab, profile, design,
                  (long long)design_stride, plan.n_lin, plan.fft_size, plan.min_value, pf);
}

int launch_design_fir(const mgb_plan& plan, double* design, int64_t design_stride, int ovs, float2* h_mid, float2* h_side,
                      double* fir_out, mgb_track_state* state, cudaStream_t stream) {
    DesignArgs a;
    memset(&a, 0, sizeof(a));
    a.scratch = design;
    a.stride = design_stride;
    a.fir_out = fir_out;
    a.h_mid = h_mid;
    a.h_side = h_side;
    a.state = state;
    a.ovs = ovs;
    if (plan.d_smooth_op && plan.d_smooth_op_rows) {
        MGB_TRY(launch("smooth_operator_kernel", smooth_operator_kernel, dim3((plan.n_lin + 3) / 4), dim3(128), 0, stream,
                       plan.d_smooth_op, (const int4*)plan.d_smooth_op_rows, a.scratch, a.stride, plan.n_lin));
        a.s_ready = 1;
    }
    return launch_design_kernel(plan, a, stream);
}

}  // namespace mgb
