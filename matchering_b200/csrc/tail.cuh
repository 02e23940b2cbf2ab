// Level statistics and RMS-correction coefficients: the tiny serial steps that follow a grid-wide
// reduction.  They are cheap enough (a few hundred numbers) that every CTA of the NEXT kernel simply
// recomputes them in its prologue from the previous kernel's partial sums -- deterministic, so all
// CTAs agree bit for bit -- instead of paying a single-CTA kernel launch or a last-block handshake
// per step on a pipeline whose whole device time is a few hundred microseconds.
// They run per WARP (lanes stride over the pieces, shuffles reduce): a dozen or so pieces do not fill a
// block, and block-wide reductions cost three barriers each -- 21 barriers for the level statistics,
// 9 per correction coefficient, which was most of the 25 us / 14 us their kernels took.
#pragma once
#include "common.cuh"

namespace mgb {

// ---- level statistics (match_levels.py:29-44, 62-71, 93-111) -------------------------------------
struct LevelsArgs {
    const double* sumsq_t;  // [div_t][slots_t] per-(piece, slot) sums of mid^2 from analyze.cu
    const double* sumsq_r;
    const float* absmax_r;  // [div_r*slots_r + 1]
    long long piece_t, piece_r;
    int div_t, slots_t, div_r, slots_r;
    double threshold, eps;
    int div_r_items_override;  // > 0: absmax_r holds this many entries (already folded), not div_r*slots_r + 1
};

struct LevelsResult {
    double peak;     // max|reference|
    double coef;     // final amplitude coefficient (dsp.normalize with normalize_clipped=False)
    double match_t;  // target match RMS
    double match_r;  // match RMS of the NORMALISED reference
    double c0;       // match_r / max(eps, match_t)
    int loud_t, loud_r;
};

__device__ __forceinline__ double piece_rms(const double* part, int p, int slots, double piece) {
    double s = 0.0;
    for (int k = 0; k < slots; ++k) s += part[(long long)p * slots + k];
    return sqrt(s / piece);  // dsp.py:86
}

__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// normalize_reference's coefficient from the reference's peak (dsp.py:96-99)
__device__ __forceinline__ double reference_coef(double peak, double threshold, double eps) {
    double coef = 1.0;
    if (peak < threshold) coef = fmax(eps, peak / threshold);
    return coef;
}

// One signal's half of the level statistics (match_levels.py:62-71): the match RMS over its loud pieces and their
// number.  All 32 lanes of ONE warp call; if `mask` is not null the warp writes the signal's loudest-piece mask there.
struct SignalLevels {
    double match;
    int loud;
};
__device__ __forceinline__ SignalLevels signal_levels_warp(const double* part, int div, int slots, double piece,
                                                           unsigned char* mask) {
    const int lane = threadIdx.x & 31;
    double acc = 0.0;
    for (int p = lane; p < div; p += 32) {
        const double r = piece_rms(part, p, slots, piece);
        acc += r * r;
    }
    const double avg = sqrt(warp_sum(acc) / (double)div);  // rms(rmses), match_levels.py:101
    double accm = 0.0, cnt = 0.0;
    for (int p = lane; p < div; p += 32) {
        const double r = piece_rms(part, p, slots, piece);
        const bool m = r >= avg;  // match_levels.py:65
        if (mask) mask[p] = m ? 1 : 0;
        if (m) {
            accm += r * r;
            cnt += 1.0;
        }
    }
    const double tm = warp_sum(accm);
    const double tc = warp_sum(cnt);
    return SignalLevels{sqrt(tm / tc), (int)tc};
}

// All 32 lanes of ONE warp call (no block barrier inside); every lane gets the result.  If `mask_t` /
// `mask_r` (shared or global, [div_t] / [div_r]) are not null the warp writes the loudest-piece masks there.
__device__ __forceinline__ LevelsResult levels_compute_warp(const LevelsArgs& a, unsigned char* mask_t, unsigned char* mask_r) {
    const int lane = threadIdx.x & 31;
    LevelsResult out;
    float pk = 0.0f;
    const int peaks = a.div_r_items_override > 0 ? a.div_r_items_override : a.div_r * a.slots_r + 1;
    for (int i = lane; i < peaks; i += 32) pk = fmaxf(pk, a.absmax_r[i]);
    out.peak = (double)warp_max_f(pk);
    out.coef = reference_coef(out.peak, a.threshold, a.eps);
    const SignalLevels t = signal_levels_warp(a.sumsq_t, a.div_t, a.slots_t, (double)a.piece_t, mask_t);
    const SignalLevels r = signal_levels_warp(a.sumsq_r, a.div_r, a.slots_r, (double)a.piece_r, mask_r);
    out.match_t = t.match;
    out.match_r = r.match / out.coef;  // the reference measures the normalised reference
    out.c0 = out.match_r / fmax(a.eps, out.match_t);
    out.loud_t = t.loud;
    out.loud_r = r.loud;
    return out;
}

__device__ __forceinline__ void levels_store(const LevelsResult& r, mgb_track_state* state) {
    state->reference_peak = r.peak;
    state->final_amplitude_coef = r.coef;
    state->target_match_rms = r.match_t;
    state->reference_match_rms = r.match_r;
    state->rms_coefficient = r.c0;
    state->gain = 1.0;
    state->result_peak = 0.0;
    state->normalize_coef = 1.0;
    state->target_loud_pieces = r.loud_t;
    state->reference_loud_pieces = r.loud_r;
    state->limiter_engaged = 1;
    state->steps_done = 0;
    for (int i = 0; i < MGB_MAX_CORRECTION_STEPS; ++i) state->correction[i] = 1.0;
}

// ---- one RMS-correction step's coefficient from its per-piece sums (stages.py:153-168) -------------
// All 32 lanes of a warp call (no block barrier); every lane -- and, the arithmetic being the same in every
// warp, every warp of every CTA -- gets the same coefficient.
__device__ __forceinline__ double correction_coefficient(const double* sums, int divisions, long long piece, double eps,
                                                         double reference_match_rms) {
    const int lane = threadIdx.x & 31;
    double acc = 0.0;
    for (int p = lane; p < divisions; p += 32) acc += sums[p] / (double)piece;  // rms^2
    const double avg = sqrt(warp_sum(acc) / (double)divisions);
    double accm = 0.0, cnt = 0.0;
    for (int p = lane; p < divisions; p += 32) {
        const double r = sqrt(sums[p] / (double)piece);
        if (r >= avg) {
            accm += r * r;
            cnt += 1.0;
        }
    }
    const double tm = warp_sum(accm);
    const double tc = warp_sum(cnt);
    return reference_match_rms / fmax(eps, sqrt(tm / tc));
}

}  // namespace mgb
