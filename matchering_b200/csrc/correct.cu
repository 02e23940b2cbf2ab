// K5 -- RMS correction and the small elementwise kernels of __finalize.
//
// Replaces (reference file:line):
//   stages.__correct_levels                       matchering/stages.py:138-170
//     dsp.clip                                    matchering/dsp.py:109-110
//     get_average_rms / get_lpis_and_match_rms    stage_helpers/match_levels.py:62-71,93-103
//     get_rms_c_and_amplify_pair                  stage_helpers/match_levels.py:114-131
//   dsp.normalize(..., normalize_clipped=True)    matchering/dsp.py:93-100 (stages.py:186-191)
//
// The reference rescales result_mid and result after every step; here the coefficients only
// accumulate in mgb_track_state::gain (a float64 on the device) and each later pass multiplies by
// it on the fly.  A step reads only the mid samples loud enough to clip (the convolution's loud
// lists, kernels.cuh) instead of three full-array passes.
#include "kernels.cuh"
#include "tail.cuh"

namespace mgb {

namespace {

// clip(mid*gain)^2 of four samples: the product and the clip in float32 (the samples are float32
// anyway), the squares summed in float64
__device__ __forceinline__ double clip_sq4(float4 v, float gain) {
    const float a = fminf(1.0f, fmaxf(-1.0f, v.x * gain)), b = fminf(1.0f, fmaxf(-1.0f, v.y * gain));
    const float c = fminf(1.0f, fmaxf(-1.0f, v.z * gain)), d = fminf(1.0f, fmaxf(-1.0f, v.w * gain));
    return (double)a * a + (double)b * b + ((double)c * c + (double)d * d);
}
__device__ __forceinline__ double clip_sq(float v, float gain) {
    const float c = fminf(1.0f, fmaxf(-1.0f, v * gain));  // dsp.clip
    return (double)c * c;
}

// A later step's per-piece sums of clip(mid*gain)^2 (kernels.cuh: kLoudMid); grid = (chunks per piece, pieces).
// From the piece's loud list when that is exact: gain^2 * S_quiet + sum over the list of clip(m*gain)^2, with
// S_quiet = step-0 sum - sum over the list of clip(m)^2 (every term exact in float64: a float squared).  Otherwise
// (the list overflowed, or quiet samples could clip at this gain) from the result, mid = (L + R) / 2.
__global__ void __launch_bounds__(256)
loud_sumsq_kernel(LoudList loud, long long piece, int divisions, int step, double eps, mgb_track_state* __restrict__ state,
                  const double* __restrict__ step0_sums, const double* __restrict__ prev_sums, double* __restrict__ sums) {
    __shared__ double red[32];
    const long long p = blockIdx.y;
    const long long n = loud.count[p];
    const bool fits = n <= loud.capacity;
    // chunk blockIdx.x takes the float4 groups [lo4, hi4) of the row; entries >= n are not part of the list
    const long long n4 = fits ? (n + 3) / 4 : 0;
    const long long per4 = (n4 + gridDim.x - 1) / gridDim.x;
    const long long lo4 = (long long)blockIdx.x * per4;
    const long long hi4 = lo4 + per4 < n4 ? lo4 + per4 : n4;
    const float4* row = reinterpret_cast<const float4*>(loud.values + p * loud.capacity);
    // the first load does not depend on the coefficient: it goes out before the prologue's chain of dependent reads
    long long i = lo4 + threadIdx.x;
    float4 v = i < hi4 ? row[i] : make_float4(0.f, 0.f, 0.f, 0.f);

    // prologue, identical in every CTA: the previous step's coefficient from its per-piece sums, and
    // the gain accumulated so far (stages.py:161-168 applied lazily)
    const double c_prev = correction_coefficient(prev_sums, divisions, piece, eps, state->reference_match_rms);  // per warp, no barrier
    double gain = c_prev;
    for (int j = 0; j < step - 1; ++j) gain *= state->correction[j];
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
        state->correction[step - 1] = c_prev;  // no CTA of this launch reads this slot
        state->steps_done = step;
    }
    const float gain_f = (float)gain;
    double acc = 0.0;
    if (fits && gain * (double)kLoudMid <= 1.0 - kLoudMargin) {
        double loud_g = 0.0, loud_1 = 0.0;
        while (i < hi4) {
            float4 w = v;
            const long long e = 4 * i;  // entry of w.x (< n)
            i += blockDim.x;
            if (i < hi4) v = row[i];  // next group in flight while this one is reduced
            if (e + 1 >= n) w.y = 0.0f;
            if (e + 2 >= n) w.z = 0.0f;
            if (e + 3 >= n) w.w = 0.0f;
            loud_g += clip_sq4(w, gain_f);
            loud_1 += clip_sq4(w, 1.0f);
        }
        // the quiet samples cannot clip: their part is gain^2 * S_quiet, in float64
        acc = loud_g - gain * gain * loud_1;
        if (blockIdx.x == 0 && threadIdx.x == 0) acc += gain * gain * step0_sums[p];
    } else {
        const float2* res = *loud.result_slot;
        const long long per = (piece + gridDim.x - 1) / gridDim.x;
        const long long lo = p * piece + (long long)blockIdx.x * per;
        const long long hi = lo + per < (p + 1) * piece ? lo + per : (p + 1) * piece;
#pragma unroll 4
        for (long long f = lo + threadIdx.x; f < hi; f += blockDim.x) {
            const float2 x = res[f];
            acc += clip_sq((x.x + x.y) * 0.5f, gain_f);
        }
    }
    const double total = block_sum(acc, red);
    if (threadIdx.x == 0 && total != 0.0) atomicAdd(&sums[p], total);
}

// after the last step: its coefficient, the total gain, the result's peak, the limiter's early-out
// flag (hyrax.py:83-85) and the normalisation coefficient (stages.py:186-191); one CTA
__global__ void __launch_bounds__(32)
correction_final_kernel(const double* __restrict__ last_sums, int divisions, long long piece, int steps, double eps,
                        double threshold, mgb_track_state* __restrict__ state) {
    double gain = 1.0;
    if (steps > 0) {
        const double c_last = correction_coefficient(last_sums, divisions, piece, eps, state->reference_match_rms);
        gain = c_last;
        for (int j = 0; j < steps - 1; ++j) gain *= state->correction[j];
        if (threadIdx.x == 0) state->correction[steps - 1] = c_last;
    }
    if (threadIdx.x == 0) {
        state->steps_done = steps;
        state->gain = gain;
        const double peak = (double)state->conv_peak_bits * gain;
        state->result_peak = peak;
        state->normalize_coef = fmax(eps, peak / threshold);  // dsp.py:99 with normalize_clipped=True
        const double r = fmax(peak, threshold) / threshold;   // dsp.py:117-121 at the loudest frame
        state->limiter_engaged = (fabs(r - 1.0) <= 1e-8 + 1e-5) ? 0 : 1;  // np.isclose defaults, hyrax.py:83
    }
}

// out = in * gain / divisor, two frames per thread
__global__ void __launch_bounds__(256)
scale_kernel(const float4* __restrict__ in, float4* __restrict__ out, long long pairs, const float2* __restrict__ in_tail,
             float2* __restrict__ out_tail, const double* __restrict__ gain, const double* __restrict__ divisor) {
    double g = gain ? *gain : 1.0;
    if (divisor) g /= *divisor;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += stride) {
        const float4 v = in[i];
        out[i] = make_float4((float)((double)v.x * g), (float)((double)v.y * g), (float)((double)v.z * g),
                             (float)((double)v.w * g));
    }
    if (in_tail && blockIdx.x == 0 && threadIdx.x == 0) {
        const float2 v = *in_tail;
        *out_tail = make_float2((float)((double)v.x * g), (float)((double)v.y * g));
    }
}

__global__ void __launch_bounds__(256)
absmax_kernel(const float2* __restrict__ in, long long frames, float* __restrict__ out_bits) {
    __shared__ float red[32];
    float pk = 0.0f;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < frames; i += stride) {
        const float2 v = in[i];
        pk = fmaxf(pk, fmaxf(fabsf(v.x), fabsf(v.y)));
    }
    pk = block_max(pk, red);
    if (threadIdx.x == 0) atomic_max_nonneg(out_bits, pk);
}

__global__ void convert_f64_f32_kernel(const double* __restrict__ in, float* __restrict__ out, long long count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) out[i] = (float)in[i];
}
__global__ void convert_f32_f64_kernel(const float* __restrict__ in, double* __restrict__ out, long long count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) out[i] = (double)in[i];
}

// ---- PCM <-> float32 at the file boundary (SURVEY.md 8f: loader / saver) ---------------------------
// decode: libsndfile's integer -> float read, x / 2^(bits-1)  (what sf.read hands the reference,
// matchering/loader.py:35).  encode: its float -> integer write, lrint(x * (2^(bits-1) - 1)) with
// clipping (matchering/saver.py:32).  24-bit samples are packed little-endian triplets.
__global__ void __launch_bounds__(256)
pcm16_decode_kernel(const short* __restrict__ in, float* __restrict__ out, long long count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long pairs = count >> 1;
    const short2* in2 = reinterpret_cast<const short2*>(in);
    float2* out2 = reinterpret_cast<float2*>(out);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += stride) {
        const short2 v = in2[i];
        out2[i] = make_float2((float)v.x * (1.0f / 32768.0f), (float)v.y * (1.0f / 32768.0f));
    }
    if ((count & 1) && blockIdx.x == 0 && threadIdx.x == 0) out[count - 1] = (float)in[count - 1] * (1.0f / 32768.0f);
}

__global__ void __launch_bounds__(256)
pcm24_decode_kernel(const unsigned char* __restrict__ in, float* __restrict__ out, long long count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
        const unsigned char* p = in + 3 * i;
        int v = (int)p[0] | ((int)p[1] << 8) | ((int)(signed char)p[2] << 16);
        out[i] = (float)v * (1.0f / 8388608.0f);
    }
}

// In double, like libsndfile's d2s/d2bet writers the reference reaches with its float64 arrays: the
// product x * top is exact in float64 (24 + 23 significant bits), so ties round exactly as lrint does
// there; a float32 product would be rounded to 24 bits first and could land one LSB away.
__device__ __forceinline__ int quantize(float x, double top) {
    const double q = rint((double)x * top);  // round half to even, like lrint
    return (int)fmin(top, fmax(-top - 1.0, q));
}

__global__ void __launch_bounds__(256)
pcm16_encode_kernel(const float* __restrict__ in, short* __restrict__ out, long long count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long pairs = count >> 1;
    const float2* in2 = reinterpret_cast<const float2*>(in);
    short2* out2 = reinterpret_cast<short2*>(out);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += stride) {
        const float2 v = in2[i];
        short2 q;
        q.x = (short)quantize(v.x, 32767.0);
        q.y = (short)quantize(v.y, 32767.0);
        out2[i] = q;
    }
    if ((count & 1) && blockIdx.x == 0 && threadIdx.x == 0) out[count - 1] = (short)quantize(in[count - 1], 32767.0);
}

__global__ void __launch_bounds__(256)
pcm24_encode_kernel(const float* __restrict__ in, unsigned char* __restrict__ out, long long count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
        const int q = quantize(in[i], 8388607.0);
        unsigned char* p = out + 3 * i;
        p[0] = (unsigned char)(q & 0xff);
        p[1] = (unsigned char)((q >> 8) & 0xff);
        p[2] = (unsigned char)((q >> 16) & 0xff);
    }
}

// ---- checker reductions (matchering/checker.py:64-88, dsp.count_max_peaks dsp.py:49-54) ------------
// number of samples with |x| "close" to `peak` in numpy.isclose's sense (rtol 1e-5, atol 1e-8)
__global__ void __launch_bounds__(256)
count_close_kernel(const float* __restrict__ x, long long count, const float* __restrict__ peak_bits,
                   unsigned long long* __restrict__ out) {
    const double peak = (double)*peak_bits;
    const double tol = 1e-8 + 1e-5 * peak;
    unsigned long long local = 0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride)
        local += (fabs(fabs((double)x[i]) - peak) <= tol) ? 1ull : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(out, local);
}

// number of samples where two equally long signals differ beyond numpy.allclose's tolerance
__global__ void __launch_bounds__(256)
count_different_kernel(const float* __restrict__ a, const float* __restrict__ b, long long count,
                       unsigned long long* __restrict__ out) {
    unsigned long long local = 0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
        const double x = a[i], y = b[i];
        local += (fabs(x - y) <= 1e-8 + 1e-5 * fabs(y)) ? 0ull : 1ull;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(out, local);
}

// ---- preview creator (matchering/preview_creator.py:30-94; dsp.strided_app_2d / batch_rms_2d / fade
// dsp.py:128-152) --------------------------------------------------------------------------------------
// energy[w] = sum over window w = [w*step, w*step + window) of L^2 + R^2 (float64): the argmax of the
// reference's per-window RMS.  grid = (slices, windows): a CTA sums one slice of one window.
__global__ void __launch_bounds__(256)
window_energy_kernel(const float2* __restrict__ x, long long window, long long step, double* __restrict__ energy) {
    __shared__ double red[32];
    const long long w = blockIdx.y;
    const long long per = (window + gridDim.x - 1) / gridDim.x;
    const long long lo = blockIdx.x * per;
    const long long hi = lo + per < window ? lo + per : window;
    const float2* src = x + w * step;
    double acc = 0.0;
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const float2 v = src[i];
        acc += (double)v.x * (double)v.x + (double)v.y * (double)v.y;
    }
    const double total = block_sum(acc, red);
    if (threadIdx.x == 0 && total != 0.0) atomicAdd(&energy[w], total);
}

// out = clip(in, +-clip_to) (clip_to <= 0: no clip) with linear fades of `fade` frames at both ends:
// fade_in = linspace(0, 1, fade), fade_out its mirror (dsp.fade).
__global__ void __launch_bounds__(256)
preview_piece_kernel(const float2* __restrict__ in, float2* __restrict__ out, long long frames, float clip_to,
                     long long fade) {
    const double ramp = fade > 1 ? 1.0 / (double)(fade - 1) : 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < frames; i += stride) {
        float2 v = in[i];
        if (clip_to > 0.0f) {
            v.x = fminf(clip_to, fmaxf(-clip_to, v.x));
            v.y = fminf(clip_to, fmaxf(-clip_to, v.y));
        }
        double g = 1.0;
        if (i < fade) g = (i == fade - 1 && fade > 1) ? 1.0 : (double)i * ramp;
        const long long j = frames - 1 - i;  // distance from the end
        if (j < fade) g *= (j == fade - 1 && fade > 1) ? 1.0 : (double)j * ramp;
        out[i] = make_float2((float)((double)v.x * g), (float)((double)v.y * g));
    }
}

unsigned grid_for(long long items, int per_block) {
    long long blocks = (items + per_block - 1) / per_block;
    const long long cap = (long long)num_sms() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (unsigned)blocks;
}

}  // namespace

int launch_loud_sumsq(const mgb_plan& plan, const mgb_track_layout& layout, const Workspace& ws, int step,
                      mgb_track_state* state, cudaStream_t stream) {
    // The grid is fixed before the device decides between list and result, so it is sized for a pass over
    // the result (three CTAs per SM); a list, at most a quarter of the piece, leaves most of them a few entries.
    const int div = layout.target_divisions;
    long long per_piece = (3LL * num_sms() + div - 1) / div;
    const long long max_useful = (layout.target_piece + 8191) / 8192;
    if (per_piece > max_useful) per_piece = max_useful;
    if (per_piece < 1) per_piece = 1;
    const LoudList loud{ws.loud_values, ws.loud_count, (long long)ws.loud_capacity, ws.result_slot};
    return launch("loud_sumsq_kernel", loud_sumsq_kernel, dim3((unsigned)per_piece, (unsigned)div), dim3(256), 0, stream, loud,
                  (long long)layout.target_piece, div, step, plan.min_value, state, (const double*)ws.piece_sums,
                  (const double*)(ws.piece_sums + (long long)(step - 1) * div), ws.piece_sums + (long long)step * div);
}

int launch_correction_final(const mgb_plan& plan, const mgb_track_layout& layout, const Workspace& ws,
                            mgb_track_state* state, cudaStream_t stream) {
    const int steps = plan.rms_correction_steps, div = layout.target_divisions;
    const double* last = ws.piece_sums + (long long)(steps > 0 ? steps - 1 : 0) * div;
    return launch("correction_final_kernel", correction_final_kernel, dim3(1), dim3(32), 0, stream, last, div,
                  (long long)layout.target_piece, steps, plan.min_value, plan.threshold, state);
}

int launch_scale(const float2* in, float2* out, int64_t frames, const double* gain, const double* divisor,
                 cudaStream_t stream) {
    const long long pairs = frames / 2;
    const float2* in_tail = (frames & 1) ? in + (frames - 1) : nullptr;
    float2* out_tail = (frames & 1) ? out + (frames - 1) : nullptr;
    return launch("scale_kernel", scale_kernel, dim3(grid_for(pairs, 256)), dim3(256), 0, stream, (const float4*)in,
                  (float4*)out, pairs, in_tail, out_tail, gain, divisor);
}

int launch_absmax(const float2* in, int64_t frames, float* out_bits, cudaStream_t stream) {
    return launch("absmax_kernel", absmax_kernel, dim3(grid_for(frames, 1024)), dim3(256), 0, stream, in,
                  (long long)frames, out_bits);
}

int launch_convert_f64_f32(const double* in, float* out, int64_t count, cudaStream_t stream) {
    return launch("convert_f64_f32_kernel", convert_f64_f32_kernel, dim3(grid_for(count, 1024)), dim3(256), 0, stream, in,
                  out, (long long)count);
}
int launch_convert_f32_f64(const float* in, double* out, int64_t count, cudaStream_t stream) {
    return launch("convert_f32_f64_kernel", convert_f32_f64_kernel, dim3(grid_for(count, 1024)), dim3(256), 0, stream, in,
                  out, (long long)count);
}

int launch_pcm_decode(const void* in, int bits, float* out, int64_t count, cudaStream_t stream) {
    if (bits == 16)
        return launch("pcm16_decode_kernel", pcm16_decode_kernel, dim3(grid_for(count / 2 + 1, 1024)), dim3(256), 0, stream,
                      (const short*)in, out, (long long)count);
    if (bits == 24)
        return launch("pcm24_decode_kernel", pcm24_decode_kernel, dim3(grid_for(count, 1024)), dim3(256), 0, stream,
                      (const unsigned char*)in, out, (long long)count);
    set_error("pcm decode: %d-bit samples have no kernel (16 and 24 do)", bits);
    return MGB_ERR_UNSUPPORTED;
}

int launch_pcm_encode(const float* in, int bits, void* out, int64_t count, cudaStream_t stream) {
    if (bits == 16)
        return launch("pcm16_encode_kernel", pcm16_encode_kernel, dim3(grid_for(count / 2 + 1, 1024)), dim3(256), 0, stream, in,
                      (short*)out, (long long)count);
    if (bits == 24)
        return launch("pcm24_encode_kernel", pcm24_encode_kernel, dim3(grid_for(count, 1024)), dim3(256), 0, stream, in,
                      (unsigned char*)out, (long long)count);
    set_error("pcm encode: %d-bit samples have no kernel (16 and 24 do)", bits);
    return MGB_ERR_UNSUPPORTED;
}

int launch_peak_count(const float* x, int64_t count, float* peak_bits, unsigned long long* n_close, cudaStream_t stream) {
    // peak_bits and n_close must be zeroed by the caller
    MGB_TRY(launch("absmax_kernel", absmax_kernel, dim3(grid_for(count / 2, 1024)), dim3(256), 0, stream, (const float2*)x,
                   (long long)(count / 2), peak_bits));
    return launch("count_close_kernel", count_close_kernel, dim3(grid_for(count, 1024)), dim3(256), 0, stream, x,
                  (long long)count, (const float*)peak_bits, n_close);
}

int launch_window_energy(const float2* x, int64_t window, int64_t step, int count, double* energy, cudaStream_t stream) {
    long long slices = (4LL * num_sms() + count - 1) / count;
    const long long useful = (window + 4095) / 4096;
    if (slices > useful) slices = useful;
    if (slices < 1) slices = 1;
    return launch("window_energy_kernel", window_energy_kernel, dim3((unsigned)slices, (unsigned)count), dim3(256), 0, stream,
                  x, (long long)window, (long long)step, energy);
}

int launch_preview_piece(const float2* in, float2* out, int64_t frames, float clip_to, int64_t fade, cudaStream_t stream) {
    return launch("preview_piece_kernel", preview_piece_kernel, dim3(grid_for(frames, 1024)), dim3(256), 0, stream, in, out,
                  (long long)frames, clip_to, (long long)fade);
}

int launch_count_different(const float* a, const float* b, int64_t count, unsigned long long* n_diff, cudaStream_t stream) {
    return launch("count_different_kernel", count_different_kernel, dim3(grid_for(count, 1024)), dim3(256), 0, stream, a, b,
                  (long long)count, n_diff);
}

}  // namespace mgb
