// K6w -- the Hyrax limiter for windows wider than the halo kernel's span (limiter.cu): slow attacks, long
// holds, coefficients close to zero and sample rates of 352.8 / 384 kHz.  Same results as limiter_kernel
// (reference file:line in limiter.cu), without the halo: every quantity that crosses a chunk is carried.
//
//   limiter_wide_gain_kernel     g = 1 - thr/max(|L|,|R|,thr) (pre_gain folded in, as in the halo kernel) -> plane g;
//                                per 32-sample block its prefix and suffix maxima -> planes, block maxima -> level 0
//   limiter_wide_sparse_kernel   level j of a sparse table over the block maxima: max of 2^j blocks (one launch
//                                per level, only the levels the widest window needs)
//   A window maximum of g over [l, r] is then max(suffix max at l, prefix max at r, two table entries for the
//   whole blocks between): four loads whatever the window's length (a window inside one block scans it).
//     A[n] = max g[n-reach .. n+reach],  H[n] = max A[n-hold+1 .. n] = max g[n-reach-hold+1 .. n+reach]
//   limiter_wide_attack_kernel   filtfilt's one-pole over the odd extension of A (scipy's 6-sample padding and
//                                steady-state initial state), float64, carries across chunks by decoupled
//                                look-back: forward launch -> float64 plane, backward launch (chunks numbered
//                                from the end, so a chunk only waits for lower block indices) -> plane g_att
//   limiter_wide_apply_kernel    hold and release sections (the halo kernel's scans and look-back), then
//                                out = x * pre * (1 - max(g, g_att, hold, rel)) * post
//
// Workspace per frame: planes g, prefix, suffix and g_att (float32, 16 B), the forward plane (float64, 8 B) and
// (levels + 1) / 8 B of sparse table.
// (included by limiter.cu: one translation unit for both limiter paths)
#pragma once
#include <math.h>

#include "limiter_scan.cuh"

namespace mgb {

namespace {

constexpr int EXT = 6;  // scipy filtfilt's padlen for a one-pole: odd extension by 6 samples at both ends

struct WidePlanes {
    float* g;        // [frames] hard-clip gain
    float* pf;       // [frames] prefix max inside the sample's 32-block
    float* sf;       // [frames] suffix max inside the sample's 32-block
    float* st;       // [levels + 1][nblocks] sparse table over the block maxima
    double* fwd;     // [frames + 2 EXT] the attack filter's forward pass over the extended signal
    float* att;      // [frames] g_att
};

struct WideGeom {
    long long frames, nblocks;
    int reach, hold, levels;
    int publish_inclusive;
};

// max g[l .. r], 0 <= l <= r < frames
__device__ __forceinline__ float range_max(const WidePlanes& p, long long nblocks, long long l, long long r) {
    const long long bl = l >> 5, br = r >> 5;
    if (bl == br) {
        float m = 0.0f;
        for (long long i = l; i <= r; ++i) m = fmaxf(m, p.g[i]);
        return m;
    }
    float m = fmaxf(p.sf[l], p.pf[r]);
    if (br - bl > 1) {
        const long long a = bl + 1, b = br - 1;
        const int j = 31 - __clz((int)(b - a + 1));
        const float* lev = p.st + (long long)j * nblocks;
        m = fmaxf(m, fmaxf(lev[a], lev[b - (1LL << j) + 1]));
    }
    return m;
}
__device__ __forceinline__ float env_a(const WidePlanes& p, const WideGeom& w, long long n) {
    return range_max(p, w.nblocks, n - w.reach > 0 ? n - w.reach : 0, n + w.reach < w.frames ? n + w.reach : w.frames - 1);
}
__device__ __forceinline__ float env_h(const WidePlanes& p, const WideGeom& w, long long n) {
    const long long l = n - w.reach - w.hold + 1;
    return range_max(p, w.nblocks, l > 0 ? l : 0, n + w.reach < w.frames ? n + w.reach : w.frames - 1);
}

__device__ __forceinline__ bool bypassed(const int* engaged) { return engaged && *engaged == 0; }

// GATED (every kernel of this path, loudness_target.cuh): the grid returns at once while *skip is set
template <bool GATED>
__device__ __forceinline__ bool skipped(const int* skip) {
    if constexpr (GATED) return *skip != 0;
    return false;
}

// TP: the true-peak mode's detector plane tp_d in place of max(|L|, |R|) (true_peak.cuh)
template <bool TP, bool GATED = false>
__global__ void __launch_bounds__(256) limiter_wide_gain_kernel(mgb_limiter_params lp, WideGeom w, const float2* __restrict__ in,
                                                                const double* __restrict__ pre_gain, const int* __restrict__ engaged,
                                                                WidePlanes p, const float* __restrict__ tp_d,
                                                                const int* __restrict__ skip) {
    if (skipped<GATED>(skip)) return;
    if (bypassed(engaged)) return;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if ((i >> 5) >= w.nblocks) return;  // (whole warps)
    const int lane = threadIdx.x & 31;
    const double pre = pre_gain ? *pre_gain : 1.0;
    float g = 0.0f;
    if (i < w.frames) {
        // exactly the halo kernel's g (limiter.cu, P1)
        double a;
        if constexpr (TP) {
            a = (double)__ldg(tp_d + i) * pre;
        } else {
            const float2 v = __ldg(in + i);
            a = (double)fmaxf(fabsf(v.x), fabsf(v.y)) * pre;
        }
        const double over = a - lp.threshold;
        if (over > 0.0) g = __fdiv_rn((float)over, (float)a);
    }
    float pf = g, sf = g;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const float up = __shfl_up_sync(0xffffffffu, pf, d);
        const float dn = __shfl_down_sync(0xffffffffu, sf, d);
        if (lane >= d) pf = fmaxf(pf, up);
        if (lane + d < 32) sf = fmaxf(sf, dn);
    }
    if (i < w.frames) {
        p.g[i] = g;
        p.pf[i] = pf;
        p.sf[i] = sf;
    }
    if (lane == 31) p.st[i >> 5] = pf;
}

template <bool GATED = false>
__global__ void __launch_bounds__(256) limiter_wide_sparse_kernel(WideGeom w, const int* __restrict__ engaged, float* st, int level,
                                                                  const int* __restrict__ skip) {
    if (skipped<GATED>(skip)) return;
    if (bypassed(engaged)) return;
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= w.nblocks) return;
    const float* prev = st + (long long)(level - 1) * w.nblocks;
    const long long half = 1LL << (level - 1);
    const float v = prev[k];
    st[(long long)level * w.nblocks + k] = k + half < w.nblocks ? fmaxf(v, prev[k + half]) : v;
}

// The attack filter y = (1-c) x + c y_prev over the extended signal (length frames + 2 EXT) as an order-1 section.
// BACKWARD = false: x = the odd extension of A, state before the first sample = x[0] (scipy's zi = c x[0]); writes the
// forward plane.  BACKWARD = true: runs over the forward plane from its end (block b owns the b-th chunk counted from
// the end), state beyond the last sample = its forward value; writes g_att for the signal's own samples.
// words: [chunks][2] look-back words, forward pass in word 0 of its chunk, backward pass in word 1.
template <bool BACKWARD, bool GATED = false>
__global__ void __launch_bounds__(NT) limiter_wide_attack_kernel(mgb_limiter_params lp, WideGeom w, const int* __restrict__ engaged,
                                                                 WidePlanes p, LookbackWord* __restrict__ words,
                                                                 const unsigned char* __restrict__ tables, const int* __restrict__ skip) {
    __shared__ SectionTab<1> tab;  // the attack pole's powers in the sections' layout
    __shared__ double scratch[32];
    __shared__ double bcast;
    if (skipped<GATED>(skip)) return;
    if (bypassed(engaged)) return;
    const int tid = threadIdx.x;
    {
        // (the tables hold the attack pole's ScanPow for CORE_EPT elements per thread on this path)
        const ScanPow* pw = reinterpret_cast<const ScanPow*>(tables);
        if (tid < CORE_EPT) tab.pe[tid][0] = pw->pe[tid + 1];
        if (tid < 33) {
            tab.ql[tid][0][0] = pw->ql[tid];
            tab.pc[tid][0][0] = pw->pc[tid];
        }
        if (tid < 17) tab.qw[tid][0][0] = pw->qw[tid];
    }
    __syncthreads();
    const int chunk = blockIdx.x;
    const long long m = w.frames + 2 * EXT;  // extended length
    const long long q0 = (long long)chunk * LC + (long long)tid * CORE_EPT;
    const double c = lp.attack_c;
    auto input = [&](long long q) -> double {  // the pass's input at its own position q (0 = where it starts)
        if (BACKWARD) return p.fwd[m - 1 - q];
        if (q < EXT) return 2.0 * (double)env_a(p, w, 0) - (double)env_a(p, w, EXT - q);
        if (q >= w.frames + EXT) return 2.0 * (double)env_a(p, w, w.frames - 1) - (double)env_a(p, w, 2 * w.frames + EXT - 2 - q);
        return (double)env_a(p, w, q - EXT);
    };
    double y[CORE_EPT];
    double acc = 0.0;
#pragma unroll
    for (int e = 0; e < CORE_EPT; ++e) {
        const long long q = q0 + e;
        acc = (1.0 - c) * (q < m ? input(q) : 0.0) + c * acc;
        y[e] = acc;
    }
    if (chunk == 0 && tid == 0) bcast = input(0);  // the state before the first sample
    StVec<1> end;
    end.v[0] = acc;
    const StVec<1> carry = section_scan<1>(end, &tab, scratch);  // (its barrier also publishes bcast)
    LookbackWord* own = words + (long long)chunk * 2 + (BACKWARD ? 1 : 0);
    double cin;
    if (chunk == 0) {
        cin = bcast;  // known at once: chunk 0 publishes its inclusive state only
    } else {
        if (tid == NT - 1) {
            StVec<1> agg = end;
            st_addmul<1>(agg, tab.ql[1], carry);
            publish_state<1>(own, agg, 1);
        }
        if (tid < 32) {
            const StVec<1> v = lookback<1>(words + (BACKWARD ? 1 : 0), chunk, &tab);
            if (tid == 0) bcast = v.v[0];
        }
        __syncthreads();
        cin = bcast;
    }
    StVec<1> cs;
    cs.v[0] = cin;
    const double prev = carry.v[0] + section_lead<1>(&tab, cs).v[0];
#pragma unroll
    for (int e = 0; e < CORE_EPT; ++e) y[e] += tab.pe[e][0] * prev;
    if (tid == NT - 1 && (chunk == 0 || w.publish_inclusive)) {
        StVec<1> fin;
        fin.v[0] = y[CORE_EPT - 1];
        publish_state<1>(own, fin, 2);
    }
#pragma unroll
    for (int e = 0; e < CORE_EPT; ++e) {
        const long long q = q0 + e;
        if (q >= m) break;
        if (!BACKWARD) {
            p.fwd[q] = y[e];
        } else {
            const long long n = m - 1 - q - EXT;  // the signal's sample
            if (n >= 0 && n < w.frames) p.att[n] = (float)y[e];
        }
    }
}

// Hold and release sections (limiter.cu, P3 / P5 / P6: the same scans and look-back) over H from the window
// maxima, then the gain and its application (P7).  GAINS (tests): write (g_att, max(hold_out, release_out)).
// VERS (linked versions): every entry of *vp (the main first) takes the same gain and the same early-out.
template <int NO, bool GAINS, bool GATED, bool VERS>
__device__ __forceinline__ void limiter_wide_apply_body(mgb_limiter_params lp, WideGeom w,
                                                        const float2* __restrict__ in, float2* __restrict__ out,
                                                        const double* __restrict__ pre_gain, const double* __restrict__ post_gain,
                                                        const int* __restrict__ engaged, WidePlanes p,
                                                        LookbackWord* __restrict__ slots, const unsigned char* __restrict__ tables,
                                                        const int* __restrict__ skip, const VersionPlanes* vp) {
    if (skipped<GATED>(skip)) return;
    constexpr int HC = CORE_EPT + NO;
    __shared__ SectionTab<1> pw_sec[2];  // (order capacity 1 only: the two sections' tables)
    __shared__ double scratch_a[32 * NO], scratch_b[32 * NO];
    __shared__ double bcast[2 * NO];
    __shared__ double gain_s[LC];  // 1 - max(g, g_att, hold, rel), filters' mapping, read back coalesced
    const SectionTab<NO>* sec_global = reinterpret_cast<const SectionTab<NO>*>(tables + sizeof(ScanPow));
    const SectionTab<NO>* tab_hold = NO == 1 ? reinterpret_cast<const SectionTab<NO>*>(&pw_sec[0]) : sec_global;
    const SectionTab<NO>* tab_rel = NO == 1 ? reinterpret_cast<const SectionTab<NO>*>(&pw_sec[1]) : sec_global + 1;
    const int tid = threadIdx.x;
    const int chunk = blockIdx.x;
    const long long s0 = (long long)chunk * LC;
    const int core_n = (int)((s0 + LC < w.frames) ? LC : w.frames - s0);
    const double pre = pre_gain ? *pre_gain : 1.0;
    const double post = post_gain ? *post_gain : 1.0;
    if (bypassed(engaged)) {  // hyrax.py:83-85: the limiter is not needed
        if constexpr (VERS) {
            for (int j = 0; j < vp->count; ++j)
                for (int k = tid; k < core_n; k += NT) {
                    const float2 v = vp->in[j][s0 + k];
                    vp->out[j][s0 + k] = make_float2((float)((double)v.x * pre * post), (float)((double)v.y * pre * post));
                }
        } else {
            for (int k = tid; k < core_n; k += NT) {
                const float2 v = in[s0 + k];
                out[s0 + k] = make_float2((float)((double)v.x * pre * post), (float)((double)v.y * pre * post));
            }
        }
        return;
    }
    if (NO == 1) {
        const double* src = reinterpret_cast<const double*>(tables + sizeof(ScanPow));
        double* dst = reinterpret_cast<double*>(pw_sec);
        for (int i = tid; i < (int)(2 * sizeof(SectionTab<1>) / sizeof(double)); i += NT) dst[i] = src[i];
    }
    // H at the thread's CORE_EPT samples and the NO before them (lfilter starts from rest: 0 before the signal)
    const long long bh = s0 + (long long)tid * CORE_EPT - NO;
    float hc[HC];
#pragma unroll
    for (int e = 0; e < HC; ++e) {
        const long long n = bh + e;
        hc[e] = (n >= 0 && n < w.frames) ? env_h(p, w, n) : 0.0f;
    }
    __syncthreads();  // the section tables are in shared memory

    // ---- hold_out = lfilter(butter(order, f_hold), H) (hyrax.py:61-66)
    LookbackWord* slot_hold = slots + (long long)chunk * (2 * NO);
    LookbackWord* slot_rel = slot_hold + NO;
    double hold_y[CORE_EPT];
#pragma unroll
    for (int e = 0; e < CORE_EPT; ++e) {
        double acc = lp.hold_b[0] * (double)hc[e + NO];
#pragma unroll
        for (int i = 1; i <= NO; ++i) acc += lp.hold_b[i] * (double)hc[e + NO - i];
#pragma unroll
        for (int i = 1; i <= NO; ++i)
            if (e - i >= 0) acc -= lp.hold_a[i] * hold_y[e - i];
        hold_y[e] = acc;
    }
    StVec<NO> hold_prev;
    {
        StVec<NO> end;
#pragma unroll
        for (int i = 0; i < NO; ++i) end.v[i] = hold_y[CORE_EPT - 1 - i];
        hold_prev = section_scan<NO>(end, tab_hold, scratch_a);
        if (tid == NT - 1) {
            st_addmul<NO>(end, tab_hold->ql[1], hold_prev);
            publish_state<NO>(slot_hold, end, 1);
        }
        if (tid < 32) {
            const StVec<NO> cin = lookback<NO>(slots, chunk, tab_hold);
            if (tid == 0) {
#pragma unroll
                for (int i = 0; i < NO; ++i) bcast[i] = cin.v[i];
            }
        }
        __syncthreads();
        StVec<NO> cin;
#pragma unroll
        for (int i = 0; i < NO; ++i) cin.v[i] = bcast[i];
        const StVec<NO> lead = section_lead<NO>(tab_hold, cin);
#pragma unroll
        for (int i = 0; i < NO; ++i) hold_prev.v[i] += lead.v[i];
#pragma unroll
        for (int e = 0; e < CORE_EPT; ++e)
#pragma unroll
            for (int i = 0; i < NO; ++i) hold_y[e] += tab_hold->pe[e][i] * hold_prev.v[i];
        if (tid == NT - 1 && w.publish_inclusive) {
#pragma unroll
            for (int i = 0; i < NO; ++i) end.v[i] = hold_y[CORE_EPT - 1 - i];
            publish_state<NO>(slot_hold, end, 2);
        }
    }

    // ---- release_out = lfilter(butter(order, f_rel), max(H, hold_out)) (hyrax.py:68-73)
    {
        double rel_y[CORE_EPT];
        double win[HC];
#pragma unroll
        for (int i = 0; i < NO; ++i) win[i] = fmax((double)hc[i], hold_prev.v[NO - 1 - i]);
#pragma unroll
        for (int e = 0; e < CORE_EPT; ++e) win[NO + e] = fmax((double)hc[NO + e], hold_y[e]);
#pragma unroll
        for (int e = 0; e < CORE_EPT; ++e) {
            double acc = lp.release_b[0] * win[e + NO];
#pragma unroll
            for (int i = 1; i <= NO; ++i) acc += lp.release_b[i] * win[e + NO - i];
#pragma unroll
            for (int i = 1; i <= NO; ++i)
                if (e - i >= 0) acc -= lp.release_a[i] * rel_y[e - i];
            rel_y[e] = acc;
        }
        StVec<NO> end;
#pragma unroll
        for (int i = 0; i < NO; ++i) end.v[i] = rel_y[CORE_EPT - 1 - i];
        StVec<NO> rel_prev = section_scan<NO>(end, tab_rel, scratch_b);
        if (tid == NT - 1) {
            st_addmul<NO>(end, tab_rel->ql[1], rel_prev);
            publish_state<NO>(slot_rel, end, 1);
        }
        if (tid < 32) {
            const StVec<NO> cr = lookback<NO>(slots + NO, chunk, tab_rel);
            if (tid == 0) {
#pragma unroll
                for (int i = 0; i < NO; ++i) bcast[NO + i] = cr.v[i];
            }
        }
        __syncthreads();
        {
            StVec<NO> cin;
#pragma unroll
            for (int i = 0; i < NO; ++i) cin.v[i] = bcast[NO + i];
            const StVec<NO> lead = section_lead<NO>(tab_rel, cin);
#pragma unroll
            for (int i = 0; i < NO; ++i) rel_prev.v[i] += lead.v[i];
        }
#pragma unroll
        for (int e = 0; e < CORE_EPT; ++e) {
#pragma unroll
            for (int i = 0; i < NO; ++i) rel_y[e] += tab_rel->pe[e][i] * rel_prev.v[i];
            const int k = tid * CORE_EPT + e;
            const double g_rel = fmax(hold_y[e], rel_y[e]);  // hyrax.py:75
            if (k < core_n) {
                const float att = p.att[s0 + k];
                if (GAINS) out[s0 + k] = make_float2(att, (float)g_rel);
                else gain_s[k] = 1.0 - fmax((double)fmaxf(p.g[s0 + k], att), g_rel);  // hyrax.py:97
            }
        }
        if (tid == NT - 1 && w.publish_inclusive) {
#pragma unroll
            for (int i = 0; i < NO; ++i) end.v[i] = rel_y[CORE_EPT - 1 - i];
            publish_state<NO>(slot_rel, end, 2);
        }
    }
    if (GAINS) return;
    __syncwarp();  // a warp applies the gains of its own 32*CORE_EPT consecutive samples

    // ---- apply (hyrax.py:99, stages.py:203), coalesced as in the halo kernel
    const double scale = pre * post;
    const int wbase = (tid >> 5) * (32 * CORE_EPT) + (tid & 31);
    if constexpr (VERS) {
        for (int j = 0; j < vp->count; ++j) {
            const float2* src = vp->in[j];
            float2* dst = vp->out[j];
#pragma unroll
            for (int q = 0; q < CORE_EPT; ++q) {
                const int k = wbase + q * 32;
                if (k < core_n) {
                    const float2 v = __ldg(src + s0 + k);
                    const double gain = gain_s[k] * scale;
                    dst[s0 + k] = make_float2((float)((double)v.x * gain), (float)((double)v.y * gain));
                }
            }
        }
    } else {
#pragma unroll
        for (int q = 0; q < CORE_EPT; ++q) {
            const int k = wbase + q * 32;
            if (k < core_n) {
                const float2 v = __ldg(in + s0 + k);
                const double gain = gain_s[k] * scale;
                out[s0 + k] = make_float2((float)((double)v.x * gain), (float)((double)v.y * gain));
            }
        }
    }
}

template <int NO, bool GAINS, bool GATED = false>
__global__ void __launch_bounds__(NT) limiter_wide_apply_kernel(mgb_limiter_params lp, WideGeom w, const float2* __restrict__ in,
                                                                float2* __restrict__ out, const double* __restrict__ pre_gain,
                                                                const double* __restrict__ post_gain, const int* __restrict__ engaged,
                                                                WidePlanes p, LookbackWord* __restrict__ slots,
                                                                const unsigned char* __restrict__ tables, const int* __restrict__ skip) {
    limiter_wide_apply_body<NO, GAINS, GATED, false>(lp, w, in, out, pre_gain, post_gain, engaged, p, slots, tables, skip, nullptr);
}

// the linked limiter's apply step (limiter_versions_kernel's P7 and early-out on the wide-window path)
template <int NO>
__global__ void __launch_bounds__(NT) limiter_wide_apply_versions_kernel(mgb_limiter_params lp, WideGeom w,
                                                                         const double* __restrict__ pre_gain,
                                                                         const double* __restrict__ post_gain,
                                                                         const int* __restrict__ engaged, WidePlanes p,
                                                                         LookbackWord* __restrict__ slots,
                                                                         const unsigned char* __restrict__ tables,
                                                                         const __grid_constant__ VersionPlanes vp) {
    limiter_wide_apply_body<NO, false, false, true>(lp, w, vp.in[0], vp.out[0], pre_gain, post_gain, engaged, p, slots, tables,
                                                    nullptr, &vp);
}

struct WideLayout {
    long long nblocks, chunks, ext_chunks;
    int levels;
    int64_t off_g, off_pf, off_sf, off_st, off_fwd, off_att, plane_bytes;
};

inline int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

WideLayout wide_layout(const mgb_limiter_params& lp, int64_t frames) {
    WideLayout L;
    L.nblocks = (frames + 31) / 32;
    L.chunks = (frames + LC - 1) / LC;
    L.ext_chunks = (frames + 2 * EXT + LC - 1) / LC;
    // whole blocks strictly inside the widest window (H: 2 reach + hold samples), at most all of them
    long long run = ((long long)2 * lp.reach + lp.hold) / 32;
    if (run > L.nblocks) run = L.nblocks;
    L.levels = 0;
    while ((2LL << L.levels) <= run) ++L.levels;
    int64_t off = 0;
    auto take = [&](int64_t bytes) {
        const int64_t o = off;
        off += align256(bytes);
        return o;
    };
    L.off_g = take(frames * 4);
    L.off_pf = take(frames * 4);
    L.off_sf = take(frames * 4);
    L.off_st = take((int64_t)(L.levels + 1) * L.nblocks * 4);
    L.off_fwd = take((frames + 2 * EXT) * 8);
    L.off_att = take(frames * 4);
    L.plane_bytes = off;
    return L;
}

}  // namespace

// [chunks][2 * order capacity] section words (the halo kernel's layout), then [ext_chunks][2] attack words
int64_t limiter_wide_lookback_bytes(const mgb_limiter_params& lp, int64_t frames, int order_capacity) {
    const WideLayout L = wide_layout(lp, frames);
    return align256((L.chunks * 2 * order_capacity + L.ext_chunks * 2) * (int64_t)sizeof(LookbackWord));
}

int64_t limiter_wide_plane_bytes(const mgb_limiter_params& lp, int64_t frames) { return wide_layout(lp, frames).plane_bytes; }

int launch_limiter_wide(const mgb_limiter_params& lp, int order_capacity, int publish_inclusive, const float2* in, float2* out,
                        int64_t frames, const double* pre_gain, const double* post_gain, const int* engaged, void* lookback,
                        void* planes, const void* tables, cudaStream_t stream, bool gains_only, const float* tp_d,
                        const int* skip, const VersionPlanes* vp) {
    MGB_REQUIRE(planes != nullptr, MGB_ERR_INVALID, "limiter (wide windows): workspace planes missing");
    const WideLayout L = wide_layout(lp, frames);
    unsigned char* base = (unsigned char*)planes;
    WidePlanes p;
    p.g = (float*)(base + L.off_g);
    p.pf = (float*)(base + L.off_pf);
    p.sf = (float*)(base + L.off_sf);
    p.st = (float*)(base + L.off_st);
    p.fwd = (double*)(base + L.off_fwd);
    p.att = (float*)(base + L.off_att);
    WideGeom w;
    w.frames = frames;
    w.nblocks = L.nblocks;
    w.reach = lp.reach;
    w.hold = lp.hold;
    w.levels = L.levels;
    w.publish_inclusive = publish_inclusive;
    const unsigned char* tab = (const unsigned char*)tables;
    LookbackWord* sec_words = (LookbackWord*)lookback;
    LookbackWord* att_words = sec_words + L.chunks * 2 * order_capacity;
    const dim3 gain_grid((unsigned)((L.nblocks * 32 + 255) / 256));
    // (skip != null: the gated instances of a loudness-target search's passes; never with gains_only)
    auto gain = [&](auto kernel) {
        return launch("limiter_wide_gain_kernel", kernel, gain_grid, dim3(256), 0, stream, lp, w, in, pre_gain, engaged, p, tp_d, skip);
    };
    if (skip) MGB_TRY(tp_d ? gain(limiter_wide_gain_kernel<true, true>) : gain(limiter_wide_gain_kernel<false, true>));
    else MGB_TRY(tp_d ? gain(limiter_wide_gain_kernel<true>) : gain(limiter_wide_gain_kernel<false>));
    for (int level = 1; level <= L.levels; ++level) {
        auto sparse = [&](auto kernel) {
            return launch("limiter_wide_sparse_kernel", kernel, dim3((unsigned)((L.nblocks + 255) / 256)), dim3(256), 0, stream, w,
                          engaged, p.st, level, skip);
        };
        MGB_TRY(skip ? sparse(limiter_wide_sparse_kernel<true>) : sparse(limiter_wide_sparse_kernel<>));
    }
    auto attack = [&](auto kernel) {
        return launch("limiter_wide_attack_kernel", kernel, dim3((unsigned)L.ext_chunks), dim3(NT), 0, stream, lp, w, engaged, p,
                      att_words, tab, skip);
    };
    MGB_TRY(skip ? attack(limiter_wide_attack_kernel<false, true>) : attack(limiter_wide_attack_kernel<false>));
    MGB_TRY(skip ? attack(limiter_wide_attack_kernel<true, true>) : attack(limiter_wide_attack_kernel<true>));
    if (vp) {
        auto linked = [&](auto kernel) {
            return launch("limiter_wide_apply_versions_kernel", kernel, dim3((unsigned)L.chunks), dim3(NT), 0, stream, lp, w,
                          pre_gain, post_gain, engaged, p, sec_words, tab, *vp);
        };
        return order_capacity == 1 ? linked(limiter_wide_apply_versions_kernel<1>)
                                   : linked(limiter_wide_apply_versions_kernel<MGB_MAX_FILTER_ORDER>);
    }
    auto go = [&](auto kernel) {
        return launch("limiter_wide_apply_kernel", kernel, dim3((unsigned)L.chunks), dim3(NT), 0, stream, lp, w, in, out, pre_gain,
                      post_gain, engaged, p, sec_words, tab, skip);
    };
    if (skip)
        return order_capacity == 1 ? go(limiter_wide_apply_kernel<1, false, true>)
                                   : go(limiter_wide_apply_kernel<MGB_MAX_FILTER_ORDER, false, true>);
    if (order_capacity == 1) return gains_only ? go(limiter_wide_apply_kernel<1, true>) : go(limiter_wide_apply_kernel<1, false>);
    return gains_only ? go(limiter_wide_apply_kernel<MGB_MAX_FILTER_ORDER, true>) : go(limiter_wide_apply_kernel<MGB_MAX_FILTER_ORDER, false>);
}

}  // namespace mgb
