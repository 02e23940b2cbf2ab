// K6 -- the Hyrax brickwall limiter as one chained-scan kernel.
//
// Replaces (reference file:line):
//   dsp.rectify, dsp.flip, dsp.max_mix            matchering/dsp.py:113-125
//   limiter.__sliding_window_fast                 matchering/limiter/hyrax.py:32-40
//   limiter.__process_attack                      matchering/limiter/hyrax.py:43-53
//     (scipy.signal.filtfilt of a one-pole: odd extension by 6, steady-state initial state)
//   limiter.__process_release                     matchering/limiter/hyrax.py:56-75
//     (two scipy.signal.lfilter first-order Butterworth sections, zero initial state)
//   limiter.limit                                 matchering/limiter/hyrax.py:78-99
//   the result scaling dsp.amplify(result, final_amplitude_coefficient)   stages.py:203
//
// One CTA masters one chunk of kLimiterCore samples, chunks are handed out in order by a ticket:
//   g      = 1 - thr/max(|L|,|R|,thr)                       (float64 math, kept as float32)
//   A      = centred running max of g over +-reach          (log-step doubling in shared memory)
//   g_att  = backward(forward(A)) one-pole, float64 state   (blocked scan; the pole is fast, so a
//            `warmup`-sample halo on both sides replaces cross-chunk carries to < 1e-10)
//   H      = trailing running max of A over `hold`
//   hold   = IIR(H), rel = IIR(max(H, hold))                (Butterworth low-passes of order 1..2 as
//            scipy.signal.lfilter runs them; float64 blocked scans over the filter's state vector --
//            the last `order` outputs -- whose carries cross chunks by decoupled look-back: aggregate
//            first, inclusive when known.  Order 1, the reference default, is a scalar scan.)
//   out    = x * (1 - max(g, g_att, hold, rel)) * post_gain
// HBM traffic: 8 B/frame read (+ the halo, which hits L2) and 8 B/frame written.
#include <math.h>
#include <string.h>

#include "limiter_scan.cuh"
#include "limiter_wide.cuh"  // the wide-window path: windows wider than this kernel's span

namespace mgb {

namespace {

constexpr int SPAN_EPT_MAX = kLimiterSpanEptMax;

// Exclusive carry of the recurrence y = u + p*y_prev across the block: given each thread's local
// end value B (zero initial state over its elements), returns the state just before the thread's
// first element when the state before the block's first element is c0.
// One barrier: warps scan their own 32 values with shuffles, publish the warp totals, and then EVERY
// warp scans the (at most 32) totals itself instead of waiting for one warp to do it.
// scratch: >= 32 doubles, and must not be the buffer the previous call used (callers alternate
// between two), which is what makes the leading "scratch is free again" barrier unnecessary.
// Every thread of the block must call.
__device__ __forceinline__ double scan_carry(double B, const ScanPow* t, double c0, double* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double v = B;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const double up = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += t->ql[d] * up;
    }
    if (lane == 31) scratch[warp] = v;
    __syncthreads();
    double w = lane < NT / 32 ? scratch[lane] : 0.0;
#pragma unroll
    for (int d = 1; d < NT / 32; d <<= 1) {
        const double up = __shfl_up_sync(0xffffffffu, w, d);
        if (lane >= d) w += t->qw[d] * up;
    }
    // state at the end of the previous warp (zero block carry): inclusive total of warps 0..warp-1
    const double warp_carry = __shfl_sync(0xffffffffu, w, (warp + 31) & 31);
    double prev = __shfl_up_sync(0xffffffffu, v, 1);
    if (lane == 0) prev = 0.0;
    return prev + t->ql[lane] * ((warp > 0 ? warp_carry : 0.0) + t->qw[warp] * c0);
}

// The same for a recurrence that runs from the block's LAST element to its first (thread NT-1 first):
// B is the thread's local end value after its elements were taken in descending order, *c0 the state
// just beyond the block's last element (read after the barrier, so the caller may have written it to
// shared memory just before the call); returns the state just beyond the thread's last element.
__device__ __forceinline__ double scan_carry_rev(double B, const ScanPow* t, const double* c0, double* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int rl = 31 - lane, rw = NT / 32 - 1 - warp;  // ranks in processing order
    double v = B;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const double up = __shfl_down_sync(0xffffffffu, v, d);
        if (rl >= d) v += t->ql[d] * up;
    }
    if (lane == 0) scratch[rw] = v;
    __syncthreads();
    double w = lane < NT / 32 ? scratch[lane] : 0.0;
#pragma unroll
    for (int d = 1; d < NT / 32; d <<= 1) {
        const double up = __shfl_up_sync(0xffffffffu, w, d);
        if (lane >= d) w += t->qw[d] * up;
    }
    const double warp_carry = __shfl_sync(0xffffffffu, w, (rw + 31) & 31);
    double prev = __shfl_down_sync(0xffffffffu, v, 1);
    if (rl == 0) prev = 0.0;
    return prev + t->ql[rl] * ((rw > 0 ? warp_carry : 0.0) + t->qw[rw] * (*c0));
}

struct LimiterGeom {
    int reach, hold, warm, left;  // left = max(warm, hold): left halo of the envelope A
    int ept;                      // span elements per thread (odd)
    int span;                     // samples of g the chunk touches
    int filt;                     // samples the attack filter needs to run over (LC + left + warm)
    int publish_inclusive;        // 0: chunks publish aggregates only (test switch: every look-back then walks to the cut-off)
    int shared_core;              // both windows are wide enough for the per-thread shared-core evaluation
    int margin;                   // zeros kept on both sides of G so that window reads need no bounds test (multiple of 4)
    int use_ticket;               // chunks handed out by an atomic ticket instead of the block index
};

// Config-only tables, computed once per parameter set (not per CTA: pow() is slow).  Order capacity 1: powers of
// the three poles, on the device.
__global__ void limiter_tables_kernel(mgb_limiter_params lp, int span_ept, unsigned char* tables) {
    const int i = threadIdx.x;
    ScanPow* att = reinterpret_cast<ScanPow*>(tables);
    {
        const double p = lp.attack_c;
        if (i < SPAN_EPT_MAX + 2) att->pe[i] = pow(p, (double)i);
        if (i < 33) att->ql[i] = pow(p, (double)(span_ept * i));
        if (i < 17) att->qw[i] = pow(p, (double)(span_ept * 32 * i));
        if (i < 33) att->pc[i] = pow(p, (double)LC * (double)i);
    }
    SectionTab<1>* sec = reinterpret_cast<SectionTab<1>*>(tables + sizeof(ScanPow));
    for (int f = 0; f < 2; ++f) {
        const double p = f == 0 ? -lp.hold_a[1] : -lp.release_a[1];
        SectionTab<1>* t = sec + f;
        if (i < CORE_EPT) t->pe[i][0] = pow(p, (double)(i + 1));
        if (i < 33) t->ql[i][0][0] = pow(p, (double)(CORE_EPT * i));
        if (i < 17) t->qw[i][0][0] = pow(p, (double)(CORE_EPT * 32 * i));
        if (i < 33) t->pc[i][0][0] = pow(p, (double)LC * (double)i);
        for (int j = i; j < kLookbackJumps; j += blockDim.x) t->pj[j][0][0] = pow(p, (double)LC * 32.0 * (double)j);
    }
}

// NO = order capacity of the hold and release sections: 1 (the reference defaults: scalar scans, tables in shared
// memory) or MGB_MAX_FILTER_ORDER = 2 (orders 1..2 zero-padded to 2; tables read through L1).
// GAINS (tests only, mgb_test_limiter_gains): instead of the limited samples, write the two float64-scan results
// per frame: (g_att, the attack filter's gain; max(hold_out, release_out), the release gain).
// TP (true-peak mode, true_peak.cuh): P1 rectifies the detector plane tp_d instead of max(|L|, |R|); the samples are
// read only where the output is formed.
// GATED (loudness targets, loudness_target.cuh): the whole grid returns at once while *skip is set -- a pass the
// search did not need.
// VERS (linked versions, mgb_finalize_versions): TP's detector plane holds D, the maximum over the main and its versions;
// every entry of *vp (the main first) takes the same gain in P7 and the same early-out.  limiter_kernel and
// limiter_versions_kernel below are this body with and without it.
template <int EPT, int NO, bool GAINS, bool TP, bool GATED, bool VERS>
__device__ __forceinline__ void
limiter_body(mgb_limiter_params lp, LimiterGeom gm, const float2* __restrict__ in, float2* __restrict__ out,
             long long frames, const double* __restrict__ pre_gain, const double* __restrict__ post_gain,
             const int* __restrict__ engaged, int* __restrict__ ticket, LookbackWord* __restrict__ slots,
             const unsigned char* __restrict__ tables, const float* __restrict__ tp_d, const int* __restrict__ skip,
             const VersionPlanes* vp) {
    if constexpr (GATED) {
        if (*skip) return;
    }
    constexpr int HC = CORE_EPT + NO;  // H samples a thread needs: its core and the NO before it
    constexpr int CAP = EPT * NT;
    MGB_DYN_SMEM(smem);
    double* Fd = reinterpret_cast<double*>(smem);                 // [CAP] float64 work plane
    float* Aenv = reinterpret_cast<float*>(smem) + CAP;           // [CAP] attack envelope, aliases Fd's upper half
    // [margin zeros][CAP hard-clip gain, later max(g, g_att)][margin zeros]: window samples outside the span read as 0
    float* G = reinterpret_cast<float*>(smem + (size_t)CAP * 8) + gm.margin;
    float* Wk = G + CAP + gm.margin;                              // [CAP] suffix maxima, later the hold envelope
    __shared__ float blockmax[NT];
    __shared__ ScanPow pw_att;
    __shared__ SectionTab<1> pw_sec[2];  // (order capacity 1 only: the two sections' tables)
    __shared__ double scratch_a[32 * NO], scratch_b[32 * NO];  // the block scans alternate between them
    __shared__ double bcast[2 + 2 * NO];
    __shared__ int chunk_s;
    const ScanPow* pow_att = &pw_att;
    const SectionTab<NO>* sec_global = reinterpret_cast<const SectionTab<NO>*>(tables + sizeof(ScanPow));
    const SectionTab<NO>* tab_hold = NO == 1 ? reinterpret_cast<const SectionTab<NO>*>(&pw_sec[0]) : sec_global;
    const SectionTab<NO>* tab_rel = NO == 1 ? reinterpret_cast<const SectionTab<NO>*>(&pw_sec[1]) : sec_global + 1;

    const int tid = threadIdx.x;
    // Which chunk: the block index (default) or an atomic ticket (option "limiter_ticket").  The look-back only ever
    // waits for LOWER chunks; with the block index that is safe as long as blocks start in index order -- what the
    // hardware does for a one-dimensional grid and what every decoupled-look-back scan relies on -- and it saves the
    // ticket's round trip through L2 plus a barrier in front of the chunk's first loads (12 % of this kernel's
    // stall samples sat there).  The ticket makes the order explicit instead.
    int chunk = blockIdx.x;
    if (gm.use_ticket) {
        if (tid == 0) chunk_s = atomicAdd(ticket, 1);
        __syncthreads();
        chunk = chunk_s;
    }
    const long long s0 = (long long)chunk * LC;
    const int core_n = (int)((s0 + LC < frames) ? LC : frames - s0);
    const int reach = gm.reach, hold = gm.hold, HL = gm.left, FL = gm.filt;
    const long long ga = s0 - HL - reach;  // sample at span index 0
    const int cidx = HL + reach;           // span index of the chunk's first sample
    // span indices that fall inside the signal: [vlo, vhi)
    const int vlo = ga < 0 ? (int)(-ga) : 0;
    const int vhi = (frames - ga < (long long)gm.span) ? (int)(frames - ga) : gm.span;
    const double thr = lp.threshold;

    // ---- P1: hard-clip gain g = 1 - thr/max(|L|,|R|,thr) over the span (dsp.py:117-121, hyrax.py:87)
    // All of the thread's loads go out first (one DRAM latency, not EPT), then the scalars and the tables: the
    // kernel's first use of anything it loaded comes after everything has been requested.
    float2 v[EPT];
    float dv[TP ? EPT : 1];
    if constexpr (TP) {
        const float* base = tp_d + ga;
#pragma unroll
        for (int k = 0; k < EPT; ++k) {
            const int i = tid + k * NT;
            dv[k] = (i >= vlo && i < vhi) ? __ldg(base + i) : 0.0f;
        }
    } else {
        const float2* base = in + ga;
#pragma unroll
        for (int k = 0; k < EPT; ++k) {
            const int i = tid + k * NT;
            v[k] = (i >= vlo && i < vhi) ? __ldg(base + i) : make_float2(0.0f, 0.0f);
        }
    }
    const double pre = pre_gain ? *pre_gain : 1.0;
    const double post = post_gain ? *post_gain : 1.0;
    const double scale = pre * post;
    const bool bypass = engaged && *engaged == 0;
    {
        const double* src = reinterpret_cast<const double*>(tables);
        double* dst = reinterpret_cast<double*>(&pw_att);
        for (int i = tid; i < (int)(sizeof(ScanPow) / sizeof(double)); i += NT) dst[i] = src[i];
        if (NO == 1) {
            src += sizeof(ScanPow) / sizeof(double);
            dst = reinterpret_cast<double*>(pw_sec);
            for (int i = tid; i < (int)(2 * sizeof(SectionTab<1>) / sizeof(double)); i += NT) dst[i] = src[i];
        }
    }
    if (bypass) {  // hyrax.py:83-85: the limiter is not needed
        if constexpr (VERS) {
            for (int j = 0; j < vp->count; ++j)
                for (int k = tid; k < core_n; k += NT) {
                    const float2 w = vp->in[j][s0 + k];
                    vp->out[j][s0 + k] = make_float2((float)((double)w.x * pre * post), (float)((double)w.y * pre * post));
                }
        } else {
            for (int k = tid; k < core_n; k += NT) {
                const float2 w = in[s0 + k];
                out[s0 + k] = make_float2((float)((double)w.x * pre * post), (float)((double)w.y * pre * post));
            }
        }
        return;
    }
    for (int i = tid; i < gm.margin; i += NT) {
        G[-1 - i] = 0.0f;
        G[CAP + i] = 0.0f;
    }
#pragma unroll
    for (int k = 0; k < EPT; ++k) {
        // g = 1 - thr/a = (a - thr)/a: the difference in float64 (it decides which frames are touched at
        // all, and cancels when a is close to thr), the quotient in float32 -- g is kept as float32 anyway
        double a;
        if constexpr (TP) a = (double)dv[k] * pre;
        else a = (double)fmaxf(fabsf(v[k].x), fabsf(v[k].y)) * pre;
        const double over = a - thr;
        float g = 0.0f;
        if (over > 0.0) g = __fdiv_rn((float)over, (float)a);
        G[tid + k * NT] = g;
    }
    __syncthreads();  // (also: the pole tables are in shared memory)

    // ---- P2: both running maxima of g ----------------------------------------------------------------
    //   A[n] = max g[n-reach .. n+reach]                                 (hyrax.py:35-37)
    //   H[n] = max A[n-hold+1 .. n] = max g[n-hold+1-reach .. n+reach]   (hyrax.py:38-40)
    // Every thread owns EPT consecutive samples: their prefix and suffix maxima inside the block
    // (PF, SF) and the block maximum.  A window [l, r] is max(SF[l], whole blocks between, PF[r]).
    float hc[HC];  // H at span indices cidx + tid*CORE_EPT - NO + e
    {
        float* PF = reinterpret_cast<float*>(smem);  // [CAP] lower half of Fd's bytes (Aenv is the upper half)
        float* SF = Wk;                              // [CAP]
        float x[EPT];
        const int base = tid * EPT;
#pragma unroll
        for (int e = 0; e < EPT; ++e) x[e] = G[base + e];
        float run = 0.0f;  // g >= 0
#pragma unroll
        for (int e = 0; e < EPT; ++e) {
            run = fmaxf(run, x[e]);
            PF[base + e] = run;
        }
        blockmax[tid] = run;
        run = 0.0f;
#pragma unroll
        for (int e = EPT - 1; e >= 0; --e) {
            run = fmaxf(run, x[e]);
            SF[base + e] = run;
        }
        __syncthreads();
        auto whole_blocks = [&](int a, int b) -> float {  // blocks a..b inclusive (a run of at most ~a dozen)
            float m = 0.0f;
            for (int q = a; q <= b; ++q) m = fmaxf(m, blockmax[q]);
            return m;
        };
        auto window = [&](int l, int r, int br, float pr) -> float {
            const int bl = l / EPT;
            if (bl == br) {  // shorter than a block: scan it
                float m = 0.0f;
                for (int i = l; i <= r; ++i) m = fmaxf(m, G[i]);
                return m;
            }
            float m = fmaxf(SF[l], pr);
            if (br - bl > 1) m = fmaxf(m, whole_blocks(bl + 1, br - 1));
            return m;
        };
        auto gat = [&](int i) -> float { return G[i]; };  // (outside the span: the zero margins; g >= 0, so 0 is neutral)
        // The thread's consecutive windows of one kind share most of their samples: for the EPT windows
        // [b+e-reach, b+e+reach] (b = base) the core [b+EPT-1-reach, b+reach] does not depend on e; what
        // lies left and right of it are EPT-1 samples each, combined by running maxima in registers.
        // One table query per thread and kind instead of one per sample.
        if (gm.shared_core) {
            float la[EPT], rt[EPT];
#pragma unroll
            for (int e = 0; e < EPT - 1; ++e) {
                la[e] = gat(base - reach + e);
                rt[e + 1] = gat(base + reach + 1 + e);
            }
            la[EPT - 1] = rt[0] = 0.0f;
#pragma unroll
            for (int e = EPT - 2; e >= 0; --e) la[e] = fmaxf(la[e], la[e + 1]);  // suffix maxima of the left part
#pragma unroll
            for (int e = 1; e < EPT; ++e) rt[e] = fmaxf(rt[e], rt[e - 1]);       // prefix maxima of the right part
            const int r = min(base + reach, CAP - 1);
            const float core = window(max(base + EPT - 1 - reach, 0), r, r / EPT, PF[r]);
#pragma unroll
            for (int e = 0; e < EPT; ++e) Aenv[base + e] = fmaxf(core, fmaxf(la[e], rt[e]));
        } else {
#pragma unroll
            for (int e = 0; e < EPT; ++e) {
                const int i = base + e;
                const int r = min(i + reach, CAP - 1);
                Aenv[i] = window(max(i - reach, 0), r, r / EPT, PF[r]);
            }
        }
        // H for the thread's own CORE_EPT core samples and the NO before them (the filters below run
        // over the core in this very mapping, so H never goes through shared memory for another thread):
        // windows [bh+e-reach-hold+1, bh+e+reach], e = 0..HC-1
        const int bh = cidx + tid * CORE_EPT - NO;
        if (gm.shared_core) {
            float lh[HC], rh[HC];
#pragma unroll
            for (int e = 0; e < HC - 1; ++e) {
                lh[e] = gat(bh - reach - hold + 1 + e);
                rh[e + 1] = gat(bh + reach + 1 + e);
            }
            lh[HC - 1] = rh[0] = 0.0f;
#pragma unroll
            for (int e = HC - 2; e >= 0; --e) lh[e] = fmaxf(lh[e], lh[e + 1]);
#pragma unroll
            for (int e = 1; e < HC; ++e) rh[e] = fmaxf(rh[e], rh[e - 1]);
            const int r = min(bh + reach, CAP - 1);
            const float core = window(max(bh + HC - reach - hold, 0), r, r / EPT, PF[r]);
#pragma unroll
            for (int e = 0; e < HC; ++e) hc[e] = fmaxf(core, fmaxf(lh[e], rh[e]));
        } else {
#pragma unroll
            for (int e = 0; e < HC; ++e) {
                const int r = min(bh + e + reach, CAP - 1);
                hc[e] = window(max(bh + e - reach - hold + 1, 0), r, r / EPT, PF[r]);
            }
        }
        // lfilter starts from rest: the envelope before the first sample is 0, not a window maximum
#pragma unroll
        for (int e = 0; e < HC; ++e)
            if (bh + e < vlo) hc[e] = 0.0f;
    }

    // ---- P3: hold_out = lfilter(butter(order, f_hold), H), zero-state pass (hyrax.py:61-66) ---------
    // The chunk's aggregate is published now; the carry from the previous chunks is only needed after
    // the attack filter below, which gives the predecessors time to publish theirs.
    LookbackWord* slot_hold = slots + (long long)chunk * (2 * NO);
    LookbackWord* slot_rel = slot_hold + NO;
    double hold_y[CORE_EPT];
    StVec<NO> hold_carry;  // hold_out just before the thread's first sample, zero carry into the chunk
    float* Hown = Wk + tid * HC;  // the thread's own H samples, parked until the release filter
    {
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
        StVec<NO> end;
#pragma unroll
        for (int i = 0; i < NO; ++i) end.v[i] = hold_y[CORE_EPT - 1 - i];
        // (the barrier inside also ends P2: every thread is done with PF, SF and the sparse table)
        hold_carry = section_scan<NO>(end, tab_hold, scratch_a);
        if (tid == NT - 1) {  // the chunk's zero-carry end state
            st_addmul<NO>(end, tab_hold->ql[1], hold_carry);
            publish_state<NO>(slot_hold, end, 1);
        }
#pragma unroll
        for (int e = 0; e < HC; ++e) Hown[e] = hc[e];  // SF (= Wk) is free now; only this thread reads these back
    }

    // ---- P4: g_att = filtfilt one-pole over A (hyrax.py:48-51) -------------------------------------
    // scipy's filtfilt runs over the odd extension by 6 samples with the steady-state initial state;
    // holding the extension's end value constant further out reproduces that state exactly.  Only
    // chunks that touch an end of the signal see the extension.
    const double c = lp.attack_c;
    const bool edge_l = vlo > reach, edge_r = vhi < reach + FL;
    if (edge_l || edge_r) {
        const int i0 = vlo, iL = vhi - 1;  // span indices of samples 0 and frames-1
        float fix[EPT];
#pragma unroll
        for (int k = 0; k < EPT; ++k) {
            const int i = tid + k * NT;
            fix[k] = Aenv[i];
            if (i < vlo) {
                const int d = (vlo - i < 6) ? vlo - i : 6;
                fix[k] = 2.0f * Aenv[i0] - Aenv[i0 + d];
            } else if (i >= vhi) {
                const int d = (i - iL < 6) ? i - iL : 6;
                fix[k] = 2.0f * Aenv[iL] - Aenv[iL - d];
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < EPT; ++k) Aenv[tid + k * NT] = fix[k];
        __syncthreads();
    }
    {
        // forward over the thread's own samples, then backward over the same samples in the same registers:
        // the backward scan runs across the block in descending thread order, so the forward result never
        // goes through shared memory
        double y[EPT];
        double acc = 0.0;
#pragma unroll
        for (int e = 0; e < EPT; ++e) {
            acc = (1.0 - c) * (double)Aenv[tid * EPT + e] + c * acc;
            y[e] = acc;
        }
        const double c0 = (double)Aenv[0];  // state before the first element: steady state
        const double carry = scan_carry(acc, pow_att, c0, scratch_b);  // barrier inside: Aenv fully read
#pragma unroll
        for (int e = 0; e < EPT; ++e) y[e] += pow_att->pe[e + 1] * carry;
        if (edge_r) {
            // past the extension's last sample (frames+5) the backward pass sees that value held
            const int ilast = (int)(frames + 5 - ga);
            if (ilast < CAP - 1) {
#pragma unroll
                for (int e = 0; e < EPT; ++e)
                    if (tid * EPT + e == ilast) bcast[1] = y[e];
                __syncthreads();
                const double held = bcast[1];
#pragma unroll
                for (int e = 0; e < EPT; ++e)
                    if (tid * EPT + e > ilast) y[e] = held;
                __syncthreads();  // bcast[1] is written again just below
            }
        }
        if (tid == NT - 1) bcast[1] = y[EPT - 1];  // the backward pass starts from the forward pass's last value
        acc = 0.0;
#pragma unroll
        for (int e = EPT - 1; e >= 0; --e) {
            acc = (1.0 - c) * y[e] + c * acc;
            y[e] = acc;
        }
        const double back = scan_carry_rev(acc, pow_att, &bcast[1], scratch_a);
#pragma unroll
        for (int e = 0; e < EPT; ++e) {
            const int i = tid * EPT + e;
            if (i >= cidx && i < cidx + LC) {
                const float att = (float)(y[e] + pow_att->pe[EPT - e] * back);
                G[i] = GAINS ? att : fmaxf(G[i], att);
            }
        }
    }

    // ---- P5: hold carry from the previous chunks (decoupled look-back), finish hold_out -------------
    if (tid < 32) {
        const StVec<NO> cin = lookback<NO>(slots, chunk, tab_hold);
        if (tid == 0) {
#pragma unroll
            for (int i = 0; i < NO; ++i) bcast[2 + i] = cin.v[i];
        }
    }
    __syncthreads();  // also: every thread is done reading Fd as the attack filter's plane
    StVec<NO> hold_prev;  // hold_out at the NO samples before the thread's first one
    {
        StVec<NO> cin;
#pragma unroll
        for (int i = 0; i < NO; ++i) cin.v[i] = bcast[2 + i];
        hold_prev = section_lead<NO>(tab_hold, cin);
#pragma unroll
        for (int i = 0; i < NO; ++i) hold_prev.v[i] += hold_carry.v[i];
#pragma unroll
        for (int e = 0; e < CORE_EPT; ++e)
#pragma unroll
            for (int i = 0; i < NO; ++i) hold_y[e] += tab_hold->pe[e][i] * hold_prev.v[i];
        if (tid == NT - 1 && gm.publish_inclusive) {
            StVec<NO> end;
#pragma unroll
            for (int i = 0; i < NO; ++i) end.v[i] = hold_y[CORE_EPT - 1 - i];
            publish_state<NO>(slot_hold, end, 2);
        }
    }

    // ---- P6: release_out = lfilter(butter(order, f_rel), max(H, hold_out)) (hyrax.py:68-73) ----------
    {
        double rel_y[CORE_EPT];
        double win[HC];  // the section's input max(H, hold_out) at the NO samples before the core and on it
#pragma unroll
        for (int i = 0; i < NO; ++i) win[i] = fmax((double)Hown[i], hold_prev.v[NO - 1 - i]);
#pragma unroll
        for (int e = 0; e < CORE_EPT; ++e) win[NO + e] = fmax((double)Hown[NO + e], hold_y[e]);
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
                for (int i = 0; i < NO; ++i) bcast[2 + NO + i] = cr.v[i];
            }
        }
        __syncthreads();
        {
            StVec<NO> cin;
#pragma unroll
            for (int i = 0; i < NO; ++i) cin.v[i] = bcast[2 + NO + i];
            const StVec<NO> lead = section_lead<NO>(tab_rel, cin);
#pragma unroll
            for (int i = 0; i < NO; ++i) rel_prev.v[i] += lead.v[i];
        }
#pragma unroll
        for (int e = 0; e < CORE_EPT; ++e) {
#pragma unroll
            for (int i = 0; i < NO; ++i) rel_y[e] += tab_rel->pe[e][i] * rel_prev.v[i];
            const int i = cidx + tid * CORE_EPT + e;
            const double g_rel = fmax(hold_y[e], rel_y[e]);            // hyrax.py:75
            Fd[tid * CORE_EPT + e] = GAINS ? g_rel : 1.0 - fmax((double)G[i], g_rel);  // hyrax.py:97
        }
        if (tid == NT - 1 && gm.publish_inclusive) {
#pragma unroll
            for (int i = 0; i < NO; ++i) end.v[i] = rel_y[CORE_EPT - 1 - i];
            publish_state<NO>(slot_rel, end, 2);
        }
    }
    if (GAINS) __syncthreads();  // (the attack gains in G were written in another mapping)
    else __syncwarp();           // a warp applies the gains of its own 32*CORE_EPT consecutive samples: no block barrier

    // ---- P7: apply (hyrax.py:99, stages.py:203) -----------------------------------------------------
    // The gains sit in shared memory in the filters' mapping (thread t: samples t*CORE_EPT ..); lane l of
    // warp w now takes samples w*32*CORE_EPT + l + 32 q, so that every global access is 32 neighbours.
    if constexpr (VERS) {  // the main's gains on every entry, the loads of one entry in flight at a time
        const int wbase = (tid >> 5) * (32 * CORE_EPT) + (tid & 31);
        for (int j = 0; j < vp->count; ++j) {
            const float2* src = vp->in[j];
            float2* dst = vp->out[j];
            float2 v[CORE_EPT];
#pragma unroll
            for (int q = 0; q < CORE_EPT; ++q) {
                const int k = wbase + q * 32;
                v[q] = k < core_n ? __ldg(src + s0 + k) : make_float2(0.0f, 0.0f);
            }
#pragma unroll
            for (int q = 0; q < CORE_EPT; ++q) {
                const int k = wbase + q * 32;
                if (k < core_n) {
                    const double gain = Fd[k] * scale;
                    dst[s0 + k] = make_float2((float)((double)v[q].x * gain), (float)((double)v[q].y * gain));
                }
            }
        }
    } else {
        const int wbase = (tid >> 5) * (32 * CORE_EPT) + (tid & 31);
        float2 v[CORE_EPT];
#pragma unroll
        for (int q = 0; q < CORE_EPT; ++q) {
            const int k = wbase + q * 32;
            v[q] = k < core_n ? __ldg(in + s0 + k) : make_float2(0.0f, 0.0f);
        }
#pragma unroll
        for (int q = 0; q < CORE_EPT; ++q) {
            const int k = wbase + q * 32;
            if (k < core_n) {
                if (GAINS) {
                    out[s0 + k] = make_float2(G[cidx + k], (float)Fd[k]);
                } else {
                    // (in float64 to the end: a frame the hard clip brings to the threshold must round to it exactly)
                    const double gain = Fd[k] * scale;
                    out[s0 + k] = make_float2((float)((double)v[q].x * gain), (float)((double)v[q].y * gain));
                }
            }
        }
    }
}

template <int EPT, int NO, bool GAINS = false, bool TP = false, bool GATED = false>
// (two CTAs per SM where the span leaves room for them: up to 17 samples per thread at order capacity 1)
__global__ void __launch_bounds__(NT, (NO == 1 && EPT <= 17) ? 2 : 1)
limiter_kernel(mgb_limiter_params lp, LimiterGeom gm, const float2* __restrict__ in, float2* __restrict__ out,
               long long frames, const double* __restrict__ pre_gain, const double* __restrict__ post_gain,
               const int* __restrict__ engaged, int* __restrict__ ticket, LookbackWord* __restrict__ slots,
               const unsigned char* __restrict__ tables, const float* __restrict__ tp_d, const int* __restrict__ skip) {
    limiter_body<EPT, NO, GAINS, TP, GATED, false>(lp, gm, in, out, frames, pre_gain, post_gain, engaged, ticket, slots, tables,
                                                   tp_d, skip, nullptr);
}

// the linked limiter: the detector plane D in, every entry of the table out (the main is entry 0)
template <int EPT, int NO>
__global__ void __launch_bounds__(NT, (NO == 1 && EPT <= 17) ? 2 : 1)
limiter_versions_kernel(mgb_limiter_params lp, LimiterGeom gm, long long frames, const double* __restrict__ pre_gain,
                        const double* __restrict__ post_gain, const int* __restrict__ engaged, int* __restrict__ ticket,
                        LookbackWord* __restrict__ slots, const unsigned char* __restrict__ tables,
                        const float* __restrict__ tp_d, const __grid_constant__ VersionPlanes vp) {
    limiter_body<EPT, NO, false, true, false, true>(lp, gm, vp.in[0], vp.out[0], frames, pre_gain, post_gain, engaged, ticket,
                                                    slots, tables, tp_d, nullptr, &vp);
}

// engaged = not all(isclose(rectified, 1.0)) with numpy's defaults rtol=1e-5, atol=1e-8
__global__ void limiter_engaged_kernel(const float* peak_bits, const double* pre_gain, double threshold, int* engaged) {
    const double pre = pre_gain ? *pre_gain : 1.0;
    const double peak = (double)(*peak_bits) * pre;
    const double r = fmax(peak, threshold) / threshold;
    *engaged = (fabs(r - 1.0) <= 1e-8 + 1e-5 * 1.0) ? 0 : 1;
}

// order capacity of the kernel that serves these parameters: 1 (scalar sections) or MGB_MAX_FILTER_ORDER
int limiter_order_capacity(const mgb_limiter_params& lp) {
    return (lp.hold_order <= 1 && lp.release_order <= 1) ? 1 : MGB_MAX_FILTER_ORDER;
}

}  // namespace

int limiter_validate(const mgb_limiter_params& lp) {
    MGB_REQUIRE(lp.reach >= 1 && lp.hold >= 3 && lp.warmup >= 8, MGB_ERR_INVALID, "limiter: bad window sizes");
    MGB_REQUIRE(lp.hold_order >= 1 && lp.hold_order <= MGB_MAX_FILTER_ORDER && lp.release_order >= 1 &&
                    lp.release_order <= MGB_MAX_FILTER_ORDER,
                MGB_ERR_UNSUPPORTED, "limiter: hold / release filter orders %d / %d, kernels exist for 1..%d", lp.hold_order,
                lp.release_order, MGB_MAX_FILTER_ORDER);
    MGB_REQUIRE(lp.attack_c > 0.0 && lp.attack_c < 1.0, MGB_ERR_INVALID, "limiter: attack pole out of (0,1)");
    MGB_REQUIRE(lp.threshold > 0.0, MGB_ERR_INVALID, "limiter: threshold must be positive");
    MGB_REQUIRE(lp.true_peak == 0 || lp.true_peak == 1 || lp.true_peak == 2 || lp.true_peak == 4, MGB_ERR_INVALID,
                "limiter: true_peak %d (0: sample peaks; 1, 2 or 4: the detector's oversampling)", lp.true_peak);
    return MGB_OK;
}

// The halo kernel serves the parameters exactly when its span fits (limiter_geometry: ept <= kLimiterSpanEptMax);
// the wide-window path (limiter_wide.cuh) serves all others.  The span in 64 bits: a slow attack's warm-up
// overflows int.  (Rounding ept up to odd, or to its minimum of 11, never crosses 25.)
bool limiter_span_too_wide(const mgb_limiter_params& lp) {
    const long long no = limiter_order_capacity(lp), warm = lp.warmup, hold = lp.hold, reach = lp.reach;
    const long long left = warm > hold + no - 1 ? warm : hold + no - 1;
    const long long span = LC + left + warm + 2 * reach;
    return (span + NT - 1) / NT > SPAN_EPT_MAX;
}

namespace {

int limiter_geometry(const mgb_limiter_params& lp, LimiterGeom* g) {
    MGB_TRY(limiter_validate(lp));
    const int no = limiter_order_capacity(lp);
    g->reach = lp.reach;
    g->hold = lp.hold;
    g->warm = lp.warmup;
    g->left = lp.warmup > lp.hold + no - 1 ? lp.warmup : lp.hold + no - 1;  // H is needed `no` samples before the core
    g->filt = LC + g->left + g->warm;
    g->span = g->filt + 2 * g->reach;
    int ept = (g->span + NT - 1) / NT;
    if (!(ept & 1)) ept += 1;  // odd stride: the blocked scans read shared memory conflict-free
    if (ept < 11) ept = 11;
    if (ept < CORE_EPT + no) ept = (CORE_EPT + no) | 1;  // every thread parks its CORE_EPT + no samples of H in one plane
    g->ept = ept;
    g->publish_inclusive = g_lookback_inclusive;
    g->use_ticket = g_limiter_ticket;
    // the cores [b+ept-1-reach, b+reach] and [b+ept-reach-hold, b+reach] must not be empty
    g->shared_core = (2 * lp.reach >= ept - 1 && 2 * lp.reach + lp.hold >= CORE_EPT + no) ? 1 : 0;
    g->margin = (lp.reach + lp.hold + ept + no + 3) / 4 * 4;  // the furthest a window part reaches outside [0, CAP)
    MGB_REQUIRE(ept <= SPAN_EPT_MAX, MGB_ERR_UNSUPPORTED,
                "limiter: halo of %d samples exceeds the kernel's span", g->span - LC);
    return MGB_OK;
}

}  // namespace

// ---- order capacity 2: powers of the sections' companion matrices, on the HOST in extended precision -------
// C = [[-a1, -a2], [1, 0]] has its two eigenvalues 3e-5 apart (a Butterworth pair at 0.27 Hz against 44.1 kHz):
// powers by repeated squaring in float64 lose a digit per squaring (measured: relative error 2e-8 at C^4608,
// 3e-3 at C^147456), and the blocked scan weighs whole chunks with exactly those powers.  In closed form,
//     C^m = [[U_m, -a2 U_(m-1)], [U_(m-1), -a2 U_(m-2)]],   U_m = r^m sin((m+1) theta) / sin(theta)
// for the pole pair r exp(+-i theta) of the ROUNDED coefficients the reference's lfilter runs with -- the
// discriminant a1^2 - 4 a2 formed exactly (fma) and everything after it in long double.
struct SectionPowers {
    long double A, B;       // z^2 - A z + B
    int kind;               // 0: B == 0 (an order-1 section padded to 2); 1: complex pair; 2: real pair; 3: double root
    long double r_log, theta, sin_theta;  // kind 1
    long double p1, p2;                   // kind 2 (p1 alone for kinds 0 and 3)
    explicit SectionPowers(const double* a) {
        A = -(long double)a[1];
        B = (long double)a[2];
        if (a[2] == 0.0) {
            kind = 0;
            p1 = A;
            return;
        }
        const double hi = a[1] * a[1];
        const double lo = fma(a[1], a[1], -hi);                       // a1^2 = hi + lo exactly
        const long double disc = ((long double)hi - 4.0L * B) + (long double)lo;  // (hi - 4 a2 is exact in double range)
        if (disc < 0) {
            kind = 1;
            r_log = 0.5L * log1pl(B - 1.0L);
            theta = atan2l(sqrtl(-disc), A);
            sin_theta = sinl(theta);
        } else if (disc > 0) {
            kind = 2;
            const long double q = sqrtl(disc);
            p1 = 0.5L * (A + q);
            p2 = 0.5L * (A - q);
        } else {
            kind = 3;
            p1 = 0.5L * A;
        }
    }
    long double U(long long m) const {  // m >= -1
        if (m < 0) return 0.0L;
        switch (kind) {
            case 0: return powl(p1, (long double)m);
            case 1: return expl((long double)m * r_log) * sinl((long double)(m + 1) * theta) / sin_theta;
            case 2: return (powl(p1, (long double)(m + 1)) - powl(p2, (long double)(m + 1))) / (p1 - p2);
            default: return (long double)(m + 1) * powl(p1, (long double)m);
        }
    }
    void power(long long m, double (*out)[2]) const {
        if (m == 0) {
            out[0][0] = out[1][1] = 1.0;
            out[0][1] = out[1][0] = 0.0;
            return;
        }
        const long double u0 = U(m), u1 = U(m - 1), u2 = U(m - 2);
        out[0][0] = (double)u0;
        out[0][1] = (double)(-B * u1);
        out[1][0] = (double)u1;
        out[1][1] = (double)(-B * u2);
    }
};

static void fill_section_tables(const double* a, SectionTab<2>* t) {
    const SectionPowers sp(a);
    double m[2][2];
    for (int e = 0; e < CORE_EPT; ++e) {
        sp.power(e + 1, m);
        t->pe[e][0] = m[0][0];
        t->pe[e][1] = m[0][1];
    }
    for (int k = 0; k < 33; ++k) sp.power((long long)CORE_EPT * k, t->ql[k]);
    for (int k = 0; k < 17; ++k) sp.power((long long)CORE_EPT * 32 * k, t->qw[k]);
    for (int k = 0; k < 33; ++k) sp.power((long long)LC * k, t->pc[k]);
    for (int j = 0; j < kLookbackJumps; ++j) sp.power((long long)LC * 32 * j, t->pj[j]);
}

static void fill_attack_tables(double p, int span_ept, ScanPow* t) {
    for (int i = 0; i < SPAN_EPT_MAX + 2; ++i) t->pe[i] = (double)powl((long double)p, (long double)i);
    for (int i = 0; i < 33; ++i) t->ql[i] = (double)powl((long double)p, (long double)(span_ept * i));
    for (int i = 0; i < 17; ++i) t->qw[i] = (double)powl((long double)p, (long double)(span_ept * 32 * i));
    for (int i = 0; i < 33; ++i) t->pc[i] = (double)powl((long double)p, (long double)LC * (long double)i);
}

int64_t limiter_lookback_bytes(int64_t frames, int order_capacity) {
    const int64_t chunks = (frames + LC - 1) / LC;
    return (chunks * 2 * order_capacity * (int64_t)sizeof(LookbackWord) + 255) / 256 * 256;
}
int64_t limiter_lookback_bytes(const mgb_limiter_params& lp, int64_t frames) {
    if (limiter_span_too_wide(lp)) return limiter_wide_lookback_bytes(lp, frames, limiter_order_capacity(lp));
    return limiter_lookback_bytes(frames, limiter_order_capacity(lp));
}
int64_t limiter_plane_bytes(const mgb_limiter_params& lp, int64_t frames) {
    return limiter_span_too_wide(lp) ? limiter_wide_plane_bytes(lp, frames) : 0;
}

int64_t limiter_tables_bytes() { return (int64_t)(sizeof(ScanPow) + 2 * sizeof(SectionTab<MGB_MAX_FILTER_ORDER>) + 255) / 256 * 256; }

int launch_limiter_tables(const mgb_limiter_params& lp, void* tables, cudaStream_t stream) {
    LimiterGeom g;
    MGB_TRY(limiter_validate(lp));
    if (limiter_span_too_wide(lp))
        g.ept = CORE_EPT;  // the wide-window path scans the attack filter over CORE_EPT samples per thread
    else
        MGB_TRY(limiter_geometry(lp, &g));
    if (limiter_order_capacity(lp) == 1)
        return launch("limiter_tables_kernel", limiter_tables_kernel, dim3(1), dim3(64), 0, stream, lp, g.ept,
                      (unsigned char*)tables);
    // order 2: host tables (see SectionPowers), one small upload; the copy from pageable memory is staged before
    // the call returns, so the local buffer may go out of scope
    struct Block {
        ScanPow attack;
        SectionTab<2> section[2];
    } block;
    static_assert(sizeof(Block) == sizeof(ScanPow) + 2 * sizeof(SectionTab<2>), "table layout");
    fill_attack_tables(lp.attack_c, g.ept, &block.attack);
    fill_section_tables(lp.hold_a, &block.section[0]);
    fill_section_tables(lp.release_a, &block.section[1]);
#ifdef MGB_EMULATE
    (void)stream;
    memcpy(tables, &block, sizeof(block));
#else
    if (cudaMemcpyAsync(tables, &block, sizeof(block), cudaMemcpyHostToDevice, stream) != cudaSuccess) return cuda_status("limiter tables");
#endif
    return MGB_OK;
}

int launch_limiter(const mgb_limiter_params& lp, const float2* in, float2* out, int64_t frames, const double* pre_gain,
                   const double* post_gain, const int* engaged, int* ticket, void* lookback, void* wide_planes,
                   const void* tables, cudaStream_t stream, bool gains_only, const float* tp_d, const int* skip) {
    MGB_TRY(limiter_validate(lp));
    MGB_REQUIRE(frames > 6, MGB_ERR_INVALID, "limiter: the input must be longer than filtfilt's padlen (6)");
    MGB_REQUIRE(tables != nullptr, MGB_ERR_INVALID, "limiter: pole tables missing");
    const bool tp = lp.true_peak != 0;
    MGB_REQUIRE(!tp || tp_d != nullptr, MGB_ERR_INVALID, "limiter: true-peak mode without the detector plane");
    if (limiter_span_too_wide(lp))  // (chunks by block index: the wide-window path has no ticket)
        return launch_limiter_wide(lp, limiter_order_capacity(lp), g_lookback_inclusive, in, out, frames, pre_gain, post_gain,
                                   engaged, lookback, wide_planes, tables, stream, gains_only, tp ? tp_d : nullptr, skip);
    LimiterGeom g;
    MGB_TRY(limiter_geometry(lp, &g));
    const int64_t chunks = (frames + LC - 1) / LC;
    const size_t smem = (size_t)g.ept * NT * 16 + (size_t)g.margin * 8;
    const int no = limiter_order_capacity(lp);
    MGB_REQUIRE(!(gains_only && skip), MGB_ERR_INVALID, "limiter: the gains test entry has no gated passes");
    if (gains_only) {  // test entry: the sample rates of the golden vectors (44.1 and 96 kHz windows), both capacities
        auto go = [&](auto kernel) {
            return launch("limiter_kernel", kernel, dim3((unsigned)chunks), dim3(NT), smem, stream, lp, g, in, out,
                          (long long)frames, pre_gain, post_gain, engaged, ticket, (LookbackWord*)lookback,
                          (const unsigned char*)tables, tp_d, skip);
        };
        if (no == 1 && g.ept == 11) return tp ? go(limiter_kernel<11, 1, true, true>) : go(limiter_kernel<11, 1, true>);
        if (no == 1 && g.ept == 13) return tp ? go(limiter_kernel<13, 1, true, true>) : go(limiter_kernel<13, 1, true>);
        if (no == MGB_MAX_FILTER_ORDER && g.ept == 11)
            return tp ? go(limiter_kernel<11, MGB_MAX_FILTER_ORDER, true, true>) : go(limiter_kernel<11, MGB_MAX_FILTER_ORDER, true>);
        set_error("limiter gains (test entry): no kernel for %d span samples per thread at order capacity %d", g.ept, no);
        return MGB_ERR_UNSUPPORTED;
    }
    auto run = [&](auto kernel) {
        return launch("limiter_kernel", kernel, dim3((unsigned)chunks), dim3(NT), smem, stream, lp, g, in, out, (long long)frames,
                      pre_gain, post_gain, engaged, ticket, (LookbackWord*)lookback, (const unsigned char*)tables, tp_d, skip);
    };
    // (gated passes of a loudness-target search: the same kernels behind the skip flag)
#define MGB_LIMITER_CASE(E)                                                                                           \
    case E:                                                                                                           \
        if (skip) {                                                                                                   \
            if (tp)                                                                                                   \
                return no == 1 ? run(limiter_kernel<E, 1, false, true, true>)                                         \
                               : run(limiter_kernel<E, MGB_MAX_FILTER_ORDER, false, true, true>);                     \
            return no == 1 ? run(limiter_kernel<E, 1, false, false, true>)                                            \
                           : run(limiter_kernel<E, MGB_MAX_FILTER_ORDER, false, false, true>);                        \
        }                                                                                                             \
        if (tp)                                                                                                       \
            return no == 1 ? run(limiter_kernel<E, 1, false, true>)                                                   \
                           : run(limiter_kernel<E, MGB_MAX_FILTER_ORDER, false, true>);                               \
        return no == 1 ? run(limiter_kernel<E, 1>) : run(limiter_kernel<E, MGB_MAX_FILTER_ORDER>);
    switch (g.ept) {
        MGB_LIMITER_CASE(11)
        MGB_LIMITER_CASE(13)
        MGB_LIMITER_CASE(15)
        MGB_LIMITER_CASE(17)
        MGB_LIMITER_CASE(19)  // slow attacks / high sample rates (the default limiter at 176.4 and 192 kHz): one CTA per SM
        MGB_LIMITER_CASE(21)
        MGB_LIMITER_CASE(23)
        MGB_LIMITER_CASE(25)
        default: break;
    }
#undef MGB_LIMITER_CASE
    set_error("limiter: no kernel for %d span samples per thread", g.ept);
    return MGB_ERR_UNSUPPORTED;
}

int launch_limiter_versions(const mgb_limiter_params& lp, const VersionPlanes& vp, int64_t frames, const double* pre_gain,
                            const double* post_gain, const int* engaged, int* ticket, void* lookback, void* wide_planes,
                            const void* tables, const float* d, cudaStream_t stream) {
    MGB_TRY(limiter_validate(lp));
    MGB_REQUIRE(frames > 6, MGB_ERR_INVALID, "limiter: the input must be longer than filtfilt's padlen (6)");
    MGB_REQUIRE(tables != nullptr && d != nullptr, MGB_ERR_INVALID, "limiter (versions): pole tables or detector plane missing");
    MGB_REQUIRE(vp.count >= 1 && vp.count <= 1 + MGB_MAX_VERSIONS, MGB_ERR_INVALID, "limiter (versions): %d entries", vp.count);
    if (limiter_span_too_wide(lp))
        return launch_limiter_wide(lp, limiter_order_capacity(lp), g_lookback_inclusive, vp.in[0], vp.out[0], frames, pre_gain,
                                   post_gain, engaged, lookback, wide_planes, tables, stream, false, d, nullptr, &vp);
    LimiterGeom g;
    MGB_TRY(limiter_geometry(lp, &g));
    const int64_t chunks = (frames + LC - 1) / LC;
    const size_t smem = (size_t)g.ept * NT * 16 + (size_t)g.margin * 8;
    const int no = limiter_order_capacity(lp);
    auto run = [&](auto kernel) {
        return launch("limiter_versions_kernel", kernel, dim3((unsigned)chunks), dim3(NT), smem, stream, lp, g, (long long)frames,
                      pre_gain, post_gain, engaged, ticket, (LookbackWord*)lookback, (const unsigned char*)tables, d, vp);
    };
#define MGB_LIMITER_CASE(E) \
    case E: return no == 1 ? run(limiter_versions_kernel<E, 1>) : run(limiter_versions_kernel<E, MGB_MAX_FILTER_ORDER>);
    switch (g.ept) {
        MGB_LIMITER_CASE(11)
        MGB_LIMITER_CASE(13)
        MGB_LIMITER_CASE(15)
        MGB_LIMITER_CASE(17)
        MGB_LIMITER_CASE(19)
        MGB_LIMITER_CASE(21)
        MGB_LIMITER_CASE(23)
        MGB_LIMITER_CASE(25)
        default: break;
    }
#undef MGB_LIMITER_CASE
    set_error("limiter (versions): no kernel for %d span samples per thread", g.ept);
    return MGB_ERR_UNSUPPORTED;
}

int launch_limiter_engaged(const float* peak_bits, const double* pre_gain, double threshold, int* engaged,
                           cudaStream_t stream) {
    return launch("limiter_engaged_kernel", limiter_engaged_kernel, dim3(1), dim3(1), 0, stream, peak_bits, pre_gain,
                  threshold, engaged);
}

}  // namespace mgb

#include "loudness.cuh"  // the loudness meter: the same scans, look-back words and section tables
#include "true_peak.cuh"  // the true-peak detector of the limiter's true-peak mode
#include "loudness_target.cuh"  // loudness targets: the search around the limiter and the meter
