// C ABI of libmatchering_b200 (include/matchering_b200.h): argument checking, workspace carving,
// stage sequencing.  No kernel lives here except the FFT test harness.
#include <math.h>
#include <stdarg.h>
#include <stddef.h>
#include <stdio.h>
#include <string.h>

#include <vector>

#include "fft.cuh"
#include "kernels.cuh"

namespace mgb {

int g_use_tma = 1;
int g_twiddle_chain = 1;
int g_analyze_chain = 1;
int g_conv_persistent = 1;
int g_conv_fused = 1;
int g_conv_ovs = 4;
int g_lookback_inclusive = 1;
int g_limiter_ticket = 0;
int g_poison_alloc = 0;

#ifndef MGB_EMULATE
long long g_launch_count = 0;
int g_profile = 0;
namespace {
struct ProfileRecord {
    const char* what;
    cudaEvent_t start, stop;
};
std::vector<ProfileRecord> g_records;
}  // namespace
void profile_mark(const char* what, cudaStream_t stream, bool begin) {
    if (begin) {
        ProfileRecord r;
        r.what = what;
        cudaEventCreate(&r.start);
        cudaEventCreate(&r.stop);
        cudaEventRecord(r.start, stream);
        g_records.push_back(r);
    } else if (!g_records.empty()) {
        cudaEventRecord(g_records.back().stop, stream);
    }
}
#endif

static thread_local char g_error[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

#ifdef MGB_EMULATE
int cuda_status(const char*) { return MGB_OK; }
int num_sms() { return 8; }
#else
int cuda_status(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) return MGB_OK;
    set_error("%s: %s", what, cudaGetErrorString(e));
    return MGB_ERR_CUDA;
}
int num_sms() {
    static int cached = 0;
    if (!cached) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
            cached = n;
        else
            cached = 132;  // the H100 SXM's SM count
    }
    return cached;
}
#endif

static inline int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

// With base_ptr == nullptr every pointer of the result holds its region's byte offset (mgb_test_workspace_regions).
Workspace carve_workspace(const mgb_plan& plan, const mgb_track_layout& L, void* base_ptr) {
    Workspace w;
    const uintptr_t base = reinterpret_cast<uintptr_t>(base_ptr);
    int64_t off = 0;
    auto take = [&](int64_t bytes) {
        unsigned char* p = reinterpret_cast<unsigned char*>(base + (uintptr_t)off);
        off += align256(bytes);
        return p;
    };
    const int64_t HB = plan.n_lin, F = plan.fft_size;
    const int64_t items_t = (int64_t)L.target_divisions * L.target_slots;
    const int64_t items_r = (int64_t)L.reference_divisions * L.reference_slots;
    w.spec_part_t = (float*)take(items_t * 2 * HB * 4);
    w.spec_part_r = (float*)take(items_r * 2 * HB * 4);
    w.sumsq_part_t = (double*)take(items_t * 8);
    w.sumsq_part_r = (double*)take(items_r * 8);
    w.absmax_part_t = (float*)take((items_t + 1) * 4);
    w.absmax_part_r = (float*)take((items_r + 1) * 4);
    w.mask_t = take(L.target_divisions);
    w.mask_r = take(L.reference_divisions);
    w.design_stride = (design_doubles_per_channel(plan) + 31) / 32 * 32;
    w.design = (double*)take(8 * w.design_stride * 8);  // 2 channels x up to 4 design CTAs
    w.h_mid = (float2*)take((2 * F + 1) * 8);           // FIR spectrum bins 0..N/2 of the N = 2F or 4F grid
    w.h_side = (float2*)take((2 * F + 1) * 8);
    w.loud_capacity = loud_capacity(L.target_piece);
    w.loud_values = (float*)take(w.loud_capacity * L.target_divisions * 4);
    w.result_slot = (const float2**)take(8);
    w.target_peak = (float*)take(4);
    w.conv_scratch = (float2*)take(conv_global_scratch_bytes(plan.fft_size, L.target_frames));
    w.zero_begin = reinterpret_cast<unsigned char*>(base + (uintptr_t)off);
    w.piece_sums = (double*)take((int64_t)MGB_MAX_CORRECTION_STEPS * L.target_divisions * 8);
    w.loud_count = (unsigned*)take((int64_t)L.target_divisions * 4);
    w.zero_end = reinterpret_cast<unsigned char*>(base + (uintptr_t)off);
    // zeroed by mgb_finalize right before every limiter launch (a second finalize on the same track
    // must not find the first one's tickets and published carries)
    const int64_t limiter_zero_from = off;
    w.tickets = (int*)take(256);
    w.lookback = take(limiter_lookback_bytes(plan.limiter, L.target_frames));
    const bool tp = plan.limiter.true_peak != 0;  // (true-peak mode only: the detector's maximum and plane)
    w.tp_peak = tp ? (float*)take(4) : nullptr;
    w.limiter_zero_bytes = off - limiter_zero_from;
    w.limiter_planes = take(limiter_plane_bytes(plan.limiter, L.target_frames));  // (empty unless the wide-window path runs)
    w.tp_plane = tp ? (float*)take(true_peak_plane_bytes(plan.limiter, L.target_frames)) : nullptr;
    // a profiled layout (no reference pieces): the copy of the profile, behind everything a paired layout has
    w.profile = L.reference_divisions == 0 ? (const mgb_reference_profile*)take(reference_profile_bytes(plan)) : nullptr;
    w.total_bytes = off;
    return w;
}

static bool layout_profiled(const mgb_track_layout& L) {
    return L.reference_divisions == 0 && L.reference_slots == 0 && L.reference_piece == 0;
}

// mgb_analyze_reference's scratch; with base_ptr == nullptr the pointers hold byte offsets
static ReferenceRegions carve_reference(const mgb_plan& plan, const ReferenceGeometry& g, void* base_ptr) {
    ReferenceRegions r;
    const uintptr_t base = reinterpret_cast<uintptr_t>(base_ptr);
    int64_t off = 0;
    auto take = [&](int64_t bytes) {
        unsigned char* p = reinterpret_cast<unsigned char*>(base + (uintptr_t)off);
        off += align256(bytes);
        return p;
    };
    const int64_t items = (int64_t)g.divisions * g.slots;
    r.spec_part = (float*)take(items * 2 * plan.n_lin * 4);
    r.sumsq_part = (double*)take(items * 8);
    r.absmax_part = (float*)take((items + 1) * 4);
    r.mask = take(g.divisions);
    r.total_bytes = off;
    return r;
}

static int check_plan(const mgb_plan* plan) {
    MGB_REQUIRE(plan != nullptr, MGB_ERR_INVALID, "plan is NULL");
    const int F = plan->fft_size;
    MGB_REQUIRE(F == 512 || F == 1024 || F == 2048 || F == 4096 || F == 8192 || F == 16384, MGB_ERR_UNSUPPORTED,
                "fft_size %d: kernels exist for 512, 1024, 2048, 4096, 8192, 16384", F);
    MGB_REQUIRE(plan->n_lin == F / 2 + 1 && plan->n_log >= 4, MGB_ERR_INVALID, "plan grid sizes inconsistent");
    MGB_REQUIRE(plan->rms_correction_steps >= 0 && plan->rms_correction_steps <= MGB_MAX_CORRECTION_STEPS,
                MGB_ERR_UNSUPPORTED, "rms_correction_steps %d > %d", plan->rms_correction_steps, MGB_MAX_CORRECTION_STEPS);
    MGB_REQUIRE(plan->lowess_k >= 2 && plan->lowess_k <= plan->n_log && plan->lowess_nfit >= 2, MGB_ERR_INVALID,
                "plan LOWESS sizes inconsistent");
    return MGB_OK;
}

static int check_aligned(const void* p, const char* name) {
    MGB_REQUIRE(p != nullptr, MGB_ERR_INVALID, "%s is NULL", name);
    MGB_REQUIRE((reinterpret_cast<uintptr_t>(p) & 15) == 0, MGB_ERR_INVALID, "%s is not 16-byte aligned", name);
    return MGB_OK;
}

// ------------------------------------------------------------------------------------------------
// FFT test harness: one frame per CTA through fft_run, global -> shared -> global
// ------------------------------------------------------------------------------------------------
template <typename T> struct TestPlanes { using type = SplitPlanes<T>; };
template <> struct TestPlanes<float> { using type = PackedPlanes; };  // what the float32 kernels use

template <int N, int DIR, typename T, int THREADS>
__global__ void __launch_bounds__(THREADS) test_fft_kernel(const cpx<T>* __restrict__ in, cpx<T>* __restrict__ out,
                                                           const cpx<T>* __restrict__ tw) {
    MGB_DYN_SMEM(smem);
    using P = typename TestPlanes<T>::type;
    P planes;
    if constexpr (sizeof(T) == 4) {
        planes.z = reinterpret_cast<float2*>(smem);
    } else {
        planes.re = reinterpret_cast<T*>(smem);
        planes.im = planes.re + P::elems(N);
    }
    const cpx<T>* src = in + (long long)blockIdx.x * N;
    cpx<T>* dst = out + (long long)blockIdx.x * N;
    auto first = [&](int i) { return src[i]; };
    auto last = [&](int i, cpx<T> v) { dst[i] = v; };
    fft_run<N, DIR, THREADS, T, sizeof(T) == 4>(planes, tw, first, last, false, false);
}

template <int N, typename T, int THREADS>
static int launch_test_fft_t(int dir, const void* in, void* out, int batch, const void* tw, cudaStream_t stream) {
    const size_t smem = TestPlanes<T>::type::bytes(N);
    if (dir > 0)
        return launch("test_fft_kernel", test_fft_kernel<N, +1, T, THREADS>, dim3(batch), dim3(THREADS), smem, stream,
                      (const cpx<T>*)in, (cpx<T>*)out, (const cpx<T>*)tw);
    return launch("test_fft_kernel", test_fft_kernel<N, -1, T, THREADS>, dim3(batch), dim3(THREADS), smem, stream,
                  (const cpx<T>*)in, (cpx<T>*)out, (const cpx<T>*)tw);
}

int launch_test_fft(int n, int is_f64, int dir, const void* in, void* out, int batch, const void* tw,
                    cudaStream_t stream) {
#define MGB_FFT_CASE(NN)                                                                                      \
    case NN:                                                                                                  \
        return is_f64 ? launch_test_fft_t<NN, double, 512>(dir, in, out, batch, tw, stream)                   \
                      : launch_test_fft_t<NN, float, NN / 16>(dir, in, out, batch, tw, stream);
    switch (n) {
        MGB_FFT_CASE(512)
        MGB_FFT_CASE(1024)
        MGB_FFT_CASE(2048)
        MGB_FFT_CASE(4096)
        MGB_FFT_CASE(8192)
        case 16384:
            if (!is_f64) return launch_test_fft_t<16384, float, 1024>(dir, in, out, batch, tw, stream);
            break;
        default: break;
    }
#undef MGB_FFT_CASE
    set_error("fft: size %d (%s) has no kernel", n, is_f64 ? "f64" : "f32");
    return MGB_ERR_UNSUPPORTED;
}

template <int N>
static void radices_of(int* npass, int r[4]) {
    *npass = Radices<N>::n;
    for (int i = 0; i < 4; ++i) r[i] = Radices<N>::r[i];
}
static bool radix_schedule(int n, int* npass, int r[4]) {
    switch (n) {
        case 512: radices_of<512>(npass, r); return true;
        case 1024: radices_of<1024>(npass, r); return true;
        case 2048: radices_of<2048>(npass, r); return true;
        case 4096: radices_of<4096>(npass, r); return true;
        case 8192: radices_of<8192>(npass, r); return true;
        case 16384: radices_of<16384>(npass, r); return true;
        case 32768: radices_of<32768>(npass, r); return true;
        default: return false;
    }
}
template <int N>
static bool inverse_radices_of(int* npass, int r[4]) {
    if constexpr (InverseRadices<N>::fused) {
        *npass = InverseRadices<N>::n;
        for (int i = 0; i < 4; ++i) r[i] = InverseRadices<N>::r[i];
        return true;
    } else {
        return false;
    }
}
// the second schedule the fused convolution keeps behind the forward one in the 2F float table
static bool inverse_schedule(int n, int* npass, int r[4]) {
    switch (n) {
        case 8192: return inverse_radices_of<8192>(npass, r);
        case 16384: return inverse_radices_of<16384>(npass, r);
        default: return false;
    }
}
static int schedule_count(int npass, const int r[4]) {
    int total = 0, ns = r[0];
    for (int p = 1; p < npass; ++p) {
        total += (r[p] - 1) * ns;
        ns *= r[p];
    }
    return total;
}
int twiddle_count(int n) {
    int npass, r[4];
    if (!radix_schedule(n, &npass, r)) return -1;
    return schedule_count(npass, r);
}
int inverse_twiddle_count(int n) {
    int npass, r[4];
    if (!inverse_schedule(n, &npass, r)) return 0;
    return schedule_count(npass, r);
}
// the 4F-point transform pair of the long-frame convolution (conv_frame_ovs == 4), kept behind the 2F tables
int long_frame_twiddle_count(int fft_size) {
    const int n4 = 4 * fft_size;
    int npass, r[4];
    if (!inverse_schedule(n4, &npass, r)) return 0;
    return twiddle_count(n4) + inverse_twiddle_count(n4);
}
int fill_twiddles(int n, int is_f64, void* table, cudaStream_t stream) {
    int npass, r[4];
    MGB_REQUIRE(radix_schedule(n, &npass, r), MGB_ERR_UNSUPPORTED, "fft: size %d has no radix schedule", n);
    if (is_f64)
        return launch("fft_twiddle_kernel", fft_twiddle_kernel<double>, dim3(16), dim3(256), 0, stream, (cpx<double>*)table,
                      npass, r[0], r[1], r[2], r[3]);
    return launch("fft_twiddle_kernel", fft_twiddle_kernel<float>, dim3(16), dim3(256), 0, stream, (cpx<float>*)table,
                  npass, r[0], r[1], r[2], r[3]);
}
int fill_inverse_twiddles(int n, cpx<float>* table, cudaStream_t stream) {
    int npass, r[4];
    if (!inverse_schedule(n, &npass, r)) return MGB_OK;
    return launch("fft_twiddle_kernel", fft_twiddle_kernel<float>, dim3(16), dim3(256), 0, stream, table + twiddle_count(n),
                  npass, r[0], r[1], r[2], r[3]);
}

}  // namespace mgb

using namespace mgb;

// ================================================================================================
extern "C" {

int mgb_version(void) { return MGB_VERSION; }
const char* mgb_last_error_string(void) { return g_error; }

int mgb_set_option(const char* name, int value) {
    MGB_REQUIRE(name != nullptr, MGB_ERR_INVALID, "option name is NULL");
    if (strcmp(name, "tma") == 0) {
        g_use_tma = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "conv_frame") == 0) {
        MGB_REQUIRE(value == 2 || value == 4, MGB_ERR_INVALID, "conv_frame must be 2 or 4 (FIR lengths per overlap-save frame)");
        g_conv_ovs = value;
        return MGB_OK;
    }
    if (strcmp(name, "conv_fused") == 0) {
        g_conv_fused = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "twiddle_chain") == 0) {
        g_twiddle_chain = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "conv_persistent") == 0) {
        g_conv_persistent = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "analyze_chain") == 0) {
        g_analyze_chain = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "lookback_inclusive") == 0) {
        g_lookback_inclusive = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "limiter_ticket") == 0) {
        g_limiter_ticket = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "design_direct") == 0) {
        g_design_direct = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "poison_alloc") == 0) {
        g_poison_alloc = value ? 1 : 0;
        return MGB_OK;
    }
    if (host_set_option(name, value)) return MGB_OK;
    set_error("unknown option '%s'", name);
    return MGB_ERR_INVALID;
}

long long mgb_launch_count(void) {
#ifdef MGB_EMULATE
    return 0;
#else
    return g_launch_count;
#endif
}

int mgb_profile_enable(int on) {
#ifndef MGB_EMULATE
    g_profile = on ? 1 : 0;
#else
    (void)on;
#endif
    return MGB_OK;
}

int mgb_profile_collect(char* names, int names_capacity, float* ms, int capacity) {
#ifdef MGB_EMULATE
    (void)names; (void)names_capacity; (void)ms; (void)capacity;
    return 0;
#else
    cudaDeviceSynchronize();
    int n = 0;
    int used = 0;
    if (names && names_capacity > 0) names[0] = 0;
    for (auto& r : g_records) {
        float t = 0.0f;
        cudaEventElapsedTime(&t, r.start, r.stop);
        if (n < capacity && ms) {
            ms[n] = t;
            if (names) {
                const int len = (int)strlen(r.what);
                if (used + len + 2 <= names_capacity) {
                    memcpy(names + used, r.what, len);
                    used += len;
                    names[used++] = '\n';
                    names[used] = 0;
                }
            }
            ++n;
        }
        cudaEventDestroy(r.start);
        cudaEventDestroy(r.stop);
    }
    g_records.clear();
    return n;
#endif
}

int mgb_plan_twiddle_bytes(int32_t fft_size, int64_t bytes_out[5]) {
    MGB_REQUIRE(bytes_out != nullptr, MGB_ERR_INVALID, "bytes_out is NULL");
    const int cf = twiddle_count(fft_size), c2 = twiddle_count(2 * fft_size);
    MGB_REQUIRE(cf > 0 && c2 > 0, MGB_ERR_UNSUPPORTED, "fft_size %d has no kernel", fft_size);
    bytes_out[0] = (int64_t)cf * 8;
    bytes_out[1] = (int64_t)(c2 + inverse_twiddle_count(2 * fft_size) + long_frame_twiddle_count(fft_size)) * 8;
    bytes_out[2] = (int64_t)cf * 16;
    // the convolution's float64 tables (convolve_precise_kernel): 2F points, and 4F behind them where 4F frames exist
    bytes_out[3] = (int64_t)(c2 + (long_frame_twiddle_count(fft_size) ? twiddle_count(4 * fft_size) : 0)) * 16;
    bytes_out[4] = limiter_tables_bytes();
    return MGB_OK;
}

int mgb_plan_fill_twiddles(const mgb_plan* plan, void* stream) {
    MGB_TRY(check_plan(plan));
    cudaStream_t st = (cudaStream_t)stream;
    MGB_TRY(check_aligned(plan->d_tw_f32_F, "d_tw_f32_F"));
    MGB_TRY(check_aligned(plan->d_tw_f32_2F, "d_tw_f32_2F"));
    MGB_TRY(check_aligned(plan->d_tw_f64_F, "d_tw_f64_F"));
    MGB_TRY(fill_twiddles(plan->fft_size, 0, plan->d_tw_f32_F, st));
    MGB_TRY(fill_twiddles(2 * plan->fft_size, 0, plan->d_tw_f32_2F, st));
    MGB_TRY(fill_inverse_twiddles(2 * plan->fft_size, (cpx<float>*)plan->d_tw_f32_2F, st));
    if (long_frame_twiddle_count(plan->fft_size)) {
        cpx<float>* tw4 = (cpx<float>*)plan->d_tw_f32_2F + twiddle_count(2 * plan->fft_size) + inverse_twiddle_count(2 * plan->fft_size);
        MGB_TRY(fill_twiddles(4 * plan->fft_size, 0, tw4, st));
        MGB_TRY(fill_inverse_twiddles(4 * plan->fft_size, tw4, st));
    }
    MGB_TRY(fill_twiddles(plan->fft_size, 1, plan->d_tw_f64_F, st));
    if (plan->d_tw_f64_2F) {
        MGB_TRY(fill_twiddles(2 * plan->fft_size, 1, plan->d_tw_f64_2F, st));
        if (long_frame_twiddle_count(plan->fft_size))
            MGB_TRY(fill_twiddles(4 * plan->fft_size, 1, (cpx<double>*)plan->d_tw_f64_2F + twiddle_count(2 * plan->fft_size), st));
    }
    if (!plan->d_limiter_tables) return MGB_OK;  // FFT-only plans (tests); mgb_finalize insists on the tables
    MGB_TRY(check_aligned(plan->d_limiter_tables, "d_limiter_tables"));
    return launch_limiter_tables(plan->limiter, plan->d_limiter_tables, st);
}

int64_t mgb_plan_operator_workspace_bytes(const mgb_plan* plan) {
    if (check_plan(plan) != MGB_OK) return -1;
    return operator_workspace_bytes(*plan);
}

int mgb_plan_build_operator(const mgb_plan* plan, double* d_operator_out, void* d_workspace, int64_t workspace_bytes,
                            void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_TRY(check_aligned(d_operator_out, "d_operator_out"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    MGB_REQUIRE(workspace_bytes >= operator_workspace_bytes(*plan), MGB_ERR_WORKSPACE, "operator workspace too small");
    return build_operator(*plan, d_operator_out, d_workspace, (cudaStream_t)stream);
}

// match_levels.py:47-59 piece geometry of one signal of n frames (n > fft_size and max_piece_size > 0 checked by the
// caller), and its analysis work items
static int signal_geometry(const mgb_plan* plan, int64_t n, ReferenceGeometry* g) {
    // match_levels.py:47-59: float division, then int() truncation
    const double q = (double)n / plan->max_piece_size;
    MGB_REQUIRE(q < 8000.0, MGB_ERR_UNSUPPORTED, "more than 8000 pieces (their statistics live in one CTA's shared memory)");
    const int32_t divisions = (int32_t)q + 1;
    const int64_t piece = (int64_t)((double)n / (double)divisions);
    MGB_REQUIRE(piece >= plan->fft_size, MGB_ERR_UNSUPPORTED,
                "piece of %lld samples is shorter than fft_size %d (the reference's STFT degenerates there)",
                (long long)piece, plan->fft_size);
    const int64_t frames_per_piece = piece / plan->fft_size;
    // analysis work items: one wave of three resident CTAs per SM (register/shared-memory limit of
    // analyze_kernel), never more items than that so that no tail wave forms
    int64_t slots = (3LL * num_sms()) / divisions;
    if (slots > frames_per_piece) slots = frames_per_piece;
    if (slots < 1) slots = 1;
    g->frames = n;
    g->piece = piece;
    g->divisions = divisions;
    g->slots = (int32_t)slots;
    return MGB_OK;
}

int mgb_track_layout_init(const mgb_plan* plan, int64_t target_frames, int64_t reference_frames,
                          mgb_track_layout* out) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(out != nullptr, MGB_ERR_INVALID, "layout is NULL");
    // core.py:69-74 guarantees both signals are longer than fft_size
    MGB_REQUIRE(target_frames > plan->fft_size && reference_frames > plan->fft_size, MGB_ERR_INVALID,
                "target (%lld) and reference (%lld) must be longer than fft_size (%d)", (long long)target_frames,
                (long long)reference_frames, plan->fft_size);
    MGB_REQUIRE(plan->max_piece_size > 0, MGB_ERR_INVALID, "max_piece_size must be positive");
    memset(out, 0, sizeof(*out));
    ReferenceGeometry t, r;
    MGB_TRY(signal_geometry(plan, target_frames, &t));
    MGB_TRY(signal_geometry(plan, reference_frames, &r));
    out->target_frames = target_frames;
    out->reference_frames = reference_frames;
    out->target_divisions = t.divisions;
    out->target_piece = t.piece;
    out->target_slots = t.slots;
    out->reference_divisions = r.divisions;
    out->reference_piece = r.piece;
    out->reference_slots = r.slots;
    out->workspace_bytes = carve_workspace(*plan, *out, nullptr).total_bytes;
    return MGB_OK;
}

int mgb_track_layout_init_profiled(const mgb_plan* plan, int64_t target_frames, mgb_track_layout* out) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(out != nullptr, MGB_ERR_INVALID, "layout is NULL");
    MGB_REQUIRE(target_frames > plan->fft_size, MGB_ERR_INVALID, "target (%lld) must be longer than fft_size (%d)",
                (long long)target_frames, plan->fft_size);
    MGB_REQUIRE(plan->max_piece_size > 0, MGB_ERR_INVALID, "max_piece_size must be positive");
    memset(out, 0, sizeof(*out));
    ReferenceGeometry t;
    MGB_TRY(signal_geometry(plan, target_frames, &t));
    out->target_frames = target_frames;
    out->target_divisions = t.divisions;
    out->target_piece = t.piece;
    out->target_slots = t.slots;
    out->workspace_bytes = carve_workspace(*plan, *out, nullptr).total_bytes;
    return MGB_OK;
}

int64_t mgb_reference_profile_bytes(const mgb_plan* plan) {
    if (check_plan(plan) != MGB_OK) return -1;
    return reference_profile_bytes(*plan);
}

static int reference_geometry(const mgb_plan* plan, int64_t reference_frames, ReferenceGeometry* g) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(reference_frames > plan->fft_size, MGB_ERR_INVALID, "reference (%lld) must be longer than fft_size (%d)",
                (long long)reference_frames, plan->fft_size);
    MGB_REQUIRE(plan->max_piece_size > 0, MGB_ERR_INVALID, "max_piece_size must be positive");
    return signal_geometry(plan, reference_frames, g);
}

int64_t mgb_reference_workspace_bytes(const mgb_plan* plan, int64_t reference_frames) {
    ReferenceGeometry g;
    if (reference_geometry(plan, reference_frames, &g) != MGB_OK) return -1;
    return carve_reference(*plan, g, nullptr).total_bytes;
}

int mgb_analyze_reference(const mgb_plan* plan, const float* d_reference_lr, int64_t reference_frames, void* d_workspace,
                          int64_t workspace_bytes, void* d_profile, void* stream) {
    ReferenceGeometry g;
    MGB_TRY(reference_geometry(plan, reference_frames, &g));
    MGB_TRY(check_aligned(d_reference_lr, "d_reference_lr"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    MGB_TRY(check_aligned(d_profile, "d_profile"));
    const ReferenceRegions need = carve_reference(*plan, g, nullptr);
    MGB_REQUIRE(workspace_bytes >= need.total_bytes, MGB_ERR_WORKSPACE, "analyze_reference: workspace of %lld bytes, need %lld",
                (long long)workspace_bytes, (long long)need.total_bytes);
    cudaStream_t st = (cudaStream_t)stream;
    const ReferenceRegions r = carve_reference(*plan, g, d_workspace);
    MGB_TRY(launch_analyze(*plan, (const float2*)d_reference_lr, g.frames, g.piece, g.divisions, g.slots, r.spec_part,
                           r.sumsq_part, r.absmax_part, st));
    return launch_reference_profile(*plan, g, r, (mgb_reference_profile*)d_profile, st);
}

int mgb_reference_profile_check(const mgb_plan* plan, const mgb_reference_profile* h) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(h != nullptr, MGB_ERR_INVALID, "profile header is NULL");
    MGB_REQUIRE(h->version == MGB_REFERENCE_PROFILE_VERSION, MGB_ERR_INVALID, "reference profile: version %d, this library reads %d",
                h->version, MGB_REFERENCE_PROFILE_VERSION);
#define MGB_PROFILE_FIELD(field, fmt, cast)                                                                             \
    MGB_REQUIRE(h->field == plan->field, MGB_ERR_INVALID, "reference profile: " #field " " fmt " differs from the Config's " fmt, \
                (cast)h->field, (cast)plan->field)
    MGB_PROFILE_FIELD(sample_rate, "%d", int);
    MGB_PROFILE_FIELD(fft_size, "%d", int);
    MGB_PROFILE_FIELD(n_lin, "%d", int);
    MGB_PROFILE_FIELD(max_piece_size, "%.17g", double);
    MGB_PROFILE_FIELD(threshold, "%.17g", double);
    MGB_PROFILE_FIELD(min_value, "%.17g", double);
#undef MGB_PROFILE_FIELD
    return MGB_OK;
}

int mgb_match_levels_profiled(const mgb_plan* plan, const mgb_track_layout* L, const float* d_target_lr, const void* d_profile,
                              void* d_workspace, mgb_track_state* d_state, void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_REQUIRE(layout_profiled(*L), MGB_ERR_INVALID,
                "match_levels_profiled: the layout has reference pieces (use mgb_track_layout_init_profiled)");
    MGB_TRY(check_aligned(d_target_lr, "d_target_lr"));
    MGB_TRY(check_aligned(d_profile, "d_profile"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    cudaStream_t st = (cudaStream_t)stream;
    Workspace ws = carve_workspace(*plan, *L, d_workspace);
    const size_t pbytes = (size_t)reference_profile_bytes(*plan);
#ifdef MGB_EMULATE
    memset(ws.zero_begin, 0, ws.zero_end - ws.zero_begin);
    memcpy((void*)ws.profile, d_profile, pbytes);
#else
    if (cudaMemsetAsync(ws.zero_begin, 0, ws.zero_end - ws.zero_begin, st) != cudaSuccess) return cuda_status("memset");
    if (cudaMemcpyAsync((void*)ws.profile, d_profile, pbytes, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        return cuda_status("profile copy");
#endif
    return launch_analyze(*plan, (const float2*)d_target_lr, L->target_frames, L->target_piece, L->target_divisions,
                          L->target_slots, ws.spec_part_t, ws.sumsq_part_t, ws.absmax_part_t, st);
}

int mgb_match_levels(const mgb_plan* plan, const mgb_track_layout* L, const float* d_target_lr,
                     const float* d_reference_lr, void* d_workspace, mgb_track_state* d_state, void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_REQUIRE(!layout_profiled(*L), MGB_ERR_INVALID,
                "match_levels: the layout is profiled (its reference comes from mgb_match_levels_profiled)");
    MGB_TRY(check_aligned(d_target_lr, "d_target_lr"));
    MGB_TRY(check_aligned(d_reference_lr, "d_reference_lr"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    cudaStream_t st = (cudaStream_t)stream;
    Workspace ws = carve_workspace(*plan, *L, d_workspace);
#ifdef MGB_EMULATE
    memset(ws.zero_begin, 0, ws.zero_end - ws.zero_begin);
#else
    if (cudaMemsetAsync(ws.zero_begin, 0, ws.zero_end - ws.zero_begin, st) != cudaSuccess) return cuda_status("memset");
#endif
    MGB_TRY(launch_analyze(*plan, (const float2*)d_target_lr, L->target_frames, L->target_piece, L->target_divisions,
                           L->target_slots, ws.spec_part_t, ws.sumsq_part_t, ws.absmax_part_t, st));
    // the level statistics themselves (masks, match RMS, c0, final amplitude coefficient) are computed
    // from these partial sums in the prologue of the next stage's first kernel and recorded in d_state
    return launch_analyze(*plan, (const float2*)d_reference_lr, L->reference_frames, L->reference_piece,
                          L->reference_divisions, L->reference_slots, ws.spec_part_r, ws.sumsq_part_r, ws.absmax_part_r,
                          st);
}

int mgb_match_frequencies(const mgb_plan* plan, const mgb_track_layout* L, const float* d_target_lr,
                          float* d_result_lr, double* d_fir_out, void* d_workspace, mgb_track_state* d_state,
                          void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_TRY(check_aligned(d_target_lr, "d_target_lr"));
    MGB_TRY(check_aligned(d_result_lr, "d_result_lr"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    MGB_TRY(mgb_design_frequencies(plan, L, d_fir_out, d_workspace, d_state, stream));
    return launch_convolve(*plan, *L, (const float2*)d_target_lr, (float2*)d_result_lr,
                           carve_workspace(*plan, *L, d_workspace), d_state, (cudaStream_t)stream);
}

int mgb_design_frequencies(const mgb_plan* plan, const mgb_track_layout* L, double* d_fir_out, void* d_workspace,
                           mgb_track_state* d_state, void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    return launch_design(*plan, *L, carve_workspace(*plan, *L, d_workspace), nullptr, d_fir_out, d_state,
                         (cudaStream_t)stream);
}

int mgb_match_frequencies_native(const mgb_plan* plan, const mgb_track_layout* L, const void* d_workspace,
                                 const mgb_track_state* d_state, const mgb_plan* native_plan,
                                 const mgb_track_layout* native_L, const float* d_native_target, float* d_native_result,
                                 double* d_fir_out, void* d_native_workspace, mgb_track_state* d_native_state,
                                 void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_TRY(check_plan(native_plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr && native_L != nullptr && d_native_state != nullptr, MGB_ERR_INVALID,
                "layout/state is NULL");
    const int R = plan->sample_rate, Rn = native_plan->sample_rate;
    MGB_REQUIRE(R > 0 && Rn > 0 && Rn != R, MGB_ERR_INVALID, "match_frequencies_native: rates %d and %d (they must differ)",
                R, Rn);
    const int octaves = (int)floor(log2((double)Rn / (double)R) + 0.5);
    const double want = ldexp((double)plan->fft_size, octaves);
    MGB_REQUIRE(want == (double)native_plan->fft_size, MGB_ERR_INVALID,
                "match_frequencies_native: fft_size %d at %d Hz, need %.0f for fft_size %d at %d Hz", native_plan->fft_size,
                Rn, want, plan->fft_size, R);
    MGB_REQUIRE(native_plan->d_native_idx != nullptr && native_plan->d_native_w != nullptr, MGB_ERR_INVALID,
                "match_frequencies_native: the native plan has no d_native_idx / d_native_w tables");
    MGB_REQUIRE(layout_profiled(*native_L) && native_L->target_frames > native_plan->fft_size &&
                    native_L->target_piece >= native_plan->fft_size,
                MGB_ERR_INVALID, "match_frequencies_native: the native layout must be a profiled layout of the native plan");
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    MGB_TRY(check_aligned(d_native_target, "d_native_target"));
    MGB_TRY(check_aligned(d_native_result, "d_native_result"));
    MGB_TRY(check_aligned(d_native_workspace, "d_native_workspace"));
    cudaStream_t st = (cudaStream_t)stream;
    const Workspace ws = carve_workspace(*plan, *L, const_cast<void*>(d_workspace));
    const Workspace nws = carve_workspace(*native_plan, *native_L, d_native_workspace);
    // the analysis job's scalars, with the quantities this job measures for itself cleared (the design kernel and
    // the convolution raise them by atomic maxima)
#ifdef MGB_EMULATE
    memset(nws.zero_begin, 0, nws.zero_end - nws.zero_begin);
    memset(nws.target_peak, 0, 4);
    memcpy(d_native_state, d_state, sizeof(mgb_track_state));
    d_native_state->conv_peak_bits = 0.0f;
    d_native_state->fir_peak_mid_bits = 0.0f;
    d_native_state->fir_peak_side_bits = 0.0f;
    d_native_state->conv_precise = 0;
#else
    if (cudaMemsetAsync(nws.zero_begin, 0, nws.zero_end - nws.zero_begin, st) != cudaSuccess ||
        cudaMemsetAsync(nws.target_peak, 0, 4, st) != cudaSuccess ||
        cudaMemcpyAsync(d_native_state, d_state, sizeof(mgb_track_state), cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
        cudaMemsetAsync(&d_native_state->conv_peak_bits, 0, sizeof(float), st) != cudaSuccess ||
        cudaMemsetAsync(&d_native_state->fir_peak_mid_bits, 0,
                        offsetof(mgb_track_state, conv_precise) + sizeof(int32_t) - offsetof(mgb_track_state, fir_peak_mid_bits),
                        st) != cudaSuccess)
        return cuda_status("match_frequencies_native: state copy");
#endif
    MGB_TRY(launch_absmax((const float2*)d_native_target, native_L->target_frames, nws.target_peak, st));
    MGB_TRY(launch_design_native(*plan, ws, *native_plan, *native_L, nws, d_fir_out, d_native_state, st));
    return launch_convolve(*native_plan, *native_L, (const float2*)d_native_target, (float2*)d_native_result, nws,
                           d_native_state, st);
}

// ---- album mastering ----------------------------------------------------------------------------------------------
// The album workspace: the design blocks of one job, then the FIR's spectra (mid, side) on the 2F-point and on the
// 4F-point grid (a track's convolution grid follows from its piece length, conv_frame_ovs).
struct AlbumRegions {
    double* design;
    int64_t design_stride;
    float2* h[2][2];  // [grid: 2F, 4F][mid, side]
    int64_t total_bytes;
};
static AlbumRegions carve_album(const mgb_plan& plan, void* base_ptr) {
    AlbumRegions r;
    const uintptr_t base = reinterpret_cast<uintptr_t>(base_ptr);
    int64_t off = 0;
    auto take = [&](int64_t bytes) {
        unsigned char* p = reinterpret_cast<unsigned char*>(base + (uintptr_t)off);
        off += align256(bytes);
        return p;
    };
    r.design_stride = (design_doubles_per_channel(plan) + 31) / 32 * 32;
    r.design = (double*)take(8 * r.design_stride * 8);
    for (int g = 0; g < 2; ++g)
        for (int c = 0; c < 2; ++c) r.h[g][c] = (float2*)take((2LL * plan.fft_size + 1) * 8);
    r.total_bytes = off;
    return r;
}

// a profiled layout of this plan for its own target length, as mgb_track_layout_init_profiled makes it
static int check_album_layout(const mgb_plan* plan, const mgb_track_layout* L, int t) {
    MGB_REQUIRE(L != nullptr, MGB_ERR_INVALID, "album: track %d has no layout", t);
    MGB_REQUIRE(layout_profiled(*L) && L->target_frames > plan->fft_size, MGB_ERR_INVALID,
                "album: track %d: the layout is not a profiled layout of this plan, or the track is not longer than fft_size", t);
    mgb_track_layout want;
    if (mgb_track_layout_init_profiled(plan, L->target_frames, &want) != MGB_OK ||
        memcmp(&want, L, sizeof(want)) != 0) {
        set_error("album: track %d: the layout is not this plan's profiled layout of %lld frames", t, (long long)L->target_frames);
        return MGB_ERR_INVALID;
    }
    return MGB_OK;
}

int64_t mgb_album_workspace_bytes(const mgb_plan* plan, int32_t tracks, const mgb_track_layout* layouts) {
    if (check_plan(plan) != MGB_OK || tracks < 1 || tracks > MGB_MAX_ALBUM_TRACKS || layouts == nullptr) return -1;
    for (int t = 0; t < tracks; ++t)
        if (check_album_layout(plan, &layouts[t], t) != MGB_OK) return -1;
    return carve_album(*plan, nullptr).total_bytes;
}

int mgb_album_match(const mgb_plan* plan, int32_t tracks, const mgb_album_track* t, const void* d_profile, double* d_fir_out,
                    void* d_album_ws, int64_t album_ws_bytes, void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(tracks >= 1 && tracks <= MGB_MAX_ALBUM_TRACKS, MGB_ERR_INVALID, "album: %d tracks (1 .. %d)", (int)tracks,
                MGB_MAX_ALBUM_TRACKS);
    MGB_REQUIRE(t != nullptr, MGB_ERR_INVALID, "album: the track table is NULL");
    std::vector<AlbumTrack> album((size_t)tracks);
    for (int k = 0; k < tracks; ++k) {
        MGB_TRY(check_album_layout(plan, t[k].layout, k));
        MGB_TRY(check_aligned(t[k].d_target_lr, "d_target_lr"));
        MGB_TRY(check_aligned(t[k].d_result_lr, "d_result_lr"));
        MGB_TRY(check_aligned(t[k].d_workspace, "d_workspace"));
        MGB_TRY(check_aligned(t[k].d_state, "d_state"));
        MGB_REQUIRE((const void*)t[k].d_result_lr != (const void*)t[k].d_target_lr, MGB_ERR_INVALID,
                    "album: track %d: d_result_lr is its d_target_lr", k);
        // (the analysis partials are addressed as 16-bit item numbers in the pooled kernel)
        MGB_REQUIRE((int64_t)t[k].layout->target_divisions * t[k].layout->target_slots < 65536, MGB_ERR_UNSUPPORTED,
                    "album: track %d has too many analysis items", k);
        album[k].layout = *t[k].layout;
        album[k].ws = carve_workspace(*plan, *t[k].layout, t[k].d_workspace);
        album[k].state = t[k].d_state;
    }
    MGB_TRY(check_aligned(d_profile, "d_profile"));
    MGB_TRY(check_aligned(d_album_ws, "d_album_ws"));
    const AlbumRegions need = carve_album(*plan, nullptr);
    MGB_REQUIRE(album_ws_bytes >= need.total_bytes, MGB_ERR_WORKSPACE, "album: workspace of %lld bytes, need %lld",
                (long long)album_ws_bytes, (long long)need.total_bytes);
    MGB_REQUIRE(album_mean_smem(album.data(), tracks) <= 227 * 1024, MGB_ERR_UNSUPPORTED,
                "album: %zu bytes of pooled piece statistics exceed one CTA's shared memory", album_mean_smem(album.data(), tracks));
    cudaStream_t st = (cudaStream_t)stream;
    {
        mgb_reference_profile h;
#ifdef MGB_EMULATE
        memcpy(&h, d_profile, sizeof(h));
#else
        if (cudaMemcpyAsync(&h, d_profile, sizeof(h), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess)
            return cuda_status("album: profile header");
#endif
        MGB_TRY(mgb_reference_profile_check(plan, &h));
    }
    // stage 1: each track's analysis, as its profiled job runs it
    for (int k = 0; k < tracks; ++k)
        MGB_TRY(mgb_match_levels_profiled(plan, t[k].layout, t[k].d_target_lr, d_profile, t[k].d_workspace, t[k].d_state,
                                          stream));
    // the album's level statistics and matching curve, then one FIR per convolution grid the tracks use; the first
    // track on a grid receives the FIR's peaks, the others copy them
    const AlbumRegions r = carve_album(*plan, d_album_ws);
    MGB_TRY(launch_album_mean(*plan, album.data(), tracks, album[0].ws.profile, r.design, r.design_stride, st));
    int leader[2] = {-1, -1};
    double* fir_out = d_fir_out;
    for (int k = 0; k < tracks; ++k) {
        const int grid = conv_frame_ovs(plan->fft_size, album[k].layout.target_piece) == 4 ? 1 : 0;
        if (leader[grid] < 0) {
            leader[grid] = k;
            MGB_TRY(launch_design_fir(*plan, r.design, r.design_stride, grid ? 4 : 2, r.h[grid][0], r.h[grid][1], fir_out,
                                      album[k].state, st));
            fir_out = nullptr;
        }
    }
    // stage 2: every track convolved with the album's FIR
    for (int k = 0; k < tracks; ++k) {
        const int grid = conv_frame_ovs(plan->fft_size, album[k].layout.target_piece) == 4 ? 1 : 0;
        if (leader[grid] != k) {
            float* dst = &album[k].state->fir_peak_mid_bits;
            const float* src = &album[leader[grid]].state->fir_peak_mid_bits;
#ifdef MGB_EMULATE
            memcpy(dst, src, 2 * sizeof(float));
#else
            if (cudaMemcpyAsync(dst, src, 2 * sizeof(float), cudaMemcpyDeviceToDevice, st) != cudaSuccess)
                return cuda_status("album: FIR peaks");
#endif
        }
        Workspace ws = album[k].ws;
        ws.h_mid = r.h[grid][0];
        ws.h_side = r.h[grid][1];
        MGB_TRY(launch_convolve(*plan, album[k].layout, (const float2*)t[k].d_target_lr, (float2*)t[k].d_result_lr, ws,
                                album[k].state, st));
    }
    // stage 3: one launch per step over the whole album
    for (int step = 1; step < plan->rms_correction_steps; ++step)
        MGB_TRY(launch_album_loud_sumsq(*plan, album.data(), tracks, step, st));
    return launch_album_correction_final(*plan, album.data(), tracks, st);
}

// ---- linked versions ----------------------------------------------------------------------------------------------
// Stage 4's scratch with versions: a copy of the main's scalars (whose normalisation coefficient and early-out flag the
// linked detector's maximum replaces), that maximum, and the linked detector plane D.
struct VersionRegions {
    mgb_track_state* state;
    float* d_max;
    float* d;
    int64_t total_bytes;
};
static VersionRegions carve_versions(const mgb_track_layout& L, void* base_ptr) {
    VersionRegions r;
    const uintptr_t base = reinterpret_cast<uintptr_t>(base_ptr);
    int64_t off = 0;
    auto take = [&](int64_t bytes) {
        unsigned char* p = reinterpret_cast<unsigned char*>(base + (uintptr_t)off);
        off += align256(bytes);
        return p;
    };
    r.state = (mgb_track_state*)take(sizeof(mgb_track_state));
    r.d_max = (float*)take(4);
    r.d = (float*)take(L.target_frames * 4);
    r.total_bytes = off;
    return r;
}

static int device_copy(void* dst, const void* src, size_t bytes, cudaStream_t st) {
#ifdef MGB_EMULATE
    (void)st;
    memcpy(dst, src, bytes);
#else
    if (cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return cuda_status("versions: copy");
#endif
    return MGB_OK;
}
static int device_zero(void* dst, size_t bytes, cudaStream_t st) {
#ifdef MGB_EMULATE
    (void)st;
    memset(dst, 0, bytes);
#else
    if (cudaMemsetAsync(dst, 0, bytes, st) != cudaSuccess) return cuda_status("versions: memset");
#endif
    return MGB_OK;
}

int64_t mgb_versions_workspace_bytes(const mgb_plan* plan, const mgb_track_layout* L) {
    if (check_plan(plan) != MGB_OK || L == nullptr || L->target_frames <= plan->fft_size) return -1;
    return carve_versions(*L, nullptr).total_bytes;
}

int mgb_version_match_frequencies(const mgb_plan* plan, const mgb_track_layout* L, const void* d_workspace,
                                  const mgb_track_state* d_state, int32_t versions, const mgb_version_track* v, void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_REQUIRE(versions >= 1 && versions <= MGB_MAX_VERSIONS, MGB_ERR_INVALID, "versions: %d versions (1 .. %d)", (int)versions,
                MGB_MAX_VERSIONS);
    MGB_REQUIRE(v != nullptr, MGB_ERR_INVALID, "versions: the version table is NULL");
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    MGB_TRY(check_aligned(d_state, "d_state"));
    for (int k = 0; k < versions; ++k) {
        const mgb_track_layout* VL = v[k].layout;
        MGB_REQUIRE(VL != nullptr && VL->target_frames == L->target_frames, MGB_ERR_INVALID,
                    "versions: version %d has no layout or not the main's %lld frames", k + 1, (long long)L->target_frames);
        mgb_track_layout want;
        if (mgb_track_layout_init_profiled(plan, VL->target_frames, &want) != MGB_OK || memcmp(&want, VL, sizeof(want)) != 0) {
            set_error("versions: version %d: the layout is not this plan's profiled layout of %lld frames", k + 1,
                      (long long)VL->target_frames);
            return MGB_ERR_INVALID;
        }
        MGB_TRY(check_aligned(v[k].d_target_lr, "d_target_lr"));
        MGB_TRY(check_aligned(v[k].d_result_lr, "d_result_lr"));
        MGB_TRY(check_aligned(v[k].d_workspace, "d_workspace"));
        MGB_TRY(check_aligned(v[k].d_state, "d_state"));
        for (int j = 0; j < versions; ++j) {
            MGB_REQUIRE((const void*)v[k].d_result_lr != (const void*)v[j].d_target_lr &&
                            (j == k || (const void*)v[k].d_result_lr != (const void*)v[j].d_result_lr),
                        MGB_ERR_INVALID, "versions: version %d's d_result_lr is a target or another result", k + 1);
        }
    }
    cudaStream_t st = (cudaStream_t)stream;
    const Workspace mws = carve_workspace(*plan, *L, const_cast<void*>(d_workspace));
    for (int k = 0; k < versions; ++k) {
        Workspace ws = carve_workspace(*plan, *v[k].layout, v[k].d_workspace);
        mgb_track_state* state = v[k].d_state;
        // the main's scalars (c0 is in the FIR spectra; the FIR's peaks choose the precision), with what the convolution
        // measures for itself cleared; the precision rule sees max(the main's peak, the version's own)
        MGB_TRY(device_zero(ws.zero_begin, ws.zero_end - ws.zero_begin, st));
        MGB_TRY(device_copy(state, d_state, sizeof(mgb_track_state), st));
        MGB_TRY(device_zero(&state->conv_peak_bits, sizeof(float), st));
        MGB_TRY(device_zero(&state->conv_precise, sizeof(int32_t), st));
        MGB_TRY(device_copy(ws.target_peak, mws.target_peak, sizeof(float), st));
        MGB_TRY(launch_absmax((const float2*)v[k].d_target_lr, v[k].layout->target_frames, ws.target_peak, st));
        ws.h_mid = mws.h_mid;
        ws.h_side = mws.h_side;
        MGB_TRY(launch_convolve(*plan, *v[k].layout, (const float2*)v[k].d_target_lr, (float2*)v[k].d_result_lr, ws, state, st));
    }
    return MGB_OK;
}

// the entries' checks shared by both stage-4 calls; loudness: every limited output required, the other two NULL
static int check_version_entries(int32_t entries, const mgb_version_entry* e, bool loudness) {
    MGB_REQUIRE(entries >= 1 && entries <= 1 + MGB_MAX_VERSIONS, MGB_ERR_INVALID, "versions: %d entries (1 .. %d)", (int)entries,
                1 + MGB_MAX_VERSIONS);
    MGB_REQUIRE(e != nullptr, MGB_ERR_INVALID, "versions: the entry table is NULL");
    for (int k = 0; k < entries; ++k) {
        MGB_TRY(check_aligned(e[k].d_result_lr, "d_result_lr"));
        const float* outs[3] = {e[k].d_out_limited, e[k].d_out_no_limiter, e[k].d_out_normalized};
        if (loudness) {
            MGB_TRY(check_aligned(outs[0], "d_out_limited"));
            MGB_REQUIRE(!outs[1] && !outs[2], MGB_ERR_INVALID,
                        "versions to loudness: entry %d: only d_out_limited is written here (the others must be NULL)", k);
        }
        for (int i = 0; i < 3; ++i) {
            if (!outs[i]) continue;
            MGB_TRY(check_aligned(outs[i], "output"));
            for (int j = 0; j < entries; ++j) {
                MGB_REQUIRE((const void*)outs[i] != (const void*)e[j].d_result_lr, MGB_ERR_INVALID,
                            "versions: an output of entry %d is the result of entry %d", k, j);
                const float* other[3] = {e[j].d_out_limited, e[j].d_out_no_limiter, e[j].d_out_normalized};
                for (int m = 0; m < 3; ++m)
                    MGB_REQUIRE((j == k && m == i) || outs[i] != other[m], MGB_ERR_INVALID,
                                "versions: an output of entry %d is another output", k);
            }
        }
    }
    return MGB_OK;
}

// the linked detector over every entry's result into r.d / r.d_max (true-peak mode: the main's detector, then each
// version's added to it)
static int versions_detect(const mgb_plan& plan, int64_t n, int32_t entries, const mgb_version_entry* e, const VersionRegions& r,
                           cudaStream_t st) {
    MGB_TRY(device_zero(r.d_max, 4, st));
    if (plan.limiter.true_peak) {
        MGB_TRY(launch_true_peak_detect(plan.limiter.true_peak, (const float2*)e[0].d_result_lr, n, r.d, r.d_max, st));
        for (int k = 1; k < entries; ++k)
            MGB_TRY(launch_true_peak_accumulate(plan.limiter.true_peak, (const float2*)e[k].d_result_lr, n, r.d, r.d_max, st));
        return MGB_OK;
    }
    VersionPlanes all;
    memset(&all, 0, sizeof(all));
    all.count = entries;
    for (int k = 0; k < entries; ++k) all.in[k] = (const float2*)e[k].d_result_lr;
    return launch_versions_detect(all, n, r.d, r.d_max, st);
}

int mgb_finalize_versions(const mgb_plan* plan, const mgb_track_layout* L, int32_t entries, const mgb_version_entry* e,
                          void* d_workspace, const mgb_track_state* d_state, void* d_versions_ws, int64_t versions_ws_bytes,
                          void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_TRY(check_version_entries(entries, e, false));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    MGB_TRY(check_aligned(d_versions_ws, "d_versions_ws"));
    const int64_t need = mgb_versions_workspace_bytes(plan, L);
    MGB_REQUIRE(need > 0, MGB_ERR_INVALID, "versions: the layout has no more than fft_size frames");
    MGB_REQUIRE(versions_ws_bytes >= need, MGB_ERR_WORKSPACE, "versions: workspace of %lld bytes, need %lld",
                (long long)versions_ws_bytes, (long long)need);
    cudaStream_t st = (cudaStream_t)stream;
    const Workspace ws = carve_workspace(*plan, *L, d_workspace);
    const VersionRegions r = carve_versions(*L, d_versions_ws);
    const int64_t n = L->target_frames;
    VersionPlanes lim;
    memset(&lim, 0, sizeof(lim));
    bool normalized = false;
    for (int k = 0; k < entries; ++k) {
        if (e[k].d_out_limited) {
            lim.in[lim.count] = (const float2*)e[k].d_result_lr;
            lim.out[lim.count++] = (float2*)e[k].d_out_limited;
        }
        normalized = normalized || e[k].d_out_normalized;
    }
    MGB_TRY(device_copy(r.state, d_state, sizeof(mgb_track_state), st));
    if (lim.count || normalized) {
        // max(D) in place of the main's own peak: the normalisation coefficient and the early-out (true_peak_final_kernel's
        // rule is correction_final_kernel's, from any peak)
        MGB_TRY(versions_detect(*plan, n, entries, e, r, st));
        MGB_TRY(launch_true_peak_final(r.d_max, plan->min_value, plan->threshold, r.state, st));
    }
    for (int k = 0; k < entries; ++k) {
        const float2* res = (const float2*)e[k].d_result_lr;
        if (e[k].d_out_normalized)
            MGB_TRY(launch_scale(res, (float2*)e[k].d_out_normalized, n, &r.state->gain, &r.state->normalize_coef, st));
        if (e[k].d_out_no_limiter) MGB_TRY(launch_scale(res, (float2*)e[k].d_out_no_limiter, n, &r.state->gain, nullptr, st));
    }
    if (!lim.count) return MGB_OK;
    MGB_REQUIRE(plan->d_limiter_tables != nullptr, MGB_ERR_INVALID, "versions: the plan has no limiter tables");
    MGB_TRY(device_zero(ws.tickets, ws.limiter_zero_bytes, st));
    return launch_limiter_versions(plan->limiter, lim, n, &r.state->gain, &r.state->final_amplitude_coef, &r.state->limiter_engaged,
                                   ws.tickets, ws.lookback, ws.limiter_planes, plan->d_limiter_tables, r.d, st);
}

int mgb_finalize_versions_to_loudness(const mgb_plan* plan, const mgb_track_layout* L, const mgb_loudness_params* meter,
                                      const mgb_loudness_target* target, int32_t entries, const mgb_version_entry* e,
                                      void* d_workspace, const mgb_track_state* d_state, void* d_versions_ws,
                                      int64_t versions_ws_bytes, void* d_search_ws, int64_t search_ws_bytes,
                                      mgb_loudness_target_report* d_report, void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_TRY(loudness_target_validate(target, meter));
    MGB_REQUIRE(meter->sample_rate == plan->sample_rate, MGB_ERR_INVALID,
                "versions to loudness: the meter's rate %d differs from the plan's %d", meter->sample_rate, plan->sample_rate);
    MGB_REQUIRE(plan->d_limiter_tables != nullptr, MGB_ERR_INVALID, "versions to loudness: the plan has no limiter tables");
    MGB_TRY(check_version_entries(entries, e, true));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    MGB_TRY(check_aligned(d_versions_ws, "d_versions_ws"));
    MGB_TRY(check_aligned(d_search_ws, "d_search_ws"));
    MGB_TRY(check_aligned(d_report, "d_report"));
    const int64_t need = mgb_versions_workspace_bytes(plan, L);
    MGB_REQUIRE(need > 0, MGB_ERR_INVALID, "versions: the layout has no more than fft_size frames");
    MGB_REQUIRE(versions_ws_bytes >= need, MGB_ERR_WORKSPACE, "versions: workspace of %lld bytes, need %lld",
                (long long)versions_ws_bytes, (long long)need);
    const int64_t n = L->target_frames;
    const int64_t search_need = loudness_target_search_bytes(*meter, n);
    MGB_REQUIRE(search_ws_bytes >= search_need, MGB_ERR_WORKSPACE,
                "versions to loudness: search workspace of %lld bytes, need %lld", (long long)search_ws_bytes,
                (long long)search_need);
    cudaStream_t st = (cudaStream_t)stream;
    const Workspace ws = carve_workspace(*plan, *L, d_workspace);
    const VersionRegions r = carve_versions(*L, d_versions_ws);
    VersionPlanes vp;
    memset(&vp, 0, sizeof(vp));
    vp.count = entries;
    for (int k = 0; k < entries; ++k) {
        vp.in[k] = (const float2*)e[k].d_result_lr;
        vp.out[k] = (float2*)e[k].d_out_limited;
    }
    MGB_TRY(device_zero(ws.tickets, ws.limiter_zero_bytes, st));
    MGB_TRY(versions_detect(*plan, n, entries, e, r, st));
    // s = result * gain of the main, metered once from its output (the first pass overwrites it)
    MGB_TRY(launch_scale(vp.in[0], vp.out[0], n, &d_state->gain, nullptr, st));
    return run_versions_loudness_search(plan->limiter, *meter, *target, vp, vp.out[0], n, &d_state->gain, r.d_max, r.d, ws.tickets,
                                        ws.limiter_zero_bytes, ws.lookback, ws.limiter_planes, plan->d_limiter_tables, d_search_ws,
                                        d_report, st);
}

int mgb_correct_levels(const mgb_plan* plan, const mgb_track_layout* L, void* d_workspace, mgb_track_state* d_state,
                       void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    cudaStream_t st = (cudaStream_t)stream;
    Workspace ws = carve_workspace(*plan, *L, d_workspace);
    // step 0's per-piece sums and loud lists come out of the convolution kernel's epilogue (gain is
    // still 1 there); each later step is one pass over the loud lists (over the result, for a piece
    // whose list overflowed or at a gain where quiet samples could clip: the result must be unchanged
    // since mgb_match_frequencies) that first derives the previous step's coefficient from that step's
    // sums; a last small kernel closes the chain and writes the scalars __finalize needs.
    for (int step = 1; step < plan->rms_correction_steps; ++step) MGB_TRY(launch_loud_sumsq(*plan, *L, ws, step, d_state, st));
    return launch_correction_final(*plan, *L, ws, d_state, st);
}

int mgb_finalize(const mgb_plan* plan, const mgb_track_layout* L, const float* d_result_lr, float* d_out_limited,
                 float* d_out_no_limiter, float* d_out_normalized, void* d_workspace, mgb_track_state* d_state,
                 void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_TRY(check_aligned(d_result_lr, "d_result_lr"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    cudaStream_t st = (cudaStream_t)stream;
    Workspace ws = carve_workspace(*plan, *L, d_workspace);
    const float2* res = (const float2*)d_result_lr;
    const bool tp = plan->limiter.true_peak != 0;
    auto clear_limiter = [&]() -> int {
#ifdef MGB_EMULATE
        memset(ws.tickets, 0, ws.limiter_zero_bytes);
#else
        if (cudaMemsetAsync(ws.tickets, 0, ws.limiter_zero_bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
        return MGB_OK;
    };
    if (tp && (d_out_limited || d_out_normalized)) {
        // true-peak mode: the detector over the result, then the normalisation coefficient and the limiter's early-out
        // from gain * max(d) in place of the sample peak's (correction_final_kernel)
        MGB_TRY(clear_limiter());
        MGB_TRY(launch_true_peak_detect(plan->limiter.true_peak, res, L->target_frames, ws.tp_plane, ws.tp_peak, st));
        MGB_TRY(launch_true_peak_final(ws.tp_peak, plan->min_value, plan->threshold, d_state, st));
    }
    if (d_out_normalized) {
        MGB_TRY(check_aligned(d_out_normalized, "d_out_normalized"));
        MGB_TRY(launch_scale(res, (float2*)d_out_normalized, L->target_frames, &d_state->gain, &d_state->normalize_coef, st));
    }
    if (d_out_no_limiter) {
        MGB_TRY(check_aligned(d_out_no_limiter, "d_out_no_limiter"));
        MGB_TRY(launch_scale(res, (float2*)d_out_no_limiter, L->target_frames, &d_state->gain, nullptr, st));
    }
    if (d_out_limited) {
        MGB_TRY(check_aligned(d_out_limited, "d_out_limited"));
        if (!tp) MGB_TRY(clear_limiter());  // (in true-peak mode, cleared before the detector, which only sets tp_peak)
        MGB_TRY(launch_limiter(plan->limiter, res, (float2*)d_out_limited, L->target_frames, &d_state->gain,
                               &d_state->final_amplitude_coef, &d_state->limiter_engaged, ws.tickets,
                               ws.lookback, ws.limiter_planes, plan->d_limiter_tables, st, false, ws.tp_plane));
    }
    return MGB_OK;
}

int mgb_finalize_to_loudness(const mgb_plan* plan, const mgb_track_layout* L, const mgb_loudness_params* meter,
                             const mgb_loudness_target* target, const float* d_result_lr, float* d_out_limited,
                             void* d_workspace, void* d_search_ws, int64_t search_ws_bytes, mgb_track_state* d_state,
                             mgb_loudness_target_report* d_report, void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_TRY(loudness_target_validate(target, meter));
    MGB_REQUIRE(meter->sample_rate == plan->sample_rate, MGB_ERR_INVALID,
                "finalize_to_loudness: the meter's rate %d differs from the plan's %d", meter->sample_rate, plan->sample_rate);
    MGB_REQUIRE(plan->d_limiter_tables != nullptr, MGB_ERR_INVALID, "finalize_to_loudness: the plan has no limiter tables");
    MGB_TRY(check_aligned(d_result_lr, "d_result_lr"));
    MGB_TRY(check_aligned(d_out_limited, "d_out_limited"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    MGB_TRY(check_aligned(d_search_ws, "d_search_ws"));
    MGB_TRY(check_aligned(d_report, "d_report"));
    // (s = result * gain is staged in d_out_limited while every pass still reads the result)
    MGB_REQUIRE((const void*)d_out_limited != (const void*)d_result_lr, MGB_ERR_INVALID,
                "finalize_to_loudness: d_out_limited must not be d_result_lr (the output is the search's scratch)");
    const int64_t need = loudness_target_search_bytes(*meter, L->target_frames);
    MGB_REQUIRE(search_ws_bytes >= need, MGB_ERR_WORKSPACE, "finalize_to_loudness: search workspace of %lld bytes, need %lld",
                (long long)search_ws_bytes, (long long)need);
    cudaStream_t st = (cudaStream_t)stream;
    Workspace ws = carve_workspace(*plan, *L, d_workspace);
    const float2* res = (const float2*)d_result_lr;
    const int64_t n = L->target_frames;
    const bool tp = plan->limiter.true_peak != 0;
    if (tp) {  // the detector once, over the result: d is linear in the input and the limiter scales it by its pre-gain
#ifdef MGB_EMULATE
        memset(ws.tickets, 0, ws.limiter_zero_bytes);
#else
        if (cudaMemsetAsync(ws.tickets, 0, ws.limiter_zero_bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
        MGB_TRY(launch_true_peak_detect(plan->limiter.true_peak, res, n, ws.tp_plane, ws.tp_peak, st));
    }
    // s = result * gain, metered once from d_out_limited (the first pass overwrites it)
    MGB_TRY(launch_scale(res, (float2*)d_out_limited, n, &d_state->gain, nullptr, st));
    return run_loudness_search(plan->limiter, *meter, *target, res, (const float2*)d_out_limited, (float2*)d_out_limited, n,
                               &d_state->gain, tp ? nullptr : &d_state->result_peak, tp ? ws.tp_peak : nullptr, ws.tickets,
                               ws.limiter_zero_bytes, nullptr, ws.lookback, ws.limiter_planes, plan->d_limiter_tables,
                               tp ? ws.tp_plane : nullptr, d_search_ws, d_report, st);
}

int mgb_album_finalize_to_loudness(const mgb_plan* plan, int32_t tracks, const mgb_album_track* t,
                                   float* const* d_out_limited, const mgb_loudness_params* meter,
                                   const mgb_loudness_target* target, void* d_search_ws, int64_t search_ws_bytes,
                                   mgb_loudness_target_report* d_report, void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(tracks >= 1 && tracks <= MGB_MAX_ALBUM_TRACKS, MGB_ERR_INVALID, "album loudness target: %d tracks (1 .. %d)",
                (int)tracks, MGB_MAX_ALBUM_TRACKS);
    MGB_REQUIRE(t != nullptr && d_out_limited != nullptr, MGB_ERR_INVALID,
                "album loudness target: the track table or the output table is NULL");
    MGB_TRY(loudness_target_validate(target, meter));
    MGB_REQUIRE(meter->sample_rate == plan->sample_rate, MGB_ERR_INVALID,
                "album loudness target: the meter's rate %d differs from the plan's %d", meter->sample_rate, plan->sample_rate);
    MGB_REQUIRE(plan->d_limiter_tables != nullptr, MGB_ERR_INVALID, "album loudness target: the plan has no limiter tables");
    std::vector<mgb_track_layout> layouts((size_t)tracks);
    for (int k = 0; k < tracks; ++k) {
        MGB_TRY(check_album_layout(plan, t[k].layout, k));
        MGB_TRY(check_aligned(t[k].d_result_lr, "d_result_lr"));
        MGB_TRY(check_aligned(t[k].d_workspace, "d_workspace"));
        MGB_TRY(check_aligned(t[k].d_state, "d_state"));
        MGB_TRY(check_aligned(d_out_limited[k], "d_out_limited"));
        // (s = result * gain is staged in the output while every pass still reads the result)
        MGB_REQUIRE((const void*)d_out_limited[k] != (const void*)t[k].d_result_lr, MGB_ERR_INVALID,
                    "album loudness target: track %d: d_out_limited is its d_result_lr (the output is the search's scratch)", k);
        layouts[k] = *t[k].layout;
    }
    MGB_TRY(check_aligned(d_search_ws, "d_search_ws"));
    MGB_TRY(check_aligned(d_report, "d_report"));
    const int64_t need = mgb_album_loudness_target_workspace_bytes(meter, tracks, layouts.data());
    MGB_REQUIRE(search_ws_bytes >= need, MGB_ERR_WORKSPACE, "album loudness target: search workspace of %lld bytes, need %lld",
                (long long)search_ws_bytes, (long long)need);
    cudaStream_t st = (cudaStream_t)stream;
    const bool tp = plan->limiter.true_peak != 0;
    std::vector<AlbumSearchTrack> album((size_t)tracks);
    for (int k = 0; k < tracks; ++k) {
        const Workspace ws = carve_workspace(*plan, layouts[k], t[k].d_workspace);
        const float2* res = (const float2*)t[k].d_result_lr;
        const int64_t n = layouts[k].target_frames;
        mgb_track_state* state = t[k].d_state;
        if (tp) {  // each track's detector once, as mgb_finalize_to_loudness runs it
#ifdef MGB_EMULATE
            memset(ws.tickets, 0, ws.limiter_zero_bytes);
#else
            if (cudaMemsetAsync(ws.tickets, 0, ws.limiter_zero_bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
            MGB_TRY(launch_true_peak_detect(plan->limiter.true_peak, res, n, ws.tp_plane, ws.tp_peak, st));
        }
        MGB_TRY(launch_scale(res, (float2*)d_out_limited[k], n, &state->gain, nullptr, st));
        AlbumSearchTrack& e = album[k];
        e.in = res;
        e.s_metered = e.out = (float2*)d_out_limited[k];
        e.frames = n;
        e.gain = &state->gain;
        e.peak_d = tp ? nullptr : &state->result_peak;
        e.peak_bits = tp ? ws.tp_peak : nullptr;
        e.zero = ws.tickets;
        e.zero_bytes = ws.limiter_zero_bytes;
        e.lookback = ws.lookback;
        e.planes = ws.limiter_planes;
        e.tp_d = tp ? ws.tp_plane : nullptr;
    }
    return run_album_loudness_search(plan->limiter, *meter, *target, album.data(), tracks, plan->d_limiter_tables,
                                     d_search_ws, d_report, st);
}

// standalone limiter workspace: [0,4): peak bits  [16,20): ticket  [32,36): the true-peak detector's maximum  [256, kLimitHeader):
// pole tables  [kLimitHeader, ...): look-back words, then the wide-window path's planes (none for the halo kernel), then the
// true-peak detector's plane (true-peak mode only)
static const int64_t kLimitHeader = 256 + 32768;

int64_t mgb_limiter_workspace_bytes(const mgb_limiter_params* params, int64_t frames) {
    if (!params) return -1;
    if (frames <= 0) return kLimitHeader;
    return kLimitHeader + limiter_lookback_bytes(*params, frames) + limiter_plane_bytes(*params, frames) +
           true_peak_plane_bytes(*params, frames);
}

static int limit_impl(const mgb_limiter_params* params, const float* d_in_lr, float* d_out_lr, int64_t frames,
                      void* d_workspace, int64_t workspace_bytes, int32_t* d_engaged, void* stream, bool gains_only) {
    MGB_REQUIRE(params != nullptr, MGB_ERR_INVALID, "params is NULL");
    MGB_TRY(limiter_validate(*params));
    MGB_TRY(check_aligned(d_in_lr, "d_in_lr"));
    MGB_TRY(check_aligned(d_out_lr, "d_out_lr"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    MGB_REQUIRE(d_engaged != nullptr, MGB_ERR_INVALID, "d_engaged is NULL");
    MGB_REQUIRE(frames > 6, MGB_ERR_INVALID, "limit: the input must be longer than filtfilt's padlen (6)");
    MGB_REQUIRE(limiter_tables_bytes() <= 32768, MGB_ERR_WORKSPACE, "limit: pole tables outgrew the workspace header");
    MGB_REQUIRE(workspace_bytes >= mgb_limiter_workspace_bytes(params, frames), MGB_ERR_WORKSPACE,
                "limit: workspace of %lld bytes, need %lld", (long long)workspace_bytes,
                (long long)mgb_limiter_workspace_bytes(params, frames));
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char* base = (unsigned char*)d_workspace;
    const int64_t zero_bytes = kLimitHeader + limiter_lookback_bytes(*params, frames);
#ifdef MGB_EMULATE
    memset(base, 0, zero_bytes);
#else
    if (cudaMemsetAsync(base, 0, zero_bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
    void* tables = base + 256;
    MGB_TRY(launch_limiter_tables(*params, tables, st));
    float* peak = (float*)base;
    int* ticket = (int*)(base + 16);
    float* tp_d = nullptr;
    if (params->true_peak) {  // the early-out on max(d) instead of the sample peak
        tp_d = (float*)(base + zero_bytes + limiter_plane_bytes(*params, frames));
        float* tp_peak = (float*)(base + 32);
        MGB_TRY(launch_true_peak_detect(params->true_peak, (const float2*)d_in_lr, frames, tp_d, tp_peak, st));
        MGB_TRY(launch_limiter_engaged(tp_peak, nullptr, params->threshold, d_engaged, st));
    } else {
        MGB_TRY(launch_absmax((const float2*)d_in_lr, frames, peak, st));
        MGB_TRY(launch_limiter_engaged(peak, nullptr, params->threshold, d_engaged, st));
    }
    return launch_limiter(*params, (const float2*)d_in_lr, (float2*)d_out_lr, frames, nullptr, nullptr, d_engaged, ticket,
                          base + kLimitHeader, base + zero_bytes, tables, st, gains_only, tp_d);
}

int mgb_limit(const mgb_limiter_params* params, const float* d_in_lr, float* d_out_lr, int64_t frames,
              void* d_workspace, int64_t workspace_bytes, int32_t* d_engaged, void* stream) {
    return limit_impl(params, d_in_lr, d_out_lr, frames, d_workspace, workspace_bytes, d_engaged, stream, false);
}

int mgb_test_limiter_gains(const mgb_limiter_params* params, const float* d_in_lr, float* d_gains_out, int64_t frames,
                           void* d_workspace, int64_t workspace_bytes, int32_t* d_engaged, void* stream) {
    return limit_impl(params, d_in_lr, d_gains_out, frames, d_workspace, workspace_bytes, d_engaged, stream, true);
}

int mgb_test_true_peak_detect(int32_t oversample, const float* d_lr, int64_t frames, float* d_out, float* d_max,
                              void* stream) {
    MGB_REQUIRE(oversample == 1 || oversample == 2 || oversample == 4, MGB_ERR_INVALID,
                "true_peak_detect: oversampling %d (1, 2 or 4)", oversample);
    MGB_TRY(check_aligned(d_lr, "d_lr"));
    MGB_TRY(check_aligned(d_out, "d_out"));
    MGB_TRY(check_aligned(d_max, "d_max"));
    MGB_REQUIRE(frames > 0, MGB_ERR_INVALID, "true_peak_detect: no frames");
    return launch_true_peak_detect(oversample, (const float2*)d_lr, frames, d_out, d_max, (cudaStream_t)stream);
}

int mgb_process_host(const mgb_plan* plan, const mgb_track_layout* L, const float* h_target_lr,
                     const float* h_reference_lr, float* h_out_limited, float* h_out_no_limiter,
                     float* h_out_normalized, float* d_target_lr, float* d_reference_lr, float* d_result_lr,
                     float* d_out_lr, void* d_workspace, mgb_track_state* d_state, mgb_track_state* h_state_out,
                     void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L && h_target_lr && h_reference_lr && d_state, MGB_ERR_INVALID, "NULL argument");
    MGB_REQUIRE(h_out_limited || h_out_no_limiter || h_out_normalized, MGB_ERR_INVALID, "no output requested");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t tbytes = (size_t)L->target_frames * 8, rbytes = (size_t)L->reference_frames * 8;
#ifdef MGB_EMULATE
    memcpy(d_target_lr, h_target_lr, tbytes);
    memcpy(d_reference_lr, h_reference_lr, rbytes);
#else
    if (cudaMemcpyAsync(d_target_lr, h_target_lr, tbytes, cudaMemcpyHostToDevice, st) != cudaSuccess) return cuda_status("H2D target");
    if (cudaMemcpyAsync(d_reference_lr, h_reference_lr, rbytes, cudaMemcpyHostToDevice, st) != cudaSuccess) return cuda_status("H2D reference");
#endif
    MGB_TRY(mgb_match_levels(plan, L, d_target_lr, d_reference_lr, d_workspace, d_state, stream));
    MGB_TRY(mgb_match_frequencies(plan, L, d_target_lr, d_result_lr, nullptr, d_workspace, d_state, stream));
    MGB_TRY(mgb_correct_levels(plan, L, d_workspace, d_state, stream));
    float* outs[3] = {h_out_limited, h_out_no_limiter, h_out_normalized};
    for (int k = 0; k < 3; ++k) {
        if (!outs[k]) continue;
        MGB_TRY(mgb_finalize(plan, L, d_result_lr, k == 0 ? d_out_lr : nullptr, k == 1 ? d_out_lr : nullptr,
                             k == 2 ? d_out_lr : nullptr, d_workspace, d_state, stream));
#ifdef MGB_EMULATE
        memcpy(outs[k], d_out_lr, tbytes);
#else
        if (cudaMemcpyAsync(outs[k], d_out_lr, tbytes, cudaMemcpyDeviceToHost, st) != cudaSuccess) return cuda_status("D2H result");
#endif
    }
#ifdef MGB_EMULATE
    if (h_state_out) memcpy(h_state_out, d_state, sizeof(mgb_track_state));
#else
    if (h_state_out && cudaMemcpyAsync(h_state_out, d_state, sizeof(mgb_track_state), cudaMemcpyDeviceToHost, st) != cudaSuccess)
        return cuda_status("D2H state");
    if (cudaStreamSynchronize(st) != cudaSuccess) return cuda_status("stream sync");
#endif
    return MGB_OK;
}

int mgb_convert_f64_to_f32(const double* d_in, float* d_out, int64_t count, void* stream) {
    MGB_REQUIRE(d_in && d_out && count >= 0, MGB_ERR_INVALID, "convert: bad arguments");
    return launch_convert_f64_f32(d_in, d_out, count, (cudaStream_t)stream);
}
int mgb_convert_f32_to_f64(const float* d_in, double* d_out, int64_t count, void* stream) {
    MGB_REQUIRE(d_in && d_out && count >= 0, MGB_ERR_INVALID, "convert: bad arguments");
    return launch_convert_f32_f64(d_in, d_out, count, (cudaStream_t)stream);
}

int mgb_pcm_decode(const void* d_pcm, int32_t bits, float* d_out, int64_t count, void* stream) {
    MGB_REQUIRE(d_pcm && d_out && count >= 0, MGB_ERR_INVALID, "pcm_decode: bad arguments");
    return launch_pcm_decode(d_pcm, bits, d_out, count, (cudaStream_t)stream);
}
int mgb_pcm_encode(const float* d_in, int32_t bits, void* d_pcm, int64_t count, void* stream) {
    MGB_REQUIRE(d_pcm && d_in && count >= 0, MGB_ERR_INVALID, "pcm_encode: bad arguments");
    return launch_pcm_encode(d_in, bits, d_pcm, count, (cudaStream_t)stream);
}

int mgb_pcm_encode_dithered(const mgb_dither_params* params, const float* d_lr, int64_t frames, int32_t bits, void* d_pcm,
                            void* stream) {
    MGB_TRY(dither_validate(params));
    MGB_REQUIRE(bits == 16 || bits == 24, MGB_ERR_UNSUPPORTED, "pcm_encode_dithered: %d-bit samples (16 and 24)", bits);
    MGB_TRY(check_aligned(d_lr, "d_lr"));
    MGB_TRY(check_aligned(d_pcm, "d_pcm"));
    MGB_REQUIRE(frames >= 0, MGB_ERR_INVALID, "pcm_encode_dithered: %lld frames", (long long)frames);
    if (frames == 0) return MGB_OK;
    return launch_pcm_encode_dithered(*params, d_lr, frames, bits, d_pcm, (cudaStream_t)stream);
}

int mgb_check_peaks(const float* d_lr, int64_t frames, void* d_scratch16, void* stream) {
    MGB_REQUIRE(d_lr && d_scratch16 && frames > 0, MGB_ERR_INVALID, "check_peaks: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
#ifdef MGB_EMULATE
    memset(d_scratch16, 0, 16);
#else
    if (cudaMemsetAsync(d_scratch16, 0, 16, st) != cudaSuccess) return cuda_status("memset");
#endif
    return launch_peak_count(d_lr, frames * 2, (float*)d_scratch16, (unsigned long long*)((char*)d_scratch16 + 8), st);
}

int mgb_check_equality(const float* d_a_lr, const float* d_b_lr, int64_t frames, void* d_scratch8, void* stream) {
    MGB_REQUIRE(d_a_lr && d_b_lr && d_scratch8 && frames > 0, MGB_ERR_INVALID, "check_equality: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
#ifdef MGB_EMULATE
    memset(d_scratch8, 0, 8);
#else
    if (cudaMemsetAsync(d_scratch8, 0, 8, st) != cudaSuccess) return cuda_status("memset");
#endif
    return launch_count_different(d_a_lr, d_b_lr, frames * 2, (unsigned long long*)d_scratch8, st);
}

int mgb_window_energy(const float* d_lr, int64_t frames, int64_t window, int64_t step, int32_t count, double* d_energy,
                      void* stream) {
    MGB_REQUIRE(d_lr && d_energy && window > 0 && step > 0 && count > 0, MGB_ERR_INVALID, "window_energy: bad arguments");
    MGB_REQUIRE((int64_t)(count - 1) * step + window <= frames, MGB_ERR_INVALID,
                "window_energy: %d windows of %lld frames every %lld do not fit in %lld frames", count, (long long)window,
                (long long)step, (long long)frames);
    MGB_REQUIRE(count <= 65535, MGB_ERR_INVALID, "window_energy: too many windows (%d)", count);
    cudaStream_t st = (cudaStream_t)stream;
#ifdef MGB_EMULATE
    memset(d_energy, 0, sizeof(double) * count);
#else
    if (cudaMemsetAsync(d_energy, 0, sizeof(double) * count, st) != cudaSuccess) return cuda_status("memset");
#endif
    return launch_window_energy((const float2*)d_lr, window, step, count, d_energy, st);
}

int mgb_preview_piece(const float* d_in_lr, float* d_out_lr, int64_t frames, double clip_to, int64_t fade_frames,
                      void* stream) {
    MGB_REQUIRE(d_in_lr && d_out_lr && frames > 0, MGB_ERR_INVALID, "preview_piece: bad arguments");
    MGB_REQUIRE(fade_frames >= 0 && 2 * fade_frames <= frames, MGB_ERR_INVALID,
                "preview_piece: two fades of %lld frames do not fit in %lld", (long long)fade_frames, (long long)frames);
    return launch_preview_piece((const float2*)d_in_lr, (float2*)d_out_lr, frames, (float)clip_to, fade_frames,
                                (cudaStream_t)stream);
}

int mgb_test_fft(int32_t n, int32_t is_f64, int32_t dir, const void* d_in, void* d_out, int32_t batch,
                 const void* d_twiddles, void* stream) {
    MGB_REQUIRE(d_in && d_out && d_twiddles && batch > 0, MGB_ERR_INVALID, "test_fft: bad arguments");
    return launch_test_fft(n, is_f64, dir, d_in, d_out, batch, d_twiddles, (cudaStream_t)stream);
}

int mgb_test_workspace_regions(const mgb_plan* plan, const mgb_track_layout* layout, int64_t out[16]) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(layout != nullptr && out != nullptr, MGB_ERR_INVALID, "test_workspace_regions: NULL argument");
    const Workspace w = carve_workspace(*plan, *layout, nullptr);  // pointers = byte offsets
    const void* regions[13] = {w.spec_part_t, w.spec_part_r, w.sumsq_part_t, w.sumsq_part_r, w.absmax_part_t,
                               w.absmax_part_r, w.mask_t, w.mask_r, w.h_mid, w.h_side, w.loud_values, w.piece_sums,
                               w.loud_count};
    for (int i = 0; i < 16; ++i) out[i] = 0;
    for (int i = 0; i < 13; ++i) out[i] = (int64_t)reinterpret_cast<uintptr_t>(regions[i]);
    out[13] = w.loud_capacity;
    out[14] = (int64_t)reinterpret_cast<uintptr_t>(w.tickets);  // the limiter's tickets and look-back words, which
    out[15] = w.limiter_zero_bytes;                              // mgb_finalize clears before every limiter launch
    return MGB_OK;
}

int mgb_test_design_fir(const mgb_plan* plan, const double* d_avg, double* d_fir_out, void* d_workspace, void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(d_avg && d_fir_out, MGB_ERR_INVALID, "test_design_fir: NULL argument");
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    // workspace: [8][stride] doubles then two (2F+1) float2 spectra
    Workspace ws;
    memset(&ws, 0, sizeof(ws));
    ws.design_stride = (design_doubles_per_channel(*plan) + 31) / 32 * 32;
    ws.design = (double*)d_workspace;
    ws.h_mid = (float2*)((unsigned char*)d_workspace + align256(8 * ws.design_stride * 8));
    ws.h_side = ws.h_mid + (2 * plan->fft_size + 1 + 31) / 32 * 32;
    mgb_track_layout L;
    memset(&L, 0, sizeof(L));
    L.target_piece = L.reference_piece = plan->fft_size;
    return launch_design(*plan, L, ws, d_avg, d_fir_out, nullptr, (cudaStream_t)stream);
}

}  // extern "C"
