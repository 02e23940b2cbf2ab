// Host transport at the reference's real seam: stages.main / limiter.limit take PAGEABLE float64 numpy
// arrays (what soundfile hands matchering/core.py:53-62) and return float64 arrays.
//
// Pageable memory cannot be DMA'd at link speed (the driver stages it through one internal bounce
// buffer, ~10 GB/s), float64 doubles the bytes, and cudaHostRegister of a 127 MB array costs more than
// the whole job.  So the library moves the data itself:
//
//   upload    P worker threads narrow (float64 -> float32) or copy the caller's array, slice by slice,
//             into a ring of pinned chunks; the calling thread issues one cudaMemcpyAsync per finished
//             chunk and recycles a chunk when its copy event has fired.  Conversion of chunk k+1 overlaps
//             the DMA of chunk k; half the bytes cross the link.
//   download  into pinned float64 memory (mgb_host_alloc): the device widens, ONE DMA, no host pass.
//             into anything else: float32 chunks through the ring, widened / copied by the workers.
//
// The worker pool is persistent (threads sleep on a condition variable between transfers and spin on
// atomics inside one).  Nothing here touches sample VALUES except the float64 <-> float32 conversion
// the reference's caller would otherwise pay for on the device.
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#include "kernels.cuh"

#if defined(__x86_64__) || defined(__i386__)
#include <immintrin.h>
#define MGB_CPU_RELAX() _mm_pause()
#else
#define MGB_CPU_RELAX() std::this_thread::yield()
#endif

#ifdef MGB_EMULATE
// The test emulator has no DMA engine: a copy is a memcpy at issue time and every event has fired.
// The ring, the worker threads and their hand-shakes below run exactly as on the device build.
#include <map>
typedef int cudaEvent_t;
enum { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaEventDisableTiming = 2, cudaHostAllocPortable = 1 };
// (MGB_EMUL_NO_COPY=1 drops the copy itself: host-side throughput measurements of the workers and the hand-shakes)
static const bool g_emul_no_copy = getenv("MGB_EMUL_NO_COPY") != nullptr;
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, int, cudaStream_t) {
    if (!g_emul_no_copy) memcpy(d, s, n);
    return cudaSuccess;
}
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, int) { *e = 1; return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaEventQuery(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static std::mutex g_pinned_mutex;
static std::map<const unsigned char*, size_t> g_pinned_blocks;  // what mgb_host_alloc / the ring handed out
static inline cudaError_t cudaHostAlloc(void** p, size_t n, int) {
    *p = aligned_alloc(256, (n + 255) / 256 * 256);
    std::lock_guard<std::mutex> lk(g_pinned_mutex);
    g_pinned_blocks[(const unsigned char*)*p] = n;
    return *p ? cudaSuccess : 1;
}
static inline cudaError_t cudaFreeHost(void* p) {
    {
        std::lock_guard<std::mutex> lk(g_pinned_mutex);
        g_pinned_blocks.erase((const unsigned char*)p);
    }
    free(p);
    return cudaSuccess;
}
#endif

namespace mgb {
namespace {

// tuning switches (mgb_set_option "host_download_ring" / "host_split_chunks" / "host_streaming_stores"; the
// environment gives their initial values)
// host_download_ring: 0 = pinned float64 results always by one DMA of device-widened data, 1 = through the ring up to
// kRingDownloadMaxSamples (default), 2 = always through the ring
int g_host_download_ring = getenv("MGB_DOWNLOAD_RING") ? atoi(getenv("MGB_DOWNLOAD_RING")) : 1;
constexpr int64_t kRingDownloadMaxSamples = 64LL << 20;  // 256 MB of float32: what has been measured to win
int g_host_split_chunks = getenv("MGB_HOST_SPLIT") && !strcmp(getenv("MGB_HOST_SPLIT"), "chunk");

class WorkerPool {
public:
    explicit WorkerPool(int n) : n_(n) {
        for (int i = 0; i < n; ++i) threads_.emplace_back([this, i] { loop(i); });
    }
    ~WorkerPool() {
        {
            std::lock_guard<std::mutex> lk(m_);
            stop_ = true;
        }
        cv_.notify_all();
        for (auto& t : threads_) t.join();
    }
    int size() const { return n_; }
    // every worker runs fn(worker_index) once; `lead` runs on the calling thread meanwhile
    void run(const std::function<void(int)>& fn, const std::function<void()>& lead) {
        {
            std::lock_guard<std::mutex> lk(m_);
            job_ = &fn;
            pending_ = n_;
            ++generation_;
        }
        cv_.notify_all();
        lead();
        std::unique_lock<std::mutex> lk(m_);
        done_cv_.wait(lk, [this] { return pending_ == 0; });
        job_ = nullptr;
    }

private:
    void loop(int index) {
        unsigned long long seen = 0;
        for (;;) {
            const std::function<void(int)>* job;
            {
                std::unique_lock<std::mutex> lk(m_);
                cv_.wait(lk, [&] { return stop_ || generation_ != seen; });
                if (stop_) return;
                seen = generation_;
                job = job_;
            }
            (*job)(index);
            {
                std::lock_guard<std::mutex> lk(m_);
                if (--pending_ == 0) done_cv_.notify_one();
            }
        }
    }
    int n_;
    std::vector<std::thread> threads_;
    std::mutex m_;
    std::condition_variable cv_, done_cv_;
    const std::function<void(int)>* job_ = nullptr;
    unsigned long long generation_ = 0;
    int pending_ = 0;
    bool stop_ = false;
};

inline void spin_until(const std::function<bool()>& ready) {
    int spins = 0;
    while (!ready()) {
        if (++spins < 4096)
            MGB_CPU_RELAX();
        else
            std::this_thread::yield();  // an oversubscribed host must not burn its time slices here
    }
}

// the two conversions (auto-vectorised: cvtpd2ps / cvtps2pd)
inline void narrow_plain(const double* __restrict__ src, float* __restrict__ dst, int64_t n) {
    for (int64_t i = 0; i < n; ++i) dst[i] = (float)src[i];
}
inline void widen_plain(const float* __restrict__ src, double* __restrict__ dst, int64_t n) {
    for (int64_t i = 0; i < n; ++i) dst[i] = (double)src[i];
}
#if defined(__x86_64__)
// Streaming variants.  The staging chunk is written once by a worker and read once by the DMA engine, the result
// array is written once and read by nobody here: a non-temporal store skips the read-for-ownership of every
// destination line and -- what matters more for the ring -- leaves the line in memory instead of dirty in the
// writing core's cache, where the DMA engine's reads would have to fetch it from (a ring drained from the
// cores' caches runs well below link speed; from memory it runs at link speed).  dst is 64-byte aligned by
// construction for the ring (slices start on 16-sample boundaries of a pinned allocation).
// MGB_HOST_NT: 0 = plain stores, 1 = 256-bit streaming stores, 2 = 512-bit where the CPU has them (default).
// MGB_HOST_PREFETCH: software prefetch distance in bytes (0 = none).
static int g_prefetch = getenv("MGB_HOST_PREFETCH") ? atoi(getenv("MGB_HOST_PREFETCH")) : 8192;
__attribute__((target("avx2"))) inline void narrow_stream(const double* __restrict__ src, float* __restrict__ dst, int64_t n) {
    int64_t i = 0;
    if ((reinterpret_cast<uintptr_t>(dst) & 31) == 0) {
        const int pf = g_prefetch;
        for (; i + 8 <= n; i += 8) {
            if (pf) _mm_prefetch((const char*)(src + i) + pf, _MM_HINT_NTA);
            const __m128 lo = _mm256_cvtpd_ps(_mm256_loadu_pd(src + i));
            const __m128 hi = _mm256_cvtpd_ps(_mm256_loadu_pd(src + i + 4));
            _mm256_stream_ps(dst + i, _mm256_set_m128(hi, lo));
        }
        _mm_sfence();
    }
    for (; i < n; ++i) dst[i] = (float)src[i];
}
__attribute__((target("avx512f"))) inline void narrow_stream512(const double* __restrict__ src, float* __restrict__ dst, int64_t n) {
    int64_t i = 0;
    if ((reinterpret_cast<uintptr_t>(dst) & 63) == 0) {
        const int pf = g_prefetch;
        for (; i + 16 <= n; i += 16) {  // one destination line per iteration, two source lines
            // the hardware's stream prefetcher stops at every 4 KB page of the source: touch the head of a page
            // further on once per page, so that its translation and first lines are there when the stream arrives
            if (pf && (i & 511) == 0) {
                const char* ahead = (const char*)(src + i) + pf;
                _mm_prefetch(ahead, _MM_HINT_T0);
                _mm_prefetch(ahead + 64, _MM_HINT_T0);
                _mm_prefetch(ahead + 128, _MM_HINT_T0);
                _mm_prefetch(ahead + 192, _MM_HINT_T0);
            }
            const __m256 lo = _mm512_cvtpd_ps(_mm512_loadu_pd(src + i));
            const __m256 hi = _mm512_cvtpd_ps(_mm512_loadu_pd(src + i + 8));
            _mm512_stream_ps(dst + i, _mm512_castpd_ps(_mm512_insertf64x4(_mm512_castpd256_pd512(_mm256_castps_pd(lo)), _mm256_castps_pd(hi), 1)));
        }
        _mm_sfence();
    }
    for (; i < n; ++i) dst[i] = (float)src[i];
}
__attribute__((target("avx2"))) inline void widen_stream(const float* __restrict__ src, double* __restrict__ dst, int64_t n) {
    int64_t i = 0;
    for (; i < n && (reinterpret_cast<uintptr_t>(dst + i) & 31) != 0; ++i) dst[i] = (double)src[i];
    for (; i + 8 <= n; i += 8) {
        const __m256 v = _mm256_loadu_ps(src + i);
        _mm256_stream_pd(dst + i, _mm256_cvtps_pd(_mm256_castps256_ps128(v)));
        _mm256_stream_pd(dst + i + 4, _mm256_cvtps_pd(_mm256_extractf128_ps(v, 1)));
    }
    _mm_sfence();
    for (; i < n; ++i) dst[i] = (double)src[i];
}
__attribute__((target("avx512f"))) inline void widen_stream512(const float* __restrict__ src, double* __restrict__ dst, int64_t n) {
    int64_t i = 0;
    for (; i < n && (reinterpret_cast<uintptr_t>(dst + i) & 63) != 0; ++i) dst[i] = (double)src[i];
    for (; i + 16 <= n; i += 16) {  // one source line, two destination lines
        const __m512 v = _mm512_loadu_ps(src + i);
        _mm512_stream_pd(dst + i, _mm512_cvtps_pd(_mm512_castps512_ps256(v)));
        _mm512_stream_pd(dst + i + 8, _mm512_cvtps_pd(_mm256_castpd_ps(_mm512_extractf64x4_pd(_mm512_castps_pd(v), 1))));
    }
    _mm_sfence();
    for (; i < n; ++i) dst[i] = (double)src[i];
}
inline int clamp_stream_stores(int want) {
    if (want >= 2 && !__builtin_cpu_supports("avx512f")) want = 1;
    if (want >= 1 && !__builtin_cpu_supports("avx2")) want = 0;
    return want < 0 ? 0 : want;
}
static int g_stream_stores = clamp_stream_stores(getenv("MGB_HOST_NT") ? atoi(getenv("MGB_HOST_NT")) : 2);
inline void narrow(const double* __restrict__ src, float* __restrict__ dst, int64_t n) {
    if (g_stream_stores == 2) narrow_stream512(src, dst, n);
    else if (g_stream_stores == 1) narrow_stream(src, dst, n);
    else narrow_plain(src, dst, n);
}
inline void widen(const float* __restrict__ src, double* __restrict__ dst, int64_t n) {
    if (g_stream_stores == 2) widen_stream512(src, dst, n);
    else if (g_stream_stores == 1) widen_stream(src, dst, n);
    else widen_plain(src, dst, n);
}
#else
static int g_stream_stores = 0;
inline void narrow(const double* __restrict__ src, float* __restrict__ dst, int64_t n) { narrow_plain(src, dst, n); }
inline void widen(const float* __restrict__ src, double* __restrict__ dst, int64_t n) { widen_plain(src, dst, n); }
#endif

}  // namespace
}  // namespace mgb

struct mgb_host_io {
    mgb::WorkerPool* pool = nullptr;
    int64_t chunk = 0;  // samples per ring chunk
    int ring = 0;
    float* staging = nullptr;  // pinned, ring * chunk floats
    std::vector<cudaEvent_t> events;
};

using namespace mgb;

namespace {

#ifdef MGB_EMULATE
bool is_pinned(const void* p) {
    std::lock_guard<std::mutex> lk(g_pinned_mutex);
    auto it = g_pinned_blocks.upper_bound((const unsigned char*)p);
    if (it == g_pinned_blocks.begin()) return false;
    --it;
    return (const unsigned char*)p < it->first + it->second;
}
#else
bool is_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeHost;
}
#endif

// One piece of an upload: a host array (float32 or float64, any memory) and the device float32 array it goes to.
struct UploadPiece {
    const void* h_src;
    float* d_dst;
    int64_t samples;
};

// host -> device float32, any number of arrays in ONE pass of the workers over one sequence of chunks: the ring
// never drains between the arrays (a drain is ~0.3 ms of link time with nobody converting) and the workers
// are woken once.
int upload(mgb_host_io* io, const UploadPiece* pieces, int npieces, int src_width, cudaStream_t st) {
    MGB_REQUIRE(src_width == 4 || src_width == 8, MGB_ERR_INVALID, "host array must be float32 or float64");
    const int64_t chunk = io->chunk;
    struct Chunk {
        const void* h_src;  // this chunk's first source sample
        float* d_dst;
        int64_t len;
    };
    std::vector<Chunk> chunks;
    for (int s = 0; s < npieces; ++s) {
        const UploadPiece& pc = pieces[s];
        if (pc.samples == 0) continue;
        if (src_width == 4 && is_pinned(pc.h_src)) {  // nothing to convert, DMA-able as it is
            if (cudaMemcpyAsync(pc.d_dst, pc.h_src, (size_t)pc.samples * 4, cudaMemcpyHostToDevice, st) != cudaSuccess) return cuda_status("H2D");
            continue;
        }
        for (int64_t base = 0; base < pc.samples; base += chunk)
            chunks.push_back(Chunk{(const unsigned char*)pc.h_src + base * src_width, pc.d_dst + base,
                                   pc.samples - base < chunk ? pc.samples - base : chunk});
    }
    const int64_t nchunks = (int64_t)chunks.size();
    if (nchunks == 0) return MGB_OK;
    const int P = io->pool->size();
    const int ring = io->ring;
    std::vector<std::atomic<int>> ready(nchunks);
    for (auto& r : ready) r.store(0, std::memory_order_relaxed);
    std::atomic<int64_t> released{0};  // chunks whose DMA has finished (their ring slot is free again)
    std::atomic<int> failed{0};
    // MGB_HOST_STATS=1: where an upload's time goes (per-worker conversion and waiting, the issuing thread's calls)
    static const bool stats = getenv("MGB_HOST_STATS") != nullptr;
    // MGB_HOST_SPLIT=chunk: a worker converts whole chunks (p, p+P, ...) instead of its slice of every chunk
    const bool whole_chunks = g_host_split_chunks != 0;
    std::vector<double> busy_us(P, 0.0), wait_us(P, 0.0);
    auto now_us = [] { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    auto work = [&](int p) {
        for (int64_t k = whole_chunks ? p : 0; k < nchunks; k += whole_chunks ? P : 1) {
            const double t0 = stats ? now_us() : 0.0;
            if (k >= ring) spin_until([&] { return released.load(std::memory_order_acquire) > k - ring || failed.load(); });
            if (failed.load()) return;
            const double t1 = stats ? now_us() : 0.0;
            const Chunk& c = chunks[k];
            // slices on 64-byte boundaries of the destination
            const int64_t per = whole_chunks ? c.len : ((c.len + P - 1) / P + 15) / 16 * 16;
            const int64_t lo = whole_chunks ? 0 : (int64_t)p * per, hi = lo + per < c.len ? lo + per : c.len;
            float* dst = io->staging + (k % ring) * chunk;
            if (lo < hi) {
                if (src_width == 8) narrow((const double*)c.h_src + lo, dst + lo, hi - lo);
                else memcpy(dst + lo, (const float*)c.h_src + lo, (size_t)(hi - lo) * 4);
            }
            ready[k].fetch_add(whole_chunks ? P : 1, std::memory_order_release);
            if (stats) {
                const double t2 = now_us();
                wait_us[p] += t1 - t0;
                busy_us[p] += t2 - t1;
            }
        }
    };
    int rc = MGB_OK;
    double issue_us = 0.0, total_us = 0.0;
    int64_t copies = 0, polls = 0;
    auto lead = [&]() {
        const double lead_t0 = stats ? now_us() : 0.0;
        int64_t issued = 0, freed = 0;
        std::vector<int64_t> group_end(nchunks);  // chunk k left the ring when the copy that ends with chunk group_end[k] has
        while (issued < nchunks) {
            if (ready[issued].load(std::memory_order_acquire) == P) {
                // every finished chunk that follows in the ring (without wrapping) and in the same device array goes
                // into the same copy: when the workers are ahead of this thread one launch moves several chunks
                int64_t last = issued;
                while (last + 1 < nchunks && (last + 1) % ring != 0 && chunks[last].len == chunk &&
                       chunks[last + 1].d_dst == chunks[last].d_dst + chunk && ready[last + 1].load(std::memory_order_acquire) == P)
                    ++last;
                const int64_t count = (last - issued) * chunk + chunks[last].len;
                const int slot = (int)(issued % ring);
                const double c0 = stats ? now_us() : 0.0;
                if (cudaMemcpyAsync(chunks[issued].d_dst, io->staging + slot * chunk, (size_t)count * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
                    cudaEventRecord(io->events[last % ring], st) != cudaSuccess) {
                    rc = cuda_status("H2D chunk");
                    failed.store(1);
                    return;
                }
                if (stats) issue_us += now_us() - c0, ++copies;
                for (int64_t k = issued; k <= last; ++k) group_end[k] = last;
                issued = last + 1;
            } else if (freed < issued && cudaEventQuery(io->events[group_end[freed] % ring]) == cudaSuccess) {
                freed = group_end[freed] + 1;
                released.store(freed, std::memory_order_release);
            } else {
                MGB_CPU_RELAX();
                ++polls;
            }
        }
        const double drain_t0 = stats ? now_us() : 0.0;
        // the ring is reused by the next transfer: its last copies must have left it
        if (cudaEventSynchronize(io->events[(nchunks - 1) % ring]) != cudaSuccess) rc = cuda_status("H2D drain");
        if (stats) {
            total_us = now_us() - lead_t0;
            fprintf(stderr, "[mgb upload] %lld chunks of %lld samples: %.0f us (drain %.0f), %lld copies issued in %.0f us, %lld idle polls\n",
                    (long long)nchunks, (long long)chunk, total_us, now_us() - drain_t0, (long long)copies, issue_us, (long long)polls);
        }
    };
    const double run_t0 = stats ? now_us() : 0.0;
    io->pool->run(work, lead);
    if (stats) {
        double b = 0.0, w = 0.0, bmax = 0.0;
        for (int p = 0; p < P; ++p) b += busy_us[p], w += wait_us[p], bmax = bmax > busy_us[p] ? bmax : busy_us[p];
        fprintf(stderr, "[mgb upload] %d workers: converting %.0f us each on average (max %.0f), waiting for a ring slot %.0f us; call %.0f us\n",
                P, b / P, bmax, w / P, now_us() - run_t0);
    }
    return rc;
}

int upload(mgb_host_io* io, const void* h_src, int src_width, float* d_dst, int64_t samples, cudaStream_t st) {
    const UploadPiece one{h_src, d_dst, samples};
    return upload(io, &one, 1, src_width, st);
}

// device float32 -> host (float32 or float64)
int download(mgb_host_io* io, const float* d_src, void* h_dst, int dst_width, int64_t samples, double* d_wide,
             cudaStream_t st) {
    MGB_REQUIRE(dst_width == 4 || dst_width == 8, MGB_ERR_INVALID, "host array must be float32 or float64");
    if (samples == 0) return MGB_OK;
    // float64 results into pinned memory, two routes.  (a) Widened on the device and copied by ONE DMA: twice the
    // bytes over the link, no host thread involved.  (b) Float32 chunks through the ring, widened by the workers
    // with streaming stores: faster for a 3-minute track (tools/seam_ab.py compares the two), slower than (a) on the
    // one-hour limiter buffer (2.5 GB: the widening competes with itself for the socket's memory bandwidth).
    // So (b) up to 256 MB of float32 and (a) beyond; option host_download_ring = 0 / 2 forces (a) / (b).
    const bool prefer_ring = mgb_host_download_through_ring(samples) != 0;
    const bool direct = is_pinned(h_dst) && (dst_width == 4 || (d_wide && !prefer_ring));
    if (direct) {
        const void* src = d_src;
        if (dst_width == 8) {
            MGB_TRY(launch_convert_f32_f64(d_src, d_wide, samples, st));
            src = d_wide;
        }
        if (cudaMemcpyAsync(h_dst, src, (size_t)samples * dst_width, cudaMemcpyDeviceToHost, st) != cudaSuccess) return cuda_status("D2H");
        if (cudaStreamSynchronize(st) != cudaSuccess) return cuda_status("D2H sync");
        return MGB_OK;
    }
    const int64_t chunk = io->chunk;
    const int64_t nchunks = (samples + chunk - 1) / chunk;
    const int P = io->pool->size();
    const int ring = io->ring;
    std::vector<std::atomic<int>> consumed(nchunks);
    for (auto& c : consumed) c.store(0, std::memory_order_relaxed);
    std::atomic<int64_t> arrived{0};
    std::atomic<int> failed{0};
    static const bool stats = getenv("MGB_HOST_STATS") != nullptr;
    std::vector<double> busy_us(P, 0.0), wait_us(P, 0.0);
    auto now_us = [] { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    auto work = [&](int p) {
        for (int64_t k = 0; k < nchunks; ++k) {
            const double t0 = stats ? now_us() : 0.0;
            spin_until([&] { return arrived.load(std::memory_order_acquire) > k || failed.load(); });
            if (failed.load()) return;
            const double t1 = stats ? now_us() : 0.0;
            const int64_t base = k * chunk;
            const int64_t len = (samples - base < chunk) ? samples - base : chunk;
            const int64_t per = ((len + P - 1) / P + 15) / 16 * 16;
            const int64_t lo = (int64_t)p * per, hi = lo + per < len ? lo + per : len;
            const float* src = io->staging + (k % ring) * chunk;
            if (lo < hi) {
                if (dst_width == 8) widen(src + lo, (double*)h_dst + base + lo, hi - lo);
                else memcpy((float*)h_dst + base + lo, src + lo, (size_t)(hi - lo) * 4);
            }
            consumed[k].fetch_add(1, std::memory_order_release);
            if (stats) {
                const double t2 = now_us();
                wait_us[p] += t1 - t0;
                busy_us[p] += t2 - t1;
            }
        }
    };
    int rc = MGB_OK;
    auto lead = [&]() {
        int64_t issued = 0, landed = 0;
        const double lead_t0 = stats ? now_us() : 0.0;
        double first_us = 0.0, issue_us = 0.0, gated_us = 0.0, gate_t0 = 0.0;
        while (landed < nchunks) {
            const bool slot_free = issued < ring || consumed[issued - ring].load(std::memory_order_acquire) == P;
            if (stats && issued < nchunks) {  // time spent with a copy to issue but no free slot
                if (!slot_free && gate_t0 == 0.0) gate_t0 = now_us();
                if (slot_free && gate_t0 != 0.0) gated_us += now_us() - gate_t0, gate_t0 = 0.0;
            }
            if (issued < nchunks && slot_free) {
                const int64_t base = issued * chunk;
                const int64_t len = (samples - base < chunk) ? samples - base : chunk;
                const int slot = (int)(issued % ring);
                const double c0 = stats ? now_us() : 0.0;
                if (cudaMemcpyAsync(io->staging + slot * chunk, d_src + base, (size_t)len * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                    cudaEventRecord(io->events[slot], st) != cudaSuccess) {
                    rc = cuda_status("D2H chunk");
                    failed.store(1);
                    return;
                }
                if (stats) issue_us += now_us() - c0;
                ++issued;
            } else if (landed < issued && cudaEventQuery(io->events[landed % ring]) == cudaSuccess) {
                if (stats && landed == 0) first_us = now_us() - lead_t0;
                arrived.store(++landed, std::memory_order_release);
            } else {
                MGB_CPU_RELAX();
            }
        }
        if (stats)
            fprintf(stderr, "[mgb download] first chunk landed after %.0f us (the kernels before it included), all after %.0f us; "
                            "copies issued in %.0f us; %.0f us with a copy held back for a free ring slot\n",
                    first_us, now_us() - lead_t0, issue_us, gated_us);
    };
    const double run_t0 = stats ? now_us() : 0.0;
    io->pool->run(work, lead);  // returns when every worker has consumed every chunk
    if (stats) {
        double b = 0.0, w = 0.0;
        for (int p = 0; p < P; ++p) b += busy_us[p], w += wait_us[p];
        fprintf(stderr, "[mgb download] %lld chunks of %lld samples, %d workers: converting %.0f us each on average, waiting for a chunk %.0f us; call %.0f us\n",
                (long long)nchunks, (long long)chunk, P, b / P, w / P, now_us() - run_t0);
    }
    return rc;
}

}  // namespace

// (called by mgb_set_option, api.cu)
bool mgb::host_set_option(const char* name, int value) {
    if (!strcmp(name, "host_download_ring")) g_host_download_ring = value;
    else if (!strcmp(name, "host_split_chunks")) g_host_split_chunks = value;
#if defined(__x86_64__)
    else if (!strcmp(name, "host_streaming_stores")) g_stream_stores = clamp_stream_stores(value);
    else if (!strcmp(name, "host_prefetch")) g_prefetch = value;
#endif
    else return false;
    return true;
}

extern "C" {

int mgb_host_io_create(int32_t threads, int64_t chunk_samples, int32_t ring, mgb_host_io** out) {
    MGB_REQUIRE(out != nullptr, MGB_ERR_INVALID, "host_io: NULL argument");
    if (threads <= 0) {
        // The conversion is what bounds a transfer (one worker narrows float64 source far slower than the link
        // takes it), so every core helps -- up to what the process may use: the affinity mask, and the cgroup's
        // CPU quota (workers that spin past the quota get the whole process throttled).  Three cores stay free for the issuing thread, the
        // driver's threads and the caller's own.
        int usable = (int)std::thread::hardware_concurrency();
#if defined(__linux__)
        cpu_set_t set;
        if (sched_getaffinity(0, sizeof(set), &set) == 0) usable = CPU_COUNT(&set);
        long long quota = 0, period = 0;
        if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {  // cgroup v2: "<quota|max> <period>"
            if (fscanf(f, "%lld %lld", &quota, &period) != 2) quota = period = 0;
            fclose(f);
        } else if (FILE* q = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) {  // cgroup v1
            FILE* p = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r");
            if (fscanf(q, "%lld", &quota) != 1) quota = 0;
            if (!p || fscanf(p, "%lld", &period) != 1) period = 0;
            fclose(q);
            if (p) fclose(p);
        }
        if (quota > 0 && period > 0) {
            const int cores = (int)(quota / period);
            if (cores >= 1 && cores < usable) usable = cores;
        }
#endif
        threads = usable >= 19 ? 16 : (usable > 4 ? usable - 3 : (usable > 1 ? usable - 1 : 1));
    }
    // A ring of six 4 MB chunks, written with streaming stores (tools/seam_ab.py and tools/seam_sweep.py compare
    // geometries): with ordinary stores the DMA engine has to pull every line out of the writing core's cache and
    // the ring drains well below link speed, whatever its size; with streaming stores the chunks sit in memory and
    // the ring drains at link speed.  Larger chunks mean fewer copies, and a download pays a fixed cost per copy.
    // With ordinary stores (MGB_HOST_NT=0) the best geometry is sixteen 256 KB chunks, which stay in the
    // cores' caches: that is what several processes sharing one socket's memory bandwidth should use
    // (tools/gpu_n4_sweep.sh compares the two with four processes on one socket).
    if (chunk_samples <= 0) chunk_samples = g_stream_stores ? 1 << 20 : 1 << 16;
    if (ring <= 0) ring = g_stream_stores ? 6 : 16;
    MGB_REQUIRE(threads <= 256 && ring <= 64 && chunk_samples % 16 == 0, MGB_ERR_INVALID, "host_io: bad geometry");
    mgb_host_io* io = new mgb_host_io();
    io->chunk = chunk_samples;
    io->ring = ring;
    if (cudaHostAlloc((void**)&io->staging, (size_t)ring * chunk_samples * 4, cudaHostAllocPortable) != cudaSuccess) {
        delete io;
        return cuda_status("host_io: pinned staging ring");
    }
    io->events.resize(ring);
    for (auto& e : io->events)
        if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) {
            mgb_host_io_destroy(io);
            return cuda_status("host_io: events");
        }
    io->pool = new WorkerPool(threads);
    *out = io;
    return MGB_OK;
}

int mgb_host_io_destroy(mgb_host_io* io) {
    if (!io) return MGB_OK;
    delete io->pool;
    for (auto e : io->events)
        if (e) cudaEventDestroy(e);
    if (io->staging) cudaFreeHost(io->staging);
    delete io;
    return MGB_OK;
}

int mgb_host_io_threads(const mgb_host_io* io) { return io && io->pool ? io->pool->size() : 0; }

int mgb_host_download_through_ring(int64_t samples) {
    return g_host_download_ring >= 2 || (g_host_download_ring == 1 && samples <= kRingDownloadMaxSamples);
}

void* mgb_host_alloc(int64_t bytes) {
    if (bytes <= 0) return nullptr;
    void* p = nullptr;
    if (cudaHostAlloc(&p, (size_t)bytes, cudaHostAllocPortable) != cudaSuccess) {
        cuda_status("host_alloc");
        return nullptr;
    }
    return p;
}

void mgb_host_free(void* p) {
    if (p) cudaFreeHost(p);
}

int mgb_host_upload(mgb_host_io* io, const void* h_src, int32_t src_width, float* d_dst, int64_t samples, void* stream) {
    MGB_REQUIRE(io && h_src && d_dst && samples >= 0, MGB_ERR_INVALID, "host_upload: bad arguments");
    return upload(io, h_src, src_width, d_dst, samples, (cudaStream_t)stream);
}

int mgb_host_download(mgb_host_io* io, const float* d_src, void* h_dst, int32_t dst_width, int64_t samples, double* d_wide,
                      void* stream) {
    MGB_REQUIRE(io && h_dst && d_src && samples >= 0, MGB_ERR_INVALID, "host_download: bad arguments");
    return download(io, d_src, h_dst, dst_width, samples, d_wide, (cudaStream_t)stream);
}

static int stages_after_levels(mgb_host_io* io, const mgb_plan* plan, const mgb_track_layout* L, void* h_out_limited,
                               void* h_out_no_limiter, void* h_out_normalized, int32_t out_width, const mgb_host_buffers* dev,
                               mgb_track_state* h_state_out, cudaStream_t st);

int mgb_stages_main_host(mgb_host_io* io, const mgb_plan* plan, const mgb_track_layout* L, const void* h_target,
                         const void* h_reference, int32_t in_width, void* h_out_limited, void* h_out_no_limiter,
                         void* h_out_normalized, int32_t out_width, const mgb_host_buffers* dev,
                         mgb_track_state* h_state_out, void* stream) {
    MGB_REQUIRE(io && plan && L && h_target && h_reference && dev, MGB_ERR_INVALID, "stages_main_host: NULL argument");
    MGB_REQUIRE(h_out_limited || h_out_no_limiter || h_out_normalized, MGB_ERR_INVALID, "no output requested");
    MGB_REQUIRE(dev->d_target_lr && dev->d_reference_lr && dev->d_result_lr && dev->d_out_lr && dev->d_workspace && dev->d_state,
                MGB_ERR_INVALID, "stages_main_host: device staging buffer missing");
    cudaStream_t st = (cudaStream_t)stream;
    const UploadPiece both[2] = {{h_target, dev->d_target_lr, L->target_frames * 2}, {h_reference, dev->d_reference_lr, L->reference_frames * 2}};
    MGB_TRY(upload(io, both, 2, in_width, st));
    MGB_TRY(mgb_match_levels(plan, L, dev->d_target_lr, dev->d_reference_lr, dev->d_workspace, dev->d_state, stream));
    return stages_after_levels(io, plan, L, h_out_limited, h_out_no_limiter, h_out_normalized, out_width, dev, h_state_out, st);
}

int mgb_stages_main_host_profiled(mgb_host_io* io, const mgb_plan* plan, const mgb_track_layout* L, const void* h_target,
                                  int32_t in_width, const void* d_profile, void* h_out_limited, void* h_out_no_limiter,
                                  void* h_out_normalized, int32_t out_width, const mgb_host_buffers* dev,
                                  mgb_track_state* h_state_out, void* stream) {
    MGB_REQUIRE(io && plan && L && h_target && d_profile && dev, MGB_ERR_INVALID, "stages_main_host_profiled: NULL argument");
    MGB_REQUIRE(h_out_limited || h_out_no_limiter || h_out_normalized, MGB_ERR_INVALID, "no output requested");
    MGB_REQUIRE(dev->d_target_lr && dev->d_result_lr && dev->d_out_lr && dev->d_workspace && dev->d_state, MGB_ERR_INVALID,
                "stages_main_host_profiled: device staging buffer missing");
    cudaStream_t st = (cudaStream_t)stream;
    const UploadPiece target{h_target, dev->d_target_lr, L->target_frames * 2};
    MGB_TRY(upload(io, &target, 1, in_width, st));
    MGB_TRY(mgb_match_levels_profiled(plan, L, dev->d_target_lr, d_profile, dev->d_workspace, dev->d_state, stream));
    return stages_after_levels(io, plan, L, h_out_limited, h_out_no_limiter, h_out_normalized, out_width, dev, h_state_out, st);
}

// stages 2-4 and the downloads of mgb_stages_main_host(_profiled), once stage 1 is on the stream
static int stages_after_levels(mgb_host_io* io, const mgb_plan* plan, const mgb_track_layout* L, void* h_out_limited,
                               void* h_out_no_limiter, void* h_out_normalized, int32_t out_width, const mgb_host_buffers* dev,
                               mgb_track_state* h_state_out, cudaStream_t st) {
    void* stream = (void*)st;
    MGB_TRY(mgb_match_frequencies(plan, L, dev->d_target_lr, dev->d_result_lr, nullptr, dev->d_workspace, dev->d_state, stream));
    MGB_TRY(mgb_correct_levels(plan, L, dev->d_workspace, dev->d_state, stream));
    void* outs[3] = {h_out_limited, h_out_no_limiter, h_out_normalized};
    for (int k = 0; k < 3; ++k) {
        if (!outs[k]) continue;
        MGB_TRY(mgb_finalize(plan, L, dev->d_result_lr, k == 0 ? dev->d_out_lr : nullptr, k == 1 ? dev->d_out_lr : nullptr,
                             k == 2 ? dev->d_out_lr : nullptr, dev->d_workspace, dev->d_state, stream));
        MGB_TRY(download(io, dev->d_out_lr, outs[k], out_width, L->target_frames * 2, dev->d_wide, st));
    }
    if (h_state_out && cudaMemcpyAsync(h_state_out, dev->d_state, sizeof(mgb_track_state), cudaMemcpyDeviceToHost, st) != cudaSuccess)
        return cuda_status("D2H state");
    if (cudaStreamSynchronize(st) != cudaSuccess) return cuda_status("stream sync");
    return MGB_OK;
}

int mgb_limit_host(mgb_host_io* io, const mgb_limiter_params* params, const void* h_in, int32_t in_width, void* h_out,
                   int32_t out_width, int64_t frames, float* d_in_lr, float* d_out_lr, double* d_wide, void* d_workspace,
                   int64_t workspace_bytes, int32_t* d_engaged, int32_t* h_engaged_out, void* stream) {
    MGB_REQUIRE(io && params && h_in && h_out && d_in_lr && d_out_lr && d_engaged && h_engaged_out, MGB_ERR_INVALID,
                "limit_host: NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    MGB_TRY(upload(io, h_in, in_width, d_in_lr, frames * 2, st));
    MGB_TRY(mgb_limit(params, d_in_lr, d_out_lr, frames, d_workspace, workspace_bytes, d_engaged, stream));
    if (cudaMemcpyAsync(h_engaged_out, d_engaged, 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) return cuda_status("D2H flag");
    if (cudaStreamSynchronize(st) != cudaSuccess) return cuda_status("stream sync");
    if (*h_engaged_out == 0) return MGB_OK;  // hyrax.py:83-85: the caller hands its input back untouched
    return download(io, d_out_lr, h_out, out_width, frames * 2, d_wide, st);
}

}  // extern "C"
