// TEST INFRASTRUCTURE ONLY -- controls of the race-checking emulator build (tests/test_emul_racecheck.py).
// Built with the kernels' header and flags into its own executable, linked with the race-checking build's
// objects: `racecheck_controls <name> <threads>` runs one tiny kernel over two blocks of <threads> threads (two
// blocks, so that both of the checker's lane groupings for blocks above 224 threads are used; cuda_emul.cpp).
// The `race_*` controls must be reported by ThreadSanitizer, the `ok_*` controls must not: together they pin
// down where the emulator gives a happens-before edge and where it does not, at every block size.
#include "../../matchering_b200/csrc/design.cu"  // block_kth_smallest (the rest of design.cu is unused here)
#include "../../matchering_b200/csrc/limiter_scan.cuh"  // publish / poll

namespace {

constexpr int kMaxThreads = 1024;
__shared__ int g_word[kMaxThreads];
int g_sink;
int g_threads = 64;

void run(void (*kernel)(bool), bool barrier) {
    emul::launch(dim3(2), dim3(g_threads), 0, [&]() { kernel(barrier); });
}

// the writer (thread w) stores, the reader (thread r) loads, with or without a barrier between
template <int W, int R>
void read_after_write(bool barrier) {
    if (threadIdx.x == W) g_word[0] = 1;
    if (barrier) __syncthreads();
    if (threadIdx.x == R) g_sink = g_word[0];
}

// thread 40 reads a word that thread 3 wrote before a barrier, and thread 3 writes it again afterwards
void write_after_read(bool barrier) {
    if (threadIdx.x == 3) g_word[0] = 1;
    __syncthreads();
    if (threadIdx.x == 40) g_sink = g_word[0];
    if (barrier) __syncthreads();
    if (threadIdx.x == 3) g_word[0] = 2;
}

// lanes 0 and 1 of one warp write one word (the same value)
void two_writers(bool barrier) {
    if (threadIdx.x == 0) g_word[0] = 7;
    if (barrier) __syncwarp();
    if (threadIdx.x == 1) g_word[0] = 7;
}

// every lane writes its own word and reads its neighbour's across __syncwarp; values also travel by shuffles
void warp_exchange(bool) {
    const int lane = threadIdx.x & 31;
    g_word[threadIdx.x] = lane;
    __syncwarp();
    int v = g_word[(threadIdx.x & ~31) | ((lane + 1) & 31)];
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_down_sync(0xffffffffu, v, 2);
    v = __shfl_sync(0xffffffffu, v, 0);
    if (__all_sync(0xffffffffu, v >= 0) && lane == 0) g_word[threadIdx.x] = v;
}

// every thread bumps one counter; thread 0 reads the total after the barrier
void atomic_counter(bool) {
    if (threadIdx.x == 0) g_word[0] = 0;
    __syncthreads();
    atomicAdd(&g_word[0], 1);
    atomicMax(&g_word[0], 1);
    __syncthreads();
    if (threadIdx.x == 0) g_sink = g_word[0];
}

// thread 0 publishes a look-back word, thread 33 (another warp) polls it until it is there
mgb::LookbackWord g_lookback;
void publish_poll(bool) {
    if (threadIdx.x == 0) mgb::publish(&g_lookback, 0.5, 2);
    if (threadIdx.x == 33) {
        double v = 0.0;
        while (mgb::poll(&g_lookback, &v) == 0) __nanosleep(20);
        g_sink = (int)(v * 4.0);
    }
}

// 10 non-negative values; the radix select of design.cu runs twice back to back on them, as
// lowess_residual_weights does for an even count
const double g_values[10] = {0.5, 3.0, 0.25, 7.0, 1.5, 0.0, 2.0, 9.0, 0.75, 4.0};

void kth_twice(bool) {
    const double a = mgb::block_kth_smallest(g_values, 10, 5), b = mgb::block_kth_smallest(g_values, 10, 4);
    if (threadIdx.x == 0) g_sink = (int)(4.0 * (a + b));
}

// The same select with its state reset by thread 0 on entry, as block_kth_smallest once did: a second call
// overwrites sel_prefix while other threads may still read the first call's result from it.
double kth_reset_on_entry(const double* v, int n, int k) {
    __shared__ unsigned hist[256];
    __shared__ unsigned long long sel_prefix;
    __shared__ int sel_rank;
    const int tid = threadIdx.x, nthr = blockDim.x;
    if (tid == 0) {
        sel_prefix = 0ull;
        sel_rank = k;
    }
    unsigned long long mask = 0ull;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int b = tid; b < 256; b += nthr) hist[b] = 0u;
        __syncthreads();
        const unsigned long long prefix = sel_prefix;
        for (int j = tid; j < n; j += nthr) {
            const unsigned long long bits = (unsigned long long)__double_as_longlong(v[j]);
            if ((bits & mask) == prefix) atomicAdd(&hist[(unsigned)(bits >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            int rank = sel_rank, b = 0;
            while (b < 255 && rank >= (int)hist[b]) {
                rank -= (int)hist[b];
                ++b;
            }
            sel_rank = rank;
            sel_prefix = prefix | ((unsigned long long)b << shift);
        }
        mask |= 0xffull << shift;
        __syncthreads();
    }
    return __longlong_as_double((long long)sel_prefix);
}

void kth_reset_twice(bool) {
    const double a = kth_reset_on_entry(g_values, 10, 5), b = kth_reset_on_entry(g_values, 10, 4);
    if (threadIdx.x == 0) g_sink = (int)(4.0 * (a + b));
}

}  // namespace

int main(int argc, char** argv) {
    if (argc != 3) return 2;
    const char* arg = argv[1];
    g_threads = std::atoi(argv[2]);
    if (g_threads < 64 || g_threads > kMaxThreads) return 2;
    auto name_is = [arg](const char* n) { return std::strcmp(arg, n) == 0; };
    mgb::publish(&g_lookback, 0.0, 0);
    if (name_is("race_reader_above_writer")) run(read_after_write<3, 40>, false);
    else if (name_is("race_reader_below_writer")) run(read_after_write<40, 3>, false);
    else if (name_is("race_write_after_read")) run(write_after_read, false);
    else if (name_is("race_two_lanes_one_word")) run(two_writers, false);
    else if (name_is("ok_reader_above_writer")) run(read_after_write<3, 40>, true);
    else if (name_is("ok_reader_below_writer")) run(read_after_write<40, 3>, true);
    else if (name_is("ok_write_after_read")) run(write_after_read, true);
    else if (name_is("ok_two_lanes_one_word")) run(two_writers, true);
    else if (name_is("ok_shuffles")) run(warp_exchange, false);
    else if (name_is("ok_atomics")) run(atomic_counter, false);
    else if (name_is("ok_publish_poll")) run(publish_poll, false);
    else if (name_is("race_kth_reset_on_entry")) run(kth_reset_twice, false);
    else if (name_is("ok_kth_twice")) run(kth_twice, false);
    else return 2;
    std::printf("%s %d\n", arg, g_sink);
    return 0;
}
