// TEST INFRASTRUCTURE ONLY -- fiber scheduler behind tests/emul/cuda_emul.h.
// Never built with -fsanitize=thread: in the race-checking build (-DMGB_EMUL_RACECHECK) this file tells
// ThreadSanitizer about fibers and happens-before edges through its interface, and the scheduler's own
// bookkeeping stays invisible to it.
#include <random>  // (before cuda_emul.h, whose CUDA keyword macros the standard headers must not see)
#ifdef MGB_EMUL_RACECHECK
#include <sanitizer/tsan_interface.h>
#endif

#include "cuda_emul.h"

#ifdef MGB_EMUL_RACECHECK
#define RC(stmt) stmt
#else
#define RC(stmt) (void)0
#endif

thread_local uint3 threadIdx;
thread_local uint3 blockIdx;
thread_local dim3 blockDim;
thread_local dim3 gridDim;

namespace emul {

static thread_local BlockState* g_block = nullptr;
static const size_t kStackBytes = 256 * 1024;

BlockState& block() { return *g_block; }
unsigned char* dyn_smem() { return g_block->dyn_smem; }

#if defined(__x86_64__)
// Minimal cooperative context switch: callee-saved registers + stack pointer.
extern "C" void mgb_emul_switch(void** save_sp, void* load_sp);
asm(R"(
.text
.globl mgb_emul_switch
.type mgb_emul_switch,@function
mgb_emul_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
.size mgb_emul_switch,.-mgb_emul_switch
)");

static void fiber_main() {
    BlockState& b = *g_block;
    RC(__tsan_acquire(&b.start_sync));
    b.body();
    Fiber& f = b.fibers[b.current];
    f.done = true;
    b.alive--;
    RC(__tsan_release(&b.exit_sync));
    RC(__tsan_release(&b.end_sync));
    // an exited thread no longer takes part in barriers: release one that is now complete
    if (b.alive > 0 && b.arrived >= b.alive && b.arrived > 0) {
        RC(__tsan_acquire(&b.exit_sync));
        RC(__tsan_release(&b.sync[b.gen & 1]));
        b.arrived = 0;
        b.gen++;
    }
    RC(__tsan_switch_to_fiber(b.sched_tsan, __tsan_switch_to_fiber_no_sync));
    void* dummy;
    mgb_emul_switch(&dummy, b.sched_sp);
    std::abort();  // never resumed
}

static void prepare(Fiber& f) {
    if (!f.stack) f.stack = (char*)std::malloc(kStackBytes);
    uintptr_t top = ((uintptr_t)f.stack + kStackBytes) & ~(uintptr_t)15;
    void** sp = (void**)(top - 8);
    *sp = nullptr;                   // fake return address of fiber_main
    *(--sp) = (void*)&fiber_main;    // popped by `ret`
    for (int i = 0; i < 6; ++i) *(--sp) = nullptr;
    f.sp = (void*)sp;
    f.done = false;
}

void yield() {
    BlockState& b = *g_block;
    Fiber& f = b.fibers[b.current];
    RC(__tsan_switch_to_fiber(b.sched_tsan, __tsan_switch_to_fiber_no_sync));
    mgb_emul_switch(&f.sp, b.sched_sp);
}

static void resume(BlockState& b, unsigned i) {
    b.current = i;
    threadIdx.x = b.fibers[i].tid % blockDim.x;
    threadIdx.y = (b.fibers[i].tid / blockDim.x) % blockDim.y;
    threadIdx.z = b.fibers[i].tid / (blockDim.x * blockDim.y);
    RC(__tsan_switch_to_fiber(b.fibers[i].tsan, __tsan_switch_to_fiber_no_sync));
    mgb_emul_switch(&b.sched_sp, b.fibers[i].sp);
}
#else
#error "the emulator's context switch is written for x86-64"
#endif

// Generation `gen` of a barrier releases into and acquires from sync[gen & 1]: a thread that has left
// generation gen and arrives at gen + 1 must not hand its new accesses to a thread still leaving gen.
// (Nobody arrives at gen + 2 before everybody has left gen.)  A thread that has exited counts as arrived:
// the arrival that completes a generation hands on what the exited threads did (exit_sync), and a thread
// that exits later is not seen by threads still leaving an earlier generation.
void syncthreads() {
    BlockState& b = *g_block;
    unsigned gen = b.gen;
    if (b.arrived + 1 >= b.alive) RC(__tsan_acquire(&b.exit_sync));
    RC(__tsan_release(&b.sync[gen & 1]));
    if (++b.arrived >= b.alive) {
        b.arrived = 0;
        b.gen++;
    } else {
        while (b.gen == gen) yield();
    }
    RC(__tsan_acquire(&b.sync[gen & 1]));
}

static void warp_barrier(WarpState& w, unsigned expected) {
    unsigned gen = w.gen;
    RC(__tsan_release(&w.sync[gen & 1]));
    if (++w.arrived >= expected) {
        w.arrived = 0;
        w.gen++;
    } else {
        while (w.gen == gen) yield();
    }
    RC(__tsan_acquire(&w.sync[gen & 1]));
}

void warp_barrier(unsigned expected) { warp_barrier(g_block->warps[threadIdx.x >> 5], expected); }

uint64_t shfl_raw(unsigned expected, uint64_t raw, unsigned src_lane) {
    WarpState& w = g_block->warps[threadIdx.x >> 5];
    w.vals[threadIdx.x & 31u] = raw;
    warp_barrier(w, expected);
    uint64_t got = w.vals[src_lane];
    warp_barrier(w, expected);
    return got;
}

#ifdef MGB_EMUL_RACECHECK
// ThreadSanitizer tells at most 256 live threads apart (its runtime has 256 clock slots; a context beyond that
// takes over a slot and inherits its history as if ordered after it), so a block of more than kMaxFibers
// threads shares fibers among lanes of one warp.  Lanes that share a fiber look program-ordered to the checker,
// so their races are not seen; two groupings alternate by block and launch so that every pair of lanes is
// told apart in one of them:
// - consecutive: lane * per_warp / 32, runs of at most ceil(32 / per_warp) adjacent lanes;
// - strided:     lane % per_warp, lanes a multiple of per_warp apart.
// No two lanes share a fiber in both as long as per_warp >= 6, i.e. for blocks of up to 1184 threads.  A
// grouping never spans two warps: a fiber's acquires from one warp's barriers would otherwise order another
// warp's lanes.
static const unsigned kMaxFibers = 224;  // (slots are also needed by the host's own threads)

static unsigned fiber_of(unsigned tid, unsigned nthreads, bool strided) {
    if (nthreads <= kMaxFibers) return tid;
    const unsigned per_warp = kMaxFibers / ((nthreads + 31) / 32), lane = tid & 31u;
    return (tid >> 5) * per_warp + (strided ? lane % per_warp : lane * per_warp / 32);
}
#endif

// ----------------------------------------------------------------------------- schedule order
enum class Order { forward, reverse, seeded };

static Order schedule_order() {
    const char* s = std::getenv("MGB_EMUL_ORDER");
    if (!s || !*s || !std::strcmp(s, "forward")) return Order::forward;
    if (!std::strcmp(s, "reverse")) return Order::reverse;
    if (!std::strcmp(s, "seeded")) return Order::seeded;
    std::fprintf(stderr, "MGB_EMUL_ORDER=%s: expected forward, reverse or seeded\n", s);
    std::abort();
}

static std::mt19937& schedule_rng() {
    static thread_local std::mt19937 rng([] {
        const char* s = std::getenv("MGB_EMUL_SEED");
        return (unsigned)(s ? std::strtoul(s, nullptr, 10) : 1ul);
    }());
    return rng;
}

void launch(dim3 grid, dim3 bdim, size_t smem_bytes, const std::function<void()>& body) {
    static thread_local BlockState state;
    BlockState* outer = g_block;
    BlockState& b = state;
    g_block = &b;
    gridDim = grid;
    blockDim = bdim;
    unsigned nthreads = bdim.x * bdim.y * bdim.z;
    if (b.fibers.size() < nthreads) b.fibers.resize(nthreads);
    b.warps.assign((nthreads + 31) / 32, WarpState());
    b.body = body;
    const Order order = schedule_order();
    std::vector<unsigned> ready;
    ready.reserve(nthreads);
    const size_t smem_alloc = (smem_bytes + 64 + 127) / 128 * 128;
#ifdef MGB_EMUL_RACECHECK
    static thread_local unsigned launches = 0;
    const unsigned launch_index = launches++;
    if ((nthreads + 31) / 32 > kMaxFibers / 6) {
        std::fprintf(stderr, "race-checking emulator: blocks of %u threads are not supported\n", nthreads);
        std::abort();
    }
    std::vector<void*> tsan_fibers;
#endif
    for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
            for (unsigned bx = 0; bx < grid.x; ++bx) {
                blockIdx.x = bx; blockIdx.y = by; blockIdx.z = bz;
                b.nthreads = b.alive = nthreads;
                b.arrived = 0;
                for (auto& w : b.warps) { w.arrived = 0; }
                // a fresh, poisoned allocation: nothing of the previous block (or launch) survives in it
                b.dyn_smem = (unsigned char*)std::aligned_alloc(128, smem_alloc);
                std::memset(b.dyn_smem, 0xFF, smem_alloc);
                for (unsigned i = 0; i < nthreads; ++i) { b.fibers[i].tid = i; prepare(b.fibers[i]); }
#ifdef MGB_EMUL_RACECHECK
                b.sched_tsan = __tsan_get_current_fiber();
                const bool strided = ((launch_index + bx + grid.x * (by + grid.y * bz)) & 1) != 0;
                const unsigned warps = (nthreads + 31) / 32;
                tsan_fibers.assign(nthreads <= kMaxFibers ? nthreads : warps * (kMaxFibers / warps), nullptr);
                for (void*& f : tsan_fibers) f = __tsan_create_fiber(0);
                for (unsigned i = 0; i < nthreads; ++i) b.fibers[i].tsan = tsan_fibers[fiber_of(i, nthreads, strided)];
#endif
                RC(__tsan_release(&b.start_sync));
                while (b.alive > 0) {
                    ready.clear();
                    for (unsigned i = 0; i < nthreads; ++i)
                        if (!b.fibers[i].done) ready.push_back(i);
                    if (ready.empty()) break;
                    if (order == Order::reverse) std::reverse(ready.begin(), ready.end());
                    if (order == Order::seeded) std::shuffle(ready.begin(), ready.end(), schedule_rng());
                    for (unsigned i : ready)
                        if (!b.fibers[i].done) resume(b, i);
                }
                RC(__tsan_acquire(&b.end_sync));
#ifdef MGB_EMUL_RACECHECK
                for (void* f : tsan_fibers) __tsan_destroy_fiber(f);
#endif
                std::free(b.dyn_smem);
                b.dyn_smem = nullptr;
            }
    g_block = outer;
}

}  // namespace emul
