// tests/emu/emu_rt.cpp — TEST INFRASTRUCTURE: fibers + cooperative scheduler + synchronous "CUDA runtime" behind
// tests/emu/cuda_runtime.h.  See that header for the model and for what it does and does not check.
#include <stdio.h>
#include <sys/mman.h>
#include <time.h>

#include <algorithm>
#include <mutex>
#include <vector>

#include "cuda_runtime.h"

// ---- context switch (x86-64 SysV: callee-saved registers + stack pointer) ----------------------------------------------
extern "C" void emu_switch(void **save_sp, void *new_sp);
asm(R"(
.text
.globl emu_switch
.type emu_switch,@function
emu_switch:
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
.size emu_switch,.-emu_switch
)");

struct EmuWarp {
    unsigned arrived = 0, part = 0, gen = 0, alive = 0, pending_mask = 0;
    int pending_kind = 0;
    uint64_t xchg[2][32];
    unsigned parts[2] = {0, 0};
};

EmuThread *emu_cur = nullptr;
// Dynamic shared memory of the CTA being run: the END of what the launch asked for touches an inaccessible page, so a kernel that
// strays past its shared-memory size faults (to 16 bytes, the alignment the base keeps).
static const size_t SMEM_MAX = 256 << 10;
static unsigned char *g_smem_region = nullptr;     // SMEM_MAX usable bytes followed by a PROT_NONE page
unsigned char *emu_smem = nullptr;
size_t emu_smem_bytes = 0;

static const size_t STACK_BYTES = 256 << 10;
static std::vector<void *> g_stacks;              // reused across launches
static std::vector<EmuThread> g_threads;
static std::vector<EmuWarp> g_warps;
static void *g_sched_sp = nullptr;
static const std::function<void()> *g_body = nullptr;
static unsigned g_block_arrived = 0, g_block_gen = 0, g_alive = 0;
static std::mutex g_launch_mutex;
static const char *g_fault = nullptr;

static void yield_to_scheduler() {
    EmuThread *me = emu_cur;
    emu_switch(&me->sp, g_sched_sp);
    emu_cur = me;
}

static void fiber_exit_check_warp(EmuWarp *w);

static void fiber_main() {
    (*g_body)();
    EmuThread *me = emu_cur;
    me->state = 3;
    g_alive--;
    EmuWarp *w = me->warp;
    w->alive &= ~(1u << me->lane);
    fiber_exit_check_warp(w);                       // a lane that exits may complete a rendezvous the others wait in
    if (g_block_arrived && g_block_arrived == g_alive) {   // ... or a block barrier
        g_block_arrived = 0; g_block_gen++;
        for (auto &t : g_threads) if (t.state == 2) t.state = 0;
    }
    emu_switch(&me->sp, g_sched_sp);
    abort();                                        // never resumed
}

static void complete_rendezvous(EmuWarp *w) {
    w->parts[w->gen & 1u] = w->arrived;
    w->arrived = 0; w->pending_mask = 0; w->gen++;
    const unsigned first = (unsigned)(w - g_warps.data()) * 32;
    for (unsigned l = 0; l < 32 && first + l < g_threads.size(); l++) {
        EmuThread &t = g_threads[first + l];
        if (t.state == 1) t.state = 0;
    }
}

static void fiber_exit_check_warp(EmuWarp *w) {
    if (w->arrived && w->arrived == (w->pending_mask & w->alive)) complete_rendezvous(w);
}

uint64_t *emu_warp_exchange(unsigned mask, uint64_t value, int kind) {
    EmuThread *me = emu_cur;
    EmuWarp *w = me->warp;
    const unsigned g = w->gen, buf = g & 1u;
    if (!((mask >> me->lane) & 1u)) { g_fault = "a lane called a *_sync collective with a mask that does not name it"; fprintf(stderr, "emu: %s\n", g_fault); abort(); }
    if (w->arrived && w->pending_mask != mask) { g_fault = "lanes of one warp met in *_sync collectives with different masks"; fprintf(stderr, "emu: %s\n", g_fault); abort(); }
    if (w->arrived && w->pending_kind != kind) {
        g_fault = "lanes of one warp met in DIFFERENT collectives (e.g. a *_sync call that only some lanes execute)";
        fprintf(stderr, "emu: %s: kinds %d and %d, block %u warp %u lane %u\n", g_fault, w->pending_kind, kind, me->bid.x, me->warp_id, me->lane);
        abort();
    }
    w->pending_mask = mask; w->pending_kind = kind;
    w->xchg[buf][me->lane] = value;
    w->arrived |= 1u << me->lane;
    if (w->arrived == (mask & w->alive)) complete_rendezvous(w);
    else {
        me->state = 1; me->wait_gen = g;
        yield_to_scheduler();
    }
    return w->xchg[buf];
}

unsigned emu_warp_arrived_mask() {
    EmuWarp *w = emu_cur->warp;
    return w->parts[(w->gen - 1u) & 1u];            // valid until this lane enters its next collective
}

void emu_block_barrier() {
    EmuThread *me = emu_cur;
    g_block_arrived++;
    if (g_block_arrived == g_alive) {
        g_block_arrived = 0; g_block_gen++;
        for (auto &t : g_threads) if (t.state == 2) t.state = 0;
    } else {
        me->state = 2;
        yield_to_scheduler();
    }
}

static void *new_stack() {
    void *p = mmap(nullptr, STACK_BYTES, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (p == MAP_FAILED) { perror("emu: mmap"); abort(); }
    mprotect(p, 4096, PROT_NONE);                   // guard page
    return p;
}

void emu_launch(unsigned grid, unsigned block, size_t smem_bytes, const std::function<void()> &body) {
    std::lock_guard<std::mutex> lock(g_launch_mutex);
    if (!g_smem_region) {
        g_smem_region = (unsigned char *)mmap(nullptr, SMEM_MAX + 4096, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
        if (g_smem_region == MAP_FAILED) { perror("emu: mmap"); abort(); }
        mprotect(g_smem_region + SMEM_MAX, 4096, PROT_NONE);
    }
    if (block == 0 || block > 1024 || smem_bytes > SMEM_MAX) { fprintf(stderr, "emu: bad launch configuration (%u threads, %zu bytes)\n", block, smem_bytes); abort(); }
    while (g_stacks.size() < block) g_stacks.push_back(new_stack());
    const unsigned n_warps = (block + 31) / 32;
    for (unsigned b = 0; b < grid; b++) {
        emu_smem_bytes = (smem_bytes + 15) & ~(size_t)15;
        emu_smem = g_smem_region + SMEM_MAX - emu_smem_bytes;
        memset(emu_smem, 0xcd, emu_smem_bytes);                           // shared memory starts undefined
        g_threads.assign(block, EmuThread());
        g_warps.assign(n_warps, EmuWarp());
        g_body = &body; g_block_arrived = 0; g_alive = block;
        for (unsigned t = 0; t < block; t++) {
            EmuThread &th = g_threads[t];
            th.tid = uint3{t, 0, 0}; th.bid = uint3{b, 0, 0}; th.bdim = uint3{block, 1, 1}; th.gdim = uint3{grid, 1, 1};
            th.lane = t & 31; th.warp_id = t >> 5; th.warp = &g_warps[t >> 5]; th.state = 0;
            g_warps[t >> 5].alive |= 1u << (t & 31);
            // initial frame: six callee-saved registers, the entry point as return address, one slot of padding for alignment
            uintptr_t top = ((uintptr_t)g_stacks[t] + STACK_BYTES) & ~(uintptr_t)15;
            void **sp = (void **)top;
            *--sp = nullptr;                         // fake return address of fiber_main (keeps rsp = 8 mod 16 at its entry)
            *--sp = (void *)fiber_main;
            for (int i = 0; i < 6; i++) *--sp = nullptr;
            th.sp = sp;
        }
        // round-robin until every thread is done.  B200_EMU_SCHED_SEED=<n>: a different random order of the fibers in every round
        // (lanes within a warp and warps within the CTA), to shake out code that only works in the default lane-0-first order
        static const char *sched_env = getenv("B200_EMU_SCHED_SEED");
        static uint64_t rng = sched_env ? (uint64_t)strtoull(sched_env, nullptr, 10) * 0x9E3779B97F4A7C15ull + 1 : 0;
        std::vector<unsigned> order(block);
        for (unsigned t = 0; t < block; t++) order[t] = t;
        while (g_alive) {
            bool progressed = false;
            if (sched_env)
                for (unsigned i = block - 1; i > 0; i--) {
                    rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;          // xorshift64
                    std::swap(order[i], order[rng % (i + 1)]);
                }
            for (unsigned oi = 0; oi < block; oi++) {
                const unsigned t = order[oi];
                EmuThread &th = g_threads[t];
                if (th.state != 0) continue;
                progressed = true;
                emu_cur = &th;
                emu_switch(&g_sched_sp, th.sp);
            }
            if (!progressed) {
                fprintf(stderr, "emu: deadlock in block %u: every live thread waits in a rendezvous (divergent *_sync / __syncthreads?)\n", b);
                for (unsigned w = 0; w < n_warps; w++)
                    fprintf(stderr, "  warp %u: alive %08x arrived %08x mask %08x\n", w, g_warps[w].alive, g_warps[w].arrived, g_warps[w].pending_mask);
                abort();
            }
        }
        emu_cur = nullptr;
    }
}

// ---- runtime ---------------------------------------------------------------------------------------------------------------
struct EmuStream { int dummy; };
struct EmuEvent { double t_ms; };

static double now_ms() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; }

cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) {
    memset(p, 0, sizeof *p);
    snprintf(p->name, sizeof p->name, "SIMT emulator (tests/emu)");
    p->major = 9; p->minor = 0;
    const char *e = getenv("B200_EMU_SMS");
    p->multiProcessorCount = e ? atoi(e) : 2;      // grid sizes follow the SM count: keep emulated grids small
    if (p->multiProcessorCount < 1) p->multiProcessorCount = 1;
    p->totalGlobalMem = (size_t)8 << 30; p->sharedMemPerBlockOptin = 227 << 10;
    return cudaSuccess;
}
cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
cudaError_t cudaDeviceGetStreamPriorityRange(int *lo, int *hi) { *lo = 0; *hi = -1; return cudaSuccess; }
cudaError_t cudaStreamCreateWithPriority(cudaStream_t *s, unsigned, int) { *s = new EmuStream(); return cudaSuccess; }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = new EmuStream(); return cudaSuccess; }
cudaError_t cudaStreamCreate(cudaStream_t *s) { *s = new EmuStream(); return cudaSuccess; }
cudaError_t cudaStreamDestroy(cudaStream_t s) { delete s; return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = new EmuEvent(); (*e)->t_ms = 0; return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { return cudaEventCreate(e); }
cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { e->t_ms = now_ms(); return cudaSuccess; }
cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(b->t_ms - a->t_ms); return cudaSuccess; }
// Fault injection for the error paths of the host code: the n-th allocation from now on fails (0 = never).
static long g_fail_after = 0;
extern "C" __attribute__((visibility("default"))) void emu_fail_alloc_after(long n) { g_fail_after = n; }
static bool alloc_should_fail() { return g_fail_after > 0 && --g_fail_after == 0; }

cudaError_t cudaMalloc(void **p, size_t n) {
    if (alloc_should_fail()) { *p = nullptr; return cudaErrorMemoryAllocation; }
    // 256-byte alignment like the real allocator; contents undefined (0xcd) so that reads of unwritten device memory show up
    if (posix_memalign(p, 256, n ? n : 1) != 0) { *p = nullptr; return cudaErrorMemoryAllocation; }
    memset(*p, 0xcd, n);
    return cudaSuccess;
}
cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
cudaError_t cudaHostAlloc(void **p, size_t n, unsigned) { if (alloc_should_fail()) { *p = nullptr; return cudaErrorMemoryAllocation; } if (posix_memalign(p, 256, n ? n : 1) != 0) { *p = nullptr; return cudaErrorMemoryAllocation; } memset(*p, 0xcd, n); return cudaSuccess; }
cudaError_t cudaMallocHost(void **p, size_t n) { return cudaHostAlloc(p, n, 0); }
cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t) { if (n) memmove(d, s, n); return cudaSuccess; }
cudaError_t cudaMemcpy2DAsync(void *d, size_t dpitch, const void *s, size_t spitch, size_t width, size_t height, cudaMemcpyKind, cudaStream_t) {
    for (size_t r = 0; r < height; r++) memmove((char *)d + r * dpitch, (const char *)s + r * spitch, width);
    return cudaSuccess;
}
cudaError_t cudaMemset(void *d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t) { if (n) memset(d, v, n); return cudaSuccess; }
cudaError_t cudaGetLastError() { return cudaSuccess; }
cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : e == cudaErrorMemoryAllocation ? "out of memory" : "emulated CUDA error"; }
