// cuda_shim.h -- enough of the CUDA device dialect to compile the kernels of lepton_b200/csrc as host C++ and run them
// with REAL 32-lane warps on the CPU.  Test infrastructure only: nothing here is part of the product.
//
// Every CUDA thread of a CTA is a fiber (own stack, hand-written context switch) inside one OS thread.  A fiber runs until
// it reaches a warp collective (__shfl*_sync, __ballot_sync, __any/__all_sync, __match_any_sync, __reduce_*_sync,
// __syncwarp) or __syncthreads, parks there, and the next fiber runs; the last lane to arrive releases the others.
// That is the execution model the kernels are written against (independent thread scheduling + explicit *_sync points),
// so divergence, votes, shuffles, shared memory and the persistent-CTA work queues behave as on the device, only
// sequentially: CTAs run one after the other, atomics are plain operations.  What it cannot show is anything that
// depends on timing or on the memory hierarchy.
//
// Collectives are supported with the full mask only (all the kernels use), and a lane that has returned counts as
// arrived, like an exited thread on the device.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
#define __constant__ const
#define __shared__ static
#define __restrict__
#define __launch_bounds__(...)
#define LEPB200_EMU 1

namespace emu {

struct Dim3 { unsigned x = 0, y = 0, z = 0; };

struct Warp {
    uint64_t slot[2][32];
    unsigned part[2] = {0, 0};             // lanes that took part in the collective whose deposits are in slot[i]
    unsigned gen = 0, exited_mask = 0;
    int arrived = 0, exited = 0, kind = 0;
    void* first_site = nullptr;             // code address of the first arrival (diagnostics)
};

struct Deposits {
    const uint64_t* v;                      // the 32 deposits (valid until the lane's next collective)
    unsigned part;                          // lanes that deposited; a lane that had returned before does not vote
};

struct Lane {
    void* sp = nullptr;
    char* stack = nullptr;
    Dim3 tid;
    int lane = 0;
    Warp* warp = nullptr;
    bool done = true;
};

struct Cta {
    std::vector<Lane> lanes;
    std::vector<Warp> warps;
    int nthreads = 0, live = 0;
    unsigned sync_gen = 0;
    int sync_arrived = 0;
    void (*body)(void*) = nullptr;
    void* arg = nullptr;
    void* main_sp = nullptr;
};

inline Cta g_cta;
inline Lane* g_cur = nullptr;
inline unsigned long long g_progress = 0;       // arrivals + exits: a wait loop that sees no progress for long is a deadlock
inline Dim3 g_block_idx, g_block_dim, g_grid_dim;
// schedule: false = CTAs in order and, inside a CTA, thread 0 first (each runs until it waits or returns); true = the
// last CTA first and the threads of a CTA from the last one down.  A kernel that is right only because of the order in
// which its threads touch shared data gives different results under the two.
inline bool g_reverse = false;

extern "C" void emu_ctx_switch(void** from_sp, void* to_sp);
#if defined(__x86_64__)
// callee-saved registers on the outgoing stack, swap stack pointers, restore (System V AMD64)
asm(R"(
    .text
    .globl emu_ctx_switch
    .type emu_ctx_switch,@function
emu_ctx_switch:
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
    .size emu_ctx_switch,.-emu_ctx_switch
)");
#else
#error "the warp emulator's context switch is written for x86-64"
#endif

// run the next fiber that has not returned; back to the launcher when none is left
inline void yield() {
    Cta& c = g_cta;
    Lane* from = g_cur;
    const int n = c.nthreads;
    int i = (int)(from - c.lanes.data());
    for (int k = 0; k < n; ++k) {
        if (g_reverse) i = i == 0 ? n - 1 : i - 1;
        else i = i + 1 == n ? 0 : i + 1;
        if (!c.lanes[i].done) {
            if (&c.lanes[i] == from) return;           // everybody else is gone: keep going (a wait loop will re-check)
            g_cur = &c.lanes[i];
            emu_ctx_switch(&from->sp, g_cur->sp);
            return;
        }
    }
    emu_ctx_switch(&from->sp, c.main_sp);
}

inline void wait_check(unsigned long long& seen, unsigned& spins, const char* what) {
    if (seen != g_progress) { seen = g_progress; spins = 0; return; }
    if (++spins > 1000000u) { fprintf(stderr, "warp emulator: deadlock, every remaining thread is parked (%s)\n", what); abort(); }
}

inline void release_if_complete(Warp& w) {
    if (w.arrived > 0 && w.arrived + w.exited == 32) { w.part[w.gen & 1] = ~w.exited_mask; w.arrived = 0; w.gen++; }
}

inline void lane_exit() {
    Cta& c = g_cta;
    Lane* me = g_cur;
    me->done = true;
    c.live--;
    g_progress++;
    me->warp->exited++;
    me->warp->exited_mask |= 1u << me->lane;
    release_if_complete(*me->warp);
    if (c.sync_arrived > 0 && c.sync_arrived == c.live) { c.sync_arrived = 0; c.sync_gen++; }
    yield();                                            // never comes back
    abort();
}

inline void trampoline() {
    g_cta.body(g_cta.arg);
    lane_exit();
}

// all lanes of the calling warp deposit `v` and get everybody's deposits back
__attribute__((noinline)) inline Deposits exchange(uint64_t v, int kind) {
    Lane* me = g_cur;
    Warp& w = *me->warp;
    const unsigned g = w.gen;
    uint64_t* buf = w.slot[g & 1];
    if (w.arrived == 0) { w.kind = kind; w.first_site = __builtin_return_address(0); }
    else if (w.kind != kind) {
        fprintf(stderr, "warp emulator: lanes of one warp are in different collectives (%d at %p vs %d at %p): thread %u, %d arrived, %d exited, generation %u\n",
                w.kind, (void*)((char*)w.first_site - (char*)&emu_ctx_switch), kind, (void*)((char*)__builtin_return_address(0) - (char*)&emu_ctx_switch), me->tid.x, w.arrived, w.exited, w.gen);
        abort();
    }
    buf[me->lane] = v;
    w.arrived++;
    g_progress++;
    release_if_complete(w);
    unsigned long long seen = g_progress;
    unsigned spins = 0;
    while (w.gen == g) { yield(); wait_check(seen, spins, "warp collective"); }
    Deposits d = {buf, w.part[g & 1]};
    return d;
}

inline void cta_barrier() {
    Cta& c = g_cta;
    const unsigned g = c.sync_gen;
    g_progress++;
    if (++c.sync_arrived == c.live) { c.sync_arrived = 0; c.sync_gen++; }
    unsigned long long seen = g_progress;
    unsigned spins = 0;
    while (c.sync_gen == g) { yield(); wait_check(seen, spins, "__syncthreads"); }
}

constexpr size_t STACK_BYTES = 128 * 1024;

// Runs grid x block CUDA threads of `body(arg)`; CTAs one after the other.
inline void launch(unsigned grid, unsigned block, void (*body)(void*), void* arg) {
    Cta& c = g_cta;
    if (block % 32 != 0 && block > 32) { fprintf(stderr, "warp emulator: block size must be <= 32 or a multiple of 32\n"); abort(); }
    if (c.lanes.size() < block) {
        const size_t old = c.lanes.size();
        c.lanes.resize(block);
        for (size_t i = old; i < block; ++i) c.lanes[i].stack = static_cast<char*>(aligned_alloc(64, STACK_BYTES));
    }
    g_block_dim.x = block; g_block_dim.y = g_block_dim.z = 1;
    g_grid_dim.x = grid; g_grid_dim.y = g_grid_dim.z = 1;
    for (unsigned bb = 0; bb < grid; ++bb) {
        const unsigned b = g_reverse ? grid - 1 - bb : bb;
        g_block_idx.x = b;
        c.nthreads = (int)block; c.live = (int)block; c.sync_gen = 0; c.sync_arrived = 0;
        c.body = body; c.arg = arg;
        c.warps.assign((block + 31) / 32, Warp());
        for (unsigned t = 0; t < block; ++t) {
            Lane& l = c.lanes[t];
            l.tid.x = t; l.tid.y = l.tid.z = 0;
            l.lane = (int)(t & 31);
            l.warp = &c.warps[t >> 5];
            l.done = false;
            // first switch pops six registers and returns into the trampoline with (rsp + 8) % 16 == 0
            uintptr_t top = (reinterpret_cast<uintptr_t>(l.stack) + STACK_BYTES) & ~uintptr_t(15);
            void** sp = reinterpret_cast<void**>(top - 64);
            for (int k = 0; k < 6; ++k) sp[k] = nullptr;
            sp[6] = reinterpret_cast<void*>(&trampoline);
            l.sp = sp;
        }
        for (unsigned t = block; t < ((block + 31) / 32) * 32; ++t) { c.warps[t >> 5].exited++; c.warps[t >> 5].exited_mask |= 1u << (t & 31); }      // lanes of a partial warp that do not exist
        g_cur = &c.lanes[g_reverse ? block - 1 : 0];
        emu_ctx_switch(&c.main_sp, g_cur->sp);
        if (c.live != 0) { fprintf(stderr, "warp emulator: CTA %u stopped with %d threads parked (deadlock)\n", b, c.live); abort(); }
    }
}

}  // namespace emu

#define threadIdx (emu::g_cur->tid)
#define blockIdx (emu::g_block_idx)
#define blockDim (emu::g_block_dim)
#define gridDim (emu::g_grid_dim)

struct uint4 { uint32_t x, y, z, w; };
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { uint4 r = {x, y, z, w}; return r; }
struct uint2 { uint32_t x, y; };
static inline uint2 make_uint2(uint32_t x, uint32_t y) { uint2 r = {x, y}; return r; }

enum { EMU_K_SYNCWARP = 1, EMU_K_VOTE, EMU_K_SHFL, EMU_K_MATCH, EMU_K_REDUCE };

static inline void __syncthreads() { emu::cta_barrier(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { emu::exchange(0, EMU_K_SYNCWARP); }
static inline void emu_check_full(unsigned mask) { if (mask != 0xffffffffu) { fprintf(stderr, "warp emulator: only full-mask collectives are modelled\n"); abort(); } }
static inline unsigned __ballot_sync(unsigned mask, int p) {
    emu_check_full(mask);
    const emu::Deposits d = emu::exchange(p ? 1 : 0, EMU_K_VOTE);
    unsigned r = 0;
    for (int i = 0; i < 32; ++i) if (d.v[i] & 1) r |= 1u << i;
    return r & d.part;
}
static inline int __any_sync(unsigned mask, int p) { return __ballot_sync(mask, p) != 0; }
static inline int __all_sync(unsigned mask, int p) { return __ballot_sync(mask, !p) == 0; }
template <class T> static inline T __shfl_sync(unsigned mask, T v, int src) {
    static_assert(sizeof(T) <= 8, "shuffle of at most 64 bits");
    emu_check_full(mask);
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    const emu::Deposits d = emu::exchange(raw, EMU_K_SHFL);
    T r;
    memcpy(&r, &d.v[src & 31], sizeof(T));
    return r;
}
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int lanemask) { return __shfl_sync(mask, v, emu::g_cur->lane ^ lanemask); }
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta) {
    const int src = emu::g_cur->lane - (int)delta;
    return __shfl_sync(mask, v, src < 0 ? emu::g_cur->lane : src);
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta) {
    const int src = emu::g_cur->lane + (int)delta;
    return __shfl_sync(mask, v, src > 31 ? emu::g_cur->lane : src);
}
static inline unsigned __match_any_sync(unsigned mask, uint32_t v) {
    emu_check_full(mask);
    const emu::Deposits d = emu::exchange(v, EMU_K_MATCH);
    unsigned r = 0;
    for (int i = 0; i < 32; ++i) if ((uint32_t)d.v[i] == v) r |= 1u << i;
    return r & d.part;
}
static inline unsigned __reduce_add_sync(unsigned mask, unsigned v) {
    emu_check_full(mask);
    const emu::Deposits d = emu::exchange(v, EMU_K_REDUCE);
    unsigned r = 0;
    for (int i = 0; i < 32; ++i) if ((d.part >> i) & 1) r += (unsigned)d.v[i];
    return r;
}
static inline int __reduce_add_sync(unsigned mask, int v) { return (int)__reduce_add_sync(mask, (unsigned)v); }
static inline unsigned __reduce_max_sync(unsigned mask, unsigned v) {
    emu_check_full(mask);
    const emu::Deposits d = emu::exchange(v, EMU_K_REDUCE);
    unsigned r = 0;
    for (int i = 0; i < 32; ++i) if (((d.part >> i) & 1) && (unsigned)d.v[i] > r) r = (unsigned)d.v[i];
    return r;
}
static inline int __reduce_max_sync(unsigned mask, int v) {
    emu_check_full(mask);
    const emu::Deposits d = emu::exchange((uint64_t)(uint32_t)v, EMU_K_REDUCE);
    int r = INT32_MIN;
    for (int i = 0; i < 32; ++i) if (((d.part >> i) & 1) && (int)(uint32_t)d.v[i] > r) r = (int)(uint32_t)d.v[i];
    return r;
}

// one OS thread: atomics are plain read-modify-writes
template <class T> static inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
template <class T> static inline T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }
template <class T> static inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }

template <class T> static inline T __ldg(const T* p) { return *p; }

static inline int __clz(uint32_t v) { return v ? __builtin_clz(v) : 32; }
static inline int __clzll(unsigned long long v) { return v ? __builtin_clzll(v) : 64; }
static inline int __popc(uint32_t v) { return __builtin_popcount(v); }
static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
static inline int __ffs(uint32_t v) { return __builtin_ffs((int)v); }
static inline uint32_t __brev(uint32_t v) { uint32_t r = 0; for (int i = 0; i < 32; ++i) if (v & (1u << i)) r |= 1u << (31 - i); return r; }
static inline uint32_t __umulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
static inline uint32_t __funnelshift_l(uint32_t lo, uint32_t hi, uint32_t shift) {
    const uint64_t v = ((uint64_t)hi << 32) | lo;
    return (uint32_t)((v << (shift & 31)) >> 32);
}
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t shift) {
    const uint64_t v = ((uint64_t)hi << 32) | lo;
    return (uint32_t)(v >> (shift & 31));
}
static inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t sel) {
    const uint64_t v = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i) r |= (uint32_t)((v >> (8 * ((sel >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
}
// cvt.rz.f32.u32: the largest float not above the integer
static inline float __uint2float_rz(uint32_t a) {
    float f = (float)a;
    if ((double)f > (double)a) f = std::nextafterf(f, 0.0f);
    return f;
}
static inline float __frcp_rn(float x) { return 1.0f / x; }          // IEEE round-to-nearest reciprocal

static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline uint32_t min(uint32_t a, uint32_t b) { return a < b ? a : b; }
static inline uint32_t max(uint32_t a, uint32_t b) { return a > b ? a : b; }
static inline unsigned long long min(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
static inline unsigned long long max(unsigned long long a, unsigned long long b) { return a > b ? a : b; }
