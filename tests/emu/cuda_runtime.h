// tests/emu/cuda_runtime.h — TEST INFRASTRUCTURE.  A stand-in for the CUDA runtime + device intrinsics that lets the
// repository's .cu sources (kernels AND the C-ABI host code) be compiled by g++ and executed on the CPU, one fiber per
// CUDA thread, so that the `-m "not gpu"` tier can run the kernels' own source through the parity tests and a kernel
// change can be checked for logic errors before GPU minutes are spent on it.
//
// This is NOT a product path: nothing under readsb_b200/ or include/ refers to it, the product library is still built by
// nvcc for sm_90a only and still has no CPU path (tests/test_abi.py).  The emulated library is built by
// tests/emu/build_emu.py into tests/emu/_build/ and is only ever loaded by tests/test_emu_kernels.py.
//
// Model: a CTA's threads are fibers scheduled cooperatively on the calling OS thread; CTAs of a grid run one after the
// other (no kernel here waits for another CTA).  Warp collectives (*_sync, __syncwarp) and __syncthreads are rendezvous
// points: a lane leaves only when every lane named in the mask has arrived, and lanes run strictly one at a time in
// between — so shared-memory communication inside a warp that lacks a __syncwarp fails deterministically here (stricter
// than the hardware).  "Device" memory is host memory; streams execute at enqueue time, in call order (a valid order for
// any correctly synchronised program; missing cross-stream dependencies are NOT detected).
#pragma once
#include <stddef.h>
#include <stdio.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

#include <functional>
#include <type_traits>

#define B200_HOST_EMU 1

// ---- qualifiers ----------------------------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define EMU_NOINLINE __attribute__((noinline))   /* build_emu.py rewrites __noinline__ to this */
#define __launch_bounds__(...)
#define __maxnreg__(...)
#define __align__(n) alignas(n)
#define __shared__ static            /* static __shared__ variables: one CTA at a time on one OS thread */

// ---- vector types ---------------------------------------------------------------------------------------------------
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
struct alignas(8) float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) int2 { int x, y; };
struct uint3 { unsigned x, y, z; };
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
static inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline int2 make_int2(int x, int y) { return int2{x, y}; }

// ---- the fiber a CUDA thread runs on ---------------------------------------------------------------------------------
struct EmuWarp;
struct EmuThread {
    uint3 tid, bid, bdim, gdim;
    unsigned lane, warp_id;
    EmuWarp *warp;
    void *sp;                 // saved stack pointer while switched out
    int state;                // 0 runnable, 1 waiting in a warp rendezvous, 2 waiting in __syncthreads, 3 done
    unsigned wait_gen;
};
extern EmuThread *emu_cur;
extern unsigned char *emu_smem;      // the CTA's dynamic shared memory (16-byte aligned; its end touches an inaccessible page)
extern size_t emu_smem_bytes;

#define threadIdx (emu_cur->tid)
#define blockIdx (emu_cur->bid)
#define blockDim (emu_cur->bdim)
#define gridDim (emu_cur->gdim)

// rendezvous primitives (emu_rt.cpp)
uint64_t *emu_warp_exchange(unsigned mask, uint64_t value, int kind);   // returns the 32 values of the lanes that took part (lane-indexed); kind: which collective (all lanes of a rendezvous must agree)
unsigned emu_warp_arrived_mask();                             // lanes that took part in the exchange just completed
void emu_block_barrier();

// ---- warp collectives ------------------------------------------------------------------------------------------------
template <class T> static inline uint64_t emu_pack(T v) { static_assert(sizeof(T) <= 8, "shuffle of > 8 bytes"); uint64_t u = 0; memcpy(&u, &v, sizeof(T)); return u; }
template <class T> static inline T emu_unpack(uint64_t u) { T v; memcpy(&v, &u, sizeof(T)); return v; }

template <class T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
    const uint64_t *x = emu_warp_exchange(mask, emu_pack(v), 1);
    const unsigned lane = emu_cur->lane, base = lane & ~(unsigned)(width - 1);
    return emu_unpack<T>(x[base + ((unsigned)src & (unsigned)(width - 1))]);
}
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    const uint64_t *x = emu_warp_exchange(mask, emu_pack(v), 2);
    const unsigned lane = emu_cur->lane, base = lane & ~(unsigned)(width - 1);
    return (lane - base) >= delta ? emu_unpack<T>(x[lane - delta]) : v;
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    const uint64_t *x = emu_warp_exchange(mask, emu_pack(v), 3);
    const unsigned lane = emu_cur->lane, base = lane & ~(unsigned)(width - 1);
    return (lane - base) + delta < (unsigned)width ? emu_unpack<T>(x[lane + delta]) : v;
}
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int lanemask, int width = 32) {
    const uint64_t *x = emu_warp_exchange(mask, emu_pack(v), 4);
    const unsigned lane = emu_cur->lane, other = lane ^ (unsigned)lanemask;
    return (other & ~(unsigned)(width - 1)) == (lane & ~(unsigned)(width - 1)) ? emu_unpack<T>(x[other]) : v;
}
static inline unsigned __ballot_sync(unsigned mask, int pred) {
    const uint64_t *x = emu_warp_exchange(mask, pred ? 1u : 0u, 5);
    const unsigned part = emu_warp_arrived_mask();
    unsigned r = 0;
    for (unsigned l = 0; l < 32; l++) if (((part >> l) & 1u) && x[l]) r |= 1u << l;
    return r;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __all_sync(unsigned mask, int pred) { const unsigned b = __ballot_sync(mask, pred); return b == (emu_warp_arrived_mask()); }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { (void)emu_warp_exchange(mask, 0, 6); }
static inline void __syncthreads() { emu_block_barrier(); }
static inline void __threadfence_block() {}
static inline void __threadfence() {}
template <class T> static inline T emu_reduce(unsigned mask, T v, int op) {
    const uint64_t *x = emu_warp_exchange(mask, emu_pack(v), 16 + op);
    const unsigned part = emu_warp_arrived_mask();
    bool first = true; T r = 0;
    for (unsigned l = 0; l < 32; l++) if ((part >> l) & 1u) {
        const T e = emu_unpack<T>(x[l]);
        if (first) { r = e; first = false; }
        else switch (op) { case 0: r = (T)(r + e); break; case 1: r = r < e ? r : e; break; case 2: r = r > e ? r : e; break;
                           case 3: r = (T)(r & e); break; case 4: r = (T)(r | e); break; default: r = (T)(r ^ e); }
    }
    return r;
}
static inline unsigned __reduce_add_sync(unsigned mask, unsigned v) { return emu_reduce<unsigned>(mask, v, 0); }
static inline int __reduce_add_sync(unsigned mask, int v) { return emu_reduce<int>(mask, v, 0); }
static inline unsigned __reduce_min_sync(unsigned mask, unsigned v) { return emu_reduce<unsigned>(mask, v, 1); }
static inline unsigned __reduce_max_sync(unsigned mask, unsigned v) { return emu_reduce<unsigned>(mask, v, 2); }
static inline unsigned __reduce_and_sync(unsigned mask, unsigned v) { return emu_reduce<unsigned>(mask, v, 3); }
static inline unsigned __reduce_or_sync(unsigned mask, unsigned v) { return emu_reduce<unsigned>(mask, v, 4); }
static inline unsigned __reduce_xor_sync(unsigned mask, unsigned v) { return emu_reduce<unsigned>(mask, v, 5); }

// ---- integer intrinsics ------------------------------------------------------------------------------------------------
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __ffsll(long long x) { return __builtin_ffsll(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline unsigned __brev(unsigned x) {
    x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1); x = ((x >> 2) & 0x33333333u) | ((x & 0x33333333u) << 2);
    x = ((x >> 4) & 0x0f0f0f0fu) | ((x & 0x0f0f0f0fu) << 4); return __builtin_bswap32(x);
}
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) { return (unsigned)((((uint64_t)hi << 32) | lo) >> (sh & 31u)); }
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned sh) { return (unsigned)(((((uint64_t)hi << 32) | lo) << (sh & 31u)) >> 32); }
static inline unsigned emu_prmt(unsigned a, unsigned b, unsigned sel, bool sign_mode) {
    const uint64_t v = ((uint64_t)b << 32) | a;
    unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        const unsigned s = (sel >> (4 * i)) & 0xfu;
        unsigned byte = (unsigned)(v >> (8 * (s & 7u))) & 0xffu;
        if (sign_mode && (s & 8u)) byte = (byte & 0x80u) ? 0xffu : 0x00u;
        r |= byte << (8 * i);
    }
    return r;
}
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned sel) { return emu_prmt(a, b, sel & 0x7777u, false); }
static inline long long __double_as_longlong(double d) { long long v; memcpy(&v, &d, 8); return v; }
static inline double __longlong_as_double(long long v) { double d; memcpy(&d, &v, 8); return d; }
static inline unsigned __float_as_uint(float f) { unsigned v; memcpy(&v, &f, 4); return v; }
static inline float __uint_as_float(unsigned v) { float f; memcpy(&f, &v, 4); return f; }
static inline int __float_as_int(float f) { int v; memcpy(&v, &f, 4); return v; }
static inline float __int_as_float(int v) { float f; memcpy(&f, &v, 4); return f; }

template <class A, class B> static inline typename std::common_type<A, B>::type min(A a, B b) { typedef typename std::common_type<A, B>::type T; return (T)a < (T)b ? (T)a : (T)b; }
template <class A, class B> static inline typename std::common_type<A, B>::type max(A a, B b) { typedef typename std::common_type<A, B>::type T; return (T)a > (T)b ? (T)a : (T)b; }

// ---- memory ------------------------------------------------------------------------------------------------------------
template <class T> static inline T __ldg(const T *p) { return *p; }
template <class T> static inline T __ldcg(const T *p) { return *p; }
template <class T> static inline T __ldcs(const T *p) { return *p; }
template <class T> static inline void __stcg(T *p, T v) { *p = v; }
template <class T> static inline void __stcs(T *p, T v) { *p = v; }
static inline size_t __cvta_generic_to_shared(const void *p) {
    const ptrdiff_t off = (const unsigned char *)p - emu_smem;
    if (off < 0 || (size_t)off >= emu_smem_bytes) { fprintf(stderr, "emu: __cvta_generic_to_shared of a pointer outside dynamic shared memory\n"); abort(); }
    return (size_t)off;
}

template <class T, class V> static inline T atomicAdd(T *p, V v) { const T o = *p; *p = (T)(o + (T)v); return o; }
template <class T, class V> static inline T atomicSub(T *p, V v) { const T o = *p; *p = (T)(o - (T)v); return o; }
template <class T, class V> static inline T atomicOr(T *p, V v) { const T o = *p; *p = (T)(o | (T)v); return o; }
template <class T, class V> static inline T atomicAnd(T *p, V v) { const T o = *p; *p = (T)(o & (T)v); return o; }
template <class T, class V> static inline T atomicXor(T *p, V v) { const T o = *p; *p = (T)(o ^ (T)v); return o; }
template <class T, class V> static inline T atomicMax(T *p, V v) { const T o = *p; if ((T)v > o) *p = (T)v; return o; }
template <class T, class V> static inline T atomicMin(T *p, V v) { const T o = *p; if ((T)v < o) *p = (T)v; return o; }
template <class T, class V> static inline T atomicExch(T *p, V v) { const T o = *p; *p = (T)v; return o; }
template <class T, class V> static inline T atomicCAS(T *p, V cmp, V v) { const T o = *p; if (o == (T)cmp) *p = (T)v; return o; }

// ---- inline PTX (build_emu.py rewrites every asm statement into a call of emu_asm_<opcode>(outputs..., inputs..., immediates...)) ----
static inline void emu_asm_dp2a_lo_u32_s32(int &d, unsigned a, unsigned b, int c) { d = c + (int)(a & 0xffffu) * (int)(int8_t)(b & 0xffu) + (int)(a >> 16) * (int)(int8_t)((b >> 8) & 0xffu); }
static inline void emu_asm_dp2a_hi_u32_s32(int &d, unsigned a, unsigned b, int c) { d = c + (int)(a & 0xffffu) * (int)(int8_t)((b >> 16) & 0xffu) + (int)(a >> 16) * (int)(int8_t)(b >> 24); }
static inline void emu_asm_min_u16x2(unsigned &d, unsigned a, unsigned b) { const unsigned lo = (a & 0xffffu) < (b & 0xffffu) ? (a & 0xffffu) : (b & 0xffffu), hi = (a >> 16) < (b >> 16) ? (a >> 16) : (b >> 16); d = lo | (hi << 16); }
static inline void emu_asm_max_u16x2(unsigned &d, unsigned a, unsigned b) { const unsigned lo = (a & 0xffffu) > (b & 0xffffu) ? (a & 0xffffu) : (b & 0xffffu), hi = (a >> 16) > (b >> 16) ? (a >> 16) : (b >> 16); d = lo | (hi << 16); }
static inline void emu_asm_prmt_b32(unsigned &d, unsigned a, unsigned b, unsigned sel) { d = emu_prmt(a, b, sel, true); }
static inline void emu_asm_mad_wide_u32(unsigned long long &acc, unsigned a, unsigned b) { acc += (unsigned long long)a * b; }
static inline void emu_asm_ld_global_nc_L1__no_allocate_v4_u32(unsigned &x, unsigned &y, unsigned &z, unsigned &w, const void *p) {
    const uint4 v = *reinterpret_cast<const uint4 *>(p); x = v.x; y = v.y; z = v.z; w = v.w;
}
static inline void emu_asm_cp_async_cg_shared_global(unsigned dst, const void *src, int bytes) { memcpy(emu_smem + dst, src, (size_t)bytes); }
static inline void emu_asm_cp_async_ca_shared_global(unsigned dst, const void *src, int bytes) { memcpy(emu_smem + dst, src, (size_t)bytes); }
static inline void emu_asm_cp_async_cg_shared_global_L2__cache_hint(unsigned dst, const void *src, unsigned long long, int bytes) { memcpy(emu_smem + dst, src, (size_t)bytes); }
static inline void emu_asm_createpolicy_fractional_L2__evict_first_b64(unsigned long long &p) { p = 1; }
static inline void emu_asm_createpolicy_fractional_L2__evict_last_b64(unsigned long long &p) { p = 2; }
static inline void emu_asm_st_global_L2__cache_hint_b32(unsigned *p, unsigned v, unsigned long long) { *p = v; }
static inline void emu_asm_bar_sync(int, unsigned) { emu_block_barrier(); }     // named barrier of the warps still alive (the others have returned)
static inline void emu_asm_cp_async_commit_group() {}
static inline void emu_asm_cp_async_wait_group(int) {}
static inline void emu_asm_prefetch_global_L2(const void *) {}

// ---- runtime API (emu_rt.cpp): synchronous, host memory ------------------------------------------------------------------
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorInvalidValue = 1, cudaErrorHostMemoryAlreadyRegistered = 712 };
enum { cudaHostRegisterDefault = 0 };
#define __grid_constant__
typedef struct EmuStream *cudaStream_t;
typedef struct EmuEvent *cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaHostAllocDefault = 0, cudaHostAllocMapped = 2, cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaEventDefault = 0 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9 };
struct cudaDeviceProp { char name[256]; int major, minor, multiProcessorCount; size_t totalGlobalMem; size_t sharedMemPerBlockOptin; };

cudaError_t cudaGetDeviceCount(int *n);
cudaError_t cudaGetDevice(int *d);
cudaError_t cudaSetDevice(int d);
cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int d);
cudaError_t cudaDeviceSynchronize();
cudaError_t cudaDeviceGetStreamPriorityRange(int *lo, int *hi);
cudaError_t cudaStreamCreateWithPriority(cudaStream_t *s, unsigned flags, int prio);
cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned flags);
cudaError_t cudaStreamCreate(cudaStream_t *s);
cudaError_t cudaStreamDestroy(cudaStream_t s);
cudaError_t cudaStreamSynchronize(cudaStream_t s);
cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned flags);
cudaError_t cudaEventCreate(cudaEvent_t *e);
cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned flags);
cudaError_t cudaEventDestroy(cudaEvent_t e);
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s);
cudaError_t cudaEventSynchronize(cudaEvent_t e);
cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b);
cudaError_t cudaMalloc(void **p, size_t n);
cudaError_t cudaFree(void *p);
cudaError_t cudaHostAlloc(void **p, size_t n, unsigned flags);
cudaError_t cudaMallocHost(void **p, size_t n);
cudaError_t cudaFreeHost(void *p);
static inline cudaError_t cudaHostRegister(void *, size_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaHostGetDevicePointer(void **d, void *h, unsigned) { *d = h; return cudaSuccess; }
static inline cudaError_t cudaHostUnregister(void *) { return cudaSuccess; }
cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind k);
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind k, cudaStream_t st = nullptr);
cudaError_t cudaMemcpy2DAsync(void *d, size_t dpitch, const void *s, size_t spitch, size_t width, size_t height, cudaMemcpyKind k, cudaStream_t st = nullptr);
cudaError_t cudaMemset(void *d, int v, size_t n);
cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t st = nullptr);
cudaError_t cudaGetLastError();
cudaError_t cudaPeekAtLastError();
const char *cudaGetErrorString(cudaError_t e);
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }

// kernel<<<grid, block, smem, stream>>>(args...) becomes EMU_LAUNCH(grid, block, smem, kernel(args...))
void emu_launch(unsigned grid, unsigned block, size_t smem_bytes, const std::function<void()> &body);
#define EMU_LAUNCH(grid, block, smem, ...) emu_launch((unsigned)(grid), (unsigned)(block), (size_t)(smem), [=]() { __VA_ARGS__; })     // (variadic: template arguments bring commas)
