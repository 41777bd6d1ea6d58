// device_utils.cuh — small device helpers shared by the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define WARP 32
#define FULLMASK 0xffffffffu

// 16-byte streaming load: read-only path, do not keep the line in L1 (every IQ byte is read once).
__device__ __forceinline__ uint4 ldg_stream_u4(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// prmt.b32 in its default mode: selector nibble bit 3 replicates the sign of the selected byte
// (the __byte_perm intrinsic masks that bit away).
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
    return d;
}

// Two uc8 IQ pairs (bytes I0 Q0 I1 Q1 of w) -> two magnitudes through the folded, bank-swizzled 128x128 table in shared
// memory (modes_tables.h; convert.c:35-62 is symmetric about 127.5 in both I and Q).
__device__ __forceinline__ void uc8_pair_to_mag(const uint16_t *lut_smem, uint32_t w, uint32_t &m0, uint32_t &m1) {
    const uint32_t sgn = prmt(w, 0, 0xba98);                // 0xff where the byte is >= 128
    const uint32_t f = (w ^ sgn) & 0x7f7f7f7fu;             // fold: v>=128 ? 255-v : v  (127 = centre, 0 = full scale; one LOP3)
    uint32_t off = f + (f & 0x007f007fu);                   // per half: fq*256 + 2*fi
    off ^= (f >> 5) & 0x00780078u;                          // bank swizzle
    m0 = *reinterpret_cast<const uint16_t *>(reinterpret_cast<const uint8_t *>(lut_smem) + (off & 0xffffu));
    m1 = *reinterpret_cast<const uint16_t *>(reinterpret_cast<const uint8_t *>(lut_smem) + (off >> 16));
}

// acc += a * b with a single IMAD.WIDE (32x32 -> 64 accumulate)
__device__ __forceinline__ void mad_wide(unsigned long long &acc, uint32_t a, uint32_t b) {
    asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc) : "r"(a), "r"(b));
}

__device__ __forceinline__ uint32_t warp_excl_scan(uint32_t v, uint32_t lane, uint32_t *total) {
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < WARP; o <<= 1) {
        uint32_t y = __shfl_up_sync(FULLMASK, x, o);
        if (lane >= (uint32_t)o) x += y;
    }
    *total = __shfl_sync(FULLMASK, x, WARP - 1);
    return x - v;
}

// Exclusive prefix sum over the block (all threads must call). scratch: >= 33 uint32 of shared memory.
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t *scratch, uint32_t *total) {
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    uint32_t wtot;
    uint32_t ex = warp_excl_scan(v, lane, &wtot);
    __syncthreads();                       // protect scratch reuse from a previous call
    if (lane == 0) scratch[wid] = wtot;
    __syncthreads();
    if (wid == 0) {
        uint32_t t = lane < nw ? scratch[lane] : 0, tt;
        uint32_t e = warp_excl_scan(t, lane, &tt);
        if (lane < nw) scratch[lane] = e;
        if (lane == 0) scratch[32] = tt;
    }
    __syncthreads();
    *total = scratch[32];
    return ex + scratch[wid];
}
