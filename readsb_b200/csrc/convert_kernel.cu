// convert_kernel.cu — the float-path IQ converters (SURVEY.md section 8f row 3): convert_sc16_nodc convert.c:212-250 and
// convert_sc16q11_nodc convert.c:329-367 (the default build has no SC16Q11 table), for bladeRF / Pluto / Soapy style input.
//
// One launch converts a whole step: every receiver's buffers (and, for a continued receiver, its 326-sample halo) into
// uint16 magnitudes, and every buffer's two float sums.
//
//   magnitudes   exactly the reference's float expression (I / 32768 or I / 2048 is an exact scaling, the two products and
//                their sum are rounded separately — the library is built with --fmad=false —, sqrtf is correctly rounded,
//                * 65535 + 0.5 are two operations).  A pure function of the sample, so a halo converted again from the raw
//                halo equals the magnitudes the previous step made of the same samples.
//   sums         the reference returns mean_level / mean_power of these formats from FLOAT accumulators added to in sample
//                order (convert.c:225,238-239).  A float sum is not associative, so each buffer's two sums are two dependent
//                chains of adds in sample order; a parallel reduction would give other bits.
//
// A CTA owns SC16_GROUP buffers of equal length and walks them in blocks of SC16_BLOCK samples.  Its eight worker warps
// convert block k data parallel (coalesced 4-byte loads and 2-byte stores; the loads of block k+1 are issued before block k
// is converted) and stage each sample's float mag / magsq in shared memory; meanwhile lane 2j / 2j+1 of the ninth warp adds
// block k-1's staged values of buffer j to its level / power sum.  One warp instruction thus advances 32 chains, and the
// chains of all buffers of a step run at the same time: the step pays one chain of buf_len dependent adds (about
// 4 cycles each), not one per buffer.
#include "common.h"
#include "device_utils.cuh"

#define SC16_GROUP   16                          // buffers per CTA: two chains each in the summing warp
#define SC16_BLOCK   512                         // samples per buffer and block
#define SC16_ROW     (SC16_BLOCK + 4)            // staged floats per chain: +4 keeps the summing warp's 16-byte reads conflict-free
#define SC16_WORKERS 256
#define SC16_PER_THREAD (SC16_GROUP * SC16_BLOCK / SC16_WORKERS)
#define SC16_SMEM    (2 * 2 * SC16_GROUP * SC16_ROW * (int)sizeof(float))    // two blocks in turn

__device__ __forceinline__ void sc16_sample(uint32_t iq, float scale, float &mag, float &magsq) {
    const float fI = (float)(int16_t)(iq & 0xffffu) * scale, fQ = (float)(int16_t)(iq >> 16) * scale;   // I / 32768.0f resp. I / 2048.0f: exact
    const float a = fI * fI, b = fQ * fQ;
    magsq = a + b;
    if (magsq > 1.0f) magsq = 1.0f;
    mag = sqrtf(magsq);
}

__device__ __forceinline__ uint16_t sc16_mag_u16(float mag) {
    const float scaled = mag * 65535.0f;
    return (uint16_t)(scaled + 0.5f);
}

// The segment that holds buffer g (the last one whose first_buf <= g): receivers present in the step hold one segment each, in order.
__device__ __forceinline__ const Segment &sc16_seg(const Sc16Params &P, uint32_t i) { return P.n_segs == 1 ? P.seg0 : P.segs[i]; }

__global__ void __launch_bounds__(SC16_WORKERS + 32, 1) sc16_convert_kernel(const __grid_constant__ Sc16Params P) {
    extern __shared__ __align__(16) float sc16_stage[];       // [2][2 * SC16_GROUP][SC16_ROW]
    __shared__ uint32_t grp_seg[SC16_GROUP];                  // segment of buffer g0 + j
    const uint32_t tid = threadIdx.x;
    const uint32_t nbuf = P.n_bufs, g0 = blockIdx.x * SC16_GROUP;
    const uint32_t n_here = min((uint32_t)SC16_GROUP, nbuf - g0);
    if (tid < n_here) {
        uint32_t lo = 0, hi = P.n_segs;                       // invariant: first_buf(lo) <= g < first_buf(hi)
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) / 2; if (sc16_seg(P, mid).first_buf <= g0 + tid) lo = mid; else hi = mid; }
        grp_seg[tid] = lo;
    }
    __syncthreads();

    // halos of the continued receivers whose first buffer is in this CTA: converted, not summed
    for (uint32_t j = 0; j < n_here; j++) {
        const Segment &sg = sc16_seg(P, grp_seg[j]);
        if (sg.first_buf != g0 + j || (sg.flags & SEG_HALO_ZERO)) continue;
        const uint32_t *in = P.iq + sg.stream * P.iq_stride - B200_TRAIL;
        uint16_t *out = P.mag + sg.stream * P.mag_stride;
        for (uint32_t i = tid; i < B200_TRAIL; i += blockDim.x) {
            float mag, magsq;
            sc16_sample(in[i], P.scale, mag, magsq);
            out[i] = sc16_mag_u16(mag);
        }
    }

    const uint32_t n_blocks = (P.buf_len + SC16_BLOCK - 1) / SC16_BLOCK;
    if (tid < SC16_WORKERS) {
        // item r of this thread: buffer r / 2 of the group, sample tid + 256 * (r & 1) of the block
        const uint32_t *src[SC16_GROUP];
        uint16_t *dst[SC16_GROUP];
#pragma unroll
        for (int j = 0; j < SC16_GROUP; j++) {
            const uint32_t jj = min((uint32_t)j, n_here - 1);
            const Segment &sg = sc16_seg(P, grp_seg[jj]);
            const uint32_t s = sg.stream, b = g0 + jj - sg.first_buf;
            src[j] = P.iq + s * P.iq_stride + (size_t)b * P.buf_len;
            dst[j] = P.mag + s * P.mag_stride + B200_TRAIL + (size_t)b * P.buf_len;
        }
        uint32_t nxt[SC16_PER_THREAD];
        auto load = [&](uint32_t k) {
#pragma unroll
            for (int r = 0; r < SC16_PER_THREAD; r++) {
                const uint32_t i = k * SC16_BLOCK + tid + SC16_WORKERS * (r & 1);
                nxt[r] = ((uint32_t)(r >> 1) < n_here && i < P.buf_len) ? __ldg(src[r >> 1] + i) : 0u;
            }
        };
        load(0);
        for (uint32_t k = 0; k <= n_blocks; k++) {
            if (k < n_blocks) {
                uint32_t cur[SC16_PER_THREAD];
#pragma unroll
                for (int r = 0; r < SC16_PER_THREAD; r++) cur[r] = nxt[r];
                if (k + 1 < n_blocks) load(k + 1);
                float *stage = sc16_stage + (k & 1) * (2 * SC16_GROUP * SC16_ROW);
#pragma unroll
                for (int r = 0; r < SC16_PER_THREAD; r++) {
                    // every item, also of absent buffers: a guard between the items costs the full groups more than it saves
                    const uint32_t x = tid + SC16_WORKERS * (r & 1), i = k * SC16_BLOCK + x;
                    float mag, magsq;
                    sc16_sample(cur[r], P.scale, mag, magsq);       // a missing sample is (0, 0): 0 + 0.0f leaves a sum as it is
                    if ((uint32_t)(r >> 1) < n_here && i < P.buf_len) dst[r >> 1][i] = sc16_mag_u16(mag);
                    stage[(2 * (r >> 1)) * SC16_ROW + x] = mag;
                    stage[(2 * (r >> 1) + 1) * SC16_ROW + x] = magsq;
                }
            }
            __syncthreads();
        }
    } else {
        const uint32_t lane = tid - SC16_WORKERS;            // chain: buffer lane / 2, level (even lane) or power (odd lane)
        float sum = 0.0f;
        for (uint32_t k = 0; k <= n_blocks; k++) {
            if (k > 0) {
                const float4 *row = reinterpret_cast<const float4 *>(sc16_stage + ((k - 1) & 1) * (2 * SC16_GROUP * SC16_ROW) + lane * SC16_ROW);
#pragma unroll 16
                for (int q = 0; q < SC16_BLOCK / 4; q++) {
                    const float4 v = row[q];
                    sum += v.x; sum += v.y; sum += v.z; sum += v.w;
                }
            }
            __syncthreads();
        }
        if (lane / 2 < n_here) {
            float *out = reinterpret_cast<float *>(P.sums + (size_t)(g0 + lane / 2) * P.sums_stride);
            out[lane & 1] = sum;
        }
    }
}

extern "C" int b200_prepare_convert(void) {      // per device, from b200_demod_create
    return (int)cudaFuncSetAttribute(sc16_convert_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SC16_SMEM);
}

extern "C" int b200_launch_sc16_convert(const Sc16Params *p, void *stream) {
    const uint32_t nbuf = p->n_bufs;
    if (!nbuf || !p->buf_len) return 0;
    sc16_convert_kernel<<<(nbuf + SC16_GROUP - 1) / SC16_GROUP, SC16_WORKERS + 32, SC16_SMEM, (cudaStream_t)stream>>>(*p);
    return (int)cudaGetLastError();
}
