// modeac_kernel.cu — Mode A/C demodulator (SURVEY.md section 8f row 2; reference demodulate2400AC, demod_2400.c:575-761).
//
// Runs only for contexts created with B200_CFG_MODE_AC (readsb --modeac), after the scan kernel of the same run:
// the reply detector needs the buffer's mean level and mean power (noise floor, demod_2400.c:580-581), i.e. the
// exact per-buffer sums the scan kernel produces, so it cannot share that kernel's single pass over the samples.
//
//   modeac_noise_kernel   one thread per reference buffer: the fp64 noise floor, once (not per position)
//   modeac_scan_kernel    stateless per position, like stage A: is there a well-formed reply whose F1 pulse starts here?
//                         Output is ONE BIT per position (1 KB per tile), so its size does not depend on the input:
//                         no candidate pool, no overflow, no repeat.
//   modeac_walk_kernel    the reference's sequential part, one warp per reference buffer (the skip state does not
//                         survive a buffer): greedy walk over the bit map (a reply hides the next 69 positions), then
//                         the lanes decode the accepted replies in parallel straight from the samples.
//   ac_prefix_kernel, ac_pack_kernel, modeac_stats_kernel   after stage B: the reply lists packed in buffer order, receiver statistics.
//
// Exactness notes: float products and divisions are single IEEE operations (--fmad=false keeps them un-fused), the
// sqrt(2) factors are fp64 exactly as the C expressions promote them, sqrt / sqrtf are the correctly rounded CUDA
// versions, `noise_level * f1f2_level` wraps in 32 bits like the reference's unsigned product, and
// (unsigned)((double)x + 0.5) of a non-negative float x is evaluated as trunc(x) + (x - trunc(x) >= 0.5), which is the
// same integer for every x (both subtractions are exact in fp32).
#include "common.h"
#include "device_utils.cuh"

#define AC_SKIP (20 * 87 / 25 + 1)   // positions hidden by an accepted reply (demod_2400.c:753 + the loop increment)

// ---- the reply detector, shared by the scan (magnitudes in shared memory) and the walk (samples from global memory) ----

struct SmemMag {              // m[k] = data[f1_sample + k]
    const uint16_t *m;
    __device__ __forceinline__ uint32_t operator()(int k) const { return m[k]; }
};

struct GlobalMag {
    const uint8_t *base;      // segment data index 0
    const uint16_t *lut;      // full 65536-entry table
    int64_t d;                // data index of f1_sample in the segment
    int64_t zero_end, data_end;
    bool is_mag;
    __device__ __forceinline__ uint32_t operator()(int k) const {
        const int64_t i = d + k;
        if (i < zero_end || i >= data_end) return 0;
        const uint32_t v = __ldg(reinterpret_cast<const uint16_t *>(base + 2 * i));
        return is_mag ? v : __ldg(&lut[v]);      // the table is symmetric in I and Q: the little-endian pair indexes it directly
    }
};

__device__ __forceinline__ uint32_t round_half_up(float x) {     // (unsigned)((double)x + 0.5), x >= 0
    const uint32_t r = (uint32_t)x;
    return r + ((x - (float)r) >= 0.5f ? 1u : 0u);
}

// demod_2400.c:630-672: F1 edge / quiet / level, clock phase, F2 edge / quiet / level.  j = f1_sample.
template <class M>
__device__ __forceinline__ bool ac_front(const M &m, uint32_t j, uint32_t noise_level, uint32_t *f1_clock_out, uint32_t *f1f2_out) {
    const uint32_t a0 = m(0), a1 = m(1), a2 = m(2);
    if (!(m(-1) < a0) || a2 > a0 || a2 > a1) return false;
    const uint32_t f1_level = (a0 + a1) / 2;
    if (noise_level * 2 > f1_level) return false;
    // :651-654 clock phase from the power that spilled into the second sample
    const float f1a = (float)a0 * (float)a0, f1b = (float)a1 * (float)a1;
    const float fraction = f1b / (f1a + f1b);
    const uint32_t f1_clock = round_half_up(25.0f * ((float)j + fraction * fraction));
    const int o2 = (int)((f1_clock + 87 * 14) / 25 - j);
    const uint32_t b0 = m(o2), b1 = m(o2 + 1), b2 = m(o2 + 2);
    if (!(m(o2 - 1) < b0) || b2 > b0 || b2 > b1) return false;
    const uint32_t f2_level = (b0 + b1) / 2;
    if (noise_level * 2 > f2_level) return false;
    *f1_clock_out = f1_clock;
    *f1f2_out = max(f1_level, f2_level);
    return true;
}

// demod_2400.c:674-731: thresholds, 20 bit cells, framing; returns the Mode A/C word or 0xffffffff.
template <class M>
__device__ __forceinline__ uint32_t ac_bits(const M &m, uint32_t j, uint32_t noise_level, uint32_t f1_clock, uint32_t f1f2) {
    const float midpoint = sqrtf((float)(noise_level * f1f2));            // :676, 32-bit wrap included
    const uint32_t signal_threshold = (uint32_t)((double)midpoint * 1.41421356237309504880 + 0.5);
    const uint32_t noise_threshold = (uint32_t)((double)midpoint / 1.41421356237309504880 + 0.5);
    uint32_t bits = 0, bad = 0, clock = f1_clock;
#pragma unroll 4
    for (int bit = 0; bit < 20; ++bit, clock += 87) {
        const int o = (int)(clock / 25 - j);
        const uint32_t s0 = m(o), s1 = m(o + 1), s2 = m(o + 2);
        bits <<= 1;
        if (s2 >= signal_threshold) bad = 1;                                   // noisy quiet period
        if (s0 >= signal_threshold || s1 >= signal_threshold) bits |= 1;
        else if (s0 > noise_threshold && s1 > noise_threshold) bad = 1;        // uncertain
    }
    if ((bits & 0x80020) != 0x80020 || (bits & 0x0101B) != 0 || bad) return 0xffffffffu;
    return ((bits & 0x40000) ? 0x0010 : 0) | ((bits & 0x20000) ? 0x1000 : 0) | ((bits & 0x10000) ? 0x0020 : 0) |      // :716-731
           ((bits & 0x08000) ? 0x2000 : 0) | ((bits & 0x04000) ? 0x0040 : 0) | ((bits & 0x02000) ? 0x4000 : 0) |
           ((bits & 0x00800) ? 0x0100 : 0) | ((bits & 0x00400) ? 0x0001 : 0) | ((bits & 0x00200) ? 0x0200 : 0) |
           ((bits & 0x00100) ? 0x0002 : 0) | ((bits & 0x00080) ? 0x0400 : 0) | ((bits & 0x00040) ? 0x0004 : 0) |
           ((bits & 0x00004) ? 0x0080 : 0);
}

// ---- noise floor per reference buffer --------------------------------------------------------------------------------
// `(unsigned)x` of the reference's noise floor as its x86-64 build evaluates it: gcc converts a double to a 32-bit unsigned
// through the 64-bit cvttsd2si, so the floor wraps modulo 2^32 below 2^63 and is 0 for NaN and beyond (0x8000000000000000
// truncated).  cvt.rzi.u32.f64 would clamp at 0xffffffff instead.  (An aarch64 build of the reference clamps too.)  The
// floor is never negative: the square root is NaN unless mean_power >= mean_level^2 >= 0.
__device__ __forceinline__ uint32_t u32_of_double_x86(double x) {
    return (x >= 0.0 && x < 9223372036854775808.0) ? (uint32_t)(uint64_t)x : 0u;
}

__global__ void modeac_noise_kernel(const AcScanParams P) {
    for (uint32_t si = blockIdx.x; si < P.n_segs; si += gridDim.x) {
        const Segment seg = P.segs[si];
        for (uint32_t b = threadIdx.x; b < seg.n_bufs; b += blockDim.x) {
            const uint32_t len = min(seg.buf_len, seg.npos - b * seg.buf_len);
            if (len == 0) { P.noise[seg.first_buf + b] = 0; continue; }       // empty buffer: nothing will ask for its noise floor
            const BufAcc &a = P.buf_acc[seg.first_buf + b];     // sum_signal_power may still be accumulating: not read
            const AcLevel lv = P.levels[seg.first_buf + b];
            double mean_level, mean_power;
            if (lv.mode == AC_LEVEL_GIVEN) { mean_level = lv.mean_level; mean_power = lv.mean_power; }
            else if (lv.mode == AC_LEVEL_FSUM) {                // `sum_level / nsamples`: a float division, widened afterwards (convert.c:243-249)
                const float2 f = P.fsum[lv.idx];
                mean_level = (double)(f.x / (float)len); mean_power = (double)(f.y / (float)len);
            } else {
                mean_level = (double)a.sum_level / 65536.0 / (double)len;            // convert.c:100-102
                mean_power = (double)a.sum_power / 65535.0 / 65535.0 / (double)len;  // convert.c:104-106
            }
            const double noise_stddev = sqrt(mean_power - mean_level * mean_level);           // demod_2400.c:580
            P.noise[seg.first_buf + b] = u32_of_double_x86((mean_power + noise_stddev) * 65535 + 0.5);   // :581
        }
    }
}

// ---- stateless scan: one bit per position ----------------------------------------------------------------------------
// Warp-autonomous, like the Mode S scan: one persistent CTA per SM shares the folded magnitude table; every warp claims scan
// tiles (2048 positions) from an atomic counter and works on them alone - no block barrier after the table is staged:
//   convert   the tile's samples (8 before, 104 after: m[-1] .. m[+75] of every position) -> magnitudes in the warp's own shared memory
//   window    16 positions per lane: the noise-independent part of the F1 test (rising edge, quiet third sample, demod_2400.c:630-640)
//             on packed 16-bit halves -> a bit per position; F2 must pass the same test 48 or 49 positions on -> 3 % candidates
//   front     the candidates 32 at a time: level against the buffer's noise floor, clock phase, F2 tests (:641-672) -> < 1 %
//   bits      those few: 20 bit cells against the thresholds, framing (:674-731) -> the position's bit in the map
// (A block-phased predecessor - load a quad, barrier, F1 tests, barrier, F2 / bit cells, barrier - needed more than twice the warp
// instructions per sample.)
#define AC2_WARPS 28
#define AC2_BEHIND 8
#define AC2_AHEAD 104
#define AC2_NMAG (AC2_BEHIND + SCAN_TILE + AC2_AHEAD)      // 2160 = 270 pieces of 8
#define AC2_Q2 64                                          // pooled over the tile and worked off 32 at a time (they are < 1 % of the positions)

struct AcWarpSmem {
    alignas(16) uint16_t mag[AC2_NMAG];      // mag[AC2_BEHIND + p] = magnitude at tile position p
    uint16_t edge[SCAN_TILE / 16 + 8];       // 16 positions per entry: bit i = position 16 e + i passes the edge / quiet-sample test
    uint16_t q1[512 + 32];                   // candidate positions (tile-relative, ascending): a chunk's, behind up to 31 left over
    uint4 q2[AC2_Q2];                        // survivors of the front tests waiting for their bit cells: position | buffer << 16, f1_sample, f1_clock, f1f2 level
    uint32_t bits[SCAN_TILE / 32];
};

struct Ac2Smem {
    uint16_t lut[128 * 128];
    AcWarpSmem w[AC2_WARPS];
};

__device__ __forceinline__ uint32_t ac_vmin2(uint32_t a, uint32_t b) { uint32_t d; asm("min.u16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }

__global__ void __launch_bounds__(AC2_WARPS * 32, 1) modeac_scan_kernel(const AcScanParams P) {
    extern __shared__ __align__(16) unsigned char ac_smem_raw[];
    Ac2Smem &S = *reinterpret_cast<Ac2Smem *>(ac_smem_raw);
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (P.ctl->overflow & OV_STAGE_A_FAILED) return;
    {   // the folded table, once per CTA
        const uint4 *src = reinterpret_cast<const uint4 *>(P.tables->lut_fold);
        uint4 *dst = reinterpret_cast<uint4 *>(S.lut);
        for (uint32_t i = tid; i < 128 * 128 * 2 / 16; i += AC2_WARPS * 32) dst[i] = src[i];
    }
    __syncthreads();          // the only block barrier
    AcWarpSmem &W = S.w[wid];
    const uint32_t lt = (1u << lane) - 1u;
    // A warp's tile costs it three dependent round trips to L2 / HBM before the first magnitude is there (claim, descriptor, samples),
    // which seven warps per scheduler do not hide: the NEXT tile is claimed while this one is worked on, the segment descriptor is kept
    // while the tiles stay in the segment (hundreds in a row), and the next tile's samples are asked into L2 half-way through this one.
    uint32_t tile = 0;
    if (lane == 0) tile = atomicAdd(&P.ctl->pad_[0], 1u);
    tile = __shfl_sync(FULLMASK, tile, 0);
    Segment seg;
    uint32_t seg_tile_end = 0;
    while (tile < P.n_tiles) {
        if (tile >= seg_tile_end) { seg = P.segs[P.tile_seg[tile] & ~TILE_QUAD_START]; seg_tile_end = seg.tile_begin + seg.n_tiles; }
        uint32_t tile_next = 0;
        if (lane == 0) tile_next = atomicAdd(&P.ctl->pad_[0], 1u);              // (waited for at the end of this tile)
        const uint32_t x0 = (tile - seg.tile_begin) * SCAN_TILE;               // tile coordinate x = data index + lead
        const uint32_t x_data_end = seg.lead + seg.npos + B200_TRAIL;
        const uint32_t x_zero_end = (seg.flags & SEG_HALO_ZERO) ? seg.lead + B200_TRAIL : seg.lead;
        const bool is_mag = seg.flags & SEG_MAG;
        __syncwarp();
        // ---- convert: magnitudes of tile coordinates [x0 - 8, x0 + 2048 + 104) ------------------------------------------
        if (x0 >= x_zero_end + AC2_BEHIND && x0 + SCAN_TILE + AC2_AHEAD <= x_data_end) {
            // a tile in the interior of the data (nearly all of them): no piece needs a bounds test
            // A sample is two bytes as uc8 IQ and two bytes as a magnitude: the input lands, asynchronously and all 4320 bytes at once
            // (one exposed memory latency per tile instead of one per pair of pieces), where its magnitudes belong, and is converted
            // in place - every lane reads back exactly the pieces it copied.  A magnitude hand-off is complete when it has landed.
            const uint8_t *src = seg.base + 2 * ((int64_t)x0 - AC2_BEHIND - (int64_t)seg.lead);
            bool convert = !is_mag;
            if (convert && P.mag_copy && x0 + SCAN_TILE + AC2_AHEAD <= seg.n_tiles * SCAN_TILE) {
                // uc8 IQ that the Mode S scan has been through: its magnitudes are there to be read (ScanParams::mag_copy)
                src = reinterpret_cast<const uint8_t *>(P.mag_copy + ((size_t)seg.tile_begin * SCAN_TILE + x0 - AC2_BEHIND));
                convert = false;
            }
            const uint32_t dst0 = (uint32_t)__cvta_generic_to_shared(W.mag);
            for (uint32_t c = lane; c < AC2_NMAG / 8; c += 32)
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst0 + c * 16), "l"(src + (size_t)c * 16) : "memory");
            asm volatile("cp.async.commit_group;" ::: "memory");
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            if (convert) {
#pragma unroll 3
                for (uint32_t c = lane; c < AC2_NMAG / 8; c += 32) {
                    const uint4 raw = *reinterpret_cast<const uint4 *>(&W.mag[c * 8]);
                    const uint32_t wv[4] = {raw.x, raw.y, raw.z, raw.w};
                    uint32_t m[8];
#pragma unroll
                    for (int i = 0; i < 4; i++) uc8_pair_to_mag(S.lut, wv[i], m[2 * i], m[2 * i + 1]);
                    uint4 packed;
                    packed.x = __byte_perm(m[0], m[1], 0x5410); packed.y = __byte_perm(m[2], m[3], 0x5410);
                    packed.z = __byte_perm(m[4], m[5], 0x5410); packed.w = __byte_perm(m[6], m[7], 0x5410);
                    *reinterpret_cast<uint4 *>(&W.mag[c * 8]) = packed;
                }
            }
        } else
        for (uint32_t c = lane; c < AC2_NMAG / 8; c += 32) {
            const int64_t xc = (int64_t)x0 - AC2_BEHIND + (int64_t)c * 8;
            uint32_t m[8];
            if (xc < 0 || xc + 8 <= (int64_t)x_zero_end || xc >= (int64_t)x_data_end) {
#pragma unroll
                for (int i = 0; i < 8; i++) m[i] = 0;
            } else {
                const uint4 raw = ldg_stream_u4(seg.base + 2 * (xc - (int64_t)seg.lead));
                const uint32_t wv[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    if (is_mag) { m[2 * i] = wv[i] & 0xffffu; m[2 * i + 1] = wv[i] >> 16; }
                    else uc8_pair_to_mag(S.lut, wv[i], m[2 * i], m[2 * i + 1]);
                }
                if (xc < (int64_t)x_zero_end || xc + 8 > (int64_t)x_data_end) {
#pragma unroll
                    for (int i = 0; i < 8; i++) if (xc + i < (int64_t)x_zero_end || xc + i >= (int64_t)x_data_end) m[i] = 0;
                }
            }
            uint4 packed;
            packed.x = __byte_perm(m[0], m[1], 0x5410); packed.y = __byte_perm(m[2], m[3], 0x5410);
            packed.z = __byte_perm(m[4], m[5], 0x5410); packed.w = __byte_perm(m[6], m[7], 0x5410);
            *reinterpret_cast<uint4 *>(&W.mag[c * 8]) = packed;
        }
        W.bits[lane] = 0; W.bits[lane + 32] = 0;
        __syncwarp();

        // position p of the tile = data index d_tile0 + p of the segment = f1_sample (d mod buf_len) of buffer d / buf_len
        const int64_t d_tile0 = (int64_t)x0 - (int64_t)seg.lead;
        const uint32_t bt = d_tile0 > 0 ? (uint32_t)d_tile0 / seg.buf_len : 0;     // buffer of the tile's first position
        const int64_t bt_d0 = (int64_t)bt * seg.buf_len;
        // the noise floors the tile's candidates are measured against: those of its first buffer and the next (a tile rarely reaches further),
        // asked for now instead of once per batch of candidates
        const uint32_t noise_b0 = bt < seg.n_bufs ? P.noise[seg.first_buf + bt] : 0u, noise_b1 = bt + 1 < seg.n_bufs ? P.noise[seg.first_buf + bt + 1] : 0u;
        auto noise_of = [&](uint32_t brel) { return brel == 0 ? noise_b0 : brel == 1 ? noise_b1 : P.noise[seg.first_buf + bt + brel]; };

        // ---- window: rising edge and quiet third sample (demod_2400.c:630-640: m[-1] < m[0], m[2] <= m[0], m[2] <= m[1]) for every
        //      position of the tile and the 64 after it, two positions per step on packed halves -> one bit each in W.edge.
        //      The F2 pulse of a reply whose F1 starts at p starts at p + 48 or p + 49 (f1_clock lies in [25 j, 25 j + 25], :651-660)
        //      and has to pass the very same three tests (:662-668): only positions with edge(p) && (edge(p+48) || edge(p+49)) can
        //      be replies - 3 % of the positions on receiver noise instead of 13 %, by bit arithmetic alone.
#pragma unroll 1
        for (uint32_t c = 0; c < SCAN_TILE / 512 + 1; c++) {
            if (c == SCAN_TILE / 512 && lane >= 4) break;                                     // look-ahead: 64 positions
            const uint32_t p0 = c * 512 + lane * 16;
            const uint4 *src = reinterpret_cast<const uint4 *>(&W.mag[p0]);                   // samples p0 - 8 .. p0 + 23
            const uint4 q0 = src[0], q1v = src[1], q2 = src[2], q3 = src[3];
            const uint32_t wv[16] = {q0.x, q0.y, q0.z, q0.w, q1v.x, q1v.y, q1v.z, q1v.w, q2.x, q2.y, q2.z, q2.w, q3.x, q3.y, q3.z, q3.w};
            // wv[4 + k] = (m[2k], m[2k+1]) relative to p0
            uint32_t acc2 = 0;
#pragma unroll
            for (int k = 7; k >= 0; k--) {
                const uint32_t bq = wv[4 + k];                                        // b: m[0] of both positions
                const uint32_t aq = __funnelshift_r(wv[3 + k], wv[4 + k], 16);        // a: m[-1]
                const uint32_t cq = __funnelshift_r(wv[4 + k], wv[5 + k], 16);        // c: m[1]
                const uint32_t eq = wv[5 + k];                                        // e: m[2]
                const uint32_t d1 = bq - ac_vmin2(aq, bq);                            // != 0  <=>  m[-1] < m[0]
                const uint32_t d2 = eq - ac_vmin2(eq, ac_vmin2(bq, cq));              // == 0  <=>  m[2] <= m[0] && m[2] <= m[1]
                const uint32_t okq = ac_vmin2(d1, 0x00010001u) & ~ac_vmin2(d2, 0x00010001u);
                acc2 = acc2 * 4u + okq;
            }
            W.edge[c * 32 + lane] = (uint16_t)((acc2 & 0xffffu) | (acc2 >> 15));
        }
        __syncwarp();
        tile_next = __shfl_sync(FULLMASK, tile_next, 0);
        if (tile_next < seg_tile_end) {    // the next tile's samples (same segment: its descriptor is at hand) on their way into L2
            const int64_t xn = (int64_t)(tile_next - seg.tile_begin) * SCAN_TILE - AC2_BEHIND - (int64_t)seg.lead;      // its first sample, as a data index
            if (xn >= B200_TRAIL && xn + AC2_NMAG <= (int64_t)seg.npos + B200_TRAIL) {      // (memory the interior path of that tile reads anyway)
                const uint32_t xt = (tile_next - seg.tile_begin) * SCAN_TILE;
                const uint8_t *pn = (!is_mag && P.mag_copy && xt + SCAN_TILE + AC2_AHEAD <= seg.n_tiles * SCAN_TILE)
                                        ? reinterpret_cast<const uint8_t *>(P.mag_copy + ((size_t)seg.tile_begin * SCAN_TILE + xt - AC2_BEHIND)) : seg.base + 2 * xn;
                asm volatile("prefetch.global.L2 [%0];" :: "l"(pn + lane * 128));
                if (lane < 2) asm volatile("prefetch.global.L2 [%0];" :: "l"(pn + 4096 + lane * 128));
            }
        }

        uint32_t n1 = 0, n2 = 0;           // candidates waiting in W.q1, front-test survivors waiting in W.q2
#pragma unroll 1
        for (uint32_t c = 0; c <= SCAN_TILE / 512; c++) {
            const bool last = c == SCAN_TILE / 512;
            if (!last) {
                // ---- candidates of this chunk, in order, behind those left over from the chunk before -----------------------
                const uint32_t p0 = c * 512 + lane * 16, e = c * 32 + lane;
                const uint32_t f2 = (uint32_t)W.edge[e + 3] | ((uint32_t)W.edge[e + 4] << 16);     // edge bits of p0 + 48 ...
                uint32_t mask = (uint32_t)W.edge[e] & (f2 | (f2 >> 1)) & 0xffffu;
                uint32_t tot;
                uint32_t off = n1 + warp_excl_scan(__popc(mask), lane, &tot);
                while (mask) { const uint32_t i = __ffs(mask) - 1; mask &= mask - 1; W.q1[off++] = (uint16_t)(p0 + i); }
                n1 += tot;
                __syncwarp();
            }
            // ---- front: level, clock phase, F2 (demod_2400.c:641-672), 32 candidates at a time (the rest waits for the next chunk) ----
            uint32_t r0 = 0;
            for (; r0 + 32 <= n1 || (last && r0 < n1); r0 += 32) {
                const bool has = r0 + lane < n1;
                const uint32_t p = has ? W.q1[r0 + lane] : 0;
                bool surv = false;
                uint32_t f1_clock = 0, f1f2 = 0, jj32 = 0, brel = 0;
                if (has) {
                    const int64_t d = d_tile0 + p;
                    if (d >= 0 && d < (int64_t)seg.npos) {
                        uint32_t b = bt;
                        int64_t jj = d - bt_d0;
                        while (jj >= (int64_t)seg.buf_len) { jj -= seg.buf_len; b++; }
                        if (jj >= 1) {                                       // f1_sample runs from 1 (demod_2400.c:612)
                            jj32 = (uint32_t)jj; brel = b - bt;
                            const uint32_t noise = noise_of(brel);
                            surv = ac_front(SmemMag{&W.mag[p + AC2_BEHIND]}, jj32, noise, &f1_clock, &f1f2);
                        }
                    }
                }
                const uint32_t bal = __ballot_sync(FULLMASK, surv);
                if (surv) W.q2[n2 + __popc(bal & lt)] = make_uint4(p | (brel << 16), jj32, f1_clock, f1f2);
                n2 += __popc(bal);
                __syncwarp();
                if (n2 >= 32) {            // bit cells of 32 pooled survivors
                    const uint4 e = W.q2[lane];
                    const uint32_t ep = e.x & 0xffffu;
                    if (ac_bits(SmemMag{&W.mag[ep + AC2_BEHIND]}, e.y, noise_of(e.x >> 16), e.z, e.w) != 0xffffffffu) atomicOr(&W.bits[ep >> 5], 1u << (ep & 31));
                    __syncwarp();
                    const uint4 mv = lane + 32 < n2 ? W.q2[lane + 32] : make_uint4(0, 0, 0, 0);
                    __syncwarp();
                    W.q2[lane] = mv;
                    n2 -= 32;
                    __syncwarp();
                }
            }
            if (r0 && r0 < n1) {           // fewer than 32 left: to the front of the queue
                const uint32_t keep = n1 - r0;
                const uint32_t v = lane < keep ? W.q1[r0 + lane] : 0;
                __syncwarp();
                if (lane < keep) W.q1[lane] = (uint16_t)v;
                n1 = keep;
            } else if (r0) n1 = 0;
            __syncwarp();
        }
        if (n2) {                          // the rest of the tile's survivors
            if (lane < n2) {
                const uint4 e = W.q2[lane];
                const uint32_t ep = e.x & 0xffffu;
                if (ac_bits(SmemMag{&W.mag[ep + AC2_BEHIND]}, e.y, noise_of(e.x >> 16), e.z, e.w) != 0xffffffffu) atomicOr(&W.bits[ep >> 5], 1u << (ep & 31));
            }
            __syncwarp();
        }
        // one bit per position of this scan tile
        uint32_t *dst = P.bitmap + (size_t)tile * (SCAN_TILE / 32);
        dst[lane] = W.bits[lane]; dst[lane + 32] = W.bits[lane + 32];
        tile = tile_next;
    }
}

// ---- the sequential part, one warp per reference buffer ---------------------------------------------------------------
__global__ void __launch_bounds__(256, 1) modeac_walk_kernel(const AcWalkParams P) {
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if (P.ctl->overflow & OV_STAGE_A_FAILED) return;
    for (uint32_t si = blockIdx.x; si < P.n_segs; si += gridDim.x) {
        const Segment seg = P.segs[si];
        const uint32_t stream_first_buf = P.segs[P.stream_seg_begin[seg.stream]].first_buf;
        const uint32_t *bits = P.bitmap + (size_t)seg.tile_begin * (SCAN_TILE / 32);    // bit x = tile coordinate x of the segment
        for (uint32_t b = wid; b < seg.n_bufs; b += nw) {
            const uint32_t len_b = min(seg.buf_len, seg.npos - b * seg.buf_len);
            if (len_b == 0) {       // an empty buffer (a frontend that had nothing to deliver): no positions, no tiles, no bit-map words
                if (lane == 0) P.ac_count[seg.first_buf + b] = 0;
                continue;
            }
            const uint32_t xa = seg.lead + b * seg.buf_len, xb = xa + len_b;
            const uint32_t w_first = xa >> 5, w_last = (xb - 1) >> 5;
            b200_modeac *out = P.ac_out + (size_t)(seg.first_buf + b) * P.per_buf_cap;
            uint32_t n = 0, next_ok = 0;
            // The map is nearly empty (a reply per 10 000 positions): a lane takes four words at a time (128 words = 4096 positions per
            // warp step) and the warp only looks closer when one of them is not zero.  The map of a segment starts at a tile boundary
            // and every tile has 64 words of its own, so groups of four words are aligned and never leave the segment's tiles.
            const uint32_t g_first = w_first >> 2, g_last = w_last >> 2;
            const uint4 *bits4 = reinterpret_cast<const uint4 *>(bits);
            uint4 grp_next = g_first + lane <= g_last ? bits4[g_first + lane] : make_uint4(0, 0, 0, 0);
            for (uint32_t g0 = g_first; g0 <= g_last; g0 += 32) {
                const uint32_t gi = g0 + lane;
                const uint4 grp = grp_next;
                grp_next = gi + 32 <= g_last ? bits4[gi + 32] : make_uint4(0, 0, 0, 0);
                if (!__any_sync(FULLMASK, (grp.x | grp.y | grp.z | grp.w) != 0)) continue;
                // words of the group outside the buffer, and the bits of its first / last word that belong to its neighbours, do not count
                auto clip = [&](uint32_t v, uint32_t wi) {
                    if (wi < w_first || wi > w_last) v = 0;
                    if (wi == w_first) v &= ~0u << (xa & 31);
                    if (wi == w_last && (xb & 31)) v &= (1u << (xb & 31)) - 1u;
                    return v;
                };
                const uint32_t wi0 = gi * 4;
                const uint32_t v0 = clip(grp.x, wi0), v1 = clip(grp.y, wi0 + 1), v2 = clip(grp.z, wi0 + 2), v3 = clip(grp.w, wi0 + 3);
                for (;;) {
                    // this lane's first position that is not hidden by the reply accepted before it (demod_2400.c:747: the next 69 are skipped)
                    auto first_in = [&](uint32_t v, uint32_t wi, uint32_t later) {
                        const uint32_t wx = wi * 32;
                        if (next_ok > wx) v = next_ok - wx >= 32 ? 0 : v & (~0u << (next_ok - wx));
                        return v ? wx + __ffs(v) - 1 : later;
                    };
                    const uint32_t mine = first_in(v0, wi0, first_in(v1, wi0 + 1, first_in(v2, wi0 + 2, first_in(v3, wi0 + 3, 0xffffffffu))));
                    const uint32_t bal = __ballot_sync(FULLMASK, mine != 0xffffffffu);
                    if (!bal) break;
                    const uint32_t pos = __shfl_sync(FULLMASK, mine, __ffs(bal) - 1);
                    if (lane == 0) { if (n < P.per_buf_cap) out[n].f1_sample = pos - xa; else atomicOr(&P.ctl->overflow, OV_MODEAC_CAP); }
                    n++;
                    next_ok = pos + AC_SKIP;
                }
            }
            n = min(n, P.per_buf_cap);
            __syncwarp();
            // decode the accepted replies, one per lane (the scan proved each of them well-formed)
            const uint32_t noise = P.noise[seg.first_buf + b];
            for (uint32_t k = lane; k < n; k += 32) {
                const uint32_t j = out[k].f1_sample;
                GlobalMag m;
                m.base = seg.base; m.lut = P.lut_full; m.d = (int64_t)b * seg.buf_len + j;
                m.zero_end = (seg.flags & SEG_HALO_ZERO) ? B200_TRAIL : 0; m.data_end = (int64_t)seg.npos + B200_TRAIL;
                m.is_mag = seg.flags & SEG_MAG;
                uint32_t f1_clock = 0, f1f2 = 0;
                ac_front(m, j, noise, &f1_clock, &f1f2);
                const uint32_t modeac = ac_bits(m, j, noise, f1_clock, f1f2);
                b200_modeac a;
                a.timestamp = seg.first_ts + (int64_t)b * seg.buf_len * 5 + (f1_clock + 87 * 14) / 5;          // demod_2400.c:745
                a.f1_sample = j; a.modeac = (uint16_t)modeac;
                a.buffer_idx = (uint16_t)(seg.first_buf + b - stream_first_buf);
                out[k] = a;
            }
            if (lane == 0) P.ac_count[seg.first_buf + b] = n;
        }
    }
}

// Exclusive prefix of the per-buffer reply counts (ac_pack_kernel packs the lists with it)
__global__ void __launch_bounds__(1024) ac_prefix_kernel(const uint32_t *count, uint32_t *prefix, uint32_t n, const RunCtl *ctl) {
    const uint32_t n_all = n;
    __shared__ uint32_t scratch[40];
    uint32_t base = 0;
    if (ctl->overflow & RUN_REPEAT_BITS) n = 0;
    for (uint32_t i0 = 0; i0 < n; i0 += blockDim.x) {
        const uint32_t i = i0 + threadIdx.x;
        const uint32_t v = i < n ? count[i] : 0;
        uint32_t total;
        const uint32_t ex = block_excl_scan(v, scratch, &total);
        if (i < n) prefix[i] = base + ex;
        base += total;
    }
    for (uint32_t i = n + threadIdx.x; i < n_all; i += blockDim.x) prefix[i] = base;
    if (threadIdx.x == 0) prefix[n_all] = base;
}

// Pack the per-buffer reply lists in buffer order (one block per buffer).
__global__ void ac_pack_kernel(const b200_modeac *ac_out, const uint32_t *count, const uint32_t *prefix, b200_modeac *packed, uint32_t cap, const RunCtl *ctl) {
    if (ctl->overflow & RUN_REPEAT_BITS) return;          // the walk did not run (this step is going to be repeated): its counts are not this run's
    const uint32_t s = blockIdx.x;
    const uint32_t n = min(count[s], cap), base = prefix[s];
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) packed[base + i] = ac_out[(size_t)s * cap + i];
}

// after the count prefix: receiver statistics (the only state Mode A/C touches; skipped with the rest of stage B on a failed run)
__global__ void modeac_stats_kernel(const AcWalkParams P, const uint32_t *prefix) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= P.n_streams || (P.ctl->overflow & (RUN_REPEAT_BITS | OV_MODEAC_CAP))) return;
    const uint32_t sb = P.stream_seg_begin[s], se = P.stream_seg_begin[s + 1];
    if (sb == se) return;
    const uint32_t b0 = P.segs[sb].first_buf, b1 = P.segs[se - 1].first_buf + P.segs[se - 1].n_bufs;
    P.state[s].stats.demod_modeac += prefix[b1] - prefix[b0];
}

extern "C" int b200_prepare_modeac(void) {      // per device, from b200_demod_create
    return (int)cudaFuncSetAttribute(modeac_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Ac2Smem));
}

extern "C" int b200_launch_modeac(const AcScanParams *sp, const AcWalkParams *wp, int n_sm, void *stream) {
    if (sp->n_segs) {       // also for a run of empty buffers only (no tiles): the walk is what sets every buffer's reply count, zero included
        modeac_noise_kernel<<<min(sp->n_segs, 1024u), 32, 0, (cudaStream_t)stream>>>(*sp);
        if (sp->n_tiles) {
            uint32_t grid = (uint32_t)n_sm;               // one persistent CTA per SM, its warps claim scan tiles
            const uint32_t need = (sp->n_tiles + AC2_WARPS - 1) / AC2_WARPS;
            if (grid > need) grid = need;
            modeac_scan_kernel<<<grid, AC2_WARPS * 32, sizeof(Ac2Smem), (cudaStream_t)stream>>>(*sp);
        }
        modeac_walk_kernel<<<wp->n_segs, 256, 0, (cudaStream_t)stream>>>(*wp);
    }
    return (int)cudaGetLastError();
}

// After the Mode S stage B of the same step, on its stream: the walk's per-buffer reply lists -> one packed array in buffer order
// (prefix, pack), then the receiver statistics.  Three launches.
extern "C" int b200_launch_modeac_pack(const AcWalkParams *wp, uint32_t n_bufs, uint32_t *prefix, b200_modeac *packed, void *stream) {
    ac_prefix_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(wp->ac_count, prefix, n_bufs, wp->ctl);
    if (n_bufs) ac_pack_kernel<<<n_bufs, 32, 0, (cudaStream_t)stream>>>(wp->ac_out, wp->ac_count, prefix, packed, wp->per_buf_cap, wp->ctl);
    modeac_stats_kernel<<<(wp->n_streams + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*wp, prefix);
    return (int)cudaGetLastError();
}
