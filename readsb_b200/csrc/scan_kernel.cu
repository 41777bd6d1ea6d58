// scan_kernel.cu — stage A of the Mode-S demodulator, warp-autonomous version: the stateless, data-parallel part of
// demodulate2400() as one persistent sm_90a kernel in which EVERY WARP owns whole tiles and never meets a block barrier.
//
// One CTA per SM shares the read-only tables (folded uc8 magnitude table 32 KB, CRC table, single-bit syndromes); each of
// its warps pulls tiles of SCAN_TILE positions from an atomic counter and walks them in chunks of 512 positions
// (16 per lane) through a private shared-memory pipeline:
//
//     iteration k:   window(k)        pre-check of the chunk's 512 positions + the TICK MAP of its 512 samples
//                    stage(k+2)       cp.async of the chunk's 1 KB of input into the warp's staging area, in flight during ...
//                    candidates(k-1)  thresholds -> DF gate -> full slice + CRC + classification -> ordered emission
//                    convert(k+2)     staged bytes -> magnitudes through the folded table into the ring, exact per-buffer sums
//
// window(k) needs the first samples of chunk k+1, candidates(k-1) need ticks up to 310 samples ahead (chunk k) and
// magnitudes 18 ahead: a ring of three magnitude chunks and two tick chunks per warp (4.8 KB) holds exactly that.  The
// warps of an SM drift apart, so table lookups (LSU), tick arithmetic (ALU / IDP) and candidate work of different
// warps overlap instead of marching through block-wide phases; nothing waits for the slowest warp of a CTA.
//
// A warp takes RUNS of consecutive tiles (guided self-scheduling: long runs first, single tiles at the end, so the last
// warps finish together) and keeps its pipeline going across tile boundaries: the look-ahead chunk is paid once per run.
// Full slices are rare (1-2 per 512 positions) and expensive, so they are deferred and pooled over the run: DF-gate
// survivors queue up until 32 lanes have work; the ticks they need are kept in a per-warp global copy (L2 resident).
//
// Output per tile is unchanged (PosEntry list in pos_pool, live records contiguous in rec_pool, TileOut): a warp stages
// the live records of its run in a small private global area and copies them to one reservation at the end of the run.
//
// No tensor cores: integer scan/correlate work bounded by HBM reads and instruction issue.
#include "common.h"
#include "device_utils.cuh"

#define SC_WARPS 28
#define SC_MAXNREG 72                         // SC_WARPS x 32 x SC_MAXNREG <= 65536 registers per SM (other splits were slower: DESIGN.md §4, "Tried and NOT in the code")
#define CHUNK 512
#define TILE_CHUNKS (SCAN_TILE / CHUNK)       // 4 chunks of positions per tile
#define RUN_MAX 8                             // a warp takes runs of up to 8 consecutive tiles of one segment (guided self-scheduling)
#define RUN_CHUNKS_MAX (RUN_MAX * TILE_CHUNKS)
#define MAG_RING (3 * CHUNK)
#define MAG_MIRROR 64                         // first samples of slot 0 again behind slot 2: reads never wrap
#define TICK_CW (5 * CHUNK / 32)              // 80 words of ticks per chunk
#define TICK_BITS (5 * CHUNK)
#define TICK_RING (2 * TICK_CW)
#define TICK_MIRROR 12
#define Q1_SMEM 128                           // pre-check passers of a chunk kept in shared memory (58 on receiver noise); the rest (dense input) spills to global memory
#define SURV_CAP 64
#define TICKG_WORDS ((RUN_CHUNKS_MAX + 1) * TICK_CW + 8)   // per-warp global copy of a whole run's ticks (slicing is deferred and pooled)

// Per-run scalars, identical in every lane; kept in shared memory so that the register budget goes to the window pass.
struct RunCtx {
    const uint8_t *tile_base;      // byte address of run coordinate 0 (= tile coordinate x0 of the segment)
    long long n_first;             // new-sample index of run coordinate 0
    long long bound;               // first new sample of the reference buffer after buffer nb
    uint32_t x0, x_zero_end, x_data_end;
    uint32_t p_lo, p_hi;           // run-relative positions that are preamble starts of the segment
    uint32_t buf_len, first_buf, npos;
    uint32_t n_chunks;             // chunks of positions; chunk n_chunks is look-ahead only
    uint32_t nb;                   // reference buffer of the chunk being converted, tracked incrementally
    uint32_t is_mag, last_tile;
    uint32_t tile0, n_tiles;
    uint32_t tile_rel0;            // tile0 - seg.tile_begin: stage B walks quads of tiles, PosEntry positions are quad-relative
    uint32_t sub_off;              // run coordinate 0 inside its tile (0 unless the tile is shared between warps, see finish_shared_tile)
};

struct WarpSmem {
    alignas(16) uint16_t mag[MAG_RING + MAG_MIRROR];
    alignas(16) uint8_t raw[2 * CHUNK];       // the next chunk's input bytes, landed here by cp.async while the candidates are worked on
    uint32_t tick[TICK_RING + TICK_MIRROR];   // tick of sample s (chunk-local) and row r at bit 5 s + r of the chunk's slot
    uint16_t q1[Q1_SMEM];                     // pre-check passers of the previous chunk (chunk-local positions, ascending)
    uint32_t pass[32];                        // threshold passers waiting for their DF gates: chunk-local position | tried << 16
    uint32_t surv[SURV_CAP];                  // DF-gate survivors waiting for a full slice: run position | ph << 14 | long << 17 | PosEntry index << 18
    uint32_t seg[16];                         // the run's Segment
    uint32_t n_pos[RUN_MAX], n_rec[RUN_MAX];  // per tile of the run
    // L2 eviction policies: the input is read once (evict first); the warp's tick copy and record staging are rewritten run after
    // run and should stay in L2 instead of being written back to HBM behind the input stream (evict last)
    unsigned long long pol_stream, pol_keep;
    RunCtx ctx;
};

struct ScanSmem {                             // the read-only tables every warp of the CTA shares
    uint16_t lut[128 * 128];                  // folded, bank-swizzled UC8 magnitude table
    uint32_t crc_tab[256];
    uint32_t bit_syn[112];
    uint32_t syn_hash[512];
    uint32_t syn_mul;
    uint32_t pad_[3];
};

struct ScanSmemFull {
    ScanSmem t;
    WarpSmem w[SC_WARPS];
};

__device__ __forceinline__ void stg_keep(uint32_t *p, uint32_t v, unsigned long long policy) {
    asm volatile("st.global.L2::cache_hint.b32 [%0], %1, %2;" :: "l"(p), "r"(v), "l"(policy) : "memory");
}

// packed unsigned 16-bit min / max (VIMNMX.U16x2): two magnitudes per instruction
__device__ __forceinline__ uint32_t vmin2(uint32_t a, uint32_t b) { uint32_t d; asm("min.u16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }
__device__ __forceinline__ uint32_t vmax2(uint32_t a, uint32_t b) { uint32_t d; asm("max.u16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }

// mixed-sign two-way dot products: a = two unsigned 16-bit magnitudes, b = four signed 8-bit coefficients
__device__ __forceinline__ int dp2a_lo(uint32_t a, uint32_t b, int c) {
    int d;
    asm("dp2a.lo.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ int dp2a_hi(uint32_t a, uint32_t b, int c) {
    int d;
    asm("dp2a.hi.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// crc.c:383-406 for nfix_crc = 1: message bit (>= 5) whose single-bit syndrome equals `syn`, or -2.
__device__ __forceinline__ int diagnose1(const ScanSmem &S, uint32_t syn, int bits) {
    uint32_t e = S.syn_hash[(syn * S.syn_mul) >> 23];
    if ((e >> 8) != syn) return -2;
    int b = (int)(e & 0xffu) - (112 - bits);
    return b >= 5 ? b : -2;
}

// Filter-independent part of scoreModesMessage (mode_s.c:309-419) for a fully sliced frame with syndrome `crc`.
// Returns RecKind, or 0 when the score is -2 whatever the filter holds.
__device__ __forceinline__ uint32_t classify(const ScanSmem &S, const ScanParams &P, const uint32_t w[4], int df, bool is_long,
                                             uint32_t crc, uint32_t *addr_out, int *fixbit_out) {
    const uint32_t aa = w[0] & 0xffffffu;
    *fixbit_out = -1;
    *addr_out = 0;
    if (is_long) {
        if (P.fixdf && P.nfix && (df == 1 || df == 25 || df == 21 || df == 19 || df == 16)) {
            // fixDF17msgtype (mode_s.c:276-301): forcing DF=17 flips exactly one DF bit, so the repaired
            // frame is CRC-clean iff the syndrome equals that bit's single-bit syndrome.
            const int bit = __clz((uint32_t)(df ^ 17)) - 27;     // 16->0, 8->1, 4->2, 2->3, 1->4
            if (crc == S.bit_syn[bit]) { *addr_out = aa; *fixbit_out = bit; return K_DFREPAIR; }
        }
        if (df == 16 || df == 20 || df == 21) { *addr_out = crc; return K_AP; }
        if (df == 17 || df == 18) {
            if (crc == 0) { *addr_out = aa; return K_ES_OK; }
            if (!P.nfix) return 0;
            const int b = diagnose1(S, crc, 112);
            if (b < 0) return 0;
            *fixbit_out = b;
            *addr_out = (b >= 8 && b <= 31) ? (aa ^ (1u << (31 - b))) : aa;   // correct_aa_field, mode_s.c:230-245
            return K_ES_FIX;
        }
        return 0;   // DF1/19/25 without a repair: unknown message type
    }
    // short frames; all-zero check mode_s.c:336-338 (only DF0 can start with a zero byte)
    if (w[0] == 0 && (w[1] >> 8) == 0) return 0;
    if (df == 11) {
        if (crc & 0xffff80u) {
            if (!P.nfix) return 0;
            const int b = diagnose1(S, crc, 56);
            if (b < 0) return 0;
            *fixbit_out = b;
            *addr_out = (b >= 8 && b <= 31) ? (aa ^ (1u << (31 - b))) : aa;
            return K_DF11_FIX;
        }
        *addr_out = aa;
        return (crc & 0x7fu) ? K_DF11_IID : K_DF11_IID0;
    }
    *addr_out = crc;   // DF0/4/5
    return K_AP;
}

// Ticks at stride 12 -> adjacent bits, earliest tick in the most significant position.
__device__ __forceinline__ uint32_t gather3(uint32_t x) {   // ticks 0, 12, 24 of x -> 3 bits
    return (((x & 0x01001001u) * 0x04002001u) >> 24) & 7u;
}
__device__ __forceinline__ uint32_t gather2(uint32_t x) {   // ticks 0, 12 of x -> 2 bits
    return (((x & 0x00001001u) * 0x00002001u) >> 12) & 3u;
}

// Thresholds of the three preamble correlations at pa = &mag[position] (demod_2400.c:330-378): phases to try.
__device__ __forceinline__ uint32_t threshold_phases(const uint16_t *pa, int thr) {
    const int base_noise = pa[5] + pa[8] + pa[16] + pa[17] + pa[18];
    const int ref_level = (base_noise * thr) >> 5;
    const int d23 = (int)pa[2] - (int)pa[3], s14 = pa[1] + pa[4], d1011 = (int)pa[10] - (int)pa[11];
    const int common = s14 - d23 + pa[9] + pa[12];
    uint32_t tried = 0;
    if (common - d1011 >= ref_level) tried |= 0x03;                        // try_phase 4, 5
    if (common + d1011 >= ref_level) tried |= 0x0c;                        // try_phase 6, 7
    if (s14 + 2 * d23 + d1011 + pa[12] >= ref_level) tried |= 0x10;        // try_phase 8
    return tried;
}

// Ring bit index of the first message tick of (chunk-local position pl, try_phase 4 + ph) for a chunk whose ticks sit in
// slot `tslot`: the closed form of slice_byte (demod_2400.c:133-213): PPM bit k is the tick 5 (p + 19) + 4 + ph + 12 k.
__device__ __forceinline__ uint32_t first_tick(uint32_t tslot, uint32_t pl, uint32_t ph) {
    uint32_t B = tslot * TICK_BITS + 5u * (pl + 19u) + 4u + ph;
    if (B >= 2 * TICK_BITS) B -= 2 * TICK_BITS;
    return B;
}

// DF gate (demod_2400.c:222-239): the five DF ticks starting at ring bit B -> keep | long << 1.
__device__ __forceinline__ uint32_t df_gate(const WarpSmem &W, const ScanParams &P, uint32_t B) {
    const uint32_t *t = &W.tick[B >> 5];
    const uint32_t sh = B & 31u, a = t[0], b = t[1], c = t[2];
    const uint32_t lo = __funnelshift_r(a, b, sh), hi = __funnelshift_r(b, c, sh);     // bit k at tick 12k: 0, 12, 24, 36, 48
    const uint32_t df = (gather3(lo) << 2) | gather2(hi >> 4);
    const uint32_t is_long = (P.long_set >> df) & 1u;
    return (is_long | ((P.short_set >> df) & 1u)) | (is_long << 1);
}

// Full slice of one (position, phase) from the warp's global tick copy (bit B = first message tick, linear over the run):
// 8 message bits per 96 ticks, CRC by table, classification; fills rw[0..7] (a Rec).
// Returns the RecKind (0 = score -2 regardless of the filter).
__device__ __forceinline__ uint32_t slice_and_classify(const ScanSmem &S, const uint32_t *tickg, const ScanParams &P, uint32_t B, bool is_long, uint32_t rw[8]) {
    const int nbytes = is_long ? 14 : 7;
    uint32_t w[4] = {0, 0, 0, 0}, rem = 0, tail = 0;
    // A message byte is 96 ticks = exactly three words further on than the one before, at the same bit offset: seven bytes need 22
    // consecutive words.  They are loaded together (one L2 round trip per half frame instead of one per byte), then the bytes are cut out.
    const uint32_t *t = &tickg[B >> 5];
    const uint32_t sh = B & 31u;
#pragma unroll
    for (int half = 0; half < 2; half++) {
        if (half == 1 && !is_long) break;
        uint32_t tw[22];
#pragma unroll
        for (int k = 0; k < 22; k++) tw[k] = __ldcg(t + 21 * half + k);
#pragma unroll
        for (int i = 0; i < 7; i++) {
            const int by = 7 * half + i;
            const uint32_t x0 = __funnelshift_r(tw[3 * i], tw[3 * i + 1], sh), x1 = __funnelshift_r(tw[3 * i + 1], tw[3 * i + 2], sh),
                           x2 = __funnelshift_r(tw[3 * i + 2], tw[3 * i + 3], sh);
            // message bits at ticks 0,12,24 | 36,48,60 | 72,84 of this 96-tick group, MSB first
            const uint32_t byte = (gather3(x0) << 5) | (gather3(x1 >> 4) << 2) | gather2(x2 >> 8);
            w[by >> 2] |= byte << (24 - 8 * (by & 3));
            if (by < nbytes - 3) rem = ((rem << 8) ^ S.crc_tab[byte ^ ((rem >> 16) & 0xffu)]) & 0xffffffu;   // crc.c:74-77
            else tail = (tail << 8) | byte;
        }
    }
    const uint32_t syn = rem ^ tail;                                                                  // crc.c:79-80
    const int df = (int)(w[0] >> 27);
    uint32_t addr; int fixbit;
    const uint32_t kind = classify(S, P, w, df, is_long, syn, &addr, &fixbit);
    // bytes 0..13 = message, byte 14 = kind, byte 15 = fixbit (little-endian words, big-endian message)
    rw[0] = __byte_perm(w[0], 0, 0x0123); rw[1] = __byte_perm(w[1], 0, 0x0123); rw[2] = __byte_perm(w[2], 0, 0x0123);
    rw[3] = (__byte_perm(w[3], 0, 0x0123) & 0xffffu) | (kind << 16) | ((uint32_t)(fixbit & 0xff) << 24);
    rw[4] = syn; rw[5] = addr; rw[6] = 0; rw[7] = 0;
    return kind;
}

// Correlator rows (demod_2400.c:74-93) NEGATED and packed as four signed bytes (c0, c1, c2, c3):
// the sign bit of the negated correlation is exactly [correlation > 0].
#define NEG_ROW0 0x00030feeu   // -18,  15,   3,  0
#define NEG_ROW1 0x000905f2u   // -14,   5,   9,  0
#define NEG_ROW2 0x0014fbf0u   // -16,  -5,  20,  0
#define NEG_ROW3 0x0012f5f9u   //  -7, -11,  18,  0
#define NEG_ROW4 0xff14f1fcu   //  -4, -15,  20, -1

// Half of a lane's window: 8 consecutive positions / samples starting at W.mag[mi0] (24 magnitudes in registers).
// Returns the 8-bit pre-check mask; a0 / a1 receive the 40 ticks of the 8 samples (a0: ticks 0..31, a1: ticks 32..39, tick n at bit n).
__device__ __forceinline__ uint32_t half_window(const WarpSmem &W, uint32_t mi0, uint32_t &a0, uint32_t &a1) {
    const uint4 *src = reinterpret_cast<const uint4 *>(&W.mag[mi0]);
    const uint4 q0 = src[0], q1v = src[1], q2 = src[2];
    const uint32_t wv[12] = {q0.x, q0.y, q0.z, q0.w, q1v.x, q1v.y, q1v.z, q1v.w, q2.x, q2.y, q2.z, q2.w};
    // xs[j] = the pair (m[2j+1], m[2j+2]): the 16-bit-shifted view of the window, used by the pre-check and by the odd samples of the tick map
    uint32_t xs[11];
#pragma unroll
    for (int j = 0; j < 11; j++) xs[j] = __funnelshift_r(wv[j], wv[j + 1], 16);
    // pre-check (demod_2400.c:311-320): pa[1] > pa[7] && pa[12] > pa[14] && pa[12] > pa[15], two positions (2k, 2k+1) per step on
    // packed halves: a > b  <=>  a - min(a, b) != 0 (no borrow between the halves: min(a, b) <= a in each); both conditions hold
    // <=> the smaller of the two differences is not zero.
    uint32_t acc2 = 0;
#pragma unroll
    for (int k = 3; k >= 0; k--) {
        const uint32_t mx = vmax2(wv[k + 7], xs[k + 7]);             // max(pa[14], pa[15]) of both positions
        const uint32_t d2 = wv[k + 6] - vmin2(wv[k + 6], mx);         // pa[12] - min(pa[12], that)
        const uint32_t d1 = xs[k] - vmin2(xs[k], xs[k + 3]);          // pa[1] - min(pa[1], pa[7])
        const uint32_t c = vmin2(vmin2(d1, d2), 0x00010001u);         // 1 per half where the position passes
        acc2 = acc2 * 4u + c;                                         // position 2k at bit 2k, position 2k+1 at bit 16 + 2k
    }
    // tick map: sample i needs the pairs (m[i], m[i+1]) and (m[i+2], m[i+3]); odd i takes them from the 16-bit-shifted words
    uint32_t acc[2] = {0, 0};
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const uint32_t A = (i & 1) ? xs[i >> 1] : wv[i >> 1];
        const uint32_t Bp = (i & 1) ? xs[(i >> 1) + 1] : wv[(i >> 1) + 1];
        const uint32_t rows[5] = {NEG_ROW0, NEG_ROW1, NEG_ROW2, NEG_ROW3, NEG_ROW4};
#pragma unroll
        for (int r = 0; r < 5; r++) {
            const int nv = dp2a_hi(Bp, rows[r], dp2a_lo(A, rows[r], 0));
            const int g = 5 * i + r;                                           // tick within these 40
            acc[g >> 5] = __funnelshift_l((uint32_t)nv, acc[g >> 5], 1);       // shift the sign bit in, earliest tick ends up highest
        }
    }
    a0 = __brev(acc[0]); a1 = __brev(acc[1]) >> 24;                            // acc[1] holds 8 ticks in its low byte
    return (acc2 & 0xffu) | ((acc2 >> 15) & 0xffu);
}

// One lane = 16 consecutive samples / positions starting at ring index mi0, in two halves of 8 (the window of a half is 24
// magnitudes: half the registers of a 16-position window, which is what lets the kernel run with more warps per SM).
// Returns the 16-bit pre-check mask; writes the 80 ticks of its samples (two lanes share five words) at tick word tw0.
__device__ __forceinline__ uint32_t window_pass(WarpSmem &W, uint32_t mi0, uint32_t tw0, uint32_t lane, bool mirror, uint32_t *tickg_chunk) {
    uint32_t h0a, h0b, h1a, h1b;
    const uint32_t m0 = half_window(W, mi0, h0a, h0b);
    const uint32_t m1 = half_window(W, mi0 + 8, h1a, h1b);
    const uint32_t mask = m0 | (m1 << 8);
    // 80 ticks: t0 = ticks 0..31, t1 = ticks 32..63, t2 = ticks 64..79 (low half)
    const uint32_t t0 = h0a, t1 = h0b | (h1a << 8), t2 = (h1a >> 24) | (h1b << 8);
    // lanes 2j, 2j+1 own 160 ticks: five words
    uint32_t *dst = &W.tick[tw0 + (lane >> 1) * 5];
    uint32_t *dg = tickg_chunk + (lane >> 1) * 5;
    const unsigned long long keep = W.pol_keep;
    const uint32_t other_t0 = __shfl_down_sync(FULLMASK, t0, 1);
    if ((lane & 1) == 0) {
        const uint32_t w2 = t2 | (other_t0 << 16);
        dst[0] = t0; dst[1] = t1; dst[2] = w2;
        stg_keep(dg, t0, keep); stg_keep(dg + 1, t1, keep); stg_keep(dg + 2, w2, keep);
        if (mirror && lane < 4) { uint32_t *m = &W.tick[TICK_RING + (lane >> 1) * 5]; m[0] = t0; m[1] = t1; m[2] = w2; }
    } else {
        const uint32_t w3 = __funnelshift_r(t0, t1, 16), w4 = __funnelshift_r(t1, t2, 16);
        dst[3] = w3; dst[4] = w4;
        stg_keep(dg + 3, w3, keep); stg_keep(dg + 4, w4, keep);
        if (mirror && lane < 4) { uint32_t *m = &W.tick[TICK_RING + (lane >> 1) * 5]; m[3] = w3; m[4] = w4; }
    }
    return mask;
}

// One chunk's samples, two 16-byte pieces per lane (samples 256 r + 8 lane .. + 8).  Holding the loaded words in registers
// across the candidate work costs more registers than the kernel has, and an L2 prefetch leaves the L2 latency of the real
// load exposed at convert time (12 % of the stall samples): the chunk is copied ASYNCHRONOUSLY into the warp's staging
// kilobyte (LDGSTS, bypassing L1) before the candidate work and read from there when it is converted.  Every lane reads
// back exactly the bytes it copied, so its own cp.async.wait_group is all the synchronisation there is.
__device__ __forceinline__ void stage_raw(WarpSmem &W, const uint8_t *src, uint32_t lane) {
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(W.raw) + lane * 16;
    const unsigned long long pol = W.pol_stream;
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" :: "r"(dst), "l"(src + lane * 16), "l"(pol) : "memory");
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" :: "r"(dst + 512), "l"(src + 512 + lane * 16), "l"(pol) : "memory");
    asm volatile("cp.async.commit_group;" ::: "memory");
}
__device__ __forceinline__ void stage_wait() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// Chunks at the edge of the data are not staged (their loads are masked piece by piece): prefetch them into L2 instead.
__device__ __forceinline__ void prefetch_raw(const RunCtx &T, uint32_t c, uint32_t lane) {
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const uint32_t xo = c * CHUNK + r * 256 + lane * 8, xc = T.x0 + xo;
        if (!(xc + 8 <= T.x_zero_end || xc >= T.x_data_end))
            asm volatile("prefetch.global.L2 [%0];" :: "l"(T.tile_base + (size_t)xo * 2));
    }
}

// keep: where the chunk's piece r of this lane goes in ScanParams::mag_copy, or null (Mode A/C off, a magnitude segment, or outside
// the segment's tiles)
__device__ __forceinline__ void store_mags(WarpSmem &W, uint32_t slot, int r, uint32_t lane, const uint32_t m[8], uint16_t *keep) {
    uint4 packed;
    packed.x = __byte_perm(m[0], m[1], 0x5410); packed.y = __byte_perm(m[2], m[3], 0x5410);      // lo | hi << 16 in one PRMT (magnitudes are < 65536)
    packed.z = __byte_perm(m[4], m[5], 0x5410); packed.w = __byte_perm(m[6], m[7], 0x5410);
    *reinterpret_cast<uint4 *>(&W.mag[slot * CHUNK + r * 256 + lane * 8]) = packed;
    if (keep) __stcs(reinterpret_cast<uint4 *>(keep), packed);
    if (slot == 0 && r == 0 && lane < MAG_MIRROR / 8) *reinterpret_cast<uint4 *>(&W.mag[MAG_RING + lane * 8]) = packed;
}

__device__ __forceinline__ void to_mags(const ScanSmem &S, bool is_mag, const uint4 &raw, uint32_t m[8]) {
    const uint32_t wv[4] = {raw.x, raw.y, raw.z, raw.w};
    if (is_mag) {
#pragma unroll
        for (int i = 0; i < 4; i++) { m[2 * i] = wv[i] & 0xffffu; m[2 * i + 1] = wv[i] >> 16; }
    } else {
#pragma unroll
        for (int i = 0; i < 4; i++) uc8_pair_to_mag(S.lut, wv[i], m[2 * i], m[2 * i + 1]);
    }
}

// ScanParams::mag_copy address of sample (chunk cn, piece r, this lane's 8) of the run, or null when it is not kept.
template <bool KEEP> __device__ __forceinline__ uint16_t *mag_keep_at(const WarpSmem &W, const ScanParams &P, uint32_t cn, int r, uint32_t lane) {
    if (!KEEP || W.ctx.is_mag) return nullptr;
    const Segment &seg = *reinterpret_cast<const Segment *>(W.seg);
    const uint32_t x = W.ctx.x0 + cn * CHUNK + r * 256 + lane * 8;
    return x < seg.n_tiles * SCAN_TILE ? P.mag_copy + ((size_t)seg.tile_begin * SCAN_TILE + x) : nullptr;
}

// Magnitudes of one chunk into ring slot `slot` + exact statistics (convert.c:64-108), chunk entirely data; if count_buf is a
// reference buffer the whole chunk lies in it and is counted: lane partials -> warp sum -> one pair of atomics.
template <bool KEEP> __device__ __forceinline__ void convert_chunk_fast(const ScanSmem &S, WarpSmem &W, const ScanParams &P, bool is_mag, uint32_t slot,
                                                   uint32_t lane, uint32_t count_buf, uint32_t cn) {
    stage_wait();
    const uint4 raw0 = *reinterpret_cast<const uint4 *>(&W.raw[lane * 16]), raw1 = *reinterpret_cast<const uint4 *>(&W.raw[512 + lane * 16]);
    uint32_t level = 0;
    unsigned long long power = 0;
#pragma unroll
    for (int r = 0; r < 2; r++) {
        uint32_t m[8];
        to_mags(S, is_mag, r ? raw1 : raw0, m);
        level += (m[0] + m[1]) + (m[2] + m[3]) + (m[4] + m[5]) + (m[6] + m[7]);
#pragma unroll
        for (int i = 0; i < 8; i++) mad_wide(power, m[i], m[i]);
        store_mags(W, slot, r, lane, m, mag_keep_at<KEEP>(W, P, cn, r, lane));
    }
    if (count_buf != 0xffffffffu) {
        // hardware warp reductions (REDUX) instead of 15 shuffle steps: a lane's level is < 2^20, its power < 2^36, so the
        // power goes in two pieces whose warp sums stay below 2^32
        const uint32_t lv = __reduce_add_sync(FULLMASK, level);
        const uint32_t plo = __reduce_add_sync(FULLMASK, (uint32_t)power & 0xfffffu), phi = __reduce_add_sync(FULLMASK, (uint32_t)(power >> 20));
        if (lane == 0) { atomicAdd(&P.buf_acc[count_buf].sum_level, (unsigned long long)lv); atomicAdd(&P.buf_acc[count_buf].sum_power, ((unsigned long long)phi << 20) + plo); }
    }
}

// The same for a chunk at the edge of the data or across a buffer boundary.  Power statistics are per reference buffer:
// new sample n = x - lead - 326 belongs to buffer n / buf_len and is counted by the run whose position range holds x
// (the last tile of a segment also owns the tail).
template <bool KEEP> __device__ __noinline__ void convert_chunk_edge(const ScanSmem &S, WarpSmem &W, const ScanParams &P, uint32_t c, uint32_t slot, uint32_t lane) {
    const RunCtx &T = W.ctx;
    const bool owned = c < T.n_chunks || T.last_tile;
    unsigned long long level = 0, power = 0;
    uint32_t buf = 0xffffffffu;
    for (int r = 0; r < 2; r++) {
        const uint32_t xo = c * CHUNK + r * 256 + lane * 8, xc = T.x0 + xo;
        uint32_t m[8];
        if (xc + 8 <= T.x_zero_end || xc >= T.x_data_end) {
#pragma unroll
            for (int i = 0; i < 8; i++) m[i] = 0;
        } else {
            to_mags(S, T.is_mag, ldg_stream_u4(T.tile_base + (size_t)xo * 2), m);
            if (xc < T.x_zero_end || xc + 8 > T.x_data_end) {   // boundary group: mask the samples that are not data
#pragma unroll
                for (int i = 0; i < 8; i++) if (xc + i < T.x_zero_end || xc + i >= T.x_data_end) m[i] = 0;
            }
            if (owned) {
                const long long n0 = T.n_first + (long long)xo;
                for (int i = 0; i < 8; i++) {
                    const long long n = n0 + i;
                    if (n >= 0 && n < (long long)T.npos) {
                        const uint32_t bb = T.first_buf + (uint32_t)n / T.buf_len;
                        if (bb != buf) {
                            if (buf != 0xffffffffu) { atomicAdd(&P.buf_acc[buf].sum_level, level); atomicAdd(&P.buf_acc[buf].sum_power, power); }
                            buf = bb; level = 0; power = 0;
                        }
                        level += m[i];
                        mad_wide(power, m[i], m[i]);
                    }
                }
            }
        }
        store_mags(W, slot, r, lane, m, mag_keep_at<KEEP>(W, P, c, r, lane));
    }
    if (buf != 0xffffffffu) { atomicAdd(&P.buf_acc[buf].sum_level, level); atomicAdd(&P.buf_acc[buf].sum_power, power); }
}

// One round of full slices: the first `cnt` (<= 32) queued survivors, one per lane; live records go to the warp's staging area.
// This warp's private global areas, recomputed from the thread index where they are needed (measured: holding them in shared
// memory puts a shared-memory load in front of every global store of the tick copy and is 1.5 % slower)
#define WARP_GLOBAL() (blockIdx.x * SC_WARPS + (threadIdx.x >> 5))
#define W_TICKG(W, P) ((P).tick_scratch + (size_t)WARP_GLOBAL() * TICKG_WORDS)
#define W_STAGE(W, P) ((P).stage_rec + (size_t)WARP_GLOBAL() * (P).stage_cap)
#define W_STAGE_KEY(W, P) ((P).stage_key + (size_t)WARP_GLOBAL() * (P).stage_cap)
#define W_Q1_OVER(W, P) ((P).q1_over + (size_t)WARP_GLOBAL() * CHUNK)

__device__ __forceinline__ void slice_round(const ScanSmem &S, WarpSmem &W, const ScanParams &P, uint32_t cnt, uint32_t lane, uint32_t &n_stage) {
    const uint32_t *tickg = W_TICKG(W, P);
    Rec *stage = W_STAGE(W, P);
    uint32_t *stage_key = W_STAGE_KEY(W, P);
    PosEntry *run_pos = P.pos_pool + (size_t)W.ctx.tile0 * SCAN_TILE;
    uint32_t rw[8];
    uint32_t kind = 0;
    if (lane < cnt) {
        const uint32_t e = W.surv[lane];
        const uint32_t p = e & 0x3fffu, ph = (e >> 14) & 7u;
        kind = slice_and_classify(S, tickg, P, 5u * (p + 19u) + 4u + ph, (e >> 17) & 1u, rw);
        if (kind) {
            const uint32_t m = p / SCAN_TILE;
            atomicOr(&run_pos[(size_t)m * SCAN_TILE + (e >> 18)], 1u << (21 + ph));      // this phase has a record
            atomicAdd(&W.n_rec[m], 1u);
        }
    }
    const uint32_t bal = __ballot_sync(FULLMASK, kind != 0);
    if (kind) {
        const uint32_t at = n_stage + __popc(bal & ((1u << lane) - 1u));
        if (at < P.stage_cap) {
            uint4 *dst = reinterpret_cast<uint4 *>(stage + at);
            dst[0] = make_uint4(rw[0], rw[1], rw[2], rw[3]); dst[1] = make_uint4(rw[4], rw[5], rw[6], rw[7]);
            const int fixbit = (int)(int8_t)(rw[3] >> 24);
            const uint32_t aa_changed = (kind == K_ES_FIX && fixbit >= 8 && fixbit <= 31) ? 1u : 0u;   // mode_s.c:560
            const uint32_t df = (rw[0] & 0xffu) >> 3;                     // byte 0 of the frame as sliced
            stage_key[at] = (aa_changed ? KEY_AA_CHANGED : 0u) | (df == 17 ? KEY_DF17 : 0u) | ((df & 0x10u) ? KEY_LONG : 0u) | (kind << 24) | (rw[5] & 0xffffffu);
            // mode_s.c:766-779: only these can teach the filter an address; counted so that stage B knows before it starts whether the
            // receiver's tables are large enough for this run (real frames only: noise does not produce CRC-clean DF11 / DF17)
            if (kind == K_DF11_IID0 || (kind == K_ES_OK && df == 17)) atomicAdd(&P.stream_addable[reinterpret_cast<const Segment *>(W.seg)->stream], 1u);
        }
    }
    n_stage += __popc(bal);
}

// Candidates of one chunk: its pre-check passers (q1, ascending) -> thresholds -> PosEntries; DF gate -> survivor queue,
// sliced 32 at a time whenever the queue fills (the rest waits for later chunks of the run).
template <bool SUB> __device__ __forceinline__ void process_candidates(const ScanSmem &S, WarpSmem &W, const ScanParams &P, uint32_t n_q1, uint32_t chunk_p0, uint32_t mslot,
                                                   uint32_t tslot, uint32_t lane, uint32_t &n_surv, uint32_t &n_stage) {
    const uint32_t lt = (1u << lane) - 1u;
    const uint32_t m = chunk_p0 / SCAN_TILE;                     // tile of the run this chunk belongs to
    PosEntry *pos_out = P.pos_pool + (size_t)(W.ctx.tile0 + m) * SCAN_TILE;
    const uint32_t pe_base = ((chunk_p0 + (SUB ? W.ctx.sub_off : 0u)) & (SCAN_TILE - 1)) | (((W.ctx.tile_rel0 + m) & 3u) * SCAN_TILE);    // PosEntry position of chunk-local position 0
    const uint16_t *mag0 = &W.mag[mslot * CHUNK];
    // Threshold passers wait in W.pass (32 entries) until the chunk's last batch is through or the next batch's passers would
    // not fit: their DF gates are evaluated five lanes per passer, and a single batch rarely has more than three.
    uint32_t n_pass = 0, pos_base = W.n_pos[m];                 // passers waiting in W.pass; PosEntry index (in the tile) of W.pass[0]
    for (uint32_t b0 = 0;; b0 += 32) {
        const bool have_batch = b0 < n_q1;
        uint32_t pl = 0, tried = 0, bal = 0;
        if (have_batch) {
            const uint32_t e = b0 + lane;
            if (e < n_q1) {
                pl = e < Q1_SMEM ? W.q1[e] : W_Q1_OVER(W, P)[e - Q1_SMEM];      // chunk-local position
                tried = threshold_phases(mag0 + pl, reinterpret_cast<const Segment *>(W.seg)->thr);     // the receiver's own threshold
            }
            bal = __ballot_sync(FULLMASK, tried != 0);
        }
        const uint32_t n_b = __popc(bal);
        if (n_pass && (!have_batch || n_pass + n_b > 32)) {      // ---- DF gates of the waiting passers
            __syncwarp();
            for (uint32_t i0 = 0; i0 < 5 * n_pass; i0 += 32) {          // five lanes per passer, one per phase
                const uint32_t i_ = i0 + lane, r = i_ / 5, gph = i_ - 5 * r;
                uint32_t g = 0, pe = 0;
                if (r < n_pass) {
                    pe = W.pass[r];
                    if ((pe >> (16 + gph)) & 1u) g = df_gate(W, P, first_tick(tslot, pe & 0xffffu, gph));
                }
                const uint32_t bal2 = __ballot_sync(FULLMASK, g & 1u);
                if (g & 1u) W.surv[n_surv + __popc(bal2 & lt)] = (chunk_p0 + (pe & 0xffffu)) | (gph << 14) | ((g >> 1) << 17) | ((pos_base + r) << 18);
                n_surv += __popc(bal2);
                __syncwarp();
                if (n_surv >= 32) {
                    slice_round(S, W, P, 32, lane, n_stage);
                    const uint32_t moved = lane + 32 < n_surv ? W.surv[lane + 32] : 0;
                    __syncwarp();
                    W.surv[lane] = moved;
                    n_surv -= 32;
                    __syncwarp();
                }
            }
            pos_base += n_pass; n_pass = 0;
            __syncwarp();                                        // W.pass is free again
        }
        if (!have_batch) break;
        if (bal) {
            if (tried) {
                const uint32_t r = n_pass + __popc(bal & lt);
                W.pass[r] = pl | (tried << 16);
                pos_out[pos_base + r] = (pe_base + pl) | (tried << 16);   // live bits are OR-ed in when its phases are sliced
            }
            n_pass += n_b;
        }
    }
    __syncwarp();                                                // (every lane has read W.n_pos[m] above; compute-sanitizer's racecheck wants the fence, not just the ballots in between)
    if (lane == 0) W.n_pos[m] = pos_base;
}

// End of a run that covers only part of a tile.  A run of a few dozen tiles (one receiver's single buffer: the drop-in's call
// shape) leaves most of the chip idle and is latency-bound in every warp, so the launcher gives each tile to one CTA and each of
// its chunks to a warp of its own: a quarter of the serial work per warp (one 65536-sample buffer: 24 -> see DESIGN.md 3.7).  Each
// warp has written its PosEntries at its chunk's offset in the tile's list and staged its records privately; here the warps of
// the CTA meet (the only barriers after table staging, and only in this mode), reserve the tile's records in one piece, copy
// their records behind those of the warps before them and close the gaps in the PosEntry list, so that the tile's output is what
// one warp would have produced.
__device__ __forceinline__ void shared_tile_barrier(uint32_t n_warps) { asm volatile("bar.sync %0, %1;" :: "r"(1), "r"(n_warps * 32) : "memory"); }

// (W0 = the first warp's area: a one-tile run uses entry 0 of its per-tile counters only, the others carry what the warps tell each other
// here - nothing is added to the shared-memory layout of the whole-tile kernel)
__device__ __noinline__ void finish_shared_tile(WarpSmem &W0, WarpSmem &W, const ScanParams &P, uint32_t lane, uint32_t wid, uint32_t n_stage) {
    static_assert(RUN_MAX >= TILE_CHUNKS + 3, "exchange area of finish_shared_tile");
    struct Exchange { uint32_t *sub_pos, *sub_rec; uint32_t &sub_rec_off, &sub_ok; } S = {&W0.n_pos[1], &W0.n_rec[1], W0.n_pos[TILE_CHUNKS + 1], W0.n_pos[TILE_CHUNKS + 2]};
    const RunCtx &T = W.ctx;
    const uint32_t n_warps = TILE_CHUNKS, tile = T.tile0;
    PosEntry *tile_pos = P.pos_pool + (size_t)tile * SCAN_TILE;
    const uint32_t my_pos = W.n_pos[0] - T.sub_off;
    if (lane == 0) { S.sub_pos[wid] = my_pos; S.sub_rec[wid] = n_stage; }
    shared_tile_barrier(n_warps);
    uint32_t pos_before = 0, rec_before = 0, pos_tot = 0, rec_tot = 0, need = 0;
    for (uint32_t w = 0; w < n_warps; w++) {
        const uint32_t a = S.sub_pos[w], b = S.sub_rec[w];
        if (w < wid) { pos_before += a; rec_before += b; }
        pos_tot += a; rec_tot += b; need = max(need, b);
    }
    if (wid == 0 && lane == 0) {
        uint32_t off = 0, ok = 1;
        if (need > P.stage_cap) { atomicOr(&P.ctl->overflow, OV_STAGING_FULL); atomicMax(&P.ctl->stage_need, need); ok = 0; }         // as at the end of a whole-tile run
        else if (rec_tot) {
            off = atomicAdd(&P.ctl->rec_alloc, rec_tot);
            if (off + rec_tot > P.rec_cap) { atomicOr(&P.ctl->overflow, OV_REC_POOL_FULL); ok = 0; }
        }
        S.sub_rec_off = off; S.sub_ok = ok;
    }
    shared_tile_barrier(n_warps);
    const uint32_t off = S.sub_rec_off, ok = S.sub_ok;
    if (ok) {
        const Rec *stage = W_STAGE(W, P);
        const uint32_t *stage_key = W_STAGE_KEY(W, P);
        for (uint32_t i = lane; i < n_stage; i += 32) {
            const uint4 *src = reinterpret_cast<const uint4 *>(stage + i);
            uint4 *dst = reinterpret_cast<uint4 *>(P.rec_pool + off + rec_before + i);
            dst[0] = __ldcg(src); dst[1] = __ldcg(src + 1);
            P.key_pool[off + rec_before + i] = __ldcg(stage_key + i);
        }
    }
    // PosEntry lists: warp w's entries move down behind those of the warps before it, one warp after the other (a warp's
    // destination may reach into the list of the warp before it, which has moved by then; within a warp the destination never
    // lies above the source, so 32 entries at a time in ascending order is a safe forward move)
    for (uint32_t w = 1; w < n_warps; w++) {
        if (wid == w && pos_before != T.sub_off) {
            for (uint32_t i0 = 0; i0 < my_pos; i0 += 32) {
                const bool has = i0 + lane < my_pos;
                PosEntry v = 0;
                if (has) v = __ldcg(&tile_pos[T.sub_off + i0 + lane]);
                __syncwarp();
                if (has) tile_pos[pos_before + i0 + lane] = v;
                __syncwarp();
            }
        }
        shared_tile_barrier(n_warps);
    }
    if (wid == 0 && lane == 0) { TileOut t; t.n_pos = pos_tot; t.n_rec = ok ? rec_tot : 0; t.rec_off = off; t.n_found = rec_tot; P.tile_out[tile] = t; }
}

// SUB: the launcher's form for a run of at most one tile per SM, a tile shared by the warps of one CTA: CTA b takes tile b without a
// claim, and its first TILE_CHUNKS warps take one chunk of it each (finish_shared_tile).  KEEP: a Mode A/C context, the magnitudes are
// also written to ScanParams::mag_copy.  Both are compile-time so that the plain kernel - the one the throughput is measured on -
// carries nothing of either (measured with them as run-time tests: 4 - 6 % slower).
template <bool SUB, bool KEEP> __global__ void __maxnreg__(SC_MAXNREG) scan_kernel(const __grid_constant__ ScanParams P, const DeviceTables *__restrict__ tables) {
    constexpr uint32_t SC_THREADS = SC_WARPS * 32;
    extern __shared__ uint4 smem_raw[];
    ScanSmemFull &F = *reinterpret_cast<ScanSmemFull *>(smem_raw);
    ScanSmem &S = F.t;
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;

    {   // one-time table staging (persistent CTA)
        const uint4 *src = reinterpret_cast<const uint4 *>(tables->lut_fold);
        uint4 *dst = reinterpret_cast<uint4 *>(S.lut);
        if (P.need_lut) for (uint32_t i = tid; i < sizeof(S.lut) / 16; i += SC_THREADS) dst[i] = src[i];
        for (uint32_t i = tid; i < 256; i += SC_THREADS) S.crc_tab[i] = tables->crc_tab[i];
        for (uint32_t i = tid; i < 112; i += SC_THREADS) S.bit_syn[i] = tables->bit_syn[i];
        for (uint32_t i = tid; i < 512; i += SC_THREADS) S.syn_hash[i] = tables->syn_hash[i];
        if (tid == 0) S.syn_mul = tables->syn_hash_mul;
    }
    __syncthreads();      // the only block barrier: from here on every warp is on its own
    if (wid >= P.warps_per_cta) return;      // small run: the launcher spread it over more SMs with fewer warps each

    WarpSmem &W = F.w[wid];
    RunCtx &T = W.ctx;
    if (lane == 0) {
        unsigned long long pol;
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
        W.pol_stream = pol;
        asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
        W.pol_keep = pol;
    }
    __syncwarp();

    uint32_t pend_tile = 0, pend_n = 0;       // tiles already claimed but not processed yet (a claim that crossed a segment boundary)
    for (;;) {
        // ---- claim a run: guided self-scheduling, then cut at the segment boundary --------------------------------------
        if (!pend_n) {
            uint32_t start = 0, n = 0;
            if (SUB) {                            // one tile per CTA (a run of a few dozen tiles): no claim, no atomic round trip
                start = blockIdx.x; n = 1;
            } else if (lane == 0) {
                const uint32_t cur = *reinterpret_cast<volatile uint32_t *>(&P.ctl->tile_counter);
                if (cur < P.n_tiles) {
                    const uint32_t workers = gridDim.x * P.warps_per_cta;
                    n = min(max((P.n_tiles - cur + workers - 1u) / workers, 1u), (uint32_t)RUN_MAX);   // ceil(remaining / warps): single tiles only for the last round
                    start = atomicAdd(&P.ctl->tile_counter, n);
                    if (start >= P.n_tiles) n = 0; else n = min(n, P.n_tiles - start);
                }
            }
            if (!SUB) { start = __shfl_sync(FULLMASK, start, 0); n = __shfl_sync(FULLMASK, n, 0); }
            pend_tile = start; pend_n = n;
            if (!pend_n) break;
        }
        __syncwarp();
        if (lane < 16) {
            const Segment *sg = P.one_seg_valid ? &P.one_seg : &P.segs[P.tile_seg[pend_tile] & ~TILE_QUAD_START];
            W.seg[lane] = reinterpret_cast<const uint32_t *>(sg)[lane];
        }
        if (lane < (SUB ? 1u : (uint32_t)RUN_MAX)) { W.n_pos[lane] = 0; W.n_rec[lane] = 0; }      // (SUB: the other entries of warp 0 are finish_shared_tile's exchange area)
        __syncwarp();
        uint32_t n_chunks;
        {
            const Segment &seg = *reinterpret_cast<const Segment *>(W.seg);
            const uint32_t tile0 = pend_tile, n_tiles_run = min(pend_n, seg.tile_begin + seg.n_tiles - tile0);
            pend_tile += n_tiles_run; pend_n -= n_tiles_run;
            n_chunks = SUB ? 1u : n_tiles_run * TILE_CHUNKS;
            const uint32_t sub_off = SUB ? wid * CHUNK : 0u;                         // a tile shared between warps: this warp's chunk of it
            if (lane == 0) {
                const uint32_t x0 = (tile0 - seg.tile_begin) * SCAN_TILE + sub_off;   // run origin in tile coordinates (x = data index + lead)
                T.x0 = x0; T.tile0 = tile0; T.n_tiles = n_tiles_run; T.n_chunks = n_chunks; T.tile_rel0 = tile0 - seg.tile_begin; T.sub_off = sub_off;
                W.n_pos[0] = sub_off;                                                 // (its PosEntries start at its own offset in the tile's list)
                T.tile_base = seg.base + 2 * ((long long)x0 - (long long)seg.lead);
                T.x_data_end = seg.lead + seg.npos + B200_TRAIL;                      // first x without data
                T.x_zero_end = (seg.flags & SEG_HALO_ZERO) ? seg.lead + B200_TRAIL : seg.lead;   // x below: magnitude 0, memory not read
                T.is_mag = (seg.flags & SEG_MAG) ? 1u : 0u;
                T.last_tile = tile0 + n_tiles_run == seg.tile_begin + seg.n_tiles && (!SUB || sub_off + n_chunks * CHUNK == SCAN_TILE);
                const long long n_first = (long long)x0 - seg.lead - B200_TRAIL;
                T.n_first = n_first;
                T.buf_len = seg.buf_len; T.first_buf = seg.first_buf; T.npos = seg.npos;
                T.p_lo = seg.lead > x0 ? seg.lead - x0 : 0;                           // first real position
                T.p_hi = min(n_chunks * CHUNK, seg.lead + seg.npos > x0 ? seg.lead + seg.npos - x0 : 0u);
                const uint32_t nb = n_first > 0 ? (uint32_t)n_first / seg.buf_len : 0;
                T.nb = nb; T.bound = (long long)(nb + 1) * seg.buf_len;
            }
        }
        __syncwarp();

        uint32_t n_q1 = 0, n_surv = 0, n_stage = 0;
        uint32_t ms = 0;          // ring slot of chunk k's magnitudes; ticks of chunk k sit in slot k & 1
        // Chunks in the interior of the data and of a reference buffer need no case analysis: `fast_left` counts how many chunks
        // after the one just classified are of the same kind (staged, converted by the fast path, counted for buffer `fast_buf`);
        // the classification below runs at the edges of the data and once per reference buffer.
        uint32_t fast_left = 0, fast_buf = 0;
        const uint32_t k_int_lo = (T.p_lo + CHUNK - 1) / CHUNK, k_int_hi = T.p_hi / CHUNK;    // chunks whose 512 positions are all preamble starts

#pragma unroll 1
        for (int k = -2; k <= (int)n_chunks; k++) {
            uint32_t mask = 0;
            if (k >= 0) {
                // ---- window(k): pre-check + tick map -----------------------------------------------------------------
                mask = window_pass(W, ms * CHUNK + lane * 16, (k & 1) * TICK_CW, lane, (k & 1) == 0, W_TICKG(W, P) + k * TICK_CW);
                if ((uint32_t)k < k_int_lo || (uint32_t)k >= k_int_hi) {      // positions outside [p_lo, p_hi) are not preamble starts
                    const uint32_t i0 = k * CHUNK + lane * 16;               // run-relative
                    const uint32_t p_lo = T.p_lo, p_hi = T.p_hi;
                    const uint32_t lo_cut = p_lo > i0 ? min(p_lo - i0, 16u) : 0u, hi_cut = p_hi > i0 ? min(p_hi - i0, 16u) : 0u;
                    mask &= (0xffffu << lo_cut) & ((1u << hi_cut) - 1u);
                }
            }
            // ---- what kind of chunk is k+2 ------------------------------------------------------------------------------
            const uint32_t cn = (uint32_t)(k + 2);
            bool more, all_data, fast;
            uint32_t count_buf;
            if (fast_left) { fast_left--; more = true; all_data = true; fast = true; count_buf = fast_buf; }
            else {
                more = cn <= n_chunks; all_data = false; fast = false; count_buf = 0xffffffffu;
                if (more) {
                    const uint32_t xs = T.x0 + cn * CHUNK;
                    all_data = xs >= T.x_zero_end && xs + CHUNK <= T.x_data_end;
                    const bool owned = cn < n_chunks || T.last_tile;
                    const long long n0 = T.n_first + (long long)cn * CHUNK;
                    uint32_t nb = T.nb;
                    long long bound = T.bound;
                    if (n0 >= bound) {
                        while (n0 >= bound) { nb++; bound += T.buf_len; }
                        __syncwarp();
                        if (lane == 0) { T.nb = nb; T.bound = bound; }
                    }
                    const long long lim = min(bound, (long long)T.npos);
                    const bool one_buf = n0 >= 0 && n0 + CHUNK <= lim;                        // every sample counted, all in buffer nb
                    fast = all_data && (one_buf || !owned || n0 >= (long long)T.npos);
                    if (owned && one_buf) {
                        count_buf = T.first_buf + nb;
                        if (all_data) {         // how many of the following chunks are owned, all data and inside the same buffer
                            const uint32_t e1 = (T.last_tile ? n_chunks : n_chunks - 1u) - cn;
                            const uint32_t e2 = (T.x_data_end - xs) / CHUNK - 1u;
                            const uint32_t e3 = (uint32_t)((lim - n0) / CHUNK) - 1u;
                            fast_left = min(e1, min(e2, e3)); fast_buf = count_buf;
                        }
                    }
                }
            }
            // ---- stage(k+2) -------------------------------------------------------------------------------------------
            if (more) { if (all_data) stage_raw(W, T.tile_base + (size_t)cn * CHUNK * 2, lane); else prefetch_raw(T, cn, lane); }
            __syncwarp();                                        // ticks of chunk k visible to the warp
            // ---- candidates(k-1) --------------------------------------------------------------------------------------
            if (n_q1) process_candidates<SUB>(S, W, P, n_q1, (uint32_t)(k - 1) * CHUNK, ms == 0 ? 2 : ms - 1, (uint32_t)(k - 1) & 1u, lane, n_surv, n_stage);
            __syncwarp();                                        // chunk k-1's magnitudes are dead now
            // ---- convert(k+2) into the slot chunk k-1 occupied ------------------------------------------------------
            if (more) {
                const uint32_t msn = k < 0 ? cn : (ms == 0 ? 2 : ms - 1);       // (ms + 2) % 3; the first two chunks fill slots 0 and 1
                if (fast) convert_chunk_fast<KEEP>(S, W, P, T.is_mag, msn, lane, count_buf, cn);
                else {
                    if (all_data) stage_wait();      // staged, but this chunk straddles a buffer boundary: the edge path loads it itself
                    convert_chunk_edge<KEEP>(S, W, P, cn, msn, lane);
                }
            }
            // ---- q1 <- pre-check passers of chunk k -------------------------------------------------------------------
            if (k >= 0) {
                uint32_t off = warp_excl_scan(__popc(mask), lane, &n_q1);
                const uint32_t i0 = lane * 16;                   // chunk-local
                uint32_t mb = mask;
                while (mb) {
                    const uint32_t b = __ffs(mb) - 1; mb &= mb - 1;
                    if (off < Q1_SMEM) W.q1[off] = (uint16_t)(i0 + b); else W_Q1_OVER(W, P)[off - Q1_SMEM] = (uint16_t)(i0 + b);
                    off++;
                }
                ms = ms == 2 ? 0 : ms + 1;
            }
            __syncwarp();
        }

        // ---- end of run: remaining slices, one record-pool reservation, copy of the staged records ------------------------
        Rec *stage = W_STAGE(W, P);
        uint32_t *stage_key = W_STAGE_KEY(W, P);
        const uint32_t tile0 = T.tile0, n_tiles_run = T.n_tiles;
        if (n_surv) slice_round(S, W, P, n_surv, lane, n_stage);
        __syncwarp();
        if (SUB) { finish_shared_tile(F.w[0], W, P, lane, wid, n_stage); break; }
        uint32_t off = 0, ok = 1;
        if (lane == 0) {
            if (n_stage > P.stage_cap) { atomicOr(&P.ctl->overflow, OV_STAGING_FULL); atomicMax(&P.ctl->stage_need, n_stage); ok = 0; }   // host grows the staging areas and reruns
            else if (n_stage) {
                off = atomicAdd(&P.ctl->rec_alloc, n_stage);
                if (off + n_stage > P.rec_cap) { atomicOr(&P.ctl->overflow, OV_REC_POOL_FULL); ok = 0; }                              // host regrows the pool and reruns
            }
        }
        off = __shfl_sync(FULLMASK, off, 0); ok = __shfl_sync(FULLMASK, ok, 0);
        if (ok) {
            for (uint32_t i = lane; i < n_stage; i += 32) {
                const uint4 *src = reinterpret_cast<const uint4 *>(stage + i);
                uint4 *dst = reinterpret_cast<uint4 *>(P.rec_pool + off + i);
                dst[0] = __ldcg(src); dst[1] = __ldcg(src + 1);
                P.key_pool[off + i] = __ldcg(stage_key + i);
            }
        }
        {   // TileOut per tile of the run: records of tile m follow those of tile m-1 in the reservation
            const uint32_t mine = lane < n_tiles_run ? W.n_rec[lane] : 0;
            uint32_t tot;
            const uint32_t before = warp_excl_scan(mine, lane, &tot);
            if (lane < n_tiles_run) { TileOut t; t.n_pos = W.n_pos[lane]; t.n_rec = ok ? mine : 0; t.rec_off = off + before; t.n_found = mine; P.tile_out[tile0 + lane] = t; }
        }
    }
}

extern "C" int b200_scan_warps(int n_sm) { return n_sm * SC_WARPS; }
extern "C" int b200_scan_tick_words(void) { return TICKG_WORDS; }

// Kernel attributes are per device: b200_demod_create calls this for the context's device (current at that point).
extern "C" int b200_prepare_scan(void) {
    const int bytes = (int)sizeof(ScanSmemFull);
    cudaError_t e = cudaFuncSetAttribute(scan_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(scan_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(scan_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(scan_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    return (int)e;
}

extern "C" int b200_launch_scan(const ScanParams *p, const DeviceTables *d_tables, int n_sm, void *stream_) {
    // One persistent CTA per SM.  A run with fewer tiles than the chip has warps is spread out: as many CTAs as there are tiles (at
    // most one per SM) and only as many warps of each as it takes - a lone warp on an SM runs several times faster than one of 28.
    if (!p->n_tiles) return 0;
    const cudaStream_t stream = (cudaStream_t)stream_;
    ScanParams q = *p;
    uint32_t grid = (uint32_t)n_sm;
    q.warps_per_cta = SC_WARPS;
    if (q.n_tiles < grid * SC_WARPS) {
        if (grid > q.n_tiles) grid = q.n_tiles;
        q.warps_per_cta = (q.n_tiles + grid - 1) / grid;
    }
    const bool shared = grid == q.n_tiles;            // as many CTAs as tiles: CTA b takes tile b, one chunk per warp (finish_shared_tile)
    if (shared) q.warps_per_cta = TILE_CHUNKS;
    const size_t smem = sizeof(ScanSmemFull);
    if (shared) { if (q.mag_copy) scan_kernel<true, true><<<grid, SC_WARPS * 32, smem, stream>>>(q, d_tables); else scan_kernel<true, false><<<grid, SC_WARPS * 32, smem, stream>>>(q, d_tables); }
    else { if (q.mag_copy) scan_kernel<false, true><<<grid, SC_WARPS * 32, smem, stream>>>(q, d_tables); else scan_kernel<false, false><<<grid, SC_WARPS * 32, smem, stream>>>(q, d_tables); }
    return (int)cudaGetLastError();
}
