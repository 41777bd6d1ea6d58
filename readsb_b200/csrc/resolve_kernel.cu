// resolve_kernel.cu — stage B, the frame finaliser and the ICAO filter's control kernels.
//
//   resolve_kernel  one CTA per receiver: the sequential part of demodulate2400() (ICAO-filter dependent
//                   scoring mode_s.c:309-419, best-phase pick demod_2400.c:241-258, the accept test of
//                   decodeModesMessage mode_s.c:443-596,:766-779, skip-ahead demod_2400.c:468, the filter flip
//                   readsb.c:1227-1231), walked speculatively 32 candidates at a time with the receiver's two
//                   filter generations (icao_filter.c) in shared memory.  The walk touches only staged data:
//                   each tile's PosEntry list and 32-bit score keys arrive through a cp.async ring three tiles
//                   ahead, so no dependent global load sits on the sequential path.
//   finalize_stream the same CTA, after its receiver is resolved, one warp per accepted frame: assembles the frame from its
//                   32-byte record (bit fix / DF17 repair, mode_s.c:443-596), signal power (demod_2400.c:436-457), per-buffer /
//                   per-receiver power statistics, packing of the frame list for a single D2H copy.
#include "common.h"
#include "device_utils.cuh"

// ------------------------------------------------------------------------------------------------
// ICAO address filter: two generations of an open-addressed set (icao_filter.c semantics)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t icao_slot(uint32_t a, uint32_t log2) { return (a * 0x9E3779B1u) >> (32 - log2); }

__device__ __forceinline__ bool gen_has(const uint32_t *g, uint32_t log2, uint32_t a) {
    const uint32_t mask = (1u << log2) - 1u;
    uint32_t h = icao_slot(a, log2);
    for (;;) {
        const uint32_t v = g[h];
        if (v == a) return true;
        if (v == ICAO_EMPTY) return false;
        h = (h + 1) & mask;
    }
}

// Inserts `a` unless it is there; true when it was new to this generation (the caller keeps the generation's count and applies
// the reference's resize rule).  Room is guaranteed: the capacity check ahead of stage B keeps every generation's load <= 1/2.
__device__ __forceinline__ bool gen_insert(uint32_t *g, uint32_t log2, uint32_t a) {
    const uint32_t mask = (1u << log2) - 1u;
    uint32_t h = icao_slot(a, log2);
    for (;;) {
        const uint32_t v = g[h];
        if (v == a) return false;
        if (v == ICAO_EMPTY) break;
        h = (h + 1) & mask;
    }
    g[h] = a;
    return true;
}

// icao_filter.c:126-128: the insertion that made the active generation `count` addresses large doubles the reference's tables
// (filterBits + 1) - and icaoFilterResize (:66-92) carries only the ACTIVE generation over: the older one is forgotten.
__device__ __forceinline__ bool ref_resize_due(uint32_t count, uint32_t bits) { return count > (1u << bits) / 3u && bits < ICAO_MAXBITS; }
// icao_filter.c:97-99: icaoFilterExpire halves the tables first when the active generation is small
__device__ __forceinline__ bool ref_shrink_due(uint32_t count, uint32_t bits) { return count < (1u << bits) / 9u && bits > ICAO_MINBITS; }

#define RS_WARPS 8            // warps per receiver: buffers of one receiver are resolved speculatively in parallel, eight at a time.
                              // 128 registers per thread: two CTAs per SM, so 256 receivers are one wave on 132 SMs (H100 SXM)
#define RS_STAGE 384          // PosEntry / score keys of one quad staged in shared memory (denser quads are read in place)
#define RS_RING  2            // staging buffers per warp: the current quad plus one in flight
#define NEW_CAP  24           // addresses one buffer may learn in deferred mode before it has to be redone in direct mode
#define OLD_BITS 8192         // membership pre-filter of the older generation: one bit per hash value

// The ACTIVE generation (the one adds go to) lives in shared memory as the exact table.  The OLDER generation is only ever
// read until the next flip: shared memory holds a bit per hash value of its entries, and the exact table in global memory
// (StreamState) is probed only where that bit is set — same answers, 17 KB instead of 32 KB.
__device__ __forceinline__ uint32_t old_bit(uint32_t a) { return (a * 0x85EBCA6Bu) >> (32 - 13); }

struct WarpRing {
    PosEntry pos[RS_RING][RS_STAGE];
    uint32_t key[RS_RING][RS_STAGE];
    uint32_t q_np[4], q_nr[4], q_ro[4];      // the current quad's four TileOuts
};

// What resolving one reference buffer produced (everything the commit step needs to apply it, or to throw it away).
struct BufResult {
    long long now_ms;          // Modes.synthetic_now at the end of the buffer (demod_2400.c:283-285, 409-414)
    uint32_t n_frames, n_new, fail;
    uint32_t skip_out;         // the reference's `pa` after the range: positions below it are inside the last accepted frame
    uint32_t n_add;            // icaoFilterAdd calls of this buffer (mode_s.c:778) whose address the ACTIVE generation did not hold when the
                               // buffer was speculated: at most so many insertions into it
    uint32_t stats[15];        // preambles, bad, unknown, accepted[2], tried phases[5], best phases[5]
    uint32_t news[NEW_CAP];    // addresses this buffer learned that the filter did not hold (deferred mode)
};

// How a buffer's walk reaches the receiver's filter.  Default tables (ICAO_CAP slots): the active generation is S.act (shared
// memory) and `act` is unused; grown tables (BIG): both generations stay in global memory.
struct FilterRef {
    uint32_t *act;             // BIG: the active generation
    uint32_t *old_gen;         // the older generation's exact table (global memory), probed where its hash bit is set
    uint32_t log2;             // slots per generation = 1 << log2
    uint32_t *counts;          // direct mode: sizes of the two generations ...
    uint32_t *bits;            // ... the reference's filterBits ...
    uint32_t active;           // ... and which generation is the active one
};

struct ResolveSmem {
    uint32_t act[ICAO_CAP];
    uint32_t old_bits[OLD_BITS / 32];
    WarpRing ring[RS_WARPS];
    BufResult res[RS_WARPS];
    uint32_t tot[16], bstat[16];             // counters of the run / of the buffer being committed (lane k owns counter k)
};

__device__ __forceinline__ void cp_async4(void *smem, const void *gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ int rec_score(uint32_t kind, bool known) {
    switch (kind) {
        case K_AP: return known ? 1000 : -1;
        case K_DFREPAIR: return known ? 900 : 700;
        case K_DF11_FIX: return known ? 800 : -1;
        case K_DF11_IID0: return known ? 1600 : 750;
        case K_DF11_IID: return known ? 1000 : -1;
        case K_ES_OK: return known ? 1800 : 1400;
        case K_ES_FIX: return known ? 900 : 700;
        default: return -2;
    }
}

// One reference buffer of one receiver: the sequential loop of demodulate2400 over the threshold-passing positions stage A
// listed (demod_2400.c:306-471), one warp, 32 positions at a time.
//   DEFER = true  (speculation): the filter is read only; addresses the buffer would teach it are kept in R.news and the
//                 frames carry B200_FRAME_ICAO_ADDED — the commit step applies them if the speculation holds.
//   DEFER = false (direct): adds go straight into the shared-memory table, exactly as the reference does.
// Frames are written to fout[0 .. n_frames); `old_gen` is the older generation's exact table in global memory.
// DEFER is a function parameter: the many-receiver kernels pass a literal and get two specialised inlined copies (measured faster
// there: 256 CTAs share the instruction cache); the one-receiver kernel runs cold every call and goes through resolve_buffer_call,
// a single real function (its fully inlined form was 64 000 instructions, most of its time instruction fetch).
template <bool BIG>
__device__ __forceinline__ void resolve_buffer(const bool DEFER, const ResolveParams &P, ResolveSmem &S, WarpRing &R, BufResult &out, const Segment &seg, uint32_t si,
                                            uint32_t b, uint32_t d_lo, uint32_t d_hi, uint32_t skip_in, uint32_t seq, const FilterRef &F,
                                            b200_frame *fout, uint32_t fcap, uint32_t lane) {
    // [d_lo, d_hi): the positions of reference buffer b this call walks - the whole buffer, or one of the sub-ranges a buffer is cut
    // into when a receiver has fewer buffers in the run than stage B has warps (a sub-range is speculated like a buffer: it assumes
    // that no frame accepted before it reaches into it, skip_in = d_lo, and is redone with the real skip_in when one does).
    const uint32_t LOG2 = BIG ? F.log2 : (uint32_t)ICAO_CAP_LOG2;
    const uint32_t tile_end = seg.tile_begin + seg.n_tiles;
    const uint32_t n_quads = (seg.n_tiles + 3) / 4;
    const uint32_t d_begin = b * seg.buf_len;
    const uint32_t d_end = d_hi;
    const int64_t buf_ts = seg.first_ts + (int64_t)d_begin * 5;
    int64_t now_ms = buf_ts / 12000;          // demod_2400.c:283-285
    uint32_t skip_until = skip_in;            // data-index form of the reference's `pa` skip
    uint32_t nframes = 0, n_new = 0, fail = 0, c_add = 0;
    uint32_t c_pre = 0, c_bad = 0, c_unk = 0, c_acc0 = 0, c_acc1 = 0, c_tp[5] = {0, 0, 0, 0, 0}, c_bp[5] = {0, 0, 0, 0, 0};

    auto known_addr = [&](uint32_t a) {
        if (BIG ? gen_has(F.act, LOG2, a) : gen_has(S.act, ICAO_CAP_LOG2, a)) return true;
        const uint32_t h = old_bit(a);
        if (((S.old_bits[h >> 5] >> (h & 31)) & 1u) && gen_has(F.old_gen, LOG2, a)) return true;
        if (DEFER) for (uint32_t i = 0; i < n_new; i++) if (out.news[i] == a) return true;
        return false;
    };

    // Quad cursor: stage B walks QUADS of four consecutive scan tiles (8192 positions; PosEntry positions are quad-relative).
    // The quad's four PosEntry / key lists are staged back to back in ring slot q % RS_RING, one quad ahead; the TileOut
    // descriptors run one more ahead in registers: lane l < 4 holds the descriptor of the quad's tile l.
    uint32_t quad = (seg.lead + d_lo) / (4 * SCAN_TILE), idx = 0, rec_rel = 0, cur_npos = 0, cur_recbase = 0, sub = 4;
    bool staged = true;
    uint4 to = make_uint4(0, 0, 0, 0), d1 = to, d2 = to;
    const PosEntry *pe_ptr = nullptr;
    const uint32_t *key_ptr = nullptr;
    auto load_desc = [&](uint32_t q) {           // this lane's piece of quad q's descriptor
        const uint32_t t = seg.tile_begin + 4 * q + lane;
        return (lane < 4 && q < n_quads && t < tile_end) ? *reinterpret_cast<const uint4 *>(&P.tile_out[t]) : make_uint4(0, 0, 0, 0);
    };
    auto issue_stage = [&](uint32_t q, const uint4 &piece) {
        // lane l < 4 holds the TileOut of the quad's tile l: totals first, then the four lists back to back
        uint32_t tp = 0, tr = 0;
#pragma unroll
        for (int i = 0; i < 4; i++) { tp += __shfl_sync(FULLMASK, piece.x, i); tr += __shfl_sync(FULLMASK, piece.y, i); }
        if (q < n_quads && tp <= RS_STAGE && tr <= RS_STAGE) {
            const uint32_t buf = q % RS_RING;
            uint32_t bp = 0, br = 0;
#pragma unroll 1                 // (unrolled, these loops were 12 000 of the kernel's 41 000 instructions)
            for (int i = 0; i < 4; i++) {
                const uint32_t np = __shfl_sync(FULLMASK, piece.x, i), nr = __shfl_sync(FULLMASK, piece.y, i), ro = __shfl_sync(FULLMASK, piece.z, i);
                const PosEntry *src = P.pos_pool + (size_t)(seg.tile_begin + 4 * q + i) * SCAN_TILE;
#pragma unroll 1
                for (uint32_t e = lane; e < np; e += 32) cp_async4(&R.pos[buf][bp + e], &src[e]);
#pragma unroll 1
                for (uint32_t e = lane; e < nr; e += 32) cp_async4(&R.key[buf][br + e], &P.key_pool[ro + e]);
                bp += np; br += nr;
            }
        }
        cp_async_commit();
    };
    auto set_sublist = [&](uint32_t i) {         // dense quad, read in place: one scan tile at a time
        sub = i;
        pe_ptr = P.pos_pool + (size_t)(seg.tile_begin + 4 * quad + i) * SCAN_TILE;
        cur_npos = R.q_np[i]; cur_recbase = R.q_ro[i]; key_ptr = P.key_pool + cur_recbase;
        idx = 0; rec_rel = 0;
    };
    auto enter_quad = [&](uint32_t q) {          // make quad q current (d1 describes it, its lists are in flight)
        to = d1; d1 = d2; d2 = load_desc(q + 2);
        cp_async_wait_all();
        __syncwarp();
        if (lane < 4) { R.q_np[lane] = to.x; R.q_nr[lane] = to.y; R.q_ro[lane] = to.z; }
        __syncwarp();
        const uint32_t tp = R.q_np[0] + R.q_np[1] + R.q_np[2] + R.q_np[3], tr = R.q_nr[0] + R.q_nr[1] + R.q_nr[2] + R.q_nr[3];
        staged = tp <= RS_STAGE && tr <= RS_STAGE;
        if (staged) { const uint32_t buf = q % RS_RING; pe_ptr = R.pos[buf]; key_ptr = R.key[buf]; cur_npos = tp; cur_recbase = 0; sub = 4; idx = 0; rec_rel = 0; }
        else set_sublist(0);
        issue_stage(q + 1, d1);                  // into the slot quad q - 1 occupied
    };
    auto advance = [&]() {                       // next list with entries left: the next scan tile of a dense quad, or the next quad
        while (idx >= cur_npos) {
            if (!staged && sub < 3) set_sublist(sub + 1);
            else if (quad + 1 < n_quads) { quad++; enter_quad(quad); }
            else return false;
        }
        return true;
    };
    if (d_lo >= d_hi) quad = n_quads;         // empty range: nothing to walk
    if (quad < n_quads) {
        d1 = load_desc(quad); d2 = load_desc(quad + 1);
        issue_stage(quad, d1);
        enter_quad(quad);
    }

    for (;;) {
        if (quad >= n_quads || !advance()) break;
        const uint32_t x0 = quad * (4 * SCAN_TILE);
        const bool has = idx + lane < cur_npos;
        const PosEntry pe = has ? pe_ptr[idx + lane] : 0;
        const uint32_t d = x0 + (pe & 0x1fffu) - seg.lead;          // data index = position in the segment
        const bool inbuf = has && d < d_end;                        // entries are ascending: a prefix of lanes
        const uint32_t n_in = __popc(__ballot_sync(FULLMASK, inbuf));
        if (n_in == 0) break;                                       // next entry belongs to the next buffer
        const uint32_t tried = (pe >> 16) & 31u, live = (pe >> 21) & 31u;
        const uint32_t nlive = inbuf ? __popc(live) : 0;
        uint32_t dummy;
        const uint32_t rprefix = warp_excl_scan(nlive, lane, &dummy);
        const bool valid = inbuf && d >= skip_until;                // also drops the entries of earlier buffers in the first quad

        // score every tried phase with the current filter; first strictly greatest wins (demod_2400.c:243)
        int best = -2; uint32_t best_rel = 0, best_phase = 0, best_key = 0; bool best_known = false;
        // The chunk's records (about one for every two positions) are scored ONE PER LANE in a single pass; then every position
        // picks its own (at most five, consecutive, in phase order) with shuffles.  Scoring per position instead walks the five
        // phases with two or three lanes active each.  More than 32 records in a chunk: further rounds.
        if (__ballot_sync(FULLMASK, valid && live)) {
            uint32_t lm = (valid && live) ? live : 0u;          // this position's phases still to pick, ascending
            uint32_t jr = rprefix;                                // chunk-relative index of its next record
            for (uint32_t r0 = 0; r0 < dummy; r0 += 32) {
                uint32_t rkey = 0, rknown = 0; int rsc = -2;
                if (r0 + lane < dummy) {
                    rkey = key_ptr[rec_rel + r0 + lane];
                    rknown = known_addr(rkey & 0xffffffu) ? 1u : 0u;
                    rsc = rec_score((rkey >> 24) & 7u, rknown != 0);
                }
#pragma unroll
                for (int j = 0; j < 5; j++) {
                    const uint32_t src = (jr - r0) & 31u;
                    const uint32_t k_ = __shfl_sync(FULLMASK, rkey, src), kn_ = __shfl_sync(FULLMASK, rknown, src);
                    const int sc_ = __shfl_sync(FULLMASK, rsc, src);
                    if (lm && jr - r0 < 32u) {                    // my next record is one of this round's
                        const uint32_t ph = (uint32_t)__ffs(lm) - 1u; lm &= lm - 1u;
                        if (sc_ > best) { best = sc_; best_rel = rec_rel + jr; best_phase = ph; best_key = k_; best_known = kn_ != 0; }
                        jr++;
                    }
                }
            }
        }
        // accept test of decodeModesMessage (mode_s.c:443-596): only a corrected AA that is unknown rejects
        const bool decode_ok = best >= 0 && !((best_key & KEY_AA_CHANGED) && !best_known);
        // Commit the chunk in order.  After an accept the skip-ahead (demod_2400.c:468) silently consumes the
        // following lanes inside the frame; the lanes beyond keep their scores as long as the accepted frame did
        // not teach the filter a NEW address, so one loaded chunk can yield several frames.
        uint32_t pending = __ballot_sync(FULLMASK, inbuf), consumed = n_in;
        for (;;) {
            const bool live_lane = ((pending >> lane) & 1u) && d >= skip_until;
            const uint32_t acc_mask = __ballot_sync(FULLMASK, live_lane && decode_ok);
            const uint32_t f = acc_mask ? (uint32_t)__ffs(acc_mask) - 1 : 32u;
            if (live_lane && lane < f) {       // rejected preambles before the next accepted one
                c_pre++;
#pragma unroll
                for (int p = 0; p < 5; p++) c_tp[p] += (tried >> p) & 1u;
                if (best == -2) c_bad++; else c_unk++;       // -1, or decode result -1
            }
            if (!acc_mask) break;
            uint32_t msglen = 0, relearn = 0, newaddr = 0xffffffffu, dropped = 0;
            if (lane == f) {
                c_pre++;
#pragma unroll
                for (int p = 0; p < 5; p++) c_tp[p] += (tried >> p) & 1u;
                const uint32_t kind = (best_key >> 24) & 7u;
                msglen = (best_key & KEY_LONG) ? 112 : 56;              // demod_2400.c:399 (DF as sliced)
                const bool corrected = kind == K_DFREPAIR || kind == K_DF11_FIX || kind == K_ES_FIX;
                // mode_s.c:766-779: clean DF17, or DF11 with IID 0, teaches the filter its address
                const bool add = kind == K_DF11_IID0 || (kind == K_ES_OK && (best_key & KEY_DF17));
                const uint32_t j = d - d_begin;
                const int64_t ts = buf_ts + (int64_t)j * 5 + (8 + 56) * 12 + (4 + best_phase);   // demod_2400.c:406
                if (nframes < fcap) {
                    // accept record; finalize_stream turns it into the full frame from the 32-byte Rec
                    b200_frame fr;
                    fr.timestamp = ts; fr.sigpow_sum = 0; fr.j = j; fr.addr = best_key & 0xffffffu; fr.score = best;
                    fr.crc = 0;
                    if (staged) {        // index in the quad's concatenated list -> index in the record pool
                        uint32_t rel = best_rel;
#pragma unroll
                        for (int i = 0; i < 4; i++) { const uint32_t n = R.q_nr[i]; if (rel < n) { fr.crc = R.q_ro[i] + rel; break; } rel -= n; }
                    } else fr.crc = cur_recbase + best_rel;
                    fr.buffer_seq = seq; fr.signal_len = (uint16_t)(msglen * 12 / 5); fr.phase = (uint8_t)(4 + best_phase);
                    fr.msgtype = 0; fr.msgbits = 0; fr.correctedbits = 0; fr.fix_bit = -1; fr.flags = add ? B200_FRAME_ICAO_ADDED : 0;
#pragma unroll
                    for (int i = 0; i < 14; i++) fr.msg[i] = 0;
                    fr.pad_[0] = 0; fr.pad_[1] = 0;
                    *reinterpret_cast<uint16_t *>(&fr.pad_[0]) = (uint16_t)(si & 0xffffu);   // segment (low 16 bits) and data index
                    *reinterpret_cast<uint32_t *>(&fr.pad_[2]) = d;
                    fout[nframes] = fr;
                } else atomicOr(&P.ctl->overflow, OV_FRAME_CAP);
                if (corrected) c_acc1++; else c_acc0++;
                c_bp[best_phase]++;
                if (add) {
                    if (DEFER) {
                        if (!best_known) newaddr = best_key & 0xffffffu;
                        if (!(BIG ? gen_has(F.act, LOG2, best_key & 0xffffffu) : gen_has(S.act, ICAO_CAP_LOG2, best_key & 0xffffffu))) c_add++;
                    }
                    else if (gen_insert(BIG ? F.act : S.act, LOG2, best_key & 0xffffffu)) {      // icaoFilterAdd, icao_filter.c:112-130
                        const uint32_t cnt = ++F.counts[F.active];
                        if (ref_resize_due(cnt, *F.bits)) { (*F.bits)++; dropped = 1; }
                    }
                    relearn = (best_known && !dropped) ? 0u : 1u;      // membership changed: later scores are stale
                }
                now_ms = buf_ts / 12000 + (ts - buf_ts) / 12000;      // demod_2400.c:409-414
            }
            __syncwarp();
            // broadcast the state the accepting lane changed
            msglen = __shfl_sync(FULLMASK, msglen, f);
            relearn = __shfl_sync(FULLMASK, relearn, f);
            now_ms = __shfl_sync(FULLMASK, now_ms, f);
            if (DEFER) {
                newaddr = __shfl_sync(FULLMASK, newaddr, f);
                if (newaddr != 0xffffffffu) {
                    if (n_new < NEW_CAP) { if (lane == 0) out.news[n_new] = newaddr; n_new++; } else fail = 1;
                    __syncwarp();
                }
            }
            if (!DEFER) {
                dropped = __shfl_sync(FULLMASK, dropped, f);
                if (dropped) {      // the reference's resize carried only the active generation over (icao_filter.c:66-92): forget the older one
                    for (uint32_t q = lane; q < OLD_BITS / 32; q += 32) S.old_bits[q] = 0;
                    for (uint32_t q = lane; q < (1u << LOG2); q += 32) F.old_gen[q] = ICAO_EMPTY;
                    if (lane == 0) F.counts[F.active ^ 1u] = 0;
                    __syncwarp();
                }
            }
            const uint32_t d_f = __shfl_sync(FULLMASK, d, f);
            skip_until = d_f + msglen * 2 + 1;                          // demod_2400.c:468 + loop increment
            nframes++;
            pending &= ~((2u << f) - 1u);                               // lanes up to the accepted one are done
            if (relearn) { consumed = f + 1; break; }                   // re-score the rest of the chunk with the new filter
            if (!pending) break;
        }
        // advance the cursors past the consumed entries
        const uint32_t last = consumed - 1;
        rec_rel += __shfl_sync(FULLMASK, rprefix + nlive, last);
        idx += consumed;
    }
    cp_async_wait_all();      // nothing may land in this warp's ring after the next buffer starts to use it
    __syncwarp();

    const uint32_t red[15] = {c_pre, c_bad, c_unk, c_acc0, c_acc1, c_tp[0], c_tp[1], c_tp[2], c_tp[3], c_tp[4], c_bp[0], c_bp[1], c_bp[2], c_bp[3], c_bp[4]};
#pragma unroll
    for (int k = 0; k < 15; k++) {
        const uint32_t t = __reduce_add_sync(FULLMASK, red[k]);       // REDUX: one instruction per counter
        if (lane == 0) out.stats[k] = t;
    }
    c_add = __reduce_add_sync(FULLMASK, c_add);
    if (lane == 0) { out.now_ms = now_ms; out.n_frames = min(nframes, fcap); out.n_new = n_new; out.fail = fail; out.n_add = c_add; out.skip_out = skip_until; }
    __syncwarp();
}

template <bool BIG>
__device__ __noinline__ void resolve_buffer_call(bool defer, const ResolveParams &P, ResolveSmem &S, WarpRing &R, BufResult &out, const Segment &seg, uint32_t si,
                                                 uint32_t b, uint32_t d_lo, uint32_t d_hi, uint32_t skip_in, uint32_t seq, const FilterRef &F,
                                                 b200_frame *fout, uint32_t fcap, uint32_t lane) {
    resolve_buffer<BIG>(defer, P, S, R, out, seg, si, b, d_lo, d_hi, skip_in, seq, F, fout, fcap, lane);
}

// The capacity check of a receiver: stream_addable (scan kernel) bounds the insertions of this run; a generation never exceeds
// (active now + that), so with 2 x that <= slots no table can fill up and stage B needs no overflow path.  A receiver that could
// exceed it gets grow_log2 set and the run OV_FILTER_GROW: the host grows its tables and repeats.  True when the tables suffice.
__device__ __forceinline__ bool tables_fit(const ResolveParams &P, StreamState *st, uint32_t log2, uint32_t g0, uint32_t g1, uint32_t add) {
    const uint32_t need = max(g0, g1) + add;
    if (2u * need <= (1u << log2)) return true;
    uint32_t lg = log2 + 1;
    while ((1u << lg) < 4u * need && lg < ICAO_MAXBITS + 1) lg++;
    st->grow_log2 = lg;
    atomicOr(&P.ctl->overflow, OV_FILTER_GROW);
    return false;
}

// The asynchronous pipeline's "the step ahead has to be repeated" test: then this run is OV_SKIPPED.
__device__ __forceinline__ bool step_ahead_repeats(const ResolveParams &P) {
    if (!P.prev_stop || !*P.prev_stop) return false;
    atomicOr(&P.ctl->overflow, OV_SKIPPED);
    return true;
}

// COMPACT (the one-receiver kernel): the capacity check (capacity_check_all) is made here, by the CTA itself, while the other
// threads already fetch the tables.  *n_frames_out (shared memory) receives the receiver's frame count, or ~0 when stage B must not run.
template <bool BIG, bool COMPACT>
__device__ __forceinline__ void resolve_stream(const ResolveParams &P, ResolveSmem &S, StreamState *st, uint32_t stream, uint32_t *n_frames_out) {
    __shared__ uint32_t s_active, s_gcount[2], s_bits, s_go;
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t LOG2 = BIG ? st->cap_log2 : (uint32_t)ICAO_CAP_LOG2, CAP = 1u << LOG2;
    uint32_t *const tab0 = st->tab[0], *const tab1 = st->tab[1];
    auto tab = [&](uint32_t g) { return g ? tab1 : tab0; };

    if (tid == 0) {
        const uint32_t g0 = st->gen_count[0], g1 = st->gen_count[1];
        s_active = st->active; s_gcount[0] = g0; s_gcount[1] = g1; s_bits = st->filter_bits;
        uint32_t go = 1;
        if (COMPACT) {
            const uint32_t add = P.stream_addable[stream];
            P.stream_addable[stream] = 0;
            if (P.ctl->overflow & RUN_REPEAT_BITS) go = 0;
            if (step_ahead_repeats(P)) go = 0;
            if (go && !tables_fit(P, st, LOG2, g0, g1, add)) go = 0;
            *P.stop_out = go ? 0u : 1u;
            if (!go) *n_frames_out = ~0u;
        }
        s_go = go;
    }
    for (uint32_t i = tid; i < OLD_BITS / 32; i += blockDim.x) S.old_bits[i] = 0;
    if (tid < 16) { S.tot[tid] = 0; S.bstat[tid] = 0; }
    // the tables, four slots per load and all of a thread's loads in flight together (a receiver's default tables: 2 x 16 KB)
    constexpr uint32_t TL = ICAO_CAP / 4 / (RS_WARPS * 32);     // uint4 loads per thread and table for the default size
    uint4 va[BIG ? 1 : TL], vo[BIG ? 1 : TL];
    const uint32_t active0 = st->active;
    if (!BIG) {
        const uint4 *ta4 = reinterpret_cast<const uint4 *>(active0 ? tab1 : tab0), *to4 = reinterpret_cast<const uint4 *>(active0 ? tab0 : tab1);
#pragma unroll
        for (uint32_t k = 0; k < TL; k++) { va[k] = ta4[tid + k * RS_WARPS * 32]; vo[k] = to4[tid + k * RS_WARPS * 32]; }
    }
    __syncthreads();
    if (COMPACT && !s_go) return;
    if (!BIG) {
#pragma unroll
        for (uint32_t k = 0; k < TL; k++) {
            reinterpret_cast<uint4 *>(S.act)[tid + k * RS_WARPS * 32] = va[k];
            const uint32_t o[4] = {vo[k].x, vo[k].y, vo[k].z, vo[k].w};
#pragma unroll
            for (int j = 0; j < 4; j++) if (o[j] != ICAO_EMPTY) { const uint32_t h = old_bit(o[j]); atomicOr(&S.old_bits[h >> 5], 1u << (h & 31)); }
        }
    } else {
        const uint32_t *to = tab(s_active ^ 1u);
        for (uint32_t i = tid; i < CAP; i += blockDim.x) {
            const uint32_t v = to[i];
            if (v != ICAO_EMPTY) { const uint32_t h = old_bit(v); atomicOr(&S.old_bits[h >> 5], 1u << (h & 31)); }
        }
    }
    __syncthreads();

    // state only warp 0 touches (the commit step)
    uint32_t armed = st->flip_armed, seq = st->buffer_seq;
    int64_t next_flip = st->next_flip_ms;
    bool dirty_act = false;                  // the shared-memory table differs from the global copy of the active generation
    unsigned long long c_samples = 0;
    uint32_t c_bufs = 0, c_flips = 0, nframes = 0;
    b200_frame *fstream = P.frames + (size_t)stream * P.frame_cap;
    uint32_t cap_base = 0;                   // frame slots handed to the units of earlier rounds (each unit speculates into a region of its own)

    const uint32_t si_begin = P.one_seg_valid ? 0u : P.stream_seg_begin[stream], si_end = P.one_seg_valid ? 1u : P.stream_seg_begin[stream + 1];
    for (uint32_t si = si_begin; si < si_end; si++) {
        const Segment seg = P.one_seg_valid ? P.one_seg : P.segs[si];
        // Work units of a round: whole buffers when the receiver has at least RS_WARPS of them in this run, otherwise every buffer is
        // cut into sub-ranges of whole scan tiles so that all warps have work (a single 65536-sample mag_buf: eight ranges of 8192).
        const uint32_t nsplit = seg.n_bufs >= RS_WARPS ? 1u : max(1u, min((uint32_t)RS_WARPS / max(seg.n_bufs, 1u), (seg.buf_len + 4 * SCAN_TILE - 1) / (4 * SCAN_TILE)));
        const uint32_t sub_len = nsplit == 1 ? seg.buf_len : (((seg.buf_len + nsplit - 1) / nsplit + SCAN_TILE - 1) & ~(uint32_t)(SCAN_TILE - 1));
        const uint32_t ucap = nsplit == 1 ? P.per_buf_cap : sub_len / 113 + 3;          // frames one unit can hold (a frame hides the next 112 positions)
        const uint32_t n_units = seg.n_bufs * nsplit;
        auto unit_range = [&](uint32_t u, uint32_t &ub, uint32_t &lo, uint32_t &hi) {
            ub = u / nsplit;
            const uint32_t d_begin = ub * seg.buf_len, d_end = min(d_begin + seg.buf_len, seg.npos);
            lo = min(d_begin + (u - ub * nsplit) * sub_len, d_end); hi = min(lo + sub_len, d_end);
        };
        // per-buffer accumulation over its units (warp 0)
        uint32_t bframes = 0, skip_prev = 0;
        int64_t buf_now = 0;

        for (uint32_t u0 = 0; u0 < n_units; u0 += RS_WARPS) {
            const uint32_t n_round = min((uint32_t)RS_WARPS, n_units - u0);
            // ---- speculation: warp w resolves unit u0 + w against the filter as it stands ---------------------------------
            if (wid < n_round) {
                uint32_t b, lo, hi;
                unit_range(u0 + wid, b, lo, hi);
                // (the host sizes frame_cap so that every round's regions fit; a unit whose region would not fit holds no frames,
                // which reports the overflow instead of writing past the receiver's slots)
                const uint32_t ucap_fit = cap_base + (wid + 1) * ucap <= P.frame_cap ? ucap : 0u;
                FilterRef F;
                F.act = tab(s_active); F.old_gen = tab(s_active ^ 1u); F.log2 = LOG2; F.counts = nullptr; F.bits = nullptr; F.active = s_active;
                if (COMPACT) resolve_buffer_call<BIG>(true, P, S, S.ring[wid], S.res[wid], seg, si, b, lo, hi, lo, 0, F, fstream + cap_base + (size_t)wid * ucap, ucap_fit, lane);
                else resolve_buffer<BIG>(true, P, S, S.ring[wid], S.res[wid], seg, si, b, lo, hi, lo, 0 /* buffer_seq is stamped at commit */, F,
                                         fstream + cap_base + (size_t)wid * ucap, ucap_fit, lane);
            }
            __syncthreads();
            // ---- commit, in order -----------------------------------------------------------------------------------------------
            if (wid == 0) {
                bool spec_ok = true;
                for (uint32_t i = 0; i < n_round; i++) {
                    uint32_t b, lo, hi;
                    unit_range(u0 + i, b, lo, hi);
                    const bool first_of_buf = (u0 + i) % nsplit == 0, last_of_buf = (u0 + i) % nsplit == nsplit - 1;
                    BufResult &r = S.res[i];
                    const uint32_t d_begin = b * seg.buf_len, d_end = min(d_begin + seg.buf_len, seg.npos);
                    if (first_of_buf) { skip_prev = d_begin; buf_now = (seg.first_ts + (int64_t)d_begin * 5) / 12000; bframes = 0; }
                    b200_frame *fdst = fstream + nframes;
                    // A speculation cannot know about the reference's table resize (icao_filter.c:126-128), which forgets the older
                    // generation in the middle of a buffer: if this unit's adds could reach the resize threshold it is resolved directly.
                    const bool resize_possible = s_bits < ICAO_MAXBITS && s_gcount[s_active] + r.n_add > (1u << s_bits) / 3u;
                    const bool skip_reaches_in = skip_prev > lo;        // a frame accepted before this range hides its first positions
                    if (spec_ok && !r.fail && !resize_possible && !skip_reaches_in) {
                        // the speculation holds: teach the filter what this unit learned, move its frames into place
                        const b200_frame *fsrc = fstream + cap_base + (size_t)i * ucap;
                        const uint32_t n = r.n_frames;
                        uint32_t *act = BIG ? tab(s_active) : S.act;
                        for (uint32_t k0 = 0; k0 < n; k0 += 32) {
                            const bool has = k0 + lane < n;
                            b200_frame fr;
                            if (has) fr = fsrc[k0 + lane];
                            const uint32_t addm = __ballot_sync(FULLMASK, has && (fr.flags & B200_FRAME_ICAO_ADDED));
                            uint32_t m = addm, inserted = 0;
                            while (m) {                                  // mode_s.c:778, in frame order
                                const uint32_t l = __ffs(m) - 1; m &= m - 1;
                                const uint32_t a = __shfl_sync(FULLMASK, fr.addr, l);
                                if (lane == 0) { if (gen_insert(act, LOG2, a)) { s_gcount[s_active]++; inserted = 1; } }
                                __syncwarp();
                            }
                            // (only a real insertion makes the shared-memory table differ from its global copy: frames of aircraft the
                            // active generation already holds - the steady state - must not cost a 16 KB write-back per run)
                            if (__shfl_sync(FULLMASK, inserted, 0)) dirty_act = true;
                            if (has && fdst != fsrc) { fr.buffer_seq = seq; fdst[k0 + lane] = fr; }
                            else if (has) { const_cast<b200_frame *>(fsrc)[k0 + lane].buffer_seq = seq; }
                            __syncwarp();
                        }
                        if (r.n_new) spec_ok = false;                   // later units of the round saw a filter without these addresses
                    } else {
                        if (!skip_reaches_in || r.fail || resize_possible || !spec_ok) spec_ok = false;      // (a skip alone does not change the filter)
                        FilterRef F;
                        F.act = tab(s_active); F.old_gen = tab(s_active ^ 1u); F.log2 = LOG2; F.counts = s_gcount; F.bits = &s_bits; F.active = s_active;
                        if (COMPACT) resolve_buffer_call<BIG>(false, P, S, S.ring[0], r, seg, si, b, lo, hi, max(skip_prev, lo), seq, F, fdst, P.frame_cap - nframes, lane);
                        else resolve_buffer<BIG>(false, P, S, S.ring[0], r, seg, si, b, lo, hi, max(skip_prev, lo), seq, F, fdst, P.frame_cap - nframes, lane);
                        dirty_act = true;
                        spec_ok = false;
                    }
                    __syncwarp();
                    if (lane < 15) { S.tot[lane] += r.stats[lane]; S.bstat[lane] += r.stats[lane]; }
                    __syncwarp();
                    nframes += r.n_frames; bframes += r.n_frames;
                    if (r.n_frames) buf_now = r.now_ms;
                    skip_prev = max(skip_prev, r.skip_out);
                    if (!last_of_buf) continue;
                    // end of buffer: readsb.c:876, then backgroundTasks' filter flip (readsb.c:1227-1231)
                    c_samples += d_end - d_begin; c_bufs++;
                    uint32_t flipped = 0;
                    const int64_t now_ms = buf_now;
                    if (P.ttl_ms > 0 && (!armed || now_ms >= next_flip)) {
                        // icaoFilterExpire (icao_filter.c:96-110): the active generation becomes the older one (its exact table in global
                        // memory, its hash bits here); the other generation is emptied and becomes active
                        const uint32_t active = s_active, other = active ^ 1u;
                        uint32_t *ta = tab(active), *to = tab(other);
                        for (uint32_t q = lane; q < OLD_BITS / 32; q += 32) S.old_bits[q] = 0;
                        __syncwarp();
                        for (uint32_t q = lane; q < CAP; q += 32) {
                            const uint32_t v = BIG ? ta[q] : S.act[q];
                            if (!BIG && dirty_act) ta[q] = v;
                            if (v != ICAO_EMPTY) { const uint32_t h = old_bit(v); atomicOr(&S.old_bits[h >> 5], 1u << (h & 31)); }
                            if (BIG) to[q] = ICAO_EMPTY; else S.act[q] = ICAO_EMPTY;
                        }
                        __syncwarp();
                        if (lane == 0) {
                            if (ref_shrink_due(s_gcount[active], s_bits)) s_bits--;
                            s_gcount[other] = 0; s_active = other;
                        }
                        dirty_act = true;
                        next_flip = now_ms + P.ttl_ms; armed = 1; flipped = 1; c_flips++;
                        spec_ok = false;                                // the rest of the round saw the filter before the flip
                        __threadfence_block();
                        __syncwarp();
                    }
                    if (lane == 0) {
                        b200_buffer_result br;
                        br.sample_timestamp = seg.first_ts + (int64_t)d_begin * 5; br.sum_level = 0; br.sum_power = 0; br.sum_signal_power = 0;
                        br.length = d_end - d_begin; br.n_frames = bframes; br.buffer_seq = seq; br.icao_flipped = flipped;
                        br.demod_preambles = S.bstat[0]; br.demod_rejected_bad = S.bstat[1]; br.demod_rejected_unknown_icao = S.bstat[2];
                        br.demod_accepted[0] = S.bstat[3]; br.demod_accepted[1] = S.bstat[4];
                        for (int p = 0; p < 5; p++) { br.demod_preamblePhase[p] = S.bstat[5 + p]; br.demod_bestPhase[p] = S.bstat[10 + p]; }
                        br.pad_ = 0;
                        P.buf_out[seg.first_buf + b] = br;
                    }
                    __syncwarp();
                    if (lane < 16) S.bstat[lane] = 0;
                    __syncwarp();
                    seq++;
                }
            }
            cap_base += n_round * ucap;
            __syncthreads();
        }
    }

    // write back
    if (wid == 0) {
        const uint32_t active = s_active;
        if (!BIG && dirty_act) { uint32_t *ta = tab(active); for (uint32_t i = lane; i < ICAO_CAP; i += 32) ta[i] = S.act[i]; }
        if (lane == 0) {
            st->gen_count[0] = s_gcount[0]; st->gen_count[1] = s_gcount[1];
            st->active = active; st->filter_bits = s_bits; st->flip_armed = armed; st->next_flip_ms = next_flip; st->buffer_seq = seq;
            // counters: reductions into memory (nothing here waits for a load; the finalizer adds to the same block with atomics too)
            // (addressed through the kernel parameter so that the compiler emits global reductions, not generic atomics)
            unsigned long long *sv = reinterpret_cast<unsigned long long *>(&P.state[stream].stats);
            const uint32_t *tot = S.tot;
#define STAT_AT(field) (sv + offsetof(b200_demod_stats, field) / 8)
            atomicAdd(STAT_AT(samples_processed), c_samples); atomicAdd(STAT_AT(demod_preambles), (unsigned long long)tot[0]);
            atomicAdd(STAT_AT(demod_rejected_bad), (unsigned long long)tot[1]); atomicAdd(STAT_AT(demod_rejected_unknown_icao), (unsigned long long)tot[2]);
            atomicAdd(STAT_AT(demod_accepted), (unsigned long long)tot[3]); atomicAdd(STAT_AT(demod_accepted) + 1, (unsigned long long)tot[4]);
#pragma unroll
            for (int p = 0; p < 5; p++) { atomicAdd(STAT_AT(demod_preamblePhase) + p, (unsigned long long)tot[5 + p]); atomicAdd(STAT_AT(demod_bestPhase) + p, (unsigned long long)tot[10 + p]); }
            atomicAdd(STAT_AT(buffers), (unsigned long long)c_bufs); atomicAdd(STAT_AT(icao_flips), (unsigned long long)c_flips);
#undef STAT_AT
            *n_frames_out = min(nframes, P.frame_cap);
        }
    }
}

// Stage B: one CTA per receiver.  The buffers of a receiver only interact through the address filter (what earlier
// buffers taught it, and the 60 s flip), so RS_WARPS of them are resolved AT THE SAME TIME against the filter as it stands,
// in deferred mode; then warp 0 commits them in order.  A buffer's speculation holds if no buffer before it in the round
// changed the filter's membership: then its adds are applied and its frames moved into place.  Otherwise it is resolved
// again, directly, with the filter as the reference would have it at that point.  In steady state (aircraft already
// known, no flip) every speculation holds; the results are the sequential ones by construction either way.
// When its receiver is resolved, the CTA reserves the receiver's range of the packed frame list and finalizes the frames into it.
__device__ __forceinline__ void finalize_stream(const ResolveParams &P, uint32_t stream, uint32_t base, uint32_t n, uint32_t warp, uint32_t n_warps, uint32_t lane);

// The capacity check of a run, for every receiver (the threads of one CTA share them): (1) the asynchronous pipeline's "the step
// ahead has to be repeated" test; (2) the filter tables.
__device__ __forceinline__ void capacity_check_all(const ResolveParams &P) {
    if (threadIdx.x == 0) step_ahead_repeats(P);
    for (uint32_t s = threadIdx.x; s < P.n_streams; s += blockDim.x) {
        const uint32_t add = P.stream_addable[s];
        P.stream_addable[s] = 0;
        StreamState *st = &P.state[s];
        tables_fit(P, st, st->cap_log2, st->gen_count[0], st->gen_count[1], add);
    }
}

// Whether stage B runs in this run: for no receiver if one of them fails the capacity check, so the check is made ONCE per run,
// before any CTA touches a receiver's state, by the CTA that claims it first; the other CTAs wait for its verdict.  A CTA only ever
// waits for a CTA that is already running and needs nothing from the others to finish the check.  The launch for grown tables
// (a second launch of the same run) finds the verdict made.
__device__ __forceinline__ bool stage_b_runs(const ResolveParams &P) {
    __shared__ uint32_t s_verdict;
    volatile uint32_t *verdict = &P.ctl->cap_check;
    if (threadIdx.x == 0) s_verdict = atomicCAS(&P.ctl->cap_check, 0u, 1u);
    __syncthreads();
    if (s_verdict == 0) {                                 // this CTA claimed the check
        capacity_check_all(P);
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t v = (atomicOr(&P.ctl->overflow, 0u) & RUN_REPEAT_BITS) ? CAP_STOP : CAP_GO;
            *P.stop_out = v == CAP_STOP ? 1u : 0u;
            __threadfence();
            *verdict = v;
            s_verdict = v;
        }
    } else if (threadIdx.x == 0) {
        uint32_t v;
        while ((v = *verdict) < CAP_STOP) { }
        __threadfence();
        s_verdict = v;
    }
    __syncthreads();
    return s_verdict == CAP_GO;
}

// Receivers with grown tables (BIG) are rare: they get an instantiation of their own, launched only when there is one, so that
// the common case does not share its register allocation; each CTA of either launch leaves the other kind alone.
#define RS_MIN_CTAS 2         // CTAs per SM the register allocation aims at (128 registers; 3 -> 85: see DESIGN.md 6, SM partition experiment)
template <bool BIG>
__global__ void __launch_bounds__(RS_WARPS * 32, RS_MIN_CTAS) resolve_kernel(const ResolveParams P) {
    extern __shared__ uint4 resolve_smem_raw[];
    ResolveSmem &S = *reinterpret_cast<ResolveSmem *>(resolve_smem_raw);
    __shared__ uint32_t s_nframes, s_base;
    const uint32_t stream = blockIdx.x;
    StreamState *st = &P.state[stream];
    // Stage A failed (record pool / staging), a receiver's filter tables have to grow first, or the step ahead of this one in the
    // asynchronous pipeline has to be repeated: leave every receiver's state untouched, report no frames; the host repairs and
    // repeats the run(s) in order.
    if (!stage_b_runs(P)) {
        if (threadIdx.x == 0) { P.frame_span[2 * stream] = 0; P.frame_span[2 * stream + 1] = 0; }
        return;
    }
    if ((st->cap_log2 != ICAO_CAP_LOG2) != BIG) return;
    resolve_stream<BIG, false>(P, S, st, stream, &s_nframes);
    __syncthreads();
    // One reservation per receiver: its frames stay together and in order.  Where the receivers' ranges lie relative to each other
    // depends on which CTA gets here first; frame_span tells every reader where each receiver's frames are.
    if (threadIdx.x == 0) {
        s_base = atomicAdd(&P.ctl->total_frames, s_nframes);
        P.frame_span[2 * stream] = s_base; P.frame_span[2 * stream + 1] = s_nframes;
    }
    __syncthreads();
    finalize_stream(P, stream, s_base, s_nframes, threadIdx.x >> 5, RS_WARPS, threadIdx.x & 31);
}

__device__ __noinline__ void resolve_stream_big(const ResolveParams &P, ResolveSmem &S, StreamState *st, uint32_t stream, uint32_t *n_frames_out) { resolve_stream<true, true>(P, S, st, stream, n_frames_out); }

// A context with ONE receiver (the drop-in's shape: one readsb process, one mag_buf per call) needs no grid-wide agreement: this
// single CTA makes the capacity check for its receiver itself, and assembles the frames when it is done - stage B, the frame
// prefix and the finalizer in one launch.
__global__ void __launch_bounds__(RS_WARPS * 32, 1) resolve_solo_kernel(const __grid_constant__ ResolveParams P) {
    extern __shared__ uint4 resolve_smem_raw[];
    ResolveSmem &S = *reinterpret_cast<ResolveSmem *>(resolve_smem_raw);
    const uint32_t stream = 0;
    StreamState *st = &P.state[0];
    __shared__ uint32_t s_nframes;
    if (st->cap_log2 == ICAO_CAP_LOG2) resolve_stream<false, true>(P, S, st, stream, &s_nframes);
    else resolve_stream_big(P, S, st, stream, &s_nframes);
    __syncthreads();
    const uint32_t n = s_nframes == ~0u ? 0u : s_nframes;         // ~0: stage B did not run (the step is going to be repeated)
    if (threadIdx.x == 0) { P.frame_span[0] = 0; P.frame_span[1] = n; P.ctl->total_frames = n; }
    finalize_stream(P, stream, 0, n, threadIdx.x >> 5, RS_WARPS, threadIdx.x & 31);
    if (P.carry_src && s_nframes != ~0u) {      // (not when the step is going to be repeated: it needs its halo again) every reader of this
                                                // run's samples - scan kernel, finalizer above - is done: move the tail to the front
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < B200_TRAIL; i += blockDim.x) P.carry_dst[i] = P.carry_src[i];
    }
    if (P.publish_dst) {
        __syncthreads();                                    // the finalizer's writes (all warps) are in place
        const uint32_t n16 = (P.publish_head + n * (uint32_t)sizeof(b200_frame)) / 16;
        for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) P.publish_dst[i] = P.publish_src[i];
        __syncthreads();
        uint4 *clr = const_cast<uint4 *>(P.publish_src);
        for (uint32_t i = threadIdx.x; i < P.publish_clear / 16; i += blockDim.x) clr[i] = make_uint4(0, 0, 0, 0);
    }
}

__device__ __forceinline__ unsigned long long dmax_bits(double v) { return (unsigned long long)__double_as_longlong(v); }

// One warp per accepted frame of receiver `stream`: the frame from its record, its signal power, the statistics (see the file
// header).  Warp `warp` of `n_warps` takes frames warp, warp + n_warps, ... of the receiver's n and writes frame k to packed[base + k].
__device__ __forceinline__ void finalize_stream(const ResolveParams &P, uint32_t stream, uint32_t base, uint32_t n, uint32_t warp, uint32_t n_warps, uint32_t lane) {
    for (uint32_t k = warp; k < n; k += n_warps) {
        const uint32_t fi = base + k;
        const b200_frame *src = &P.frames[(size_t)stream * P.frame_cap + k];
        const uint32_t d = *reinterpret_cast<const uint32_t *>(&src->pad_[2]);
        // locate the segment: accept records carry the low 16 bits of the segment index; a stream has few segments
        uint32_t seg_i = P.one_seg_valid ? 0u : P.stream_seg_begin[stream];
        {
            const uint32_t low = *reinterpret_cast<const uint16_t *>(&src->pad_[0]);
            while ((seg_i & 0xffffu) != low) seg_i++;
        }
        const Segment seg = P.one_seg_valid ? P.one_seg : P.segs[seg_i];
        const uint32_t len = src->signal_len;                    // 134 or 268 samples (demod_2400.c:439): at most 9 per lane
        // the samples are fetched with all loads of a lane in flight at once (then the table lookups, likewise)
        constexpr int FIN_PER_LANE = 9;
        uint32_t raw[FIN_PER_LANE];
#pragma unroll
        for (int u = 0; u < FIN_PER_LANE; u++) {
            const uint32_t i = lane + 32u * u, dd = d + 19 + i;  // data index of the sample (demod_2400.c:443)
            const bool live = i < len && !((seg.flags & SEG_HALO_ZERO) && dd < B200_TRAIL);
            raw[u] = live ? (uint32_t)*reinterpret_cast<const uint16_t *>(seg.base + 2 * (size_t)dd) : 0xffffffffu;
        }
        unsigned long long sum = 0;
#pragma unroll
        for (int u = 0; u < FIN_PER_LANE; u++) {
            uint32_t m = 0;
            if (raw[u] != 0xffffffffu) m = (seg.flags & SEG_MAG) ? raw[u] : P.lut_full[(raw[u] & 0xffu) * 256 + (raw[u] >> 8)];
            sum += (unsigned long long)(m * m);
        }
        for (uint32_t i = lane + 32u * FIN_PER_LANE; i < len; i += 32) {      // (not reached with the reference's frame lengths)
            const uint32_t dd = d + 19 + i;
            uint32_t m;
            if ((seg.flags & SEG_HALO_ZERO) && dd < B200_TRAIL) m = 0;
            else {
                const uint16_t r16 = *reinterpret_cast<const uint16_t *>(seg.base + 2 * (size_t)dd);
                m = (seg.flags & SEG_MAG) ? r16 : P.lut_full[(r16 & 0xffu) * 256 + (r16 >> 8)];
            }
            sum += (unsigned long long)(m * m);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(FULLMASK, sum, o);
        if (lane == 0) {
            b200_frame fr = *src;
            // the accept part of decodeModesMessage (mode_s.c:443-596) on the record the resolver picked
            const uint4 r0 = reinterpret_cast<const uint4 *>(&P.rec_pool[fr.crc])[0];
            const uint4 r1 = reinterpret_cast<const uint4 *>(&P.rec_pool[fr.crc])[1];
            uint8_t msg[16];
            *reinterpret_cast<uint4 *>(msg) = r0;
            const uint32_t kind = msg[14];
            const int rec_fix = (int)(int8_t)msg[15];
            uint32_t msgtype = msg[0] >> 3, corrected = 0, crc = r1.x;
            int fix_bit = -1;
            if (kind == K_DFREPAIR) { msg[0] = (uint8_t)((msg[0] & 7) | (17 << 3)); msgtype = 17; corrected = 1; fix_bit = rec_fix; crc = 0; }   // mode_s.c:276-301
            else if (kind == K_DF11_FIX || kind == K_ES_FIX) { corrected = 1; fix_bit = rec_fix; msg[fix_bit >> 3] ^= (uint8_t)(1u << (7 - (fix_bit & 7))); }   // crc.c:410-418
            const uint32_t msgbits = (msgtype & 0x10) ? 112 : 56;
            const uint32_t aa = ((uint32_t)msg[1] << 16) | ((uint32_t)msg[2] << 8) | msg[3];
            fr.crc = crc; fr.addr = kind == K_AP ? crc : aa;
            fr.msgtype = (uint8_t)msgtype; fr.msgbits = (uint8_t)msgbits; fr.correctedbits = (uint8_t)corrected; fr.fix_bit = (int8_t)fix_bit;
#pragma unroll
            for (int i = 0; i < 14; i++) fr.msg[i] = (uint32_t)i < msgbits / 8 ? msg[i] : 0;
            fr.sigpow_sum = sum;
#pragma unroll
            for (int i = 0; i < 6; i++) fr.pad_[i] = 0;
            P.packed[fi] = fr;
            const uint32_t b = seg.first_buf + d / seg.buf_len;
            atomicAdd(&P.buf_acc[b].sum_signal_power, sum);
            b200_demod_stats &s = P.state[stream].stats;
            atomicAdd((unsigned long long *)&s.signal_power_count, (unsigned long long)len);
            atomicAdd((unsigned long long *)&s.sum_signal_power, sum);
            const double level = (double)sum / 65535.0 / 65535.0 / (double)len;      // demod_2400.c:448-449
            if (level > 0.50119) atomicAdd((unsigned long long *)&s.strong_signal_count, 1ull);
            atomicMax((unsigned long long *)&s.peak_signal_power, dmax_bits(level));
        }
    }
}

// ------------------------------------------------------------------------------------------------
// tiny control-plane kernels: ICAO filter operations from the host API
// ------------------------------------------------------------------------------------------------
__global__ void icao_op_kernel(StreamState *state, uint32_t stream, int op, uint32_t addr, int *result) {
    StreamState *st = &state[stream];
    const uint32_t log2 = st->cap_log2, cap = 1u << log2;
    int r = 0;
    if (op == 0) {            // add (icao_filter.c:112-130)
        const uint32_t a = st->active;
        __shared__ int s_dropped;
        if (threadIdx.x == 0) {
            s_dropped = 0;
            if (!gen_has(st->tab[a], log2, addr)) {
                if (2u * (st->gen_count[a] + 1u) > cap) { st->grow_log2 = log2 + 1; r = -1; }       // the host grows the tables and asks again
                else {
                    gen_insert(st->tab[a], log2, addr);
                    const uint32_t cnt = ++st->gen_count[a];
                    if (ref_resize_due(cnt, st->filter_bits)) { st->filter_bits++; st->gen_count[a ^ 1u] = 0; s_dropped = 1; }
                }
            }
        }
        __syncthreads();
        if (s_dropped) for (uint32_t i = threadIdx.x; i < cap; i += blockDim.x) st->tab[a ^ 1u][i] = ICAO_EMPTY;      // icaoFilterResize, :66-92
    } else if (op == 1) {     // test (icao_filter.c:132-154)
        if (threadIdx.x == 0) r = (gen_has(st->tab[0], log2, addr) || gen_has(st->tab[1], log2, addr)) ? 1 : 0;
    } else if (op == 2) {     // expire (icao_filter.c:96-110)
        const uint32_t other = st->active ^ 1u;
        for (uint32_t i = threadIdx.x; i < cap; i += blockDim.x) st->tab[other][i] = ICAO_EMPTY;
        __syncthreads();
        if (threadIdx.x == 0) {
            if (ref_shrink_due(st->gen_count[other ^ 1u], st->filter_bits)) st->filter_bits--;
            st->gen_count[other] = 0; st->active = other; st->stats.icao_flips++;
        }
    } else if (op == 3) {     // reset (icaoFilterInit)
        for (uint32_t i = threadIdx.x; i < cap; i += blockDim.x) { st->tab[0][i] = ICAO_EMPTY; st->tab[1][i] = ICAO_EMPTY; }
        if (threadIdx.x == 0) { st->gen_count[0] = st->gen_count[1] = 0; st->active = 0; st->filter_bits = ICAO_MINBITS; st->flip_armed = 0; st->next_flip_ms = 0; }
    }
    if (result && threadIdx.x == 0) *result = r;
}

// A receiver's tables move to larger ones (host: b200 grow_icao_tables): both generations are re-inserted.
__global__ void icao_rehash_kernel(StreamState *state, uint32_t stream, uint32_t *new0, uint32_t *new1, uint32_t new_log2) {
    StreamState *st = &state[stream];
    const uint32_t old_cap = 1u << st->cap_log2, new_cap = 1u << new_log2, mask = new_cap - 1u;
    for (uint32_t i = threadIdx.x; i < new_cap; i += blockDim.x) { new0[i] = ICAO_EMPTY; new1[i] = ICAO_EMPTY; }
    __syncthreads();
    for (int g = 0; g < 2; g++) {
        const uint32_t *from = st->tab[g];
        uint32_t *to = g ? new1 : new0;
        for (uint32_t i = threadIdx.x; i < old_cap; i += blockDim.x) {
            const uint32_t v = from[i];
            if (v == ICAO_EMPTY) continue;
            uint32_t h = icao_slot(v, new_log2);
            while (atomicCAS(&to[h], ICAO_EMPTY, v) != ICAO_EMPTY) h = (h + 1) & mask;       // addresses of one generation are distinct
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) { st->tab[0] = new0; st->tab[1] = new1; st->cap_log2 = new_log2; st->grow_log2 = 0; }
}

__global__ void init_state_kernel(StreamState *st, uint32_t n, uint32_t *slab) {
    const uint32_t s = blockIdx.x;
    if (s >= n) return;
    uint32_t *t0 = slab + (size_t)s * 2 * ICAO_CAP;
    for (uint32_t i = threadIdx.x; i < 2 * ICAO_CAP; i += blockDim.x) t0[i] = ICAO_EMPTY;
    if (threadIdx.x == 0) {
        StreamState z;
        memset(&z, 0, sizeof z);
        z.tab[0] = t0; z.tab[1] = t0 + ICAO_CAP; z.cap_log2 = ICAO_CAP_LOG2; z.filter_bits = ICAO_MINBITS;
        st[s] = z;
    }
}

// ------------------------------------------------------------------------------------------------
// launch wrappers
// ------------------------------------------------------------------------------------------------
extern "C" int b200_prepare_resolve(void) {      // per device, from b200_demod_create
    cudaError_t e = cudaFuncSetAttribute(resolve_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ResolveSmem));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(resolve_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ResolveSmem));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(resolve_solo_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ResolveSmem));
    return (int)e;
}

// any_grown: some receiver of the context has filter tables of its own (then the second instantiation runs too)
extern "C" int b200_launch_resolve(const ResolveParams *p, int any_grown, void *stream) {
    if (p->solo) {          // one receiver: capacity check, stage B, frame placement and finalizer in one launch
        resolve_solo_kernel<<<1, RS_WARPS * 32, sizeof(ResolveSmem), (cudaStream_t)stream>>>(*p);
        return (int)cudaGetLastError();
    }
    resolve_kernel<false><<<p->n_streams, RS_WARPS * 32, sizeof(ResolveSmem), (cudaStream_t)stream>>>(*p);
    if (any_grown) resolve_kernel<true><<<p->n_streams, RS_WARPS * 32, sizeof(ResolveSmem), (cudaStream_t)stream>>>(*p);
    return (int)cudaGetLastError();
}

extern "C" int b200_launch_init_state(StreamState *state, uint32_t n, uint32_t *slab, void *stream) {
    init_state_kernel<<<n, 256, 0, (cudaStream_t)stream>>>(state, n, slab);
    return (int)cudaGetLastError();
}

extern "C" int b200_launch_icao_rehash(StreamState *state, uint32_t stream, uint32_t *new0, uint32_t *new1, uint32_t new_log2, void *cstream) {
    icao_rehash_kernel<<<1, 1024, 0, (cudaStream_t)cstream>>>(state, stream, new0, new1, new_log2);
    return (int)cudaGetLastError();
}

extern "C" int b200_launch_icao_op(StreamState *state, uint32_t stream, int op, uint32_t addr, int *d_result, void *cstream) {
    icao_op_kernel<<<1, 256, 0, (cudaStream_t)cstream>>>(state, stream, op, addr, d_result);
    return (int)cudaGetLastError();
}
