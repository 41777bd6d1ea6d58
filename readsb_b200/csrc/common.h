// common.h — structures shared by the kernels (*_kernel.cu) and the C ABI (demod_api.cu).
//
// Data layout in HBM (see DESIGN.md):
//   * input: 2 bytes per sample either way (uc8 I,Q pair, or one uint16 magnitude), so one
//     address rule serves both: byte address of data index d = seg.base + 2*d, where data index 0 is
//     the first of the 326 halo samples (readsb.h:450-464 `mag_buf.data`).
//   * a SEGMENT is a run of consecutive preamble start positions of one receiver whose samples are
//     contiguous in memory; it may span several reference "buffers" (boundary every buf_len
//     positions) because consecutive mag_bufs tile the sample axis without gaps
//     (sdr_ifile.c:209-213: the halo of buffer b+1 is the tail of buffer b).
//   * stage A (scan kernel) is stateless per position and writes, per tile of TILE positions, an
//     ordered list of PosEntry (every position that passed a preamble threshold) and an ordered
//     list of Rec (every sliced phase whose score depends on the ICAO filter).
//   * stage B (resolve kernel) walks those lists sequentially per receiver with the receiver's
//     ICAO filter and emits frames.
#pragma once
#include <stdint.h>
#include "b200_demod.h"

#define B200_TRAIL 326

// ---- stage A tiling ----------------------------------------------------------------------------
#define TILE_QUAD_START 0x80000000u  // tile_seg flag: first tile of a quad (four consecutive tiles of a segment, counted from its first tile)
#define SCAN_TILE      2048          // preamble start positions per tile (the unit of stage A output and of stage B's walk)

// ---- segment descriptor ------------------------------------------------------------------------
#define SEG_MAG        0x1u   // input samples are uint16 magnitudes (demodulate2400 hand-off), not uc8 IQ
#define SEG_HALO_ZERO  0x2u   // data indices [0,326) are zeros (first buffer of a stream); memory not read

struct Segment {
    const uint8_t *base;   // byte address of data index 0 (may be unaligned by a multiple of 2)
    int64_t  first_ts;     // 12 MHz timestamp of the first NEW sample (data index 326)
    uint32_t npos;         // preamble start positions = new samples in the segment
    uint32_t buf_len;      // reference buffer length: skip state resets every buf_len positions
    uint32_t lead;         // ((uintptr_t)base & 15) / 2: dummy positions so tile origins are 16B aligned
    uint32_t flags;        // SEG_*
    uint32_t stream;
    uint32_t first_buf;    // index of this segment's first buffer in the run's BufAcc / BufOut arrays
    uint32_t n_bufs;
    uint32_t tile_begin;   // global index of this segment's first tile
    uint32_t n_tiles;
    uint32_t first_seq;    // buffer_seq of the segment's first buffer
    int32_t  thr;          // the receiver's Modes.preambleThreshold for this segment (demod_2400.c:334-338)
    uint32_t pad_;
};

// One position whose preamble correlation reached the threshold (demod_2400.c:344-378).
//   bits 0..12  position relative to the origin of the tile's QUAD (four consecutive tiles of a segment, the unit stage B walks)
//   bits 16..20 phases tried  (bit p = try_phase 4+p)
//   bits 21..25 phases whose score depends on the filter (a Rec follows for each, ascending phase)
typedef uint32_t PosEntry;

// Stateless result of slicing one phase (demod_2400.c:215-258 up to the filter lookups).
enum RecKind : uint8_t {
    K_AP = 1,        // DF0/4/5/16/20/21: score = known(crc) ? 1000 : -1
    K_DFREPAIR = 2,  // DF one bit away from 17 and CRC clean as DF17: known(AA) ? 900 : 700
    K_DF11_FIX = 3,  // DF11, 1-bit error under IID=0: known(AA') ? 800 : -1
    K_DF11_IID0 = 4, // DF11, syndrome 0: known(AA) ? 1600 : 750
    K_DF11_IID = 5,  // DF11, only the IID bits set: known(AA) ? 1000 : -1
    K_ES_OK = 6,     // DF17/18, syndrome 0: known(AA) ? 1800 : 1400
    K_ES_FIX = 7     // DF17/18, 1-bit error: known(AA') ? 900 : 700; rejected later if AA changed and unknown
};

struct __align__(16) Rec {
    uint8_t  msg[14];  // as sliced (uncorrected); bytes 7..13 zero for short frames
    uint8_t  kind;     // RecKind
    int8_t   fixbit;   // K_*_FIX: corrected message bit; K_DFREPAIR: repaired DF bit; else -1
    uint32_t crc;      // syndrome over the frame length of the DF as sliced
    uint32_t addr;     // 24-bit address the filter is asked about
    uint32_t pad_[2];
};

// Score key of a Rec (key_pool, parallel to rec_pool): everything the sequential resolver needs.
#define KEY_AA_CHANGED 0x80000000u   // K_ES_FIX whose corrected bit lies in the AA field (mode_s.c:560)
#define KEY_DF17       0x10000000u   // DF as sliced is 17
#define KEY_LONG       0x08000000u   // DF as sliced is a 112-bit type (demod_2400.c:399)
// bits 24..26 RecKind, bits 0..23 the address the filter is asked about

struct TileOut {
    uint32_t n_pos;    // PosEntry count; entries live at pos_pool[tile * SCAN_TILE ...]
    uint32_t n_rec;
    uint32_t rec_off;  // first Rec in rec_pool
    uint32_t n_found;  // records the tile produced, also when the run's reservation failed (n_rec is 0 then)
};

struct BufAcc {        // exact per-buffer sums (convert.c:75-79), zeroed at the start of a run
    unsigned long long sum_level;
    unsigned long long sum_power;
    unsigned long long sum_signal_power;
    float2 fsum;       // sc16 steps: the converter's float sums (sum_level, sum_power), written by sc16_convert_kernel
};

// ---- per-receiver persistent state (device) -----------------------------------------------------
// The address filter (icao_filter.c): two generations of an open-addressed set.  A receiver starts with tables of
// ICAO_CAP slots (a slab of the context; stage B keeps such a table in shared memory).  The load is kept <= 1/2; a receiver that
// needs more gets tables of its own, as large as it takes (the reference grows to 2^20 buckets, icao_filter.c:45-46), and stage B
// then works on them in global memory.  What the reference's own table SIZE makes observable is modelled exactly: `filter_bits`
// follows icao_filter.c:97-99 and :126-128, and the older generation is dropped when the reference's resize drops it (:66-92).
#define ICAO_CAP_LOG2 12
#define ICAO_CAP      (1u << ICAO_CAP_LOG2)   // slots per generation of the default tables
#define ICAO_EMPTY    0xffffffffu
#define ICAO_MINBITS  8
#define ICAO_MAXBITS  20

struct StreamState {
    uint32_t *tab[2];            // the two generations
    uint32_t cap_log2;           // slots per generation = 1 << cap_log2
    uint32_t grow_log2;          // set by the capacity check when this run could fill a generation beyond 1/2: what the host should grow to
    uint32_t gen_count[2];
    uint32_t active;             // generation that receives adds
    uint32_t filter_bits;        // the reference's filterBits (8..20)
    uint32_t flip_armed;         // 0 until the first flip (readsb.c:1227: next_flip starts at 0)
    uint32_t buffer_seq;         // running buffer number
    int64_t  next_flip_ms;
    b200_demod_stats stats;
};

// ---- run-wide control block (device) ------------------------------------------------------------
struct RunCtl {
    uint32_t rec_alloc;      // atomic bump pointer into rec_pool
    uint32_t pad0_;
    uint32_t overflow;       // OV_* bits
    uint32_t tile_counter;   // dynamic tile scheduler
    uint32_t total_frames;
    uint32_t stage_need;     // with OV_STAGING_FULL: the largest number of live records one tile produced (staging areas too small)
    uint32_t pad_[2];
    uint32_t cap_check;      // stage B's capacity check of this run (resolve_kernel): 0 not yet, 1 in progress, CAP_GO / CAP_STOP made
    uint32_t pad1_[3];
};
#define CAP_STOP 2u          // cap_check: made, stage B must not run (this step is going to be repeated)
#define CAP_GO   3u          // cap_check: made, stage B runs

// RunCtl.overflow
#define OV_REC_POOL_FULL 0x01u   // stage A: rec_pool exhausted
#define OV_STAGING_FULL  0x02u   // stage A: a run of tiles has more live records than the per-warp staging areas hold (RunCtl.stage_need)
#define OV_FRAME_CAP     0x04u   // stage B: a receiver's frame slots exceeded
#define OV_FILTER_GROW   0x08u   // a receiver's ICAO tables have to grow before this run (StreamState.grow_log2)
#define OV_SKIPPED       0x10u   // stage B skipped because the step ahead has to be repeated
#define OV_MODEAC_CAP    0x20u   // Mode A/C candidate / output capacity exceeded
#define OV_STAGE_A_FAILED (OV_REC_POOL_FULL | OV_STAGING_FULL)   // stage A's output is incomplete
#define RUN_REPEAT_BITS (OV_STAGE_A_FAILED | OV_FILTER_GROW | OV_SKIPPED)   // stage B did not run (or must not): the host repairs and repeats the step

struct ScanParams {
    const Segment *segs;
    const uint32_t *tile_seg;    // tile -> segment index | TILE_QUAD_START
    uint32_t n_tiles;
    PosEntry *pos_pool;
    Rec *rec_pool;
    uint32_t *key_pool;          // per Rec: aa_changed << 31 | kind << 24 | addr — all stage B needs to score it
    TileOut *tile_out;
    BufAcc *buf_acc;
    RunCtl *ctl;
    uint32_t rec_cap;            // records rec_pool / key_pool hold
    // A run of ONE segment (one receiver, one buffer: the drop-in's call shape) carries its descriptor in the kernel parameters: no
    // descriptor upload in front of the kernels.  one_seg_valid: segs / tile_seg are not read, every tile belongs to one_seg.
    Segment one_seg;
    uint32_t one_seg_valid;
    uint32_t warps_per_cta;      // set by the launcher: warps of each CTA that take work (a small run is spread over many SMs, few warps each)
    uint32_t need_lut;           // some segment holds uc8 IQ: the magnitude table has to be staged (a pure magnitude hand-off skips it)
    uint32_t long_set, short_set; // valid DF bitsets (demod_2400.c:98-128)
    int32_t nfix, fixdf;
    // per-warp private areas in global memory
    Rec *stage_rec;              // [warp][stage_cap] live records of the tile in progress
    uint32_t *stage_key;
    uint32_t stage_cap;
    uint16_t *q1_over;           // [warp][512] pre-check passers beyond the shared-memory queue (dense input)
    uint32_t *tick_scratch;      // [warp][b200_scan_tick_words()] the ticks of the run in progress (deferred, pooled slicing)
    uint32_t *stream_addable;    // [stream] records of this run that could teach the receiver's filter an address (clean DF17, DF11 with IID 0)
    // Mode A/C contexts: the magnitudes this kernel makes from uc8 IQ anyway, kept for modeac_scan_kernel (which would otherwise run
    // every sample through the table a second time): sample x (tile coordinate) of a segment at mag_copy[seg.tile_begin * SCAN_TILE + x],
    // for the x inside the segment's tiles.  Null: not kept.
    uint16_t *mag_copy;
};

struct ResolveParams {
    const Segment *segs;
    const uint32_t *stream_seg_begin; // per stream: first segment index (segments sorted by stream); [n_streams+1]
    uint32_t n_streams;
    const PosEntry *pos_pool;
    const Rec *rec_pool;
    const uint32_t *key_pool;
    const TileOut *tile_out;
    BufAcc *buf_acc;
    b200_buffer_result *buf_out;      // per run buffer results (n_frames, flip flag, ...)
    StreamState *state;
    b200_frame *frames;               // [n_streams][frame_cap]
    uint32_t frame_cap;
    uint32_t per_buf_cap;             // frames one reference buffer can hold (buf_samples / 113 + 2); frame_cap = buffers per run x this
    RunCtl *ctl;
    const uint32_t *prev_stop;        // asynchronous pipeline: the stop_out of the step ahead of this one (or nullptr)
    uint32_t *stop_out;               // set to 1 when this run's stage B does not run (the run is going to be repeated), else to 0
    int32_t ttl_ms;
    uint32_t *stream_addable;         // [n_streams] upper bound of the filter adds of this run (scan kernel); read and zeroed by the capacity check
    Segment one_seg;                  // (see ScanParams) the run's only segment, when one_seg_valid
    uint32_t one_seg_valid;
    uint32_t solo;                    // one receiver in the context: resolve_solo_kernel (see resolve_kernel.cu)
    uint32_t *frame_span;             // [n_streams][2]: where the receiver's frames start in `packed`, and how many there are
    b200_frame *packed;               // all frames of the run: each receiver's in order, in one contiguous range (frame_span)
    const uint16_t *lut_full;         // 65536-entry UC8 table in global memory (the finalizer's signal power)
    // (solo, optional) the kernel PUBLISHES the run's result block itself: copies publish_head bytes + the packed frames from
    // publish_src (device) to publish_dst (the host's pinned copy, mapped into the device's address space) - no device-to-host
    // copy operation in the stream - and then zeroes the control block and the per-buffer sums for the next run (no memset either)
    const uint4 *publish_src;
    uint4 *publish_dst;
    uint32_t publish_head;            // bytes in front of the packed frames
    uint32_t publish_clear;           // bytes at the start of the block (RunCtl + BufAcc[]) to zero afterwards
    uint16_t *carry_dst;              // (solo, optional) the receiver's arena region: its last 326 samples go to the front for the next run
    const uint16_t *carry_src;        //   (the mag_buf overlap copy, sdr_ifile.c:209-213), or null
};


// ---- Mode A/C (modeac_kernel.cu) -------------------------------------------------------------------
struct DeviceTables;
// Where a reference buffer's Mode A/C noise floor comes from: demodulate2400AC reads mag_buf.mean_level / mean_power
// (demod_2400.c:580-581), i.e. whatever the converter that filled the buffer returned.
#define AC_LEVEL_SUMS   0u   // uc8 input or a plain magnitude hand-off: the scan kernel's exact integer sums (convert.c:100-107)
#define AC_LEVEL_GIVEN  1u   // the caller's mag_buf.mean_level / mean_power (b200_demod_submit_mag_u16_levels)
#define AC_LEVEL_FSUM   2u   // sc16 input: the converter's float accumulators at fsum[idx], divided in float (convert.c:243-249)
struct AcLevel {
    double mean_level, mean_power;
    uint32_t mode, idx;
};

struct AcScanParams {
    const Segment *segs;
    uint32_t n_segs;
    const uint32_t *tile_seg;
    uint32_t n_tiles;
    const BufAcc *buf_acc;            // the scan kernel's exact per-buffer sums: noise floor of demodulate2400AC
    const DeviceTables *tables;
    uint32_t *noise;                  // [buffer] noise_level (demod_2400.c:581)
    uint32_t *bitmap;                 // [tile][SCAN_TILE/32]: bit p = a well-formed reply's F1 pulse starts at position p of the tile
    RunCtl *ctl;
    const AcLevel *levels;            // [buffer]
    const float2 *fsum;               // sc16 float sums (sum_level, sum_power), or null
    const uint16_t *mag_copy;         // (ScanParams) the Mode S scan's magnitudes of the uc8 segments, or null
};

struct AcWalkParams {
    const Segment *segs;
    uint32_t n_segs;
    const uint32_t *stream_seg_begin;
    uint32_t n_streams;
    const uint32_t *bitmap;
    const uint32_t *noise;
    const uint16_t *lut_full;
    b200_modeac *ac_out;              // [buffer][per_buf_cap]
    uint32_t *ac_count;               // [buffer]
    uint32_t per_buf_cap;             // buf_samples / 70 + 2: an accepted reply hides the next 69 positions
    StreamState *state;
    RunCtl *ctl;
};

// ---- sc16 / sc16q11 input (convert_kernel.cu) ----------------------------------------------------
// Buffer g of a step belongs to the segment whose buffers [first_buf, first_buf + n_bufs) hold it: receiver seg.stream, its buffer
// g - seg.first_buf.  Samples are interleaved int16 I,Q (one 32-bit word each).
struct Sc16Params {
    const uint32_t *iq;               // receiver s's first new sample at iq + s * iq_stride; unless its segment has SEG_HALO_ZERO, its 326 raw
                                      // halo samples precede it and are converted too
    uint16_t *mag;                    // receiver s's data index 0 (first halo magnitude) at mag + s * mag_stride
    float2 *sums;                     // buffer g's float sums (sum_level, sum_power) at sums[g * sums_stride]
    const Segment *segs;              // the step's segments (one per receiver present), ascending first_buf; not read when n_segs == 1
    Segment seg0;                     // ... the only one when n_segs == 1 (its descriptors may not be on the device)
    uint64_t iq_stride, mag_stride;   // in samples
    uint32_t sums_stride, n_segs, n_bufs, buf_len;
    float scale;                      // 1 / 32768 (sc16) or 1 / 2048 (sc16q11)
};

enum { ENC_BEAST = 0, ENC_RAW = 1 };

struct EncodeParams {                // beast_kernel.cu: one wire format of a run's records
    const Segment *segs;
    const uint32_t *stream_seg_begin;
    const b200_frame *frames;         // packed (ResolveParams::packed)
    const uint32_t *frame_span;       // [stream][2]: first frame, frame count
    const b200_buffer_result *buf_out;
    const b200_modeac *ac;            // packed in buffer order, or null
    const uint32_t *ac_prefix;        // [buffer + 1], or null
    uint8_t *out;
    uint32_t *stream_off, *stream_len;
    uint32_t *total;
    uint32_t cap;
    uint32_t format;                  // ENC_BEAST or ENC_RAW
    uint32_t flags;                   // B200_BEAST_* or B200_RAW_* of the format
};

// ---- host-built constant tables, uploaded once ---------------------------------------------------
struct DeviceTables {
    uint16_t lut_fold[128 * 128];  // folded + bank-swizzled UC8 magnitude table (see modes_tables.h)
    uint32_t crc_tab[256];         // byte-wise CRC-24 table (crc.c:46-57)
    uint32_t bit_syn[112];         // syndrome of each single bit of a 112-bit frame (crc.c:59-64)
    uint32_t syn_hash[512];        // perfect hash: (syndrome*mul)>>23 -> syndrome<<8 | bit
    uint32_t syn_hash_mul;
    uint32_t pad_[3];
};

#ifdef __cplusplus
extern "C" {
#endif
// kernel launch wrappers implemented in the *_kernel.cu files (stream is a cudaStream_t)
int b200_scan_warps(int n_sm);      // warps of the (persistent) scan kernel's grid
int b200_scan_tick_words(void);     // words of tick scratch per warp
int b200_launch_scan(const ScanParams *p, const DeviceTables *d_tables, int n_sm, void *stream);
int b200_prepare_scan(void);       // per-device kernel attributes (dynamic shared memory opt-in): call with the device current
int b200_prepare_resolve(void);
int b200_prepare_modeac(void);
int b200_launch_resolve(const ResolveParams *p, int any_grown, void *stream);
int b200_launch_init_state(StreamState *state, uint32_t n, uint32_t *slab, void *stream);
int b200_launch_icao_rehash(StreamState *state, uint32_t stream, uint32_t *new0, uint32_t *new1, uint32_t new_log2, void *stream_);
int b200_launch_modeac(const AcScanParams *sp, const AcWalkParams *wp, int n_sm, void *stream);
int b200_prepare_convert(void);
int b200_launch_sc16_convert(const Sc16Params *p, void *stream);
int b200_launch_encode(const EncodeParams *p, uint32_t n_streams, void *stream);
int b200_launch_modeac_pack(const AcWalkParams *wp, uint32_t n_bufs, uint32_t *prefix, b200_modeac *packed, void *stream);
int b200_launch_icao_op(StreamState *state, uint32_t stream, int op, uint32_t addr, int *d_result, void *cstream);
#ifdef __cplusplus
}
#endif
