/*
 * b200_demod.h — C ABI of the Hopper-native Mode-S demodulator.
 *
 * This library replaces exactly one path of wiedehopf/readsb: the 2.4 MSPS Mode-S
 * demodulator (uc8 IQ -> magnitude -> preamble detect -> 5-phase bit slice ->
 * CRC-24 + 1-bit fix -> accepted frames).  Everything else in readsb stays the
 * unchanged C host.  Reference interfaces replaced (file:line in the reference tree):
 *
 *   convert.h:34-39      iq_convert_fn(void *iq, uint16_t *mag, unsigned n, state*,
 *                        double *mean_level, double *mean_power)      -> b200_demod_submit_iq_uc8
 *   demod_2400.h:38      void demodulate2400(struct mag_buf *mag)    -> b200_demod_submit_mag_u16
 *                                                                       + b200_demod_run + b200_demod_fetch
 *   readsb.h:450-464     struct mag_buf {sampleTimestamp, mean_level, mean_power, length, data}
 *                                                                    -> submit arguments + b200_buffer_result
 *   demod_2400.c:401-471 netGetMM / fill timestamp,score,msg,signalLevel / decodeModesMessage
 *                        accept test / netUseMessage                 -> b200_frame (one per accepted frame)
 *   icao_filter.h        icaoFilterAdd / icaoFilterTest / icaoFilterExpire
 *                                                                    -> b200_demod_icao_*
 *   stats.h:62-83        struct stats demod_* counters              -> b200_demod_stats
 *
 * All entry points are plain C (extern "C"), take plain pointers and sizes, and return 0 on
 * success or a negative B200_E_* code; b200_demod_last_error() gives the text.  There is no CPU
 * fallback: if no sm_90 (H100-class) CUDA device is usable, b200_demod_create() fails.
 */
#ifndef B200_DEMOD_H
#define B200_DEMOD_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_DEMOD_ABI_VERSION 2

/* readsb.c:288  trailing_samples = (8 + 112 + 16) us * 2.4 = 326 */
#define B200_TRAILING_SAMPLES 326
/* demod_2400.h:31 PREAMBLE_THRESHOLD_DEFAULT */
#define B200_PREAMBLE_THRESHOLD_DEFAULT 58
/* readsb.h MODES_ICAO_FILTER_TTL: two tables flipped every 60 s (readsb.c:1227-1231) */
#define B200_ICAO_TTL_MS 60000

enum {
    B200_OK = 0,
    B200_E_INVAL = -1,      /* bad argument */
    B200_E_NODEV = -2,      /* no usable CUDA device (no CPU fallback exists) */
    B200_E_CUDA = -3,       /* CUDA runtime error, see b200_demod_last_error */
    B200_E_NOMEM = -4,
    B200_E_STATE = -5,      /* call sequence error (e.g. submit queue full) */
    B200_E_OVERFLOW = -6    /* caller-provided output array too small */
};

/* One accepted Mode-S frame: what demodulate2400() hands to netUseMessage()
 * (demod_2400.c:401-471) restricted to the fields the demodulator itself produces. */
typedef struct b200_frame {
    int64_t  timestamp;     /* 12 MHz: sampleTimestamp + j*5 + (8+56)*12 + phase   (demod_2400.c:406) */
    uint64_t sigpow_sum;    /* sum of mag^2 over signal_len samples from data[j+19] (demod_2400.c:443-446);
                               signalLevel = sigpow_sum / 65535.0 / 65535.0 / signal_len */
    uint32_t j;             /* preamble start: index into mag_buf.data (halo included) */
    uint32_t crc;           /* mm->crc: syndrome after DF repair, before the bit fix (mode_s.c:466) */
    uint32_t addr;          /* mm->addr: AA (DF11/17/18) or CRC-derived address (DF0/4/5/16/20/21) */
    int32_t  score;         /* scoreModesMessage() value of the winning phase (mode_s.c:309) */
    uint32_t buffer_seq;    /* per-stream running number of the buffer this frame was found in */
    uint16_t signal_len;    /* msglen*12/5 with msglen taken from the UNrepaired DF (demod_2400.c:399,439) */
    uint8_t  phase;         /* winning try_phase 4..8 */
    uint8_t  msgtype;       /* DF after DF17 repair (mm->msgtype) */
    uint8_t  msgbits;       /* 56 or 112 (mm->msgbits) */
    uint8_t  correctedbits; /* 0 or 1 (mm->correctedbits) */
    int8_t   fix_bit;       /* -1: none; 0..4: repaired DF bit; 5..111: CRC-corrected bit.
                               raw (as-received) frame = msg with this message bit flipped back */
    uint8_t  flags;         /* B200_FRAME_* */
    uint8_t  msg[14];       /* corrected frame (mm->msg after decodeModesMessage); bytes >= msgbits/8 are 0 */
    uint8_t  pad_[6];
} b200_frame;

#define B200_FRAME_ICAO_ADDED 0x01 /* this frame caused icaoFilterAdd(addr) (mode_s.c:766-779) */

/* One Mode A/C reply found by demodulate2400AC() (demod_2400.c:575-761): what it hands to decodeModeAMessage(). */
typedef struct b200_modeac {
    int64_t  timestamp;     /* 12 MHz: sampleTimestamp + f2_clock/5, i.e. at the F2 framing pulse (demod_2400.c:745) */
    uint32_t f1_sample;     /* index into mag_buf.data of the F1 pulse */
    uint16_t modeac;        /* 00 A4 A2 A1 00 B4 B2 B1 SPI C4 C2 C1 00 D4 D2 D1 (demod_2400.c:716-731) */
    uint16_t buffer_idx;    /* which buffer of the run (index into b200_demod_buffer_results) */
} b200_modeac;

/* Per (stream, buffer) scalars: what convert_uc8_nodc() returns (convert.c:100-107) and what
 * demodulate2400() folds into noise stats (demod_2400.c:474-479), kept as exact integers. */
typedef struct b200_buffer_result {
    int64_t  sample_timestamp;  /* as submitted */
    uint64_t sum_level;         /* sum of mag over the buffer's new samples; mean_level = sum/65536.0/length */
    uint64_t sum_power;         /* sum of mag^2;  mean_power = sum/65535.0/65535.0/length */
    uint64_t sum_signal_power;  /* sum of sigpow_sum over frames accepted in this buffer */
    uint32_t length;            /* new samples in this buffer */
    uint32_t n_frames;          /* frames accepted in this buffer */
    uint32_t buffer_seq;
    uint32_t icao_flipped;      /* 1 if the ICAO filter tables were flipped after this buffer */
    /* what demodulate2400() added to Modes.stats_current while it worked on this buffer (stats.h:62-83): a caller that keeps
     * readsb's statistics needs no second call per buffer */
    uint32_t demod_preambles;
    uint32_t demod_rejected_bad;
    uint32_t demod_rejected_unknown_icao;
    uint32_t demod_accepted[2];         /* by correctedbits */
    uint32_t demod_preamblePhase[5];    /* every phase tried (demod_2400.c:216) */
    uint32_t demod_bestPhase[5];
    uint32_t pad_;
} b200_buffer_result;

/* Cumulative per-stream counters = Modes.stats_current demod_* (stats.h:62-83). */
typedef struct b200_demod_stats {
    uint64_t samples_processed;
    uint64_t demod_preambles;
    uint64_t demod_rejected_bad;
    uint64_t demod_rejected_unknown_icao;
    uint64_t demod_accepted[2];       /* by correctedbits */
    uint64_t demod_preamblePhase[5];  /* every phase tried (demod_2400.c:216) */
    uint64_t demod_bestPhase[5];
    uint64_t signal_power_count;      /* sum of signal_len */
    uint64_t sum_signal_power;        /* sum of sigpow_sum (integer form of signal_power_sum) */
    uint64_t strong_signal_count;     /* signalLevel > 0.50119 */
    double   peak_signal_power;       /* highest signalLevel seen (stats.h peak_signal_power) */
    uint64_t demod_modeac;            /* Mode A/C replies (stats.h demod_modeac) */
    uint64_t buffers;
    uint64_t icao_flips;
} b200_demod_stats;

typedef struct b200_demod_config {
    uint32_t struct_size;           /* = sizeof(b200_demod_config) */
    int32_t  device;                /* CUDA ordinal; -1 = current device */
    uint32_t n_streams;             /* independent receivers handled by this context */
    uint32_t buf_samples;           /* Modes.sdr_buf_samples: max new samples per buffer (readsb.c:2212) */
    uint32_t max_buffers_per_run;   /* how many buffers per stream one b200_demod_run may process */
    int32_t  preamble_threshold;    /* Modes.preambleThreshold, 0 -> 58 (readsb.c:2268-2270) */
    int32_t  nfix_crc;              /* 0 or 1 (--fix / --no-fix, readsb.c:1460-1464) */
    int32_t  fix_df;                /* 0 or 1 (--no-fix-df, readsb.c:1467) */
    int32_t  icao_ttl_ms;           /* automatic filter flip period in stream time, <0 = never, 0 -> 60000 */
    uint32_t flags;                 /* B200_CFG_* */
} b200_demod_config;

#define B200_CFG_MODE_AC 0x1u   /* also run the Mode A/C demodulator on every buffer (--modeac, readsb.c:872-874) */
#define B200_CFG_NO_TIMING 0x2u /* blocking runs record no CUDA events between the kernels (b200_demod_last_timing then reports zeros): every
                                   event is an operation of its own in the stream, and a one-buffer run is short enough for that to show */

typedef struct b200_demod_ctx b200_demod_ctx;

/* lifecycle ------------------------------------------------------------------------------------ */
int  b200_demod_abi_version(void);
int  b200_demod_create(const b200_demod_config *cfg, b200_demod_ctx **out);
void b200_demod_destroy(b200_demod_ctx *ctx);
const char *b200_demod_last_error(const b200_demod_ctx *ctx); /* ctx may be NULL: last create error */

/* Modes.preambleThreshold for the runs that follow (create() took the initial value from the config).  The reference
 * re-reads it for every buffer and raises it to at least 75 while its 15-minute statistics show dropped samples
 * (demod_2400.c:334-338, PREAMBLE_THRESHOLD_PIZERO): a live-SDR caller applies that rule here, buffer by buffer. */
int b200_demod_set_preamble_threshold(b200_demod_ctx *ctx, int32_t preamble_threshold);

/* Run all work of this context on the caller's CUDA stream (a cudaStream_t passed as void*; NULL = the
 * context's own stream).  Lets a caller bracket runs with its own events. */
int b200_demod_set_stream(b200_demod_ctx *ctx, void *cuda_stream);

/* pinned host memory for zero-staging submits (optional; any host pointer is accepted) */
void *b200_demod_host_alloc(size_t bytes);
void  b200_demod_host_free(void *p);
/* ... or page-lock memory the caller already owns - e.g. readsb's ring of mag_bufs (readsb.h:113,855), allocated once at start-up:
 * a submit from pageable memory is staged by the driver and costs several times the copy itself. */
int   b200_demod_host_register(void *p, size_t bytes);
int   b200_demod_host_unregister(void *p);

/* host-buffer path (the drop-in) ---------------------------------------------------------------
 * submit_iq_uc8 replaces the converter call a frontend makes (sdr_ifile.c:241, sdr_rtlsdr.c:395):
 * `iq` holds nsamples interleaved unsigned 8-bit I,Q pairs; the halo of 326 preceding samples is
 * kept by the library (zeros for the first buffer of a stream, sdr_ifile.c:209-213).
 * submit_mag_u16 replaces demodulate2400(mag): `data` is mag_buf.data, i.e. 326 halo magnitudes
 * followed by `length` new ones.  Buffers of one stream are processed in submission order.
 * A stream must not mix the two submit kinds. */
int b200_demod_submit_iq_uc8(b200_demod_ctx *ctx, uint32_t stream, const uint8_t *iq,
                             uint32_t nsamples, int64_t sample_timestamp);
int b200_demod_submit_mag_u16(b200_demod_ctx *ctx, uint32_t stream, const uint16_t *data,
                              uint32_t length, int64_t sample_timestamp);
/* The same hand-off with mag_buf.mean_level / mean_power (readsb.h:452-453) as the converter that filled the buffer
 * returned them.  demodulate2400AC derives its noise floor from these two fields (demod_2400.c:580-581); for a uc8
 * frontend they equal what the library computes itself from the magnitudes (convert.c:100-107), so submit_mag_u16 is
 * enough there; the sc16 converters return float-accumulated means (convert.c:243-249) and DC-filtered ones differ too —
 * with B200_CFG_MODE_AC and such a frontend hand the buffer over with this call.  Without B200_CFG_MODE_AC the levels
 * are not used by the library (demodulate2400 itself only needs mean_power for its noise statistics, on the caller's side). */
int b200_demod_submit_mag_u16_levels(b200_demod_ctx *ctx, uint32_t stream, const uint16_t *data,
                                     uint32_t length, int64_t sample_timestamp, double mean_level, double mean_power);
/* Many receivers in one call (a multi-channel frontend's slab): stream first_stream+i has n_buffers*buf_len
 * samples at iq + i*host_stride_bytes, submitted as n_buffers consecutive buffers with timestamps
 * first_sample_timestamp + b*buf_len*5.  One strided DMA instead of n_streams*n_buffers copies. */
int b200_demod_submit_iq_uc8_strided(b200_demod_ctx *ctx, uint32_t first_stream, uint32_t n_streams,
                                     const uint8_t *iq, uint64_t host_stride_bytes, uint32_t n_buffers,
                                     uint32_t buf_len, int64_t first_sample_timestamp);
/* The float-path converters for 16-bit frontends (bladeRF, Pluto, Soapy): replaces iq_convert_fn for INPUT_SC16
 * (convert_sc16_nodc, convert.c:212-250: I / 32768) and, with q11 != 0, INPUT_SC16Q11 (convert_sc16q11_nodc,
 * convert.c:329-367: I / 2048; the default build has no table path).  `iq` holds nsamples interleaved little-endian
 * int16 I,Q pairs; halo handling as for submit_iq_uc8.  Magnitudes are the reference's, bit for bit.  The reference
 * returns mean_level / mean_power of these formats from float accumulators added to in sample order: for buffers
 * submitted here b200_buffer_result.sum_level / sum_power hold the IEEE-754 bit patterns of those two float sums
 * (mean_level = (double)(sum_level_f / (float)length), likewise mean_power); with B200_CFG_MODE_AC the Mode A/C noise
 * floor of such a buffer is derived from exactly these means, as the reference does.  Not combinable with other submit
 * kinds on the same stream in one run. */
int b200_demod_submit_iq_sc16(b200_demod_ctx *ctx, uint32_t stream, const int16_t *iq, uint32_t nsamples,
                              int64_t sample_timestamp, int q11);
/* Process everything submitted since the last run; returns when frames are in host memory. */
int b200_demod_run(b200_demod_ctx *ctx);

/* device-resident path (inputs already in HBM) ------------------------------------------------
 * d_iq: device pointer; stream s starts at d_iq + s*stream_stride_bytes and holds
 * n_buffers*buf_len contiguous uc8 IQ samples which are processed as n_buffers consecutive
 * buffers of buf_len samples.  `continues` != 0 means the 326 samples before each stream's first
 * sample (at negative offset) are valid halo from the previous call; 0 means stream start (zero halo).
 * first_sample_timestamp applies to every stream.  Frames are fetched as for b200_demod_run. */
int b200_demod_run_device_uc8(b200_demod_ctx *ctx, const uint8_t *d_iq, uint64_t stream_stride_bytes,
                              uint32_t n_buffers, uint32_t buf_len, int continues,
                              int64_t first_sample_timestamp);

/* Asynchronous form of the call above: returns once the step is enqueued; at most three steps may be in flight.
 * b200_demod_wait() completes the OLDEST step in flight and makes its results current for the fetch calls below.
 * The GPU never waits for the host between steps: the scan of step n+1 is queued behind the scan of step n, stage B of
 * step n runs as soon as its scan ends; per-receiver state still advances strictly in step order.
 * The host-buffer calls, get_stats and the icao_* calls need an empty pipeline. */
int b200_demod_run_device_uc8_async(b200_demod_ctx *ctx, const uint8_t *d_iq, uint64_t stream_stride_bytes,
                                    uint32_t n_buffers, uint32_t buf_len, int continues,
                                    int64_t first_sample_timestamp);
int b200_demod_wait(b200_demod_ctx *ctx);

/* Pipelined host-buffer step: what readsb's reader thread / decode thread pair does with its ring of mag_bufs
 * (sdr_ifile.c:194-259 fills the next buffers while readsb.c:871 demodulates the current one), for all receivers of the
 * context at once.  h_iq is a HOST slab laid out like submit_iq_uc8_strided's (receiver s at h_iq + s*host_stride_bytes,
 * n_buffers*buf_len uc8 IQ samples, first_sample_timestamp for every receiver); pin it (b200_demod_host_alloc) or the
 * copy is synchronous.  The call returns once the step is enqueued: the slab goes to one of three library-owned device
 * buffers on a copy stream of its own, so the copies of later steps overlap the kernels of earlier ones; the slab may be reused
 * after the b200_demod_wait() that completes this step.  At most three steps in flight, completed in order by
 * b200_demod_wait(), results fetched as usual.  `continues` != 0: these samples follow the previous run_host_uc8_async
 * step's without a gap (its last 326 samples become the halo, sdr_ifile.c:209-213; that step must have held >= 326
 * samples per receiver); 0: receiver start (zero halo).  buf_len must be a multiple of 8.  This path keeps its own halo:
 * it does not continue receivers fed through submit_* / run. */
int b200_demod_run_host_uc8_async(b200_demod_ctx *ctx, const uint8_t *h_iq, uint64_t host_stride_bytes,
                                  uint32_t n_buffers, uint32_t buf_len, int continues,
                                  int64_t first_sample_timestamp);

/* The three calls above for 16-bit frontends (INPUT_SC16: Pluto, SoapySDR devices such as Airspy and SDRplay; INPUT_SC16Q11:
 * bladeRF), argument for argument, plus q11 as in b200_demod_submit_iq_sc16 (0: convert_sc16_nodc, I / 32768; nonzero:
 * convert_sc16q11_nodc, I / 2048).  Each receiver's samples are interleaved little-endian int16 I,Q pairs, 4 bytes per sample,
 * so stream_stride_bytes / host_stride_bytes must be at least n_buffers * buf_len * 4; d_iq and stream_stride_bytes 16-byte
 * aligned and buf_len a multiple of 8, as for uc8.  continues != 0 means: device path, the 326 samples (1304 bytes) before each
 * receiver's first sample are valid halo; host path, the previous run_host_sc16_async step's last 326 samples become the halo
 * (a previous run_host_uc8_async step does not count: B200_E_STATE).
 * One converter launch per step turns every receiver's halo and buffers into magnitudes, bit for bit the reference's, in a
 * library-owned slab (allocated on the first such step), ahead of the scan on the same stream; a repeated step converts again.
 * b200_buffer_result.sum_level / sum_power hold the IEEE-754 bit patterns of the reference's two float sums of each buffer, as for
 * submit_iq_sc16; with B200_CFG_MODE_AC they give the Mode A/C noise floor.  Steps of both formats share the three pipeline
 * slots, b200_demod_wait and the fetch calls. */
int b200_demod_run_device_sc16(b200_demod_ctx *ctx, const int16_t *d_iq, uint64_t stream_stride_bytes,
                               uint32_t n_buffers, uint32_t buf_len, int continues,
                               int64_t first_sample_timestamp, int q11);
int b200_demod_run_device_sc16_async(b200_demod_ctx *ctx, const int16_t *d_iq, uint64_t stream_stride_bytes,
                                     uint32_t n_buffers, uint32_t buf_len, int continues,
                                     int64_t first_sample_timestamp, int q11);
int b200_demod_run_host_sc16_async(b200_demod_ctx *ctx, const int16_t *h_iq, uint64_t host_stride_bytes,
                                   uint32_t n_buffers, uint32_t buf_len, int continues,
                                   int64_t first_sample_timestamp, int q11);

/* independent live receivers in one step ------------------------------------------------------
 * The calls above give every receiver of a step the same buffer count, timestamp, halo rule and threshold.  Live SDRs are not in
 * lockstep: they start at different times, their sample clocks drift, and each drops blocks on its own when readsb's FIFO is full
 * (sdr_rtlsdr.c:345-359; the buffer after a drop starts with a zero halo, sdr_rtlsdr.c:381-385, and while samples were dropped
 * recently the receiver's preamble threshold is at least 75, demod_2400.c:334-338).  The _rx calls take one descriptor per receiver
 * of the context (rx[0 .. n_streams-1]). */
typedef struct b200_rx_step {
    int64_t  first_sample_timestamp; /* this receiver's 12 MHz clock at its first new sample */
    uint32_t n_buffers;              /* buffers this receiver delivers in this step, 0 .. max_buffers_per_run; 0 = not in this step */
    uint32_t flags;                  /* B200_RX_CONTINUES: these samples follow this receiver's previous ones without a gap */
    int32_t  preamble_threshold;     /* 0: the context's (b200_demod_set_preamble_threshold); else this receiver's, > 0 */
    uint32_t reserved_;              /* must be 0 */
} b200_rx_step;                      /* 24 bytes */
#define B200_RX_CONTINUES 0x1u
enum { B200_FORMAT_UC8 = 0, B200_FORMAT_SC16 = 1, B200_FORMAT_SC16Q11 = 2 };

/* format: B200_FORMAT_UC8 (uc8 I,Q, 2 bytes per sample), _SC16 or _SC16Q11 (int16 I,Q, 4 bytes per sample, converted as by
 * b200_demod_run_device_sc16 with q11 = 0 / 1).  Receiver s's rx[s].n_buffers * buf_len samples start at d_iq + s * stream_stride_bytes
 * (h_iq + s * host_stride_bytes) and are processed as rx[s].n_buffers consecutive buffers of buf_len samples with timestamps
 * rx[s].first_sample_timestamp + b * buf_len * 5; the stride must hold the largest count of the step.  d_iq and stream_stride_bytes
 * 16-byte aligned, buf_len a multiple of 8, at most buf_samples, as for the calls above.
 *   B200_RX_CONTINUES, device path: the 326 samples in front of the receiver's first sample are valid halo (else: zero halo).
 *   B200_RX_CONTINUES, host path: the receiver's last run_host_* step of the same sample width (uc8 or sc16) gives the halo, also if the
 *     receiver was absent from the steps in between; that step must have left it >= 326 samples, else B200_E_STATE.  The library keeps
 *     every receiver's last 326 raw samples in a store of its own (allocated with the pipelined input buffers).  The host slab is copied
 *     in one strided copy of the largest count's bytes per receiver: every row must be readable that far.
 *   n_buffers == 0: the receiver is absent: no buffer results, no frames; its filter, flip clock, buffer sequence and (host path)
 *     stored halo stay as they are.  A step may leave every receiver absent.
 *   preamble_threshold: what demod_2400.c:334-338 uses for this receiver's buffers of this step (e.g. max(75, threshold) while its
 *     samples_dropped is non-zero); 0 = the context's.
 * Refused with B200_E_INVAL before anything is enqueued or changed (no halo stored, no pipeline slot taken): a bad format, n_buffers
 * above max_buffers_per_run, a negative threshold, non-zero reserved_ or unknown flag bits, a stride too small for the largest count,
 * the alignment / buf_len rules, and buffers shorter than the 326-sample halo other than one per step without B200_RX_CONTINUES (the
 * reference gives the buffer after a short one a zero halo, sdr_ifile.c:207-212).  Results, waits and pipelining as for the calls
 * above; the uniform calls are these calls with one descriptor repeated. */
int b200_demod_run_device_rx(b200_demod_ctx *ctx, int format, const void *d_iq, uint64_t stream_stride_bytes, uint32_t buf_len,
                             const b200_rx_step *rx);
int b200_demod_run_device_rx_async(b200_demod_ctx *ctx, int format, const void *d_iq, uint64_t stream_stride_bytes, uint32_t buf_len,
                                   const b200_rx_step *rx);
int b200_demod_run_host_rx_async(b200_demod_ctx *ctx, int format, const void *h_iq, uint64_t host_stride_bytes, uint32_t buf_len,
                                 const b200_rx_step *rx);
/* The host-buffer path's form of a dropped block (sdr_rtlsdr.c:381-385, oracle_stream_restart): the receiver's next buffer given to
 * submit_iq_uc8 / submit_iq_uc8_strided / submit_iq_sc16 starts with a zero halo instead of the previous buffer's tail.  Buffers of
 * the same run already pending keep theirs; the restart falls between them and the next one.  No effect on magnitude hand-offs,
 * which bring their halo with them. */
int b200_demod_restart_stream(b200_demod_ctx *ctx, uint32_t stream);

/* results of the last run ---------------------------------------------------------------------- */
int b200_demod_frame_count(b200_demod_ctx *ctx, uint32_t stream, uint32_t *n);
int b200_demod_fetch(b200_demod_ctx *ctx, uint32_t stream, b200_frame *out, uint32_t cap, uint32_t *n);
int b200_demod_buffer_results(b200_demod_ctx *ctx, uint32_t stream, b200_buffer_result *out,
                              uint32_t cap, uint32_t *n);
int b200_demod_total_frames(b200_demod_ctx *ctx, uint64_t *n); /* all streams, last run */
/* Mode A/C replies of the last run (contexts created with B200_CFG_MODE_AC), in order */
int b200_demod_fetch_modeac(b200_demod_ctx *ctx, uint32_t stream, b200_modeac *out, uint32_t cap, uint32_t *n);
int b200_demod_get_stats(b200_demod_ctx *ctx, uint32_t stream, b200_demod_stats *out);

/* Beast binary records of the last run's accepted frames of one stream, encoded on the device, byte-identical to what
 * modesSendBeastOutput (net_io.c:1655-1714, netTimestamp :1617-1648) writes to a beast_out client for the same frames:
 * 0x1a, '2' | '3' | '1', 6-byte big-endian 12 MHz timestamp, signal byte, frame bytes, 0x1a doubled.  Order as the
 * reference emits them: per buffer the Mode S frames, then (B200_CFG_MODE_AC) the Mode A/C replies (readsb.c:871-874).
 * flags: B200_BEAST_VERBATIM = bytes as received (Modes.net_verbatim / mm->verbatim) instead of the corrected frame.
 * The forwarding policy of outputMessage (net_io.c:5820-5880: first message of an aircraft suppressed unless CRC-clean,
 * --net-verbatim, ...) belongs to the tracker and is not applied: every accepted frame is encoded.
 * *nbytes = size of the stream's records; B200_E_OVERFLOW if cap is smaller (nothing copied). */
#define B200_BEAST_VERBATIM 0x1u
#define B200_BEAST_MAX_RECORD 44
int b200_demod_fetch_beast(b200_demod_ctx *ctx, uint32_t stream, uint32_t flags, uint8_t *out, uint32_t cap, uint32_t *nbytes);

/* Raw (AVR) text records of the same frames and replies, encoded on the device, byte-identical to what readsb writes for them:
 * by default the network record of modesSendRawOutput (net_io.c:1837-1863, a raw_out client / --net-ro-port), with
 * B200_RAW_STDOUT the frame line of --raw on standard output (displayModesMessage, mode_s.c:1835-1841).
 *   prefix   '*'; with B200_RAW_MLAT (Modes.mlat) and a non-zero timestamp '@' + "%012" PRIX64 of the 12 MHz timestamp.
 *            A timestamp of 13 or more hex digits (>= 2^48, or negative, printed as unsigned) keeps only its first 12 digits
 *            in the network record (the reference steps 13 bytes past the sprintf and the frame hex overwrites the rest);
 *            the stdout line prints every digit.
 *   frame    network: uppercase hex of the corrected frame, or with B200_RAW_VERBATIM (Modes.net_verbatim) of the bytes as
 *            received; stdout: lowercase hex of the corrected frame.  A Mode A/C reply is two bytes (msgbits 16, mode_ac.c:171-173).
 *   end      ";\n".
 * Order, coverage and the cache of the encoded run are those of b200_demod_fetch_beast: the last run or the last completed
 * step (also while the next asynchronous step is in flight), per buffer the Mode S frames then the Mode A/C replies; an absent
 * receiver has 0 bytes.  The forwarding policy of outputMessage (first message of an aircraft held back, 2-bit repairs only
 * with --net-verbatim, no MLAT-sourced frames) belongs to the tracker and is not applied: every accepted frame is encoded.
 * *nbytes = size of the stream's records; B200_E_OVERFLOW if cap is smaller (nothing copied).  B200_E_INVAL for unknown flag
 * bits and for B200_RAW_STDOUT | B200_RAW_VERBATIM (the stdout line always prints the corrected frame). */
#define B200_RAW_MLAT       0x1u
#define B200_RAW_VERBATIM   0x2u
#define B200_RAW_STDOUT     0x4u
#define B200_RAW_MAX_RECORD 48
int b200_demod_fetch_raw(b200_demod_ctx *ctx, uint32_t stream, uint32_t flags, uint8_t *out, uint32_t cap, uint32_t *nbytes);

/* ICAO address filter (icao_filter.h) — per stream, lives next to the resolver on the device.
 * Capacity: 2048 addresses per generation (two generations, entries live for one to two flip periods like the reference's).
 * The reference's tables grow instead (icao_filter.c:47-90, up to 2^20 buckets): a receiver never comes near the limit here
 * (a few hundred aircraft in two minutes), but a process that forwards an aggregator's network-input addresses with
 * b200_demod_icao_add can; B200_E_OVERFLOW from add / run then says so — nothing is dropped silently. */
int b200_demod_icao_add(b200_demod_ctx *ctx, uint32_t stream, uint32_t addr);
int b200_demod_icao_test(b200_demod_ctx *ctx, uint32_t stream, uint32_t addr, int *present);
int b200_demod_icao_expire(b200_demod_ctx *ctx, uint32_t stream);
int b200_demod_icao_reset(b200_demod_ctx *ctx, uint32_t stream);

/* instrumentation: device time (ms) of the last run, by CUDA events on the library's stream:
 * [0] whole run, [1] scan kernel (stage A; in an sc16 step the converter and the scan), [2] resolve kernel (stage B), [3] H2D, [4] D2H.
 * kernel_launches = number of the library's own kernel launches in the last run. */
int b200_demod_last_timing(b200_demod_ctx *ctx, float ms[5], uint32_t *kernel_launches);

/* test instrumentation: [0] tiles, [1] threshold-passing positions, [2] filter-dependent records,
 * [3] record pool use, [4] overflow flags, [5] segments, [6] buffers, [7] frames — of the last run */
int b200_demod_debug_counters(b200_demod_ctx *ctx, uint64_t out[8]);

/* UC8 lookup table the device uses (convert.c:35-62), 65536 entries, index = I*256+Q. */
int b200_demod_uc8_lut(uint16_t *out65536);

#ifdef __cplusplus
}
#endif
#endif /* B200_DEMOD_H */
