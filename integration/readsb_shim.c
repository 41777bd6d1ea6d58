/*
 * readsb_shim.c — the reference-side binding for the demodulator path.
 *
 * Not part of the library and not built by this repository's build(): it is glue a readsb maintainer adds,
 * compiled against readsb's own headers.  Link an UNMODIFIED readsb with
 *
 *     gcc -c -I<readsb> -I<this repo>/include readsb_shim.c
 *     ... readsb objects ... readsb_shim.o -Wl,--wrap=demodulate2400 -Wl,--wrap=demodulate2400AC \
 *         -Wl,--wrap=icaoFilterAdd -Wl,--wrap=icaoFilterExpire -L<this repo>/readsb_b200 -lb200demod
 *
 * (`make -C oracle readsb-pair` does exactly that where the reference tree is present and leaves
 * oracle/_ref/readsb_cpu — the stock build — and oracle/_ref/readsb_b200 side by side; tests/test_gpu_shim.py
 * replays the same capture through both and diffs every frame line and every demodulator counter.)
 *
 * readsb.o's calls `demodulate2400(buf)` / `demodulate2400AC(buf)` (readsb.c:871-874) then resolve to the
 * __wrap_ functions below; every other symbol of demod_2400.o stays as it is, and __real_demodulate2400
 * remains available (it is never used as a fallback here: if the GPU path fails the shim calls setExit(2),
 * readsb.h:406-409 style).
 *
 * What stays on the host, unchanged: netGetMM / decodeModesMessage (field decoding, comm_b, CPR) /
 * netUseMessage / netDrainMessageBuffers, the tracker, all network I/O.  What moves to the GPU: everything
 * demodulate2400() computes up to the accept decision, including the ICAO filter lookups.  The host filter
 * (icao_filter.c) keeps existing for network-input decoding (net_io.c:3916); the two are kept in step by
 * forwarding host-side adds and the 60 s flip (readsb.c:1227-1231) to the library.
 */
#include "readsb.h"
#include "b200_demod.h"

static b200_demod_ctx *g_ctx;
static int g_in_shim;                /* adds that come from our own decodeModesMessage calls are already on the device */
static b200_frame g_frames[2048];
static b200_modeac *g_ac;            /* replies of the buffer demodulate2400 just handed to the library */
static uint32_t g_ac_cap;
static int32_t g_thr;                /* threshold the library currently uses */
static void *g_pinned[MODES_MAG_BUFFERS + 4];   /* mag_buf.data arrays already page-locked for the GPU's copy engine */
static int g_npinned;

/* readsb allocates its ring of mag_bufs once (readsb.c:283-300) and re-uses the same `data` arrays for ever: page-lock each one the
 * first time it is handed over, so that the upload is a direct DMA instead of a staged copy. */
static void pin_once(struct mag_buf *mag) {
    for (int i = 0; i < g_npinned; i++) if (g_pinned[i] == (void *) mag->data) return;
    if (g_npinned >= (int) (sizeof g_pinned / sizeof g_pinned[0])) return;
    if (b200_demod_host_register(mag->data, ((size_t) Modes.sdr_buf_samples + Modes.trailing_samples) * sizeof(uint16_t)) == B200_OK)
        g_pinned[g_npinned++] = mag->data;
}

/* readsb_shim_iq.c (optional, -Wl,--wrap=init_converter): the raw IQ the converter hook kept for a mag_buf */
int b200_shim_iq_lookup(const uint16_t *mag_data, const uint8_t **iq, unsigned *n) __attribute__((weak));

void __real_icaoFilterAdd(uint32_t addr);
void __real_icaoFilterExpire(void);

void __wrap_icaoFilterAdd(uint32_t addr) {
    __real_icaoFilterAdd(addr);
    if (g_ctx && !g_in_shim) b200_demod_icao_add(g_ctx, 0, addr);      /* learned from network input */
}

void __wrap_icaoFilterExpire(void) {
    __real_icaoFilterExpire();
    if (g_ctx) b200_demod_icao_expire(g_ctx, 0);
}

static int shim_open(void) {
    b200_demod_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.struct_size = sizeof cfg;
    cfg.device = -1;
    cfg.n_streams = 1;                                   /* one receiver per readsb process */
    cfg.buf_samples = Modes.sdr_buf_samples;             /* readsb.c:2212 */
    cfg.max_buffers_per_run = 1;                         /* the decode loop hands over one mag_buf at a time */
    cfg.preamble_threshold = (int32_t) Modes.preambleThreshold;
    cfg.nfix_crc = Modes.nfix_crc ? 1 : 0;
    cfg.fix_df = Modes.fixDF;
    cfg.icao_ttl_ms = -1;                                /* flips are driven by backgroundTasks through the wrap above */
    cfg.flags |= B200_CFG_NO_TIMING;                     /* one buffer per call: keep CUDA events out of the stream */
    if (Modes.mode_ac || Modes.mode_ac_auto) {           /* readsb.c:872: Mode A/C runs on the same buffers */
        cfg.flags |= B200_CFG_MODE_AC;
        g_ac_cap = cfg.buf_samples / 70 + 2;
        g_ac = malloc(g_ac_cap * sizeof *g_ac);
        if (!g_ac) return -1;
    }
    if (b200_demod_create(&cfg, &g_ctx) != B200_OK) {
        fprintf(stderr, "b200 demodulator: %s\n", b200_demod_last_error(NULL));
        return -1;
    }
    g_thr = cfg.preamble_threshold;
    return 0;
}

void __wrap_demodulate2400(struct mag_buf *mag) {
    if (!g_ctx && shim_open() < 0) { setExit(2); return; }

    /* demod_2400.c:283-285 */
    if (Modes.sdr_type == SDR_IFILE && Modes.synthetic_now) Modes.synthetic_now = mag->sysTimestamp;

    /* demod_2400.c:334-338: fewer preamble detections while samples were dropped recently (live SDRs) */
    int32_t thr = (int32_t) Modes.preambleThreshold;
    if (Modes.stats_15min.samples_dropped && thr < PREAMBLE_THRESHOLD_PIZERO) thr = PREAMBLE_THRESHOLD_PIZERO;
    if (thr != g_thr && b200_demod_set_preamble_threshold(g_ctx, thr) == B200_OK) g_thr = thr;

    uint32_t n = 0;
    const uint8_t *iq = NULL;
    unsigned iq_n = 0;
    int rc_submit;
    if (b200_shim_iq_lookup && b200_shim_iq_lookup(mag->data + Modes.trailing_samples, &iq, &iq_n) && iq_n == mag->length) {
        /* converter hook active: the frontend's raw uc8 IQ goes up, convert_uc8_nodc (convert.c:64-108) runs on the GPU.  The library
         * keeps the halo on this branch: after dropped samples it must start from zeros, as sdr_rtlsdr.c:381-385 does */
        rc_submit = mag->dropped ? b200_demod_restart_stream(g_ctx, 0) : B200_OK;
        if (rc_submit == B200_OK) rc_submit = b200_demod_submit_iq_uc8(g_ctx, 0, iq, mag->length, mag->sampleTimestamp);
    } else {
        iq = NULL;
        pin_once(mag);
        /* mean_level / mean_power travel with the buffer: demodulate2400AC's noise floor is made from them (demod_2400.c:580-581),
         * whatever converter filled the mag_buf */
        rc_submit = b200_demod_submit_mag_u16_levels(g_ctx, 0, mag->data, mag->length, mag->sampleTimestamp, mag->mean_level, mag->mean_power);
    }
    if (rc_submit != B200_OK ||
        b200_demod_run(g_ctx) != B200_OK ||
        b200_demod_fetch(g_ctx, 0, g_frames, sizeof g_frames / sizeof g_frames[0], &n) != B200_OK) {
        fprintf(stderr, "b200 demodulator: %s\n", b200_demod_last_error(g_ctx));
        setExit(2);
        return;
    }

    uint64_t sum_scaled_signal_power = 0;
    for (uint32_t i = 0; i < n; i++) {
        const b200_frame *f = &g_frames[i];
        struct modesMessage *mm = netGetMM(&Modes.netMessageBuffer[0]);          /* demod_2400.c:401 */
        mm->timestamp = f->timestamp;                                            /* :406 */
        mm->sysTimestamp = mag->sysTimestamp + receiveclock_ms_elapsed(mag->sampleTimestamp, mm->timestamp);
        if (Modes.sdr_type == SDR_IFILE && Modes.synthetic_now) Modes.synthetic_now = mm->sysTimestamp;
        mm->score = f->score;
        /* decodeModesMessage wants the frame as received: undo the library's correction */
        memcpy(mm->msg, f->msg, MODES_LONG_MSG_BYTES);
        if (f->fix_bit >= 0) mm->msg[f->fix_bit >> 3] ^= (unsigned char) (1 << (7 - (f->fix_bit & 7)));
        g_in_shim = 1;
        int result = decodeModesMessage(mm);                                     /* :421, field decoding stays on the host */
        g_in_shim = 0;
        if (result < 0) {
            /* The library's filter follows icao_filter.c's semantics (table resize included), so its accept decision is
             * decodeModesMessage's.  Should the two ever disagree (a host-side filter change that was not forwarded), count
             * the frame the way demod_2400.c:422-428 counts a rejected message instead of losing it silently. */
            if (result == -1) Modes.stats_current.demod_rejected_unknown_icao++;
            else Modes.stats_current.demod_rejected_bad++;
            continue;
        }
        Modes.stats_current.demod_accepted[mm->correctedbits]++;
        Modes.stats_current.demod_bestPhase[f->phase - 4]++;
        double signal_power = f->sigpow_sum / 65535.0 / 65535.0;                 /* :448-457 */
        mm->signalLevel = signal_power / f->signal_len;
        Modes.stats_current.signal_power_sum += signal_power;
        Modes.stats_current.signal_power_count += f->signal_len;
        sum_scaled_signal_power += f->sigpow_sum;
        if (mm->signalLevel > Modes.stats_current.peak_signal_power) Modes.stats_current.peak_signal_power = mm->signalLevel;
        if (mm->signalLevel > 0.50119) Modes.stats_current.strong_signal_count++;
        netUseMessage(mm);                                                       /* :471 */
    }

    /* the counters the scan itself increments (stats.h:62-83): what this call added, delivered with the buffer's result */
    b200_buffer_result br;
    uint32_t nbr = 0;
    if (b200_demod_buffer_results(g_ctx, 0, &br, 1, &nbr) == B200_OK && nbr == 1) {
        if (iq && mag->length) {          /* what convert_uc8_nodc would have returned (convert.c:100-107), from the GPU's exact sums */
            mag->mean_level = br.sum_level / 65536.0 / mag->length;
            mag->mean_power = br.sum_power / 65535.0 / 65535.0 / mag->length;
        }
        Modes.stats_current.demod_preambles += br.demod_preambles;
        Modes.stats_current.demod_rejected_bad += br.demod_rejected_bad;
        Modes.stats_current.demod_rejected_unknown_icao += br.demod_rejected_unknown_icao;
        for (int p = 0; p < 5; p++) Modes.stats_current.demod_preamblePhase[p] += br.demod_preamblePhase[p];
    }
    /* demod_2400.c:474-479 */
    double sum_signal_power = sum_scaled_signal_power / 65535.0 / 65535.0;
    Modes.stats_current.noise_power_sum += (mag->mean_power * mag->length - sum_signal_power);
    Modes.stats_current.noise_power_count += mag->length;

    netDrainMessageBuffers();                                                    /* :481 */
}

/* demod_2400.c:575-761: the replies were found by the run __wrap_demodulate2400 started for this same buffer. */
void __wrap_demodulate2400AC(struct mag_buf *mag) {
    uint32_t n = 0;
    if (!g_ctx || !g_ac || b200_demod_fetch_modeac(g_ctx, 0, g_ac, g_ac_cap, &n) != B200_OK) {
        fprintf(stderr, "b200 demodulator (Mode A/C): %s\n", b200_demod_last_error(g_ctx));
        setExit(2);
        return;
    }
    for (uint32_t i = 0; i < n; i++) {
        struct modesMessage *mm = netGetMM(&Modes.netMessageBuffer[0]);          /* :736 */
        mm->timestamp = g_ac[i].timestamp;                                       /* :740, at the F2 pulse */
        mm->sysTimestamp = mag->sysTimestamp + receiveclock_ms_elapsed(mag->sampleTimestamp, mm->timestamp);
        decodeModeAMessage(mm, g_ac[i].modeac);                                  /* :745 */
        netUseMessage(mm);
        Modes.stats_current.demod_modeac++;
    }
    netDrainMessageBuffers();
}
