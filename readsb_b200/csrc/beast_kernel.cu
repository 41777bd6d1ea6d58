// beast_kernel.cu — the wire formats of the accepted-frame stream, encoded on the device so that a GPU box can feed any
// readsb / dump1090 aggregator or raw-line consumer without the tracking layer, and the D2H traffic is the wire record
// instead of the 64-byte frame (SURVEY.md section 8f row 4).
//
// Beast binary (reference modesSendBeastOutput net_io.c:1655-1714 with netTimestamp :1617-1648): 0x1a, type ('2' 56 bit,
// '3' 112 bit, '1' Mode A/C), 6-byte big-endian 12 MHz timestamp, signal byte nearbyint(sqrt(signalLevel) * 255) clamped to
// [1 if signalLevel > 0, 255], the frame bytes; every 0x1a after the type byte is doubled.
//
// Raw / AVR text: the network record of modesSendRawOutput (net_io.c:1837-1863) or the --raw stdout line of
// displayModesMessage (mode_s.c:1835-1841).  '*', or with MLAT and a non-zero timestamp '@' + "%012" PRIX64 of the timestamp;
// the frame bytes in hex (network: uppercase, mm->msg or mm->verbatim; stdout: lowercase, always mm->msg); ";\n".  A timestamp
// of 13 or more hex digits (>= 2^48, or negative) keeps only its first 12 in the network record, because the reference steps
// p by 13 after the sprintf and the frame hex overwrites the rest; the stdout line prints every digit.
//
// One block per receiver, one kernel for both formats (templated on the encoder).  Records leave in the reference's output
// order: per reference buffer the Mode S frames (demodulate2400), then the Mode A/C replies (demodulate2400AC,
// readsb.c:871-874).  Two passes over the receiver's records: lengths -> one atomic reservation in the packed output, then the
// bytes.
#include "common.h"
#include "device_utils.cuh"

#define BEAST_THREADS 128
#define BEAST_MAX_RECORD 44        // 2 + 2 * (6 + 1 + 14)
#define RAW_MAX_RECORD 48          // '@' + 16 timestamp digits + 28 hex + ";\n" = 47 (stdout, negative timestamp)
static_assert(BEAST_MAX_RECORD == B200_BEAST_MAX_RECORD && RAW_MAX_RECORD == B200_RAW_MAX_RECORD, "record bounds of the ABI");

template <int MAX> struct WireRec { uint8_t b[MAX]; uint32_t n; };       // one record being built by one thread

// ---- Beast -------------------------------------------------------------------------------------------------------
typedef WireRec<BEAST_MAX_RECORD> Rec44;

__device__ __forceinline__ void put(Rec44 &r, uint8_t ch) { r.b[r.n++] = ch; if (ch == 0x1a) r.b[r.n++] = ch; }

__device__ __forceinline__ void head(Rec44 &r, char type, int64_t timestamp, double signal_level) {
    r.n = 0;
    r.b[r.n++] = 0x1a; r.b[r.n++] = (uint8_t)type;
#pragma unroll
    for (int sh = 40; sh >= 0; sh -= 8) put(r, (uint8_t)(timestamp >> sh));
    int sig = (int)rint(sqrt(signal_level) * 255);                       // net_io.c:1696-1700
    if (signal_level > 0 && sig < 1) sig = 1;
    if (sig > 255) sig = 255;
    put(r, (uint8_t)sig);
}

__device__ __forceinline__ void frame_bytes(uint8_t (&msg)[14], const b200_frame &f, bool verbatim) {
#pragma unroll
    for (int i = 0; i < 14; i++) msg[i] = f.msg[i];
    if (verbatim && f.fix_bit >= 0) msg[f.fix_bit >> 3] ^= (uint8_t)(1u << (7 - (f.fix_bit & 7)));    // mm->verbatim: as received
}

struct BeastEncoder {
    typedef Rec44 Record;
    __device__ static void frame(Rec44 &r, const b200_frame &f, uint32_t flags) {
        uint8_t msg[14];
        frame_bytes(msg, f, (flags & B200_BEAST_VERBATIM) != 0);
        const int len = f.msgbits / 8;
        const double signal_level = (double)f.sigpow_sum / 65535.0 / 65535.0 / (double)f.signal_len;   // demod_2400.c:448-457
        head(r, len == 7 ? '2' : '3', f.timestamp, signal_level);
        for (int i = 0; i < len; i++) put(r, msg[i]);
    }
    __device__ static void modeac(Rec44 &r, const b200_modeac &a, uint32_t) {
        head(r, '1', a.timestamp, 0.0);                                  // mode_ac.c:171-173; signalLevel stays 0
        put(r, (uint8_t)(a.modeac >> 8));
        put(r, (uint8_t)a.modeac);
    }
};

// ---- raw / AVR -----------------------------------------------------------------------------------------------------
typedef WireRec<RAW_MAX_RECORD> Rec48;

__device__ __forceinline__ uint8_t hex_digit(uint32_t d, bool lower) { return (uint8_t)(d < 10 ? '0' + d : (lower ? 'a' : 'A') + d - 10); }

__device__ __forceinline__ void raw_head(Rec48 &r, int64_t timestamp, uint32_t flags) {
    r.n = 0;
    if ((flags & B200_RAW_MLAT) && timestamp) {
        const uint64_t u = (uint64_t)timestamp;
        int nd = 12;                                                     // digits "%012" PRIX64 prints
        while (nd < 16 && (u >> (4 * nd))) nd++;
        const int keep = (flags & B200_RAW_STDOUT) ? nd : 12;           // network: p += 13, the frame hex overwrites the rest
        r.b[r.n++] = '@';
        for (int k = nd - 1; k >= nd - keep; k--) r.b[r.n++] = hex_digit((uint32_t)(u >> (4 * k)) & 15, false);
    } else {
        r.b[r.n++] = '*';
    }
}

__device__ __forceinline__ void raw_hex(Rec48 &r, uint8_t v, uint32_t flags) {
    const bool lower = (flags & B200_RAW_STDOUT) != 0;                  // printf("%02x") on stdout, printHexDigit on the network
    r.b[r.n++] = hex_digit(v >> 4, lower);
    r.b[r.n++] = hex_digit(v & 15, lower);
}

struct RawEncoder {
    typedef Rec48 Record;
    __device__ static void frame(Rec48 &r, const b200_frame &f, uint32_t flags) {
        uint8_t msg[14];
        frame_bytes(msg, f, (flags & B200_RAW_VERBATIM) != 0);
        raw_head(r, f.timestamp, flags);
        const int len = f.msgbits / 8;
        for (int i = 0; i < len; i++) raw_hex(r, msg[i], flags);
        r.b[r.n++] = ';'; r.b[r.n++] = '\n';
    }
    __device__ static void modeac(Rec48 &r, const b200_modeac &a, uint32_t flags) {
        raw_head(r, a.timestamp, flags);                                 // msgbits 16, verbatim == msg (mode_ac.c:171-173)
        raw_hex(r, (uint8_t)(a.modeac >> 8), flags);
        raw_hex(r, (uint8_t)a.modeac, flags);
        r.b[r.n++] = ';'; r.b[r.n++] = '\n';
    }
};

// ---- the walk: every record of one receiver, in output order --------------------------------------------------------
template <class Enc>
__global__ void __launch_bounds__(BEAST_THREADS) encode_kernel(const EncodeParams P) {
    __shared__ uint32_t scratch[40];
    __shared__ uint32_t s_base;
    const uint32_t s = blockIdx.x, tid = threadIdx.x;
    const uint32_t sb = P.stream_seg_begin[s], se = P.stream_seg_begin[s + 1];
    if (sb == se) { if (tid == 0) { P.stream_off[s] = 0; P.stream_len[s] = 0; } return; }
    const uint32_t b0 = P.segs[sb].first_buf, b1 = P.segs[se - 1].first_buf + P.segs[se - 1].n_bufs;
    uint32_t running = 0;
    for (int pass = 0; pass < 2; pass++) {
        uint32_t fcur = P.frame_span[2 * s];
        running = 0;
        for (uint32_t b = b0; b < b1; b++) {
            const uint32_t nf = P.buf_out[b].n_frames;
            const uint32_t a0 = P.ac_prefix ? P.ac_prefix[b] : 0, na = P.ac_prefix ? P.ac_prefix[b + 1] - a0 : 0;
            for (uint32_t i0 = 0; i0 < nf + na; i0 += BEAST_THREADS) {
                const uint32_t i = i0 + tid;
                typename Enc::Record r; r.n = 0;
                if (i < nf) Enc::frame(r, P.frames[fcur + i], P.flags);
                else if (i < nf + na) Enc::modeac(r, P.ac[a0 + i - nf], P.flags);
                uint32_t total;
                const uint32_t off = block_excl_scan(r.n, scratch, &total);
                if (pass == 1 && r.n) {
                    const uint32_t at = s_base + running + off;
                    if (at + r.n <= P.cap) for (uint32_t k = 0; k < r.n; k++) P.out[at + k] = r.b[k];
                }
                running += total;
            }
            fcur += nf;
        }
        if (pass == 0) {
            if (tid == 0) { s_base = atomicAdd(P.total, running); P.stream_off[s] = s_base; P.stream_len[s] = running; }
            __syncthreads();
        }
    }
}

extern "C" int b200_launch_encode(const EncodeParams *p, uint32_t n_streams, void *stream) {
    if (p->format == ENC_RAW) encode_kernel<RawEncoder><<<n_streams, BEAST_THREADS, 0, (cudaStream_t)stream>>>(*p);
    else encode_kernel<BeastEncoder><<<n_streams, BEAST_THREADS, 0, (cudaStream_t)stream>>>(*p);
    return (int)cudaGetLastError();
}
