// beast_kernel.cu — Beast binary output of the accepted-frame stream (SURVEY.md section 8f row 4; reference
// modesSendBeastOutput net_io.c:1655-1714 with netTimestamp :1617-1648), so that a GPU box can feed any readsb / dump1090
// aggregator without the tracking layer, and the D2H traffic is the 23-30 byte wire record instead of the 64-byte frame.
//
// One block per receiver.  Records leave in the reference's output order: per reference buffer the Mode S frames
// (demodulate2400), then the Mode A/C replies (demodulate2400AC, readsb.c:871-874).  Record: 0x1a, type ('2' 56 bit,
// '3' 112 bit, '1' Mode A/C), 6-byte big-endian 12 MHz timestamp, signal byte nearbyint(sqrt(signalLevel) * 255) clamped to
// [1 if signalLevel > 0, 255], the frame bytes; every 0x1a after the type byte is doubled.  Two passes over the receiver's
// records: lengths -> one atomic reservation in the packed output, then the bytes.
#include "common.h"
#include "device_utils.cuh"

#define BEAST_THREADS 128
#define BEAST_MAX_RECORD 44        // 2 + 2 * (6 + 1 + 14)

struct Rec44 { uint8_t b[BEAST_MAX_RECORD]; uint32_t n; };

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

__device__ void encode_frame(Rec44 &r, const b200_frame &f, bool verbatim) {
    uint8_t msg[14];
#pragma unroll
    for (int i = 0; i < 14; i++) msg[i] = f.msg[i];
    if (verbatim && f.fix_bit >= 0) msg[f.fix_bit >> 3] ^= (uint8_t)(1u << (7 - (f.fix_bit & 7)));    // mm->verbatim: as received
    const int len = f.msgbits / 8;
    const double signal_level = (double)f.sigpow_sum / 65535.0 / 65535.0 / (double)f.signal_len;       // demod_2400.c:448-457
    head(r, len == 7 ? '2' : '3', f.timestamp, signal_level);
    for (int i = 0; i < len; i++) put(r, msg[i]);
}

__device__ void encode_modeac(Rec44 &r, const b200_modeac &a) {
    head(r, '1', a.timestamp, 0.0);                                      // mode_ac.c:171-173; signalLevel stays 0
    put(r, (uint8_t)(a.modeac >> 8));
    put(r, (uint8_t)a.modeac);
}

__global__ void __launch_bounds__(BEAST_THREADS) beast_encode_kernel(const BeastParams P) {
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
                Rec44 r; r.n = 0;
                if (i < nf) encode_frame(r, P.frames[fcur + i], P.verbatim != 0);
                else if (i < nf + na) encode_modeac(r, P.ac[a0 + i - nf]);
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

extern "C" int b200_launch_beast(const BeastParams *p, uint32_t n_streams, void *stream) {
    beast_encode_kernel<<<n_streams, BEAST_THREADS, 0, (cudaStream_t)stream>>>(*p);
    return (int)cudaGetLastError();
}
