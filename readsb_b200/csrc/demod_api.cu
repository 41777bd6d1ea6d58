// demod_api.cu — the C ABI declared in include/b200_demod.h: context, device memory, the
// host-buffer (drop-in) path and the device-resident path around the kernels in scan_kernel.cu / resolve_kernel.cu.
//
// Host side of the boundary (reference tree): a frontend's converter call + mag_buf hand-off
// (sdr_ifile.c:194-259, convert.h:34-39) becomes b200_demod_submit_iq_uc8; the decode thread's
// demodulate2400(buf) (readsb.c:871, demod_2400.h:38) becomes submit_mag_u16 / run / fetch.
//
// A run owns one SLOT (segment tables, candidate pools, result buffers).  The blocking calls use slot 0 on one
// CUDA stream.  The asynchronous calls (run_device_*_async / run_host_*_async / wait) cycle through NSLOT slots: the
// scan kernels of consecutive steps run back to back on the scan stream, stage B (one launch: capacity check, stage B, frame
// placement, finalizer) + D2H of each step follow on the resolve stream (higher priority) as soon as its scan has ended; stage B
// kernels stay ordered among themselves, which is all the per-receiver state needs.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <string>
#include <vector>

#include "common.h"
#include "modes_tables.h"

#define API extern "C" __attribute__((visibility("default")))

static std::string g_create_error;

struct Pending {
    uint32_t n;          // new samples
    int64_t ts;
    size_t off;          // byte offset of data index 0 (mag) or of the first new sample (iq) in the stream's arena region
    int fsum = -1;       // sc16 input: index of the buffer's float sums in d_fsum
    bool restart = false;                // iq input: b200_demod_restart_stream came before this buffer (zero halo)
    bool has_levels = false;             // magnitude hand-off with the mag_buf's own mean_level / mean_power (Mode A/C noise floor)
    double mean_level = 0, mean_power = 0;
};

// sample format of a device-resident or pipelined step
enum IqFormat { FMT_UC8 = 0, FMT_SC16 = 1, FMT_SC16Q11 = 2 };
static inline uint32_t fmt_bytes(int fmt) { return fmt == FMT_UC8 ? 2u : 4u; }     // bytes per raw sample

struct Slot {
    bool allocated = false, in_flight = false, completed = false;
    uint32_t rec_cap = 0;
    // Descriptors of a run travel in ONE host-to-device copy and its results in ONE device-to-host copy: two blocks per slot, laid
    // out per run (layout_run); the d_* / h_* members below point into them.
    //   descriptor block  [stream_seg_begin (S+1) | segs (nseg) | tile_seg (ntile)]
    //   result block      [RunCtl | buf_acc (nbuf) | frame_span (2S) | buf_out (nbuf) | packed frames ...]
    uint8_t *d_desc = nullptr, *h_desc = nullptr, *d_res = nullptr, *h_res = nullptr;
    uint8_t *d_res_host = nullptr;    // h_res as the device sees it (mapped pinned memory): the one-receiver kernel publishes its results there
    bool res_clean = false;           // RunCtl + BufAcc[0 .. clean_bufs) in d_res are zero (the one-receiver kernel cleans up after itself)
    uint32_t clean_bufs = 0;
    size_t desc_cap = 0, res_cap = 0, res_head = 0;     // res_head: bytes in front of the packed frames in this run's result block
    Segment *d_segs = nullptr, *h_segs = nullptr;       // h_segs / h_tile_seg / h_stream_seg_begin: where the host BUILDS the run (copied into h_desc)
    uint32_t *d_tile_seg = nullptr, *h_tile_seg = nullptr;
    uint32_t *d_stream_seg_begin = nullptr, *h_stream_seg_begin = nullptr;
    uint32_t cached_tiles = 0;        // tile_seg on the device is valid for this many tiles (device-resident path)
    uint64_t cached_layout_key = 0;
    std::vector<uint32_t> cached_counts;      // ... and these per-receiver buffer counts
    RunCtl *d_ctl = nullptr, *h_ctl = nullptr;
    PosEntry *d_pos_pool = nullptr;
    Rec *d_rec_pool = nullptr;
    uint32_t *d_key_pool = nullptr;
    TileOut *d_tile_out = nullptr;
    BufAcc *d_buf_acc = nullptr, *h_buf_acc = nullptr;
    b200_buffer_result *d_buf_out = nullptr, *h_buf_out = nullptr;
    b200_frame *d_frames = nullptr, *d_packed = nullptr, *h_packed = nullptr;
    uint32_t *d_frame_span = nullptr, *h_frame_span = nullptr;    // per receiver: first packed frame, frame count (FinalizeParams)
    uint32_t *d_addable = nullptr;    // [S] filter adds this run can make at most (scan kernel -> capacity check, which zeroes it again)
    // Mode A/C (contexts created with B200_CFG_MODE_AC)
    uint32_t *d_ac_bitmap = nullptr, *d_ac_noise = nullptr;
    uint16_t *d_mag_copy = nullptr;   // Mode A/C: the Mode S scan's magnitudes of the run's uc8 tiles (ScanParams::mag_copy)
    uint32_t *d_ac_count = nullptr, *d_ac_prefix = nullptr, *h_ac_prefix = nullptr;   // per reference buffer of the run
    b200_modeac *d_ac_out = nullptr, *d_ac_packed = nullptr, *h_ac_packed = nullptr;
    AcLevel *d_ac_levels = nullptr, *h_ac_levels = nullptr;                           // per reference buffer of the run: source of the noise floor
    // the run this slot holds
    uint32_t nseg = 0, ntile = 0, nbuf = 0, run_frames = 0;
    size_t desc_bytes = 0;            // bytes of the descriptor block this run uploads
    bool upload_tiles = true;
    std::vector<uint32_t> stream_buf_begin;   // [n_streams+1] into h_buf_out
    cudaEvent_t ev[8] = {};                   // 0 scan begin, 1 scan end, 2 resolve end, 3 finalize end, 4 results on host,
                                              // 5 result copies done, 6 Mode A/C scan + walk done, 7 descriptors uploaded
    float ms[5] = {0, 0, 0, 0, 0};
    uint32_t launches = 0;
    uint32_t first_frames = 0;        // packed frames that came with the result block's copy
    uint32_t carry_in_kernel = 0xffffffffu;   // one-receiver host run: byte offset of the tail the stage B kernel carries to the front
    bool desc_on_device = true;       // false: this run's descriptors went as kernel parameters (b200_demod_fetch_beast uploads them if asked)
    int scan_grid = 0;                // CTAs the scan kernel of this run was launched with
    bool published = false, timed = true;   // this run: results published by the kernel / events recorded between the kernels
    // sc16 / sc16q11 steps: the run's magnitudes, made by sc16_convert_kernel on the scan stream ahead of the scan (again when the
    // step is repeated); its float sums go to BufAcc::fsum of the run's buffers and come back with the result block
    bool sc16 = false;
    Sc16Params conv = {};
    uint16_t *d_slab = nullptr;       // receiver s at d_slab + s * slab_stride: 2 samples of padding (new samples 16-byte aligned),
    size_t slab_stride = 0;           // 326 halo magnitudes, max_buffers_per_run * buf_samples magnitudes; allocated on the first sc16 step
};

#define FIRST_COPY_FRAMES 16

#define NSLOT 3      // steps in flight in the asynchronous modes; the blocking calls use slot 0

// measurement of the scan's share of the SMs in a pipelined session (tune_partition)
struct PartCal {
    enum { SAMPLES = 12 };
    int grids[4] = {0, 0, 0, 0};      // candidates: the whole chip, 85 %, 82 % of the SMs; [3] = the winner, measured again
    int phase = 0, n = 0, skip = 0;
    double dt[SAMPLES] = {}, mean[4] = {0, 0, 0, 0};
    uint32_t ntile = 0;               // size of the runs being measured
    std::chrono::steady_clock::time_point last;
    bool have_last = false, locked = false;
};

struct b200_demod_ctx {
    b200_demod_config cfg;
    int device = 0, n_sm = 0;
    int n_sm_scan = 0;                // CTAs of the persistent scan kernel (one per SM) in blocking runs
    // Pipelined steps: how the SMs are shared between the scan of step n+1 and stage B + finalizer of step n (tune_partition)
    int part_n = 0;                   // CTAs of the scan kernel in pipelined runs; 0 = the whole chip (the two alternate on all SMs)
    bool part_debug = false;
    bool part_fixed = false, part_off = false;     // B200_SCAN_SMS given: no tuning; B200_SCAN_PART=0: always the whole chip
    PartCal cal;
    int cal_restarts = 0;
    int scan_sub = 1;                 // chunks per warp when a run is small enough for one CTA per tile (scan_kernel.cu, finish_shared_tile); B200_SCAN_SUB: 0 = whole tiles
    int n_sm_scan_async = 0;          // ... in pipelined runs, unless the session's measurement chose fewer (part_n, tune_partition) or B200_SCAN_SMS fixed it
    cudaStream_t stream = nullptr, own_stream = nullptr, res_stream = nullptr, copy_stream = nullptr, in_stream = nullptr;
    std::string err;

    DeviceTables *d_tables = nullptr;
    uint16_t *d_lut_full = nullptr;
    StreamState *d_state = nullptr;
    uint32_t *d_icao_slab = nullptr;              // default filter tables of all receivers: [S][2][ICAO_CAP]
    std::vector<uint32_t *> icao_grown;           // tables of receivers that outgrew them (freed at destroy)
    std::vector<StreamState> h_state;             // scratch for growing

    uint8_t *d_arena = nullptr;
    size_t stream_stride = 0;
    std::vector<std::vector<Pending>> pending;
    std::vector<uint8_t> kind;        // per stream this run: 0 none, 1 uc8 iq, 2 mag hand-off, 3 sc16 iq (magnitudes made by the library)
    std::vector<uint8_t> halo_valid;  // iq streams: saved 326-sample tail is valid
    std::vector<uint8_t> restart_next;  // iq streams: the next submitted buffer starts with a zero halo (b200_demod_restart_stream)
    std::vector<size_t> cursor;       // append offset in the stream's arena region

    uint32_t seg_cap = 0, tile_cap = 0, buf_cap = 0, frame_cap = 0, ac_cap = 0;
    Slot slot[NSLOT];
    int cur = 0;                      // slot whose results fetch / buffer_results / timing report
    int next_async = 0;               // slot the next asynchronous step takes
    int head = 0, n_flight = 0;       // oldest step in flight, number of steps in flight (slots head, head+1, ... mod NSLOT)
    uint32_t *d_carry_src = nullptr, *h_carry_src = nullptr;
    uint32_t *d_stop = nullptr;       // [NSLOT] per slot: 1 when its last run's stage B did not run (ResolveParams::stop_out)
    uint8_t *h_zero = nullptr;        // pinned zeros: a run's control block and per-buffer sums are cleared by a copy from here (enqueue)
    // scan kernel: per-warp staging of a run's live records, spill of the pre-check queue, ticks of the run in progress
    Rec *d_stage_rec = nullptr; uint32_t *d_stage_key = nullptr; uint16_t *d_q1_over = nullptr; uint32_t *d_tick_scratch = nullptr;
    uint32_t stage_cap = 0;
    // Beast encoding (on demand, b200_demod_fetch_beast): packed records of every stream of one run
    uint8_t *d_beast = nullptr, *h_beast = nullptr;
    uint32_t *d_beast_meta = nullptr, *h_beast_meta = nullptr;   // [S] offsets, [S] lengths, [1] total
    uint32_t beast_cap = 0;
    int beast_slot = -1; uint32_t beast_flags = 0;               // which run the buffers hold
    // sc16 input: staging of one raw buffer, float sums of the buffers queued for the next run
    uint8_t *d_raw16 = nullptr;
    float2 *d_fsum = nullptr, *h_fsum = nullptr;
    uint32_t n_fsum = 0;
    int *d_result = nullptr;
    // pipelined host-buffer path (run_host_uc8_async): two device input buffers, one per pipeline slot, filled on in_stream
    uint8_t *d_pipe[NSLOT] = {};
    size_t pipe_stride = 0;
    uint8_t *d_pipe16[NSLOT] = {};    // ... the same for run_host_sc16_async (int16 samples), allocated on its first step
    size_t pipe16_stride = 0;
    cudaEvent_t ev_in[NSLOT] = {};
    // ... and each receiver's halo between its host-buffer steps: its last 326 raw samples (halo_store_kernel)
    uint16_t *d_halo_store = nullptr;                // [S][326 * 4 bytes]
    uint32_t *d_halo_op = nullptr, *h_halo_op = nullptr;     // [NSLOT][S] what halo_store_kernel does for each receiver in that slot's step
    std::vector<uint8_t> halo_bytes;  // per receiver: bytes per sample of its stored halo (2 uc8, 4 sc16), 0 = none; a halo only
                                      // continues a step of the same input width
    std::vector<b200_rx_step> rx_uniform;     // the uniform calls' descriptor array
};

static int fail(b200_demod_ctx *c, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (c) c->err = buf; else g_create_error = buf;
    return code;
}

#define CU(c, call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(c, B200_E_CUDA, "%s: %s", #call, cudaGetErrorString(e_)); } while (0)

template <class T> static cudaError_t dev_alloc(T **p, size_t n) { return cudaMalloc((void **)p, n * sizeof(T)); }
template <class T> static cudaError_t pin_alloc(T **p, size_t n) { return cudaHostAlloc((void **)p, n * sizeof(T), cudaHostAllocDefault); }

// Copies each IQ stream's last 326 samples to the front of its arena region (the mag_buf overlap copy,
// sdr_ifile.c:209-213), one block per stream; src[s] = byte offset of the tail, 0xffffffff = nothing to do.
__global__ void carry_halo_kernel(uint8_t *arena, size_t stride, const uint32_t *src, uint32_t n_streams) {
    const uint32_t s = blockIdx.x;
    if (s >= n_streams || src[s] == 0xffffffffu) return;
    uint8_t *region = arena + (size_t)s * stride;
    const uint16_t *from = reinterpret_cast<const uint16_t *>(region + src[s]);
    uint16_t *to = reinterpret_cast<uint16_t *>(region);
    for (uint32_t i = threadIdx.x; i < B200_TRAIL; i += blockDim.x) to[i] = from[i];
}

// Host-buffer steps (run_host_*_async): the mag_buf overlap copy (sdr_ifile.c:209-213) of every receiver through a halo store of its
// own, so that a receiver continues its own last step whatever steps it was absent from.  One block per receiver; its first new
// sample at slab + s * stride, op[s] = new samples << 1 | continues, 0 = absent.  A continued receiver first gets its stored
// 326 raw samples in front of its new ones; a receiver with >= 326 new samples then stores its last 326 for its next step.
__global__ void halo_store_kernel(uint8_t *slab, size_t stride, uint16_t *store, const uint32_t *op, uint32_t bps) {
    const uint32_t s = blockIdx.x, o = op[s], n = o >> 1, n16 = B200_TRAIL * bps / 2;
    uint16_t *halo = reinterpret_cast<uint16_t *>(slab + (size_t)s * stride) - n16;      // the halo, then the new samples
    uint16_t *st = store + (size_t)s * (B200_TRAIL * 2);
    if (o & 1u) for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) halo[i] = st[i];
    __syncthreads();
    if (n >= B200_TRAIL) for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) st[i] = halo[n * bps / 2 + i];
}

API int b200_demod_abi_version(void) { return B200_DEMOD_ABI_VERSION; }

API const char *b200_demod_last_error(const b200_demod_ctx *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

API void *b200_demod_host_alloc(size_t bytes) {
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    return p;
}
API void b200_demod_host_free(void *p) { if (p) cudaFreeHost(p); }
API int b200_demod_host_register(void *p, size_t bytes) {
    if (!p || !bytes) return B200_E_INVAL;
    const cudaError_t e = cudaHostRegister(p, bytes, cudaHostRegisterDefault);
    if (e == cudaErrorHostMemoryAlreadyRegistered) { cudaGetLastError(); return B200_OK; }
    return e == cudaSuccess ? B200_OK : B200_E_CUDA;
}
API int b200_demod_host_unregister(void *p) { return p && cudaHostUnregister(p) == cudaSuccess ? B200_OK : B200_E_INVAL; }

API int b200_demod_uc8_lut(uint16_t *out) {
    if (!out) return B200_E_INVAL;
    b200_build_uc8_lut(out);
    return B200_OK;
}

static inline size_t pad16(size_t n) { return (n + 15) & ~(size_t)15; }

// Lays this run's descriptors and results out in the slot's two blocks (nseg / ntile / nbuf are final) and copies what the host
// built into the descriptor block's host copy.
static void layout_run(b200_demod_ctx *c, Slot &sl);

static void free_slot(Slot &s) {
    cudaFree(s.d_desc); cudaFree(s.d_res); cudaFreeHost(s.h_desc); cudaFreeHost(s.h_res); cudaFree(s.d_pos_pool);
    cudaFree(s.d_rec_pool); cudaFree(s.d_key_pool); cudaFree(s.d_tile_out);
    cudaFree(s.d_frames); cudaFree(s.d_addable);
    cudaFree(s.d_mag_copy); cudaFree(s.d_ac_bitmap); cudaFree(s.d_ac_noise); cudaFree(s.d_ac_count); cudaFree(s.d_ac_prefix); cudaFree(s.d_ac_out); cudaFree(s.d_ac_packed);
    cudaFreeHost(s.h_ac_prefix); cudaFreeHost(s.h_ac_packed);
    cudaFree(s.d_ac_levels); cudaFreeHost(s.h_ac_levels);
    cudaFree(s.d_slab);
    free(s.h_segs); free(s.h_tile_seg); free(s.h_stream_seg_begin);
    for (auto &e : s.ev) if (e) cudaEventDestroy(e);
    s = Slot();
}

static cudaError_t alloc_slot(b200_demod_ctx *c, Slot &s, uint32_t rec_cap) {
    const uint32_t S = c->cfg.n_streams;
#define A(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return e_; } while (0)
    for (auto &e : s.ev) A(cudaEventCreate(&e));
    s.rec_cap = rec_cap;
    s.h_segs = (Segment *)malloc((size_t)c->seg_cap * sizeof(Segment));
    s.h_tile_seg = (uint32_t *)malloc((size_t)c->tile_cap * 4);
    s.h_stream_seg_begin = (uint32_t *)malloc(((size_t)S + 1) * 4);
    if (!s.h_segs || !s.h_tile_seg || !s.h_stream_seg_begin) return cudaErrorMemoryAllocation;
    s.desc_cap = pad16(((size_t)S + 1) * 4) + (size_t)c->seg_cap * sizeof(Segment) + (size_t)c->tile_cap * 4 + 64;
    s.res_cap = sizeof(RunCtl) + (size_t)c->buf_cap * (sizeof(BufAcc) + sizeof(b200_buffer_result)) + pad16((size_t)S * 8)
              + (size_t)S * c->frame_cap * sizeof(b200_frame) + 64;
    A(cudaMalloc((void **)&s.d_desc, s.desc_cap)); A(cudaHostAlloc((void **)&s.h_desc, s.desc_cap, cudaHostAllocDefault));
    A(cudaMalloc((void **)&s.d_res, s.res_cap)); A(cudaHostAlloc((void **)&s.h_res, s.res_cap, cudaHostAllocMapped));
    A(cudaHostGetDevicePointer((void **)&s.d_res_host, s.h_res, 0));
    A(cudaMemset(s.d_res, 0, sizeof(RunCtl)));
    memset(s.h_res, 0, sizeof(RunCtl) + pad16((size_t)S * 8));
    s.d_ctl = reinterpret_cast<RunCtl *>(s.d_res); s.h_ctl = reinterpret_cast<RunCtl *>(s.h_res);
    A(dev_alloc(&s.d_pos_pool, (size_t)c->tile_cap * SCAN_TILE));
    A(dev_alloc(&s.d_rec_pool, s.rec_cap)); A(dev_alloc(&s.d_key_pool, s.rec_cap));
    A(dev_alloc(&s.d_tile_out, c->tile_cap));
    A(dev_alloc(&s.d_frames, (size_t)S * c->frame_cap));
    A(dev_alloc(&s.d_addable, S)); A(cudaMemset(s.d_addable, 0, S * 4));

    if (c->cfg.flags & B200_CFG_MODE_AC) {
        // one bit per position, and room for every reply a buffer can hold: nothing here depends on the input
        const size_t ac_total = (size_t)c->buf_cap * c->ac_cap;
        A(dev_alloc(&s.d_ac_bitmap, (size_t)c->tile_cap * (SCAN_TILE / 32)));
        A(dev_alloc(&s.d_mag_copy, (size_t)c->tile_cap * SCAN_TILE));
        A(dev_alloc(&s.d_ac_noise, c->buf_cap)); A(dev_alloc(&s.d_ac_count, c->buf_cap));
        A(cudaMemset(s.d_ac_count, 0, (size_t)c->buf_cap * 4)); A(cudaMemset(s.d_ac_noise, 0, (size_t)c->buf_cap * 4));
        A(dev_alloc(&s.d_ac_out, ac_total)); A(dev_alloc(&s.d_ac_packed, ac_total)); A(pin_alloc(&s.h_ac_packed, ac_total));
        A(dev_alloc(&s.d_ac_prefix, c->buf_cap + 1)); A(pin_alloc(&s.h_ac_prefix, c->buf_cap + 1));
        A(dev_alloc(&s.d_ac_levels, c->buf_cap)); A(pin_alloc(&s.h_ac_levels, c->buf_cap));
        memset(s.h_ac_levels, 0, (size_t)c->buf_cap * sizeof(AcLevel));
        memset(s.h_ac_prefix, 0, (S + 1) * 4);
    }
#undef A
    s.stream_buf_begin.assign(S + 1, 0);
    layout_run(c, s);       // results of "no run yet": zero frames, zero buffers
    s.allocated = true;
    return cudaSuccess;
}

static void layout_run(b200_demod_ctx *c, Slot &sl) {
    const size_t S = c->cfg.n_streams;
    size_t o = 0;
    const size_t o_ssb = o; o += pad16((S + 1) * 4);
    const size_t o_seg = o; o += (size_t)sl.nseg * sizeof(Segment);
    const size_t o_tile = o;
    sl.d_stream_seg_begin = reinterpret_cast<uint32_t *>(sl.d_desc + o_ssb);
    sl.d_segs = reinterpret_cast<Segment *>(sl.d_desc + o_seg);
    sl.d_tile_seg = reinterpret_cast<uint32_t *>(sl.d_desc + o_tile);
    memcpy(sl.h_desc + o_ssb, sl.h_stream_seg_begin, (S + 1) * 4);
    if (sl.nseg) memcpy(sl.h_desc + o_seg, sl.h_segs, (size_t)sl.nseg * sizeof(Segment));
    if (sl.upload_tiles && sl.ntile) memcpy(sl.h_desc + o_tile, sl.h_tile_seg, (size_t)sl.ntile * 4);
    sl.desc_bytes = o_tile + (sl.upload_tiles ? (size_t)sl.ntile * 4 : 0);
    size_t r = sizeof(RunCtl);
    sl.d_buf_acc = reinterpret_cast<BufAcc *>(sl.d_res + r); sl.h_buf_acc = reinterpret_cast<BufAcc *>(sl.h_res + r); r += (size_t)sl.nbuf * sizeof(BufAcc);
    sl.d_frame_span = reinterpret_cast<uint32_t *>(sl.d_res + r); sl.h_frame_span = reinterpret_cast<uint32_t *>(sl.h_res + r); r += pad16(S * 8);
    sl.d_buf_out = reinterpret_cast<b200_buffer_result *>(sl.d_res + r); sl.h_buf_out = reinterpret_cast<b200_buffer_result *>(sl.h_res + r); r += (size_t)sl.nbuf * sizeof(b200_buffer_result);
    r = pad16(r);
    sl.d_packed = reinterpret_cast<b200_frame *>(sl.d_res + r); sl.h_packed = reinterpret_cast<b200_frame *>(sl.h_res + r);
    sl.res_head = r;
}

API void b200_demod_destroy(b200_demod_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    cudaFree(c->d_tables); cudaFree(c->d_lut_full); cudaFree(c->d_state); cudaFree(c->d_arena); cudaFree(c->d_icao_slab);
    for (uint32_t *t : c->icao_grown) cudaFree(t);
    cudaFree(c->d_carry_src); cudaFree(c->d_result); cudaFree(c->d_stop);
    cudaFree(c->d_stage_rec); cudaFree(c->d_stage_key); cudaFree(c->d_q1_over); cudaFree(c->d_tick_scratch);
    cudaFreeHost(c->h_carry_src); cudaFreeHost(c->h_zero);
    cudaFree(c->d_raw16); cudaFree(c->d_fsum); cudaFreeHost(c->h_fsum);
    cudaFree(c->d_halo_store); cudaFree(c->d_halo_op); cudaFreeHost(c->h_halo_op);
    cudaFree(c->d_beast); cudaFree(c->d_beast_meta); cudaFreeHost(c->h_beast); cudaFreeHost(c->h_beast_meta);
    for (Slot &sl : c->slot) free_slot(sl);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    if (c->res_stream) cudaStreamDestroy(c->res_stream);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    if (c->in_stream) cudaStreamDestroy(c->in_stream);
    for (int i = 0; i < NSLOT; i++) { cudaFree(c->d_pipe[i]); cudaFree(c->d_pipe16[i]); if (c->ev_in[i]) cudaEventDestroy(c->ev_in[i]); }
    delete c;
}

API int b200_demod_create(const b200_demod_config *cfg, b200_demod_ctx **out) {
    if (!cfg || !out || cfg->struct_size != sizeof(b200_demod_config)) return fail(nullptr, B200_E_INVAL, "bad config (struct_size)");
    if (cfg->n_streams == 0 || cfg->buf_samples == 0 || cfg->max_buffers_per_run == 0) return fail(nullptr, B200_E_INVAL, "n_streams, buf_samples and max_buffers_per_run must be > 0");
    if (cfg->nfix_crc < 0 || cfg->nfix_crc > 1) return fail(nullptr, B200_E_INVAL, "nfix_crc must be 0 or 1 (2-bit --aggressive tables are not on this path)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(nullptr, B200_E_NODEV, "no CUDA device: this library has no CPU path");
    b200_demod_ctx *c = new b200_demod_ctx();
    c->cfg = *cfg;
    if (c->cfg.preamble_threshold == 0) c->cfg.preamble_threshold = B200_PREAMBLE_THRESHOLD_DEFAULT;
    if (c->cfg.icao_ttl_ms == 0) c->cfg.icao_ttl_ms = B200_ICAO_TTL_MS;
    int dev = cfg->device;
    if (dev < 0 && cudaGetDevice(&dev) != cudaSuccess) { delete c; return fail(nullptr, B200_E_NODEV, "cudaGetDevice failed"); }
    if (dev >= ndev) { delete c; return fail(nullptr, B200_E_INVAL, "device %d out of range", dev); }
    c->device = dev;
#define CUC(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { fail(nullptr, B200_E_CUDA, "%s: %s", #call, cudaGetErrorString(e_)); b200_demod_destroy(c); return e_ == cudaErrorMemoryAllocation ? B200_E_NOMEM : B200_E_CUDA; } } while (0)
    CUC(cudaSetDevice(dev));
    cudaDeviceProp prop;
    CUC(cudaGetDeviceProperties(&prop, dev));
    // sm_90a code runs on compute capability 9.0 and nothing else (arch-specific features are not forward compatible)
    if (prop.major != 9 || prop.minor != 0) { fail(nullptr, B200_E_NODEV, "device %d is sm_%d%d; the kernels are built for sm_90a only", dev, prop.major, prop.minor); b200_demod_destroy(c); return B200_E_NODEV; }
    c->n_sm = prop.multiProcessorCount;
    c->n_sm_scan = c->n_sm;
    // Pipelined steps start with the whole chip for the scan; the session then measures whether a smaller grid - stage B + finalizer
    // of the step before on the remaining SMs - is faster (tune_partition).  B200_SCAN_SMS fixes the grid of both kinds of run.
    c->n_sm_scan_async = c->n_sm;
    if (const char *e = getenv("B200_SCAN_SMS")) {       // experiment knob (tools/gpu_partition.sh)
        const int v = atoi(e);
        if (v >= 1 && v <= c->n_sm) { c->n_sm_scan = c->n_sm_scan_async = v; c->part_fixed = true; }
    }
    if (const char *e = getenv("B200_SCAN_PART")) { c->part_off = atoi(e) == 0; c->part_debug = atoi(e) == 2; }
    if (const char *e = getenv("B200_SCAN_SUB")) { const int v = atoi(e); if (v >= 0 && v <= 2) c->scan_sub = v; }     // experiment knob (tools/gpu_latency.py)
    {   // With several steps in flight the scan kernels of later steps are already queued when a scan ends; stage B of the step
        // that just finished scanning must not wait behind them (its results gate the host), so its stream has the higher
        // priority: the block scheduler places stage B's CTAs first, the next scan's persistent CTAs follow as SMs drain, and
        // the small finalize CTAs fit next to them.
        int prio_lo = 0, prio_hi = 0;
        CUC(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
        const bool scan_first = getenv("B200_SCAN_PRIO") != nullptr;        // experiment knob (tools/gpu_partition.sh): the scan's stream gets the high priority
        CUC(cudaStreamCreateWithPriority(&c->own_stream, cudaStreamNonBlocking, scan_first ? prio_hi : prio_lo));
        CUC(cudaStreamCreateWithPriority(&c->res_stream, cudaStreamNonBlocking, scan_first ? prio_lo : prio_hi));
        CUC(cudaStreamCreateWithPriority(&c->copy_stream, cudaStreamNonBlocking, prio_lo));
        CUC(cudaStreamCreateWithPriority(&c->in_stream, cudaStreamNonBlocking, prio_lo));
    }
    c->stream = c->own_stream;

    const uint32_t S = cfg->n_streams, K = cfg->max_buffers_per_run, BUF = cfg->buf_samples;
    // tables
    {
        DeviceTables *t = new DeviceTables();
        std::vector<uint16_t> lut(65536);
        if (b200_build_tables(t, lut.data()) != 0) { delete t; fail(nullptr, B200_E_INVAL, "syndrome hash construction failed"); b200_demod_destroy(c); return B200_E_INVAL; }
        // the table must be bit-identical to the reference's (SURVEY.md 8a, a1): CRC32 of the LE table
        if (b200_crc32_ieee(lut.data(), 65536 * 2) != 0x8e9d21e1u) { delete t; fail(nullptr, B200_E_INVAL, "UC8 lookup table does not match the reference arithmetic (host FP contraction?)"); b200_demod_destroy(c); return B200_E_INVAL; }
        CUC(dev_alloc(&c->d_tables, 1));
        CUC(dev_alloc(&c->d_lut_full, 65536));
        CUC(cudaMemcpy(c->d_tables, t, sizeof(DeviceTables), cudaMemcpyHostToDevice));
        CUC(cudaMemcpy(c->d_lut_full, lut.data(), 65536 * 2, cudaMemcpyHostToDevice));
        delete t;
    }
    // kernel attributes (dynamic shared memory opt-in) are per device: set them for this context's device, every time
    CUC((cudaError_t)b200_prepare_scan()); CUC((cudaError_t)b200_prepare_resolve()); CUC((cudaError_t)b200_prepare_modeac());
    CUC((cudaError_t)b200_prepare_convert());
    CUC(dev_alloc(&c->d_state, S));
    CUC(dev_alloc(&c->d_icao_slab, (size_t)S * 2 * ICAO_CAP));
    CUC((cudaError_t)b200_launch_init_state(c->d_state, S, c->d_icao_slab, c->stream));
    CUC(dev_alloc(&c->d_result, 1));
    CUC(dev_alloc(&c->d_stop, NSLOT)); CUC(cudaMemsetAsync(c->d_stop, 0, NSLOT * 4, c->stream));

    // arena for host submits: [326-sample halo][K buffers, each with room for its own halo when magnitudes are submitted]
    c->stream_stride = (((size_t)K * ((size_t)BUF + B200_TRAIL + 16) * 2 + 1024) + 255) & ~(size_t)255;
    CUC(cudaMalloc((void **)&c->d_arena, c->stream_stride * S + 256));
    CUC(cudaMemsetAsync(c->d_arena, 0, c->stream_stride * S + 256, c->stream));
    c->pending.resize(S); c->kind.assign(S, 0); c->halo_valid.assign(S, 0); c->cursor.assign(S, 0);
    c->restart_next.assign(S, 0); c->halo_bytes.assign(S, 0); c->rx_uniform.resize(S);

    const uint32_t tiles_per_buf = (BUF + 16 + SCAN_TILE - 1) / SCAN_TILE + 1;
    c->seg_cap = S * K;
    c->tile_cap = S * K * tiles_per_buf;
    c->buf_cap = S * K;
    // Stage B speculates every sub-range of a buffer into a region of its own (resolve_stream): up to 8 sub-ranges, each rounded
    // up to whole scan tiles and holding len/113 + 3 frames, so a buffer can reserve BUF/113 + 8 * (2048/113 + 4) slots.
    c->frame_cap = K * (BUF / 113 + 2 + 8 * (2048 / 113 + 4));
    c->ac_cap = BUF / 70 + 2;                       // per reference buffer: a Mode A/C reply hides the next 69 positions
    {
        const size_t warps = (size_t)b200_scan_warps(c->n_sm);
        c->stage_cap = 1024;
        CUC(dev_alloc(&c->d_stage_rec, warps * c->stage_cap)); CUC(dev_alloc(&c->d_stage_key, warps * c->stage_cap));
        CUC(dev_alloc(&c->d_q1_over, warps * 512));
        CUC(dev_alloc(&c->d_tick_scratch, warps * (size_t)b200_scan_tick_words()));
    }
    const size_t positions = (size_t)S * K * BUF;
    CUC(alloc_slot(c, c->slot[0], (uint32_t)std::max<size_t>(65536, positions / 16)));
    CUC(dev_alloc(&c->d_carry_src, S)); CUC(pin_alloc(&c->h_carry_src, S));
    CUC(pin_alloc(&c->h_zero, sizeof(RunCtl) + (size_t)c->buf_cap * sizeof(BufAcc)));
    memset(c->h_zero, 0, sizeof(RunCtl) + (size_t)c->buf_cap * sizeof(BufAcc));
    CUC(cudaStreamSynchronize(c->stream));
#undef CUC
    *out = c;
    return B200_OK;
}

static bool any_in_flight(const b200_demod_ctx *c) { return c->n_flight > 0; }

// ---- submits ---------------------------------------------------------------------------------
static int submit_common(b200_demod_ctx *c, uint32_t s, const void *host, uint32_t n, int64_t ts, bool mag, const double *levels = nullptr) {
    if (!c) return B200_E_INVAL;
    if (s >= c->cfg.n_streams || (!host && n)) return fail(c, B200_E_INVAL, "bad stream or buffer");
    if (n > c->cfg.buf_samples) return fail(c, B200_E_INVAL, "buffer of %u samples exceeds buf_samples=%u", n, c->cfg.buf_samples);
    if (c->pending[s].size() >= c->cfg.max_buffers_per_run) return fail(c, B200_E_STATE, "stream %u already has max_buffers_per_run buffers queued", s);
    if (any_in_flight(c)) return fail(c, B200_E_STATE, "asynchronous steps are in flight: call b200_demod_wait first");
    const uint8_t want = mag ? 2 : 1;
    if (c->kind[s] && c->kind[s] != want) return fail(c, B200_E_STATE, "stream %u mixes submit kinds in one run", s);
    CU(c, cudaSetDevice(c->device));
    if (!c->kind[s]) { c->kind[s] = want; c->cursor[s] = mag ? 0 : (size_t)B200_TRAIL * 2; }
    uint8_t *region = c->d_arena + (size_t)s * c->stream_stride;
    Pending p;
    p.n = n; p.ts = ts; p.restart = c->restart_next[s] != 0;
    c->restart_next[s] = 0;               // (a magnitude hand-off brings its own halo: nothing to restart)
    if (levels) { p.has_levels = true; p.mean_level = levels[0]; p.mean_power = levels[1]; }
    if (mag) {
        p.off = (c->cursor[s] + 15) & ~(size_t)15;
        const size_t bytes = ((size_t)n + B200_TRAIL) * 2;
        CU(c, cudaMemcpyAsync(region + p.off, host, bytes, cudaMemcpyHostToDevice, c->stream));
        c->cursor[s] = p.off + bytes;
    } else {
        p.off = c->cursor[s];
        if (n) CU(c, cudaMemcpyAsync(region + p.off, host, (size_t)n * 2, cudaMemcpyHostToDevice, c->stream));
        c->cursor[s] = p.off + (size_t)n * 2;
    }
    c->pending[s].push_back(p);
    return B200_OK;
}

API int b200_demod_set_stream(b200_demod_ctx *c, void *cuda_stream) {
    if (!c) return B200_E_INVAL;
    if (any_in_flight(c)) return fail(c, B200_E_STATE, "asynchronous steps are in flight: call b200_demod_wait first");
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaStreamSynchronize(c->stream));
    c->stream = cuda_stream ? (cudaStream_t)cuda_stream : c->own_stream;
    return B200_OK;
}

API int b200_demod_submit_iq_uc8_strided(b200_demod_ctx *c, uint32_t first, uint32_t ns, const uint8_t *iq, uint64_t host_stride,
                                         uint32_t n_buffers, uint32_t buf_len, int64_t ts) {
    if (!c || !iq) return B200_E_INVAL;
    if (ns == 0 || first + ns > c->cfg.n_streams || n_buffers == 0 || buf_len == 0 || buf_len > c->cfg.buf_samples) return fail(c, B200_E_INVAL, "bad stream range or buffer length");
    if (n_buffers > 1 && buf_len != c->cfg.buf_samples) return fail(c, B200_E_INVAL, "several buffers per call need buf_len == buf_samples");
    if (any_in_flight(c)) return fail(c, B200_E_STATE, "asynchronous steps are in flight: call b200_demod_wait first");
    const size_t row = (size_t)n_buffers * buf_len * 2;
    if (host_stride < row) return fail(c, B200_E_INVAL, "host_stride_bytes smaller than one stream's data");
    for (uint32_t s = first; s < first + ns; s++) {
        if (c->kind[s] >= 2) return fail(c, B200_E_STATE, "stream %u mixes submit kinds in one run", s);
        if (c->pending[s].size() + n_buffers > c->cfg.max_buffers_per_run) return fail(c, B200_E_STATE, "stream %u would exceed max_buffers_per_run", s);
        if (c->kind[s] && c->cursor[s] != c->cursor[first]) return fail(c, B200_E_STATE, "strided submit needs all streams of the range at the same fill level");
    }
    CU(c, cudaSetDevice(c->device));
    const size_t off0 = c->kind[first] ? c->cursor[first] : (size_t)B200_TRAIL * 2;
    CU(c, cudaMemcpy2DAsync(c->d_arena + (size_t)first * c->stream_stride + off0, c->stream_stride, iq, host_stride, row, ns,
                            cudaMemcpyHostToDevice, c->stream));
    for (uint32_t s = first; s < first + ns; s++) {
        c->kind[s] = 1;
        for (uint32_t b = 0; b < n_buffers; b++) {
            Pending p; p.n = buf_len; p.ts = ts + (int64_t)b * buf_len * 5; p.off = off0 + (size_t)b * buf_len * 2;
            p.restart = b == 0 && c->restart_next[s];
            c->pending[s].push_back(p);
        }
        c->restart_next[s] = 0;
        c->cursor[s] = off0 + row;
    }
    return B200_OK;
}

API int b200_demod_submit_iq_sc16(b200_demod_ctx *c, uint32_t s, const int16_t *iq, uint32_t n, int64_t ts, int q11) {
    if (!c) return B200_E_INVAL;
    if (s >= c->cfg.n_streams || (!iq && n)) return fail(c, B200_E_INVAL, "bad stream or buffer");
    if (n > c->cfg.buf_samples) return fail(c, B200_E_INVAL, "buffer of %u samples exceeds buf_samples=%u", n, c->cfg.buf_samples);
    if (c->pending[s].size() >= c->cfg.max_buffers_per_run) return fail(c, B200_E_STATE, "stream %u already has max_buffers_per_run buffers queued", s);
    if (any_in_flight(c)) return fail(c, B200_E_STATE, "asynchronous steps are in flight: call b200_demod_wait first");
    if (c->kind[s] && c->kind[s] != 3) return fail(c, B200_E_STATE, "stream %u mixes submit kinds in one run", s);
    CU(c, cudaSetDevice(c->device));
    const uint32_t S = c->cfg.n_streams, K = c->cfg.max_buffers_per_run;
    if (!c->d_raw16) {
        CU(c, cudaMalloc((void **)&c->d_raw16, (size_t)c->cfg.buf_samples * 4 + 16));
        CU(c, dev_alloc(&c->d_fsum, (size_t)S * K)); CU(c, pin_alloc(&c->h_fsum, (size_t)S * K));
    }
    if (!c->kind[s]) { c->kind[s] = 3; c->cursor[s] = (size_t)B200_TRAIL * 2; }
    uint8_t *region = c->d_arena + (size_t)s * c->stream_stride;
    Pending p;
    p.n = n; p.ts = ts; p.off = c->cursor[s]; p.fsum = (int)c->n_fsum++; p.restart = c->restart_next[s] != 0;
    // one staging buffer: the copy and the converter of this submit are ordered on the stream before the next submit's copy
    if (n) CU(c, cudaMemcpyAsync(c->d_raw16, iq, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    Sc16Params cp = {};
    cp.iq = reinterpret_cast<const uint32_t *>(c->d_raw16); cp.mag = reinterpret_cast<uint16_t *>(region + p.off) - B200_TRAIL;
    cp.sums = c->d_fsum + p.fsum; cp.sums_stride = 1; cp.n_segs = 1; cp.n_bufs = 1; cp.buf_len = n;
    cp.seg0.flags = SEG_HALO_ZERO;        // buffer 0 of receiver 0 (here: this buffer); its halo is already in the arena
    cp.scale = q11 ? 1.0f / 2048.0f : 1.0f / 32768.0f;
    { int r = b200_launch_sc16_convert(&cp, c->stream);
      if (r) return fail(c, B200_E_CUDA, "sc16 convert launch: %s", cudaGetErrorString((cudaError_t)r)); }
    c->cursor[s] = p.off + (size_t)n * 2;
    c->pending[s].push_back(p);
    c->restart_next[s] = 0;
    return B200_OK;
}

API int b200_demod_restart_stream(b200_demod_ctx *c, uint32_t s) {
    if (!c) return B200_E_INVAL;
    if (s >= c->cfg.n_streams) return fail(c, B200_E_INVAL, "bad stream");
    c->restart_next[s] = 1;               // read by the next submit_iq_* of this receiver (oracle_stream_restart)
    return B200_OK;
}

API int b200_demod_submit_iq_uc8(b200_demod_ctx *c, uint32_t s, const uint8_t *iq, uint32_t n, int64_t ts) { return submit_common(c, s, iq, n, ts, false); }
API int b200_demod_submit_mag_u16(b200_demod_ctx *c, uint32_t s, const uint16_t *data, uint32_t n, int64_t ts) { return submit_common(c, s, data, n, ts, true); }
API int b200_demod_submit_mag_u16_levels(b200_demod_ctx *c, uint32_t s, const uint16_t *data, uint32_t n, int64_t ts, double mean_level, double mean_power) {
    const double lv[2] = {mean_level, mean_power};
    return submit_common(c, s, data, n, ts, true, lv);
}

API int b200_demod_set_preamble_threshold(b200_demod_ctx *c, int32_t thr) {
    if (!c) return B200_E_INVAL;
    if (thr <= 0) return fail(c, B200_E_INVAL, "preamble threshold must be > 0");
    if (any_in_flight(c)) return fail(c, B200_E_STATE, "asynchronous steps are in flight: call b200_demod_wait first");
    c->cfg.preamble_threshold = thr;      // read when the next run is enqueued
    return B200_OK;
}

// ---- the pipeline ------------------------------------------------------------------------------
static void add_segment(Slot &sl, uint32_t stream, const uint8_t *base, uint32_t npos, uint32_t buf_len, uint32_t n_bufs,
                        uint32_t flags, int64_t first_ts, int32_t thr) {
    Segment &g = sl.h_segs[sl.nseg];
    memset(&g, 0, sizeof g);
    g.base = base; g.first_ts = first_ts; g.thr = thr; g.npos = npos; g.buf_len = buf_len ? buf_len : 1;
    g.lead = (uint32_t)(((uintptr_t)base & 15) / 2); g.flags = flags; g.stream = stream;
    g.first_buf = sl.nbuf; g.n_bufs = n_bufs; g.tile_begin = sl.ntile;
    g.n_tiles = npos ? (g.lead + npos + SCAN_TILE - 1) / SCAN_TILE : 0;
    for (uint32_t t = 0; t < g.n_tiles; t++) sl.h_tile_seg[sl.ntile + t] = sl.nseg | ((t & 3u) == 0 ? TILE_QUAD_START : 0u);
    sl.ntile += g.n_tiles; sl.nbuf += n_bufs; sl.nseg++;
}

// Enqueue one run held by `sl`: tables up, stage A on `scan`, stage B (with the finalizer) + first result copy on `res`
// (the same stream in blocking mode).  `prev_stop`: stop word of the step in flight before this one (async mode), see stop_out.
static int enqueue(b200_demod_ctx *c, Slot &sl, cudaStream_t scan, cudaStream_t res, const uint32_t *prev_stop) {
    const uint32_t S = c->cfg.n_streams;
    // The run's descriptors.  Pipelined: they go up on the copy stream right now, while the step before this one is still
    // scanning, so that this step's scan kernel is ready the moment that one ends — together with the other step's stage B,
    // and placed before it (stream priority): one persistent CTA per SM first, stage B's small CTAs into what is left.
    // (Nothing on the device still reads this slot's blocks: its previous run was collected.  The step after that run learns whether
    // it has to be skipped from the slot's stop word, which this run's stage B overwrites only after that step's stage B - same stream.)
    cudaStream_t pre = scan != res ? c->copy_stream : scan;
    layout_run(c, sl);
    // One receiver, one segment, no Mode A/C (the drop-in's call shape): the descriptor rides in the kernel parameters
    const bool one_seg = S == 1 && sl.nseg == 1 && !(c->cfg.flags & B200_CFG_MODE_AC) && scan == res;
    sl.desc_on_device = !one_seg;
    if (!one_seg) CU(c, cudaMemcpyAsync(sl.d_desc, sl.h_desc, sl.desc_bytes, cudaMemcpyHostToDevice, pre));
    if (c->beast_slot == (int)(&sl - c->slot)) c->beast_slot = -1;      // the encoded records belong to the run being replaced
    // One receiver, no Mode A/C: the stage B kernel publishes the results into the host's (mapped) copy itself and zeroes the control
    // block and the per-buffer sums when it is done - no memset, no device-to-host copy in the stream.
    const bool publish = S == 1 && !(c->cfg.flags & B200_CFG_MODE_AC) && scan == res;
    const bool timing = !((c->cfg.flags & B200_CFG_NO_TIMING) && scan == res);
    // Control block + per-buffer sums: zeroed by a copy engine.  (A memset runs on the SMs, and while the step before this one keeps
    // them busy it would hold this step's scan kernel back.)
    if (!(publish && sl.res_clean && sl.nbuf <= sl.clean_bufs))
        CU(c, cudaMemcpyAsync(sl.d_res, c->h_zero, sizeof(RunCtl) + (size_t)sl.nbuf * sizeof(BufAcc), cudaMemcpyHostToDevice, pre));
    sl.res_clean = false; sl.published = publish; sl.timed = timing;
    if (pre != scan) { CU(c, cudaEventRecord(sl.ev[7], pre)); CU(c, cudaStreamWaitEvent(scan, sl.ev[7], 0)); }
    sl.launches = 0;

    ScanParams sp;
    sp.segs = sl.d_segs; sp.tile_seg = sl.d_tile_seg; sp.n_tiles = sl.ntile; sp.pos_pool = sl.d_pos_pool; sp.rec_pool = sl.d_rec_pool;
    sp.key_pool = sl.d_key_pool; sp.tile_out = sl.d_tile_out; sp.buf_acc = sl.d_buf_acc; sp.ctl = sl.d_ctl;
    sp.rec_cap = sl.rec_cap; sp.warps_per_cta = 0; sp.static_tiles = 0; sp.need_lut = 0; sp.sub_chunks = (uint32_t)c->scan_sub;
    sp.one_seg_valid = one_seg ? 1u : 0u;
    if (sl.nseg) sp.one_seg = sl.h_segs[0]; else memset(&sp.one_seg, 0, sizeof sp.one_seg);
    for (uint32_t i = 0; i < sl.nseg; i++) if (!(sl.h_segs[i].flags & SEG_MAG)) sp.need_lut = 1;
    sp.nfix = c->cfg.nfix_crc; sp.fixdf = c->cfg.fix_df;
    sp.stage_rec = c->d_stage_rec; sp.stage_key = c->d_stage_key; sp.stage_cap = c->stage_cap; sp.q1_over = c->d_q1_over; sp.tick_scratch = c->d_tick_scratch;
    sp.stream_addable = sl.d_addable;
    sp.mag_copy = (c->cfg.flags & B200_CFG_MODE_AC) ? sl.d_mag_copy : nullptr;
    // demod_2400.c:112-127
    sp.short_set = (1u << 0) | (1u << 4) | (1u << 5) | (1u << 11);
    sp.long_set = (1u << 16) | (1u << 17) | (1u << 18) | (1u << 20) | (1u << 21);
    if (sp.nfix && sp.fixdf) for (int b = 0; b < 5; b++) sp.long_set |= 1u << (17 ^ (1 << b));
    if (timing) CU(c, cudaEventRecord(sl.ev[0], scan));
    if (sl.sc16) {          // after the zeroing of the per-buffer sums above: the converter writes BufAcc::fsum
        sl.conv.sums = &sl.d_buf_acc->fsum; sl.conv.sums_stride = sizeof(BufAcc) / sizeof(float2); sl.conv.segs = sl.d_segs;
        int r = b200_launch_sc16_convert(&sl.conv, scan); if (r) return fail(c, B200_E_CUDA, "sc16 convert launch: %s", cudaGetErrorString((cudaError_t)r));
        sl.launches++;
    }
    sl.scan_grid = scan != res ? ((c->part_fixed || !c->part_n) ? c->n_sm_scan_async : c->part_n) : c->n_sm_scan;
    if (sl.ntile) { int r = b200_launch_scan(&sp, c->d_tables, sl.scan_grid, scan); if (r) return fail(c, B200_E_CUDA, "scan launch: %s", cudaGetErrorString((cudaError_t)r)); sl.launches++; }
    if (timing) CU(c, cudaEventRecord(sl.ev[1], scan));
    if (res != scan) CU(c, cudaStreamWaitEvent(res, sl.ev[1], 0));

    // demodulate2400AC on the same buffers (readsb.c:872-874).  Its scan and walk are stateless, so they stay on the
    // scan stream, where they overlap stage B of this step when the two streams differ.
    const bool mode_ac = (c->cfg.flags & B200_CFG_MODE_AC) != 0;
    AcWalkParams aw = {};
    if (mode_ac) {
        if (sl.nbuf) CU(c, cudaMemcpyAsync(sl.d_ac_levels, sl.h_ac_levels, (size_t)sl.nbuf * sizeof(AcLevel), cudaMemcpyHostToDevice, scan));
        AcScanParams as;
        as.levels = sl.d_ac_levels; as.fsum = sl.sc16 ? &sl.d_buf_acc->fsum : c->d_fsum;
        as.segs = sl.d_segs; as.n_segs = sl.nseg; as.tile_seg = sl.d_tile_seg; as.n_tiles = sl.ntile; as.buf_acc = sl.d_buf_acc;
        as.tables = c->d_tables; as.noise = sl.d_ac_noise; as.bitmap = sl.d_ac_bitmap; as.ctl = sl.d_ctl; as.mag_copy = sl.d_mag_copy;
        aw.segs = sl.d_segs; aw.n_segs = sl.nseg; aw.stream_seg_begin = sl.d_stream_seg_begin; aw.n_streams = S; aw.bitmap = sl.d_ac_bitmap;
        aw.noise = sl.d_ac_noise; aw.lut_full = c->d_lut_full; aw.ac_out = sl.d_ac_out; aw.ac_count = sl.d_ac_count; aw.per_buf_cap = c->ac_cap;
        aw.state = c->d_state; aw.ctl = sl.d_ctl;
        { int r = b200_launch_modeac(&as, &aw, c->n_sm, scan); if (r) return fail(c, B200_E_CUDA, "mode a/c launch: %s", cudaGetErrorString((cudaError_t)r)); sl.launches += 3; }
        CU(c, cudaEventRecord(sl.ev[6], scan));
    }

    FinalizeParams fp;
    fp.segs = sl.d_segs; fp.stream_seg_begin = sl.d_stream_seg_begin; fp.n_streams = S; fp.frames = sl.d_frames;
    fp.frame_span = sl.d_frame_span; fp.frame_cap = c->frame_cap; fp.packed = sl.d_packed;
    fp.buf_acc = sl.d_buf_acc; fp.state = c->d_state; fp.lut_full = c->d_lut_full; fp.rec_pool = sl.d_rec_pool;
    fp.one_seg = sp.one_seg; fp.one_seg_valid = sp.one_seg_valid;
    const bool solo = S == 1;          // one receiver: resolve_solo_kernel (also publishes its results / carries the halo)
    ResolveParams rp;
    rp.segs = sl.d_segs; rp.stream_seg_begin = sl.d_stream_seg_begin; rp.n_streams = S; rp.pos_pool = sl.d_pos_pool;
    rp.rec_pool = sl.d_rec_pool; rp.key_pool = sl.d_key_pool; rp.tile_out = sl.d_tile_out; rp.buf_acc = sl.d_buf_acc; rp.buf_out = sl.d_buf_out;
    rp.state = c->d_state; rp.frames = sl.d_frames; rp.frame_cap = c->frame_cap; rp.per_buf_cap = c->cfg.buf_samples / 113 + 2;
    rp.ctl = sl.d_ctl; rp.prev_stop = prev_stop; rp.stop_out = c->d_stop + (&sl - c->slot); rp.ttl_ms = c->cfg.icao_ttl_ms; rp.stream_addable = sl.d_addable;
    rp.one_seg = sp.one_seg; rp.one_seg_valid = sp.one_seg_valid;
    rp.solo = solo ? 1u : 0u; rp.fin = fp;
    rp.publish_src = nullptr; rp.publish_dst = nullptr; rp.publish_head = 0; rp.publish_clear = 0;
    rp.carry_dst = nullptr; rp.carry_src = nullptr;
    if (solo && sl.carry_in_kernel != 0xffffffffu) {      // host-buffer run of one receiver: the halo carry rides in the stage B kernel
        rp.carry_dst = reinterpret_cast<uint16_t *>(c->d_arena);
        rp.carry_src = reinterpret_cast<const uint16_t *>(c->d_arena + sl.carry_in_kernel);
    }
    if (publish) {
        rp.publish_src = reinterpret_cast<const uint4 *>(sl.d_res); rp.publish_dst = reinterpret_cast<uint4 *>(sl.d_res_host);
        rp.publish_head = (uint32_t)sl.res_head; rp.publish_clear = (uint32_t)(sizeof(RunCtl) + (size_t)sl.nbuf * sizeof(BufAcc));
    }
    { const int grown = !c->icao_grown.empty();
      int r = b200_launch_resolve(&rp, grown, res); if (r) return fail(c, B200_E_CUDA, "resolve launch: %s", cudaGetErrorString((cudaError_t)r)); sl.launches += solo ? 1 : 1 + grown; }
    if (timing) { CU(c, cudaEventRecord(sl.ev[2], res)); CU(c, cudaEventRecord(sl.ev[3], res)); }     // (stage B and finalizer: one launch)

    if (mode_ac) {      // per-buffer reply lists -> one packed array in buffer order, receiver statistics
        if (res != scan) CU(c, cudaStreamWaitEvent(res, sl.ev[6], 0));
        { int r = b200_launch_ac_pack(sl.d_ac_out, sl.d_ac_count, sl.d_ac_prefix, sl.d_ac_packed, sl.nbuf, c->ac_cap, sl.d_ctl, res); if (r) return fail(c, B200_E_CUDA, "mode a/c pack launch: %s", cudaGetErrorString((cudaError_t)r)); sl.launches += 2; }
        { int r = b200_launch_modeac_stats(&aw, sl.d_ac_prefix, res); if (r) return fail(c, B200_E_CUDA, "mode a/c stats launch: %s", cudaGetErrorString((cudaError_t)r)); sl.launches++; }
        CU(c, cudaMemcpyAsync(sl.h_ac_prefix, sl.d_ac_prefix, ((size_t)sl.nbuf + 1) * 4, cudaMemcpyDeviceToHost, res));
    }

    // control block, per-buffer sums, frame prefix, buffer results and the first frames: one copy (small runs need no second one)
    sl.first_frames = (uint32_t)std::min<size_t>(FIRST_COPY_FRAMES, (size_t)S * c->frame_cap);
    if (publish) sl.first_frames = 0xffffffffu;          // the kernel has put every frame into the host's copy
    else CU(c, cudaMemcpyAsync(sl.h_res, sl.d_res, sl.res_head + (size_t)sl.first_frames * sizeof(b200_frame), cudaMemcpyDeviceToHost, res));
    if (timing) CU(c, cudaEventRecord(sl.ev[4], res));
    return B200_OK;
}

// Second half: wait for the first result copy, fetch the frames, derive the timings.  Returns B200_OK, or a positive
// value when the run has to be repeated: 1 = record pool too small, 2 = dense-tile scratch arena needed, 3 = skipped
// because the step before it had to be repeated, 4 = a receiver's ICAO filter tables have to grow first.
static int collect(b200_demod_ctx *c, Slot &sl, cudaStream_t res) {
    if (sl.timed) CU(c, cudaEventSynchronize(sl.ev[4])); else CU(c, cudaStreamSynchronize(res));
    if (sl.published) { sl.res_clean = true; sl.clean_bufs = sl.nbuf; }     // the kernel zeroed RunCtl + BufAcc[] after publishing them
    const uint32_t ov = sl.h_ctl->overflow;
    if (ov & 1u) return 1;
    if ((ov & 2u) && sl.h_ctl->stage_need > c->stage_cap) return 2;
    if (ov & 16u) return 3;
    if (ov & 8u) return 4;
    if (ov & 2u) return fail(c, B200_E_OVERFLOW, "a run of tiles exceeded the record staging capacity even after regrowth");
    if (ov & 4u) return fail(c, B200_E_OVERFLOW, "per-stream frame capacity exceeded");
    if (ov & 32u) return fail(c, B200_E_OVERFLOW, "Mode A/C candidate capacity exceeded");
    const bool mode_ac = (c->cfg.flags & B200_CFG_MODE_AC) != 0;
    const uint32_t total_ac = mode_ac ? sl.h_ac_prefix[sl.nbuf] : 0;
    sl.ms[3] = 0;
    if (mode_ac && sl.timed) cudaEventElapsedTime(&sl.ms[3], sl.ev[1], sl.ev[6]);       // Mode A/C noise + scan + walk kernels
    if (total_ac) CU(c, cudaMemcpyAsync(sl.h_ac_packed, sl.d_ac_packed, (size_t)total_ac * sizeof(b200_modeac), cudaMemcpyDeviceToHost, c->copy_stream));
    const uint32_t total = sl.h_ctl->total_frames;
    sl.run_frames = total;
    if (total_ac && total <= sl.first_frames) { CU(c, cudaEventRecord(sl.ev[5], c->copy_stream)); CU(c, cudaEventSynchronize(sl.ev[5])); }
    const bool more_frames = total > sl.first_frames;
    if (more_frames) {
        // The frame copy must not queue behind the NEXT step's stage B on the resolve stream: its own stream,
        // ordered after this slot's finalize only (ev[4] already completed: finalize is done).
        (void)res;
        CU(c, cudaMemcpyAsync(sl.h_packed + sl.first_frames, sl.d_packed + sl.first_frames, (size_t)(total - sl.first_frames) * sizeof(b200_frame),
                              cudaMemcpyDeviceToHost, c->copy_stream));
        CU(c, cudaEventRecord(sl.ev[5], c->copy_stream));
        CU(c, cudaEventSynchronize(sl.ev[5]));
    }
    for (uint32_t b = 0; b < sl.nbuf; b++) {
        sl.h_buf_out[b].sum_level = sl.h_buf_acc[b].sum_level;
        sl.h_buf_out[b].sum_power = sl.h_buf_acc[b].sum_power;
        sl.h_buf_out[b].sum_signal_power = sl.h_buf_acc[b].sum_signal_power;
    }
    if (sl.sc16) for (uint32_t b = 0; b < sl.nbuf; b++) {     // the reference's float accumulators instead of the integer sums
        uint32_t lv, pw;
        memcpy(&lv, &sl.h_buf_acc[b].fsum.x, 4); memcpy(&pw, &sl.h_buf_acc[b].fsum.y, 4);
        sl.h_buf_out[b].sum_level = lv; sl.h_buf_out[b].sum_power = pw;
    }
    if (sl.timed) {
        cudaEventElapsedTime(&sl.ms[1], sl.ev[0], sl.ev[1]);
        cudaEventElapsedTime(&sl.ms[2], sl.ev[1], sl.ev[2]);
        cudaEventElapsedTime(&sl.ms[0], sl.ev[0], (more_frames || total_ac) ? sl.ev[5] : sl.ev[4]);
        cudaEventElapsedTime(&sl.ms[4], sl.ev[3], (more_frames || total_ac) ? sl.ev[5] : sl.ev[4]);
    } else sl.ms[0] = sl.ms[1] = sl.ms[2] = sl.ms[4] = 0;
    return B200_OK;
}

// Every receiver whose capacity check (or b200_demod_icao_add) asked for larger filter tables gets them: both generations are
// re-inserted on the device; the default tables stay part of the context's slab, grown ones are freed when replaced.
static int grow_icao_tables(b200_demod_ctx *c) {
    const uint32_t S = c->cfg.n_streams;
    c->h_state.resize(S);
    CU(c, cudaStreamSynchronize(c->stream));
    CU(c, cudaMemcpy(c->h_state.data(), c->d_state, (size_t)S * sizeof(StreamState), cudaMemcpyDeviceToHost));
    for (uint32_t s = 0; s < S; s++) {
        const StreamState &st = c->h_state[s];
        if (st.grow_log2 <= st.cap_log2) continue;
        if (st.grow_log2 > ICAO_MAXBITS + 1) return fail(c, B200_E_OVERFLOW, "receiver %u: ICAO filter beyond 2^%d slots", s, ICAO_MAXBITS + 1);
        uint32_t *t0 = nullptr, *t1 = nullptr;
        const size_t n = (size_t)1 << st.grow_log2;
        if (dev_alloc(&t0, n) != cudaSuccess || dev_alloc(&t1, n) != cudaSuccess) { cudaFree(t0); return fail(c, B200_E_NOMEM, "receiver %u: cannot grow the ICAO filter to 2 x %zu slots", s, n); }
        int r = b200_launch_icao_rehash(c->d_state, s, t0, t1, st.grow_log2, c->stream);
        if (r) return fail(c, B200_E_CUDA, "icao rehash launch: %s", cudaGetErrorString((cudaError_t)r));
        CU(c, cudaStreamSynchronize(c->stream));
        for (uint32_t *old : {st.tab[0], st.tab[1]}) {
            auto it = std::find(c->icao_grown.begin(), c->icao_grown.end(), old);
            if (it != c->icao_grown.end()) { cudaFree(old); c->icao_grown.erase(it); }
        }
        c->icao_grown.push_back(t0); c->icao_grown.push_back(t1);
    }
    return B200_OK;
}

// Repairs after collect() asked for a repeat.  Every slot gets the new capacity so that later steps do not trip again.
static int regrow(b200_demod_ctx *c, Slot &sl, int why) {
    if (why == 4) return grow_icao_tables(c);
    if (why == 1) {
        const uint32_t need = std::max(sl.h_ctl->rec_alloc + sl.h_ctl->rec_alloc / 4 + 65536, sl.rec_cap);
        for (Slot &s : c->slot) {
            if (!s.allocated || s.rec_cap >= need) continue;
            cudaFree(s.d_rec_pool); s.d_rec_pool = nullptr;
            cudaFree(s.d_key_pool); s.d_key_pool = nullptr;
            s.rec_cap = need;
            if (dev_alloc(&s.d_rec_pool, s.rec_cap) != cudaSuccess || dev_alloc(&s.d_key_pool, s.rec_cap) != cudaSuccess)
                return fail(c, B200_E_NOMEM, "cannot grow the record pool to %u records", need);
        }
    } else if (why == 2) {       // a run of tiles with more live records than the per-warp staging areas hold: grow them to what it needs
        const uint32_t need = sl.h_ctl->stage_need + sl.h_ctl->stage_need / 8 + 64;
        cudaFree(c->d_stage_rec); cudaFree(c->d_stage_key); c->d_stage_rec = nullptr; c->d_stage_key = nullptr; c->stage_cap = 0;
        const size_t warps = (size_t)b200_scan_warps(c->n_sm);
        if (dev_alloc(&c->d_stage_rec, warps * need) != cudaSuccess || dev_alloc(&c->d_stage_key, warps * need) != cudaSuccess)
            return fail(c, B200_E_NOMEM, "cannot grow the record staging areas to %u records per warp", need);
        c->stage_cap = need;
    }
    return B200_OK;
}

// Blocking execution of the run held by `sl` on the context's stream, repeated after pool regrowth (stage A is
// stateless and stage B refuses to run after a stage A failure, so a repeat is exact).
static int execute_blocking(b200_demod_ctx *c, Slot &sl) {
    for (int attempt = 0; attempt < 8; attempt++) {
        int rc = enqueue(c, sl, c->stream, c->stream, nullptr);
        if (rc != B200_OK) return rc;
        rc = collect(c, sl, c->stream);
        if (rc <= 0) return rc;
        rc = regrow(c, sl, rc);
        if (rc != B200_OK) return rc;
    }
    return fail(c, B200_E_NOMEM, "record pool still too small after regrowth");
}

API int b200_demod_run(b200_demod_ctx *c) {
    if (!c) return B200_E_INVAL;
    if (any_in_flight(c)) return fail(c, B200_E_STATE, "asynchronous steps are in flight: call b200_demod_wait first");
    CU(c, cudaSetDevice(c->device));
    const uint32_t S = c->cfg.n_streams, BUF = c->cfg.buf_samples;
    Slot &sl = c->slot[0];
    c->cur = 0;
    sl.nseg = sl.ntile = sl.nbuf = 0; sl.upload_tiles = true; sl.cached_tiles = 0; sl.sc16 = false;
    const int32_t thr = c->cfg.preamble_threshold;
    std::vector<std::pair<uint32_t, int>> fsum_of_buf;      // (buffer of the run, float-sum slot) for sc16 buffers
    std::vector<std::pair<uint32_t, const Pending *>> given_levels;   // (buffer of the run, hand-off that brought its own mean_level / mean_power)
    std::vector<uint8_t> halo_after(c->halo_valid);        // committed only when the run succeeded (a failed run leaves no halo behind)
    for (uint32_t s = 0; s < S; s++) {
        sl.h_stream_seg_begin[s] = sl.nseg;
        sl.stream_buf_begin[s] = sl.nbuf;
        c->h_carry_src[s] = 0xffffffffu;
        const auto &pl = c->pending[s];
        if (pl.empty()) continue;
        const uint8_t *region = c->d_arena + (size_t)s * c->stream_stride;
        if (c->kind[s] == 2) {
            for (const Pending &p : pl) {
                if (p.has_levels) given_levels.push_back({sl.nbuf, &p});
                add_segment(sl, s, region + p.off, p.n, p.n, 1, SEG_MAG, p.ts, thr);
            }
        } else {
            // consecutive full buffers with contiguous timestamps form one segment; a partial buffer ends it, and so does every buffer
            // shorter than the halo: the buffer after it starts with a zero halo (sdr_ifile.c:207-212), not with its samples
            size_t i = 0;
            bool halo_ok = c->halo_valid[s];
            while (i < pl.size()) {
                size_t j = i;
                uint32_t npos = 0;
                if (pl[i].restart) halo_ok = false;        // sdr_rtlsdr.c:381-385: a buffer after dropped samples starts with a zero halo
                for (;;) {
                    npos += pl[j].n;
                    const bool more = j + 1 < pl.size() && pl[j].n == BUF && BUF >= B200_TRAIL && pl[j + 1].ts == pl[j].ts + (int64_t)BUF * 5 && !pl[j + 1].restart;
                    if (!more) break;
                    j++;
                }
                const uint32_t nb = (uint32_t)(j - i + 1);
                add_segment(sl, s, region + pl[i].off - (size_t)B200_TRAIL * 2, npos, nb > 1 ? BUF : pl[i].n, nb,
                            (halo_ok ? 0 : SEG_HALO_ZERO) | (c->kind[s] == 3 ? SEG_MAG : 0), pl[i].ts, thr);
                if (c->kind[s] == 3) for (size_t q = i; q <= j; q++) fsum_of_buf.push_back({sl.nbuf - nb + (uint32_t)(q - i), pl[q].fsum});
                halo_ok = pl[j].n >= B200_TRAIL;      // sdr_ifile.c:209-213
                i = j + 1;
            }
            halo_after[s] = halo_ok;
            if (halo_ok) c->h_carry_src[s] = (uint32_t)(c->cursor[s] - (size_t)B200_TRAIL * 2);
        }
    }
    sl.h_stream_seg_begin[S] = sl.nseg;
    sl.stream_buf_begin[S] = sl.nbuf;
    if (c->cfg.flags & B200_CFG_MODE_AC) {                  // demod_2400.c:580-581: the noise floor comes from the mag_buf's own levels
        memset(sl.h_ac_levels, 0, (size_t)sl.nbuf * sizeof(AcLevel));
        for (const auto &g : given_levels) { AcLevel &l = sl.h_ac_levels[g.first]; l.mode = AC_LEVEL_GIVEN; l.mean_level = g.second->mean_level; l.mean_power = g.second->mean_power; }
        for (const auto &bf : fsum_of_buf) { AcLevel &l = sl.h_ac_levels[bf.first]; l.mode = AC_LEVEL_FSUM; l.idx = (uint32_t)bf.second; }
    }
    sl.carry_in_kernel = S == 1 ? c->h_carry_src[0] : 0xffffffffu;
    int rc = execute_blocking(c, sl);
    if (rc == B200_OK && !fsum_of_buf.empty()) {      // sc16 input: the reference's float accumulators instead of the integer sums
        if (cudaMemcpyAsync(c->h_fsum, c->d_fsum, (size_t)c->n_fsum * sizeof(float2), cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
            cudaStreamSynchronize(c->stream) != cudaSuccess) rc = fail(c, B200_E_CUDA, "sc16 sums copy failed");
        else for (const auto &bf : fsum_of_buf) {
            uint32_t lv, pw;
            memcpy(&lv, &c->h_fsum[bf.second].x, 4); memcpy(&pw, &c->h_fsum[bf.second].y, 4);
            sl.h_buf_out[bf.first].sum_level = lv; sl.h_buf_out[bf.first].sum_power = pw;
        }
    }
    c->n_fsum = 0;
    // next run: move each IQ stream's tail to the front of its region
    bool any_carry = false;
    for (uint32_t s = 0; s < S; s++) any_carry = any_carry || c->h_carry_src[s] != 0xffffffffu;
    if (S == 1) any_carry = false;             // carried by the stage B kernel itself (enqueue: carry_in_kernel)
    sl.carry_in_kernel = 0xffffffffu;
    if (rc == B200_OK && any_carry) {          // (magnitude hand-offs bring their halo with them: nothing to carry)
        cudaMemcpyAsync(c->d_carry_src, c->h_carry_src, S * 4, cudaMemcpyHostToDevice, c->stream);
        carry_halo_kernel<<<S, 128, 0, c->stream>>>(c->d_arena, c->stream_stride, c->d_carry_src, S);
        sl.launches++;
        if (cudaStreamSynchronize(c->stream) != cudaSuccess) rc = fail(c, B200_E_CUDA, "halo carry failed");
    }
    for (uint32_t s = 0; s < S; s++) {
        // after a failed run the tail was not carried: the receiver's next buffer starts like a fresh stream (zero halo) instead of
        // reading stale arena bytes
        if (!c->pending[s].empty() && c->kind[s] != 2) c->halo_valid[s] = rc == B200_OK ? halo_after[s] : 0;
        c->pending[s].clear(); c->kind[s] = 0; c->cursor[s] = 0;
    }
    return rc;
}

// Checks a step's arguments before anything is enqueued or changed: `fmt`, the alignment and length rules, every receiver's descriptor and
// a stride that holds the largest count (*max_n).  `device`: d_iq / stream_stride_bytes must be 16-byte aligned.
static int check_rx(b200_demod_ctx *c, int fmt, const void *iq, uint64_t stride, uint32_t buf_len, const b200_rx_step *rx, bool device,
                    uint32_t *max_n) {
    const uint32_t S = c->cfg.n_streams;
    if (!iq || !rx) return fail(c, B200_E_INVAL, "null sample or descriptor pointer");
    if (fmt != FMT_UC8 && fmt != FMT_SC16 && fmt != FMT_SC16Q11) return fail(c, B200_E_INVAL, "format %d is not B200_FORMAT_UC8, _SC16 or _SC16Q11", fmt);
    if (device && (((uintptr_t)iq & 15) || (stride & 15))) return fail(c, B200_E_INVAL, "d_iq and stream_stride_bytes must be 16-byte aligned");
    if (buf_len == 0 || buf_len > c->cfg.buf_samples || (buf_len & 7)) return fail(c, B200_E_INVAL, "buf_len must be 1 .. buf_samples and a multiple of 8");
    uint32_t m = 0;
    for (uint32_t s = 0; s < S; s++) {
        const b200_rx_step &r = rx[s];
        if (r.n_buffers > c->cfg.max_buffers_per_run) return fail(c, B200_E_INVAL, "receiver %u: %u buffers exceed max_buffers_per_run=%u", s, r.n_buffers, c->cfg.max_buffers_per_run);
        if (r.preamble_threshold < 0) return fail(c, B200_E_INVAL, "receiver %u: negative preamble threshold", s);
        if (r.reserved_ || (r.flags & ~B200_RX_CONTINUES)) return fail(c, B200_E_INVAL, "receiver %u: reserved_ and unknown flag bits must be 0", s);
        m = std::max(m, r.n_buffers);
        // a buffer shorter than the halo leaves the next one a zero halo (sdr_ifile.c:207-212), which a step's segment cannot express
        if (buf_len < B200_TRAIL && (r.n_buffers > 1 || (r.n_buffers && (r.flags & B200_RX_CONTINUES))))
            return fail(c, B200_E_INVAL, "receiver %u: buffers of %u < %u samples go one per step, without B200_RX_CONTINUES", s, buf_len, (unsigned)B200_TRAIL);
    }
    if ((uint64_t)m * buf_len * fmt_bytes(fmt) > stride && S > 1) return fail(c, B200_E_INVAL, "stride smaller than the largest receiver's data");
    *max_n = m;
    return B200_OK;
}

// Builds a device-resident step in `sl` from checked arguments: one segment per receiver present, none for an absent one.
static int build_device_run(b200_demod_ctx *c, Slot &sl, int fmt, const uint8_t *d_iq, uint64_t stride, uint32_t buf_len, const b200_rx_step *rx) {
    const uint32_t S = c->cfg.n_streams;
    sl.sc16 = fmt != FMT_UC8;
    if (sl.sc16 && !sl.d_slab) {
        const size_t stride16 = ((size_t)2 + B200_TRAIL + (size_t)c->cfg.max_buffers_per_run * c->cfg.buf_samples + 32 + 127) & ~(size_t)127;
        if (dev_alloc(&sl.d_slab, stride16 * S) != cudaSuccess) { sl.d_slab = nullptr; return fail(c, B200_E_NOMEM, "sc16 magnitude slab (%zu bytes)", stride16 * S * 2); }
        sl.slab_stride = stride16;
    }
    sl.nseg = sl.ntile = sl.nbuf = 0;
    bool same_counts = sl.cached_counts.size() == S;
    sl.cached_counts.resize(S);
    for (uint32_t s = 0; s < S; s++) {
        sl.h_stream_seg_begin[s] = sl.nseg;
        sl.stream_buf_begin[s] = sl.nbuf;
        const b200_rx_step &r = rx[s];
        same_counts = same_counts && sl.cached_counts[s] == r.n_buffers;
        sl.cached_counts[s] = r.n_buffers;
        if (!r.n_buffers) continue;
        const uint8_t *base = sl.sc16 ? reinterpret_cast<const uint8_t *>(sl.d_slab + s * sl.slab_stride + 2) : d_iq + (size_t)s * stride - (size_t)B200_TRAIL * 2;
        add_segment(sl, s, base, r.n_buffers * buf_len, buf_len, r.n_buffers, ((r.flags & B200_RX_CONTINUES) ? 0 : SEG_HALO_ZERO) | (sl.sc16 ? SEG_MAG : 0),
                    r.first_sample_timestamp, r.preamble_threshold ? r.preamble_threshold : c->cfg.preamble_threshold);
    }
    sl.h_stream_seg_begin[S] = sl.nseg;
    sl.stream_buf_begin[S] = sl.nbuf;
    if (c->cfg.flags & B200_CFG_MODE_AC) {
        memset(sl.h_ac_levels, 0, (size_t)sl.nbuf * sizeof(AcLevel));      // uc8 input: the exact sums
        if (sl.sc16) for (uint32_t b = 0; b < sl.nbuf; b++) {               // sc16: the converter's float sums, BufAcc::fsum of the buffer
            sl.h_ac_levels[b].mode = AC_LEVEL_FSUM; sl.h_ac_levels[b].idx = b * (uint32_t)(sizeof(BufAcc) / sizeof(float2));
        }
    }
    if (sl.sc16) {
        Sc16Params &p = sl.conv;
        p = Sc16Params();
        p.iq = reinterpret_cast<const uint32_t *>(d_iq); p.iq_stride = stride / 4;
        p.mag = sl.d_slab + 2; p.mag_stride = sl.slab_stride;
        p.n_segs = sl.nseg; p.n_bufs = sl.nbuf; p.buf_len = buf_len;
        if (sl.nseg) p.seg0 = sl.h_segs[0];
        p.scale = fmt == FMT_SC16Q11 ? 1.0f / 2048.0f : 1.0f / 32768.0f;
    }
    // the tile -> segment table only depends on the layout; skip its upload when nothing changed
    const uint64_t key = ((uint64_t)buf_len << 8) ^ (((uintptr_t)d_iq >> 4) & 15) ^ (stride << 20) ^ ((uint64_t)sl.sc16 << 63);
    sl.upload_tiles = !(sl.cached_tiles == sl.ntile && sl.cached_layout_key == key && same_counts);
    sl.cached_tiles = sl.ntile; sl.cached_layout_key = key;
    return B200_OK;
}

// The uniform calls: every receiver delivers n_buffers buffers from first_ts on, all continue or none, the context's threshold.
static const b200_rx_step *uniform_rx(b200_demod_ctx *c, uint32_t n_buffers, int continues, int64_t first_ts) {
    for (b200_rx_step &r : c->rx_uniform) { r = b200_rx_step(); r.first_sample_timestamp = first_ts; r.n_buffers = n_buffers; r.flags = continues ? B200_RX_CONTINUES : 0u; }
    return c->rx_uniform.data();
}

static int run_device_rx(b200_demod_ctx *c, int fmt, const uint8_t *d_iq, uint64_t stride, uint32_t buf_len, const b200_rx_step *rx) {
    if (!c) return B200_E_INVAL;
    if (any_in_flight(c)) return fail(c, B200_E_STATE, "asynchronous steps are in flight: call b200_demod_wait first");
    uint32_t max_n;
    int rc = check_rx(c, fmt, d_iq, stride, buf_len, rx, true, &max_n);
    if (rc != B200_OK) return rc;
    CU(c, cudaSetDevice(c->device));
    Slot &sl = c->slot[0];
    c->cur = 0;
    rc = build_device_run(c, sl, fmt, d_iq, stride, buf_len, rx);
    if (rc != B200_OK) return rc;
    return execute_blocking(c, sl);
}

static int run_device(b200_demod_ctx *c, const uint8_t *d_iq, uint64_t stride, uint32_t n_buffers, uint32_t buf_len,
                      int continues, int64_t first_ts, int fmt) {
    if (!c || !d_iq) return B200_E_INVAL;
    if (n_buffers == 0) return fail(c, B200_E_INVAL, "n_buffers/buf_len exceed the context's configuration");
    return run_device_rx(c, fmt, d_iq, stride, buf_len, uniform_rx(c, n_buffers, continues, first_ts));
}

API int b200_demod_run_device_uc8(b200_demod_ctx *c, const uint8_t *d_iq, uint64_t stride, uint32_t n_buffers, uint32_t buf_len,
                                  int continues, int64_t first_ts) {
    return run_device(c, d_iq, stride, n_buffers, buf_len, continues, first_ts, FMT_UC8);
}

API int b200_demod_run_device_sc16(b200_demod_ctx *c, const int16_t *d_iq, uint64_t stride, uint32_t n_buffers, uint32_t buf_len,
                                   int continues, int64_t first_ts, int q11) {
    return run_device(c, reinterpret_cast<const uint8_t *>(d_iq), stride, n_buffers, buf_len, continues, first_ts, q11 ? FMT_SC16Q11 : FMT_SC16);
}

API int b200_demod_run_device_rx(b200_demod_ctx *c, int format, const void *d_iq, uint64_t stride, uint32_t buf_len, const b200_rx_step *rx) {
    return run_device_rx(c, format, static_cast<const uint8_t *>(d_iq), stride, buf_len, rx);
}

// ---- asynchronous steps: at most NSLOT in flight ------------------------------------------------------------------------
// Enqueues the run built in slot next_async behind the steps already in flight and advances the ring.
static int launch_async(b200_demod_ctx *c, Slot &sl) {
    Slot &before = c->slot[(c->next_async + NSLOT - 1) % NSLOT];      // the step enqueued just before this one
    int rc = enqueue(c, sl, c->stream, c->res_stream, before.in_flight ? c->d_stop + (&before - c->slot) : nullptr);
    if (rc != B200_OK) return rc;
    if (c->n_flight == 0) c->head = c->next_async;
    sl.in_flight = true; sl.completed = false;
    c->next_async = (c->next_async + 1) % NSLOT;
    c->n_flight++;
    return B200_OK;
}

// The slot the next asynchronous step takes, allocated on first use.
static int async_slot(b200_demod_ctx *c, Slot **out) {
    Slot &sl = c->slot[c->next_async];
    if (sl.in_flight) return fail(c, B200_E_STATE, "%d steps are already in flight: call b200_demod_wait", NSLOT);
    if (!sl.allocated) {
        cudaError_t e = alloc_slot(c, sl, c->slot[0].rec_cap);
        if (e != cudaSuccess) return fail(c, B200_E_NOMEM, "pipeline slot %d: %s", c->next_async, cudaGetErrorString(e));
    }
    *out = &sl;
    return B200_OK;
}

static int run_device_rx_async(b200_demod_ctx *c, int fmt, const uint8_t *d_iq, uint64_t stride, uint32_t buf_len, const b200_rx_step *rx) {
    if (!c) return B200_E_INVAL;
    uint32_t max_n;
    int rc = check_rx(c, fmt, d_iq, stride, buf_len, rx, true, &max_n);
    if (rc != B200_OK) return rc;
    CU(c, cudaSetDevice(c->device));
    Slot *sl = nullptr;
    if ((rc = async_slot(c, &sl)) != B200_OK) return rc;
    if ((rc = build_device_run(c, *sl, fmt, d_iq, stride, buf_len, rx)) != B200_OK) return rc;
    return launch_async(c, *sl);
}

static int run_device_async(b200_demod_ctx *c, const uint8_t *d_iq, uint64_t stride, uint32_t n_buffers, uint32_t buf_len,
                            int continues, int64_t first_ts, int fmt) {
    if (!c || !d_iq) return B200_E_INVAL;
    if (n_buffers == 0) return fail(c, B200_E_INVAL, "n_buffers/buf_len exceed the context's configuration");
    return run_device_rx_async(c, fmt, d_iq, stride, buf_len, uniform_rx(c, n_buffers, continues, first_ts));
}

API int b200_demod_run_device_uc8_async(b200_demod_ctx *c, const uint8_t *d_iq, uint64_t stride, uint32_t n_buffers, uint32_t buf_len,
                                        int continues, int64_t first_ts) {
    return run_device_async(c, d_iq, stride, n_buffers, buf_len, continues, first_ts, FMT_UC8);
}

API int b200_demod_run_device_sc16_async(b200_demod_ctx *c, const int16_t *d_iq, uint64_t stride, uint32_t n_buffers, uint32_t buf_len,
                                         int continues, int64_t first_ts, int q11) {
    return run_device_async(c, reinterpret_cast<const uint8_t *>(d_iq), stride, n_buffers, buf_len, continues, first_ts, q11 ? FMT_SC16Q11 : FMT_SC16);
}

API int b200_demod_run_device_rx_async(b200_demod_ctx *c, int format, const void *d_iq, uint64_t stride, uint32_t buf_len, const b200_rx_step *rx) {
    return run_device_rx_async(c, format, static_cast<const uint8_t *>(d_iq), stride, buf_len, rx);
}

// ---- asynchronous host-buffer steps: the device-resident pipeline fed from library-owned input buffers ----------------
#define PIPE_LEAD 1024        // bytes in front of each receiver's samples: the 326-sample halo sits right before them
#define PIPE_LEAD16 2048      // ... for int16 I,Q samples (326 * 4 bytes)

static int run_host_rx_async(b200_demod_ctx *c, int fmt, const uint8_t *h_iq, uint64_t host_stride, uint32_t buf_len, const b200_rx_step *rx) {
    if (!c) return B200_E_INVAL;
    uint32_t max_n;
    int rc = check_rx(c, fmt, h_iq, host_stride, buf_len, rx, false, &max_n);
    if (rc != B200_OK) return rc;
    CU(c, cudaSetDevice(c->device));
    const uint32_t S = c->cfg.n_streams, K = c->cfg.max_buffers_per_run, BUF = c->cfg.buf_samples, bps = fmt_bytes(fmt);
    for (uint32_t s = 0; s < S; s++) if (!c->pending[s].empty()) return fail(c, B200_E_STATE, "buffers submitted for b200_demod_run are pending: run them first");
    const int pi = c->next_async;
    if (c->slot[pi].in_flight) return fail(c, B200_E_STATE, "%d steps are already in flight: call b200_demod_wait", NSLOT);
    for (uint32_t s = 0; s < S; s++)
        if (rx[s].n_buffers && (rx[s].flags & B200_RX_CONTINUES) && c->halo_bytes[s] != bps)
            return fail(c, B200_E_STATE, "receiver %u continues, but its last %s step did not leave >= 326 samples", s,
                        fmt == FMT_UC8 ? "uc8 host-buffer" : "sc16 host-buffer");
    Slot *slp = nullptr;
    if ((rc = async_slot(c, &slp)) != B200_OK) return rc;
    Slot &sl = *slp;
    const size_t lead = fmt == FMT_UC8 ? PIPE_LEAD : PIPE_LEAD16;
    uint8_t **pipe = fmt == FMT_UC8 ? c->d_pipe : c->d_pipe16;
    size_t &pipe_stride = fmt == FMT_UC8 ? c->pipe_stride : c->pipe16_stride;
    if (!pipe[0]) {
        pipe_stride = (lead + (size_t)K * BUF * bps + 64 + 255) & ~(size_t)255;
        for (int i = 0; i < NSLOT; i++) {
            if (cudaMalloc((void **)&pipe[i], pipe_stride * S + 256) != cudaSuccess) {
                for (int j = 0; j < i; j++) { cudaFree(pipe[j]); pipe[j] = nullptr; }
                pipe[i] = nullptr;
                return fail(c, B200_E_NOMEM, "pipelined input buffers (%d x %zu bytes)", NSLOT, pipe_stride * S);
            }
            if (!c->ev_in[i]) CU(c, cudaEventCreateWithFlags(&c->ev_in[i], cudaEventDisableTiming));
        }
    }
    if (!c->d_halo_store) {
        if (dev_alloc(&c->d_halo_store, (size_t)S * B200_TRAIL * 2) != cudaSuccess || dev_alloc(&c->d_halo_op, (size_t)NSLOT * S) != cudaSuccess ||
            pin_alloc(&c->h_halo_op, (size_t)NSLOT * S) != cudaSuccess) {
            cudaFree(c->d_halo_store); cudaFree(c->d_halo_op); cudaFreeHost(c->h_halo_op);
            c->d_halo_store = nullptr; c->d_halo_op = nullptr; c->h_halo_op = nullptr;
            return fail(c, B200_E_NOMEM, "halo store of %u receivers", S);
        }
    }
    uint8_t *dst = pipe[pi] + lead;
    if ((rc = build_device_run(c, sl, fmt, dst, pipe_stride, buf_len, rx)) != B200_OK) return rc;
    // The slot's previous step (NSLOT steps ago) has been collected, so nothing reads pipe[pi] or this slot's halo_op any more; the
    // copies and halo_store_kernel of consecutive steps are ordered on in_stream, so a receiver's stored halo is the one its last
    // step left.
    sl.cached_tiles = 0;                  // (until the step is enqueued: a failure below leaves no valid tile table behind)
    const size_t row = (size_t)max_n * buf_len * bps;
    if (row) CU(c, cudaMemcpy2DAsync(dst, pipe_stride, h_iq, host_stride, row, S, cudaMemcpyHostToDevice, c->in_stream));
    uint32_t *op = c->h_halo_op + (size_t)pi * S;
    for (uint32_t s = 0; s < S; s++)
        op[s] = rx[s].n_buffers ? (rx[s].n_buffers * buf_len) << 1 | ((rx[s].flags & B200_RX_CONTINUES) ? 1u : 0u) : 0u;
    CU(c, cudaMemcpyAsync(c->d_halo_op + (size_t)pi * S, op, (size_t)S * 4, cudaMemcpyHostToDevice, c->in_stream));
    halo_store_kernel<<<S, 128, 0, c->in_stream>>>(dst, pipe_stride, c->d_halo_store, c->d_halo_op + (size_t)pi * S, bps);
    CU(c, cudaGetLastError());
    CU(c, cudaEventRecord(c->ev_in[pi], c->in_stream));
    CU(c, cudaStreamWaitEvent(c->stream, c->ev_in[pi], 0));
    for (uint32_t s = 0; s < S; s++)
        if (rx[s].n_buffers) c->halo_bytes[s] = rx[s].n_buffers * buf_len >= B200_TRAIL ? (uint8_t)bps : 0;
    sl.cached_tiles = sl.ntile;
    return launch_async(c, sl);
}

static int run_host_async(b200_demod_ctx *c, const uint8_t *h_iq, uint64_t host_stride, uint32_t n_buffers, uint32_t buf_len,
                          int continues, int64_t first_ts, int fmt) {
    if (!c || !h_iq) return B200_E_INVAL;
    if (n_buffers == 0) return fail(c, B200_E_INVAL, "n_buffers/buf_len exceed the context's configuration (buf_len must be a multiple of 8)");
    return run_host_rx_async(c, fmt, h_iq, host_stride, buf_len, uniform_rx(c, n_buffers, continues, first_ts));
}

API int b200_demod_run_host_uc8_async(b200_demod_ctx *c, const uint8_t *h_iq, uint64_t host_stride, uint32_t n_buffers, uint32_t buf_len,
                                      int continues, int64_t first_ts) {
    return run_host_async(c, h_iq, host_stride, n_buffers, buf_len, continues, first_ts, FMT_UC8);
}

API int b200_demod_run_host_sc16_async(b200_demod_ctx *c, const int16_t *h_iq, uint64_t host_stride, uint32_t n_buffers, uint32_t buf_len,
                                       int continues, int64_t first_ts, int q11) {
    return run_host_async(c, reinterpret_cast<const uint8_t *>(h_iq), host_stride, n_buffers, buf_len, continues, first_ts, q11 ? FMT_SC16Q11 : FMT_SC16);
}

API int b200_demod_run_host_rx_async(b200_demod_ctx *c, int format, const void *h_iq, uint64_t host_stride, uint32_t buf_len, const b200_rx_step *rx) {
    return run_host_rx_async(c, format, static_cast<const uint8_t *>(h_iq), host_stride, buf_len, rx);
}

// Pipelined steps keep three kernels' worth of work in flight: the scan of step n+1 (one persistent CTA per SM, the whole SM each)
// and stage B + finalizer of step n (one CTA of 8 warps per receiver, two per SM, latency-bound: a third of the issue slots).
// Launched over the whole chip they take turns on all SMs.  With a scan grid smaller than the chip the scan runs back to back on
// its SMs and stage B lives on the rest, in several waves.  Which is faster depends on whether stage B fits into the SMs the scan
// leaves free (then the step costs what the scan costs on its SMs) or holds the scans up (then taking turns is better), and on the
// workload: on the dense stress stage B is a large share of the step and wants the whole chip (tools/gpu_partition.sh times fixed
// grids).  The kernels' event times say little while they overlap, so a pipelined session MEASURES it: after its first
// steps it runs with the whole chip, then with 85 % and 82 % of the SMs for the scan (twelve step periods each: host clock between
// completed steps, the longest dropped), measures the winner once more and keeps it - the whole chip unless a partition wins by
// 1.5 % and again by 1 %.  A run of a different size (tiles +- 1/8) starts over, up to four times per session.
static void tune_partition(b200_demod_ctx *c, Slot &sl) {
    // (sc16 steps carry a converter in front of the scan: they are not measured, as Mode A/C contexts are not)
    if (c->part_fixed || c->part_off || (c->cfg.flags & B200_CFG_MODE_AC) || sl.sc16 || !sl.ntile || c->n_sm < 16) return;
    PartCal &k = c->cal;
    const auto now = std::chrono::steady_clock::now();
    if (!k.grids[0]) { k.grids[0] = c->n_sm; k.grids[1] = (c->n_sm * 85 + 50) / 100; k.grids[2] = (c->n_sm * 82 + 50) / 100; k.grids[3] = c->n_sm; k.skip = 8; }
    if (k.locked) {
        const uint32_t d = sl.ntile > k.ntile ? sl.ntile - k.ntile : k.ntile - sl.ntile;
        if (d * 8 > k.ntile) {                                          // another workload: measure again - a few times; a session whose
            k = PartCal(); c->part_n = 0;                               // runs keep changing size stays with the whole chip
            if (++c->cal_restarts > 4) c->part_off = true;
        }
        return;
    }
    const double dt = k.have_last ? std::chrono::duration<double, std::milli>(now - k.last).count() : 0.0;
    const bool first = !k.have_last;
    k.last = now; k.have_last = true;
    if (first || sl.scan_grid != k.grids[k.phase]) { if (k.skip < 2) k.skip = 2; return; }     // a step launched before the grid was switched
    if (k.n == 0 && !k.skip) k.ntile = sl.ntile;
    if (k.skip) { k.skip--; return; }                     // (the session's first steps, the first periods with a new grid: not steady yet)
    if (sl.ntile != k.ntile) { k.n = 0; return; }          // the size changed in the middle of a measurement: start this phase over
    k.dt[k.n++] = dt;
    if (k.n < PartCal::SAMPLES) return;
    std::sort(k.dt, k.dt + PartCal::SAMPLES);
    double sum = 0;
    for (int i = 0; i < PartCal::SAMPLES - 1; i++) sum += k.dt[i];           // (the longest one may hold a pause of the caller)
    k.mean[k.phase] = sum / (PartCal::SAMPLES - 1);
    k.n = 0; k.phase++;
    if (k.phase < 3) { c->part_n = k.grids[k.phase]; return; }
    if (k.phase == 3) {                                    // candidates measured: the better partition, if it wins by 1.5 %, is measured once more
        int best = 0;
        for (int i = 1; i < 3; i++) if (k.mean[i] < 0.985 * k.mean[0] && (best == 0 || k.mean[i] < k.mean[best])) best = i;
        k.grids[3] = k.grids[best];
        c->part_n = best ? k.grids[best] : 0;
        if (best) return;
        k.mean[3] = k.mean[0];
    }
    if (k.mean[3] >= 0.99 * k.mean[0]) c->part_n = 0;      // ... and kept only if it wins again
    k.locked = true;
    if (c->part_debug) fprintf(stderr, "b200 partition: %u tiles: step period %.4f ms on %d SMs, %.4f on %d, %.4f on %d, again %.4f on %d -> scan grid %d\n", k.ntile,
                               k.mean[0], k.grids[0], k.mean[1], k.grids[1], k.mean[2], k.grids[2], k.mean[3], k.grids[3], c->part_n ? c->part_n : c->n_sm);
}

API int b200_demod_wait(b200_demod_ctx *c) {
    if (!c) return B200_E_INVAL;
    CU(c, cudaSetDevice(c->device));
    if (c->n_flight == 0) return fail(c, B200_E_STATE, "no asynchronous step in flight");
    const int idx = c->head;                 // the oldest step in flight
    Slot &sl = c->slot[idx];
    c->cur = idx;
    int rc = B200_OK;
    if (!sl.completed) {                     // (completed: already repeated synchronously, see below)
        rc = collect(c, sl, c->res_stream);
        if (rc > 0) {
            // This step (and therefore the ones behind it, which saw the failure flag of the step ahead and skipped their
            // stage B) must be repeated.  Drain the pipeline and redo all of them, in order, synchronously.
            for (int k = 1; k < c->n_flight; k++) CU(c, cudaEventSynchronize(c->slot[(idx + k) % NSLOT].ev[4]));
            CU(c, cudaStreamSynchronize(c->stream));
            CU(c, cudaStreamSynchronize(c->res_stream));
            rc = regrow(c, sl, rc);
            if (rc == B200_OK) rc = execute_blocking(c, sl);
            for (int k = 1; k < c->n_flight && rc == B200_OK; k++) {
                Slot &next = c->slot[(idx + k) % NSLOT];
                rc = execute_blocking(c, next);
                if (rc == B200_OK) next.completed = true;
            }
        }
    }
    if (rc == B200_OK && !sl.completed) tune_partition(c, sl);
    sl.in_flight = false;
    c->head = (idx + 1) % NSLOT;
    c->n_flight--;
    return rc;
}

// ---- results -----------------------------------------------------------------------------------
API int b200_demod_total_frames(b200_demod_ctx *c, uint64_t *n) { if (!c || !n) return B200_E_INVAL; *n = c->slot[c->cur].run_frames; return B200_OK; }

API int b200_demod_frame_count(b200_demod_ctx *c, uint32_t s, uint32_t *n) {
    if (!c || !n || s >= c->cfg.n_streams) return B200_E_INVAL;
    const Slot &sl = c->slot[c->cur];
    *n = sl.h_frame_span[2 * s + 1];
    return B200_OK;
}

API int b200_demod_fetch(b200_demod_ctx *c, uint32_t s, b200_frame *out, uint32_t cap, uint32_t *n) {
    if (!c || !n || s >= c->cfg.n_streams) return B200_E_INVAL;
    const Slot &sl = c->slot[c->cur];
    const uint32_t cnt = sl.h_frame_span[2 * s + 1];
    *n = cnt;
    if (cnt > cap) return fail(c, B200_E_OVERFLOW, "stream %u has %u frames, output holds %u", s, cnt, cap);
    if (cnt) memcpy(out, sl.h_packed + sl.h_frame_span[2 * s], (size_t)cnt * sizeof(b200_frame));
    return B200_OK;
}

API int b200_demod_fetch_modeac(b200_demod_ctx *c, uint32_t s, b200_modeac *out, uint32_t cap, uint32_t *n) {
    if (!c || !n || s >= c->cfg.n_streams) return B200_E_INVAL;
    if (!(c->cfg.flags & B200_CFG_MODE_AC)) return fail(c, B200_E_STATE, "context was created without B200_CFG_MODE_AC");
    const Slot &sl = c->slot[c->cur];
    const uint32_t first = sl.h_ac_prefix[sl.stream_buf_begin[s]], cnt = sl.h_ac_prefix[sl.stream_buf_begin[s + 1]] - first;
    *n = cnt;
    if (cnt > cap) return fail(c, B200_E_OVERFLOW, "stream %u has %u Mode A/C replies, output holds %u", s, cnt, cap);
    if (cnt) memcpy(out, sl.h_ac_packed + first, (size_t)cnt * sizeof(b200_modeac));
    return B200_OK;
}

API int b200_demod_fetch_beast(b200_demod_ctx *c, uint32_t s, uint32_t flags, uint8_t *out, uint32_t cap, uint32_t *nbytes) {
    if (!c || !nbytes || s >= c->cfg.n_streams || (flags & ~B200_BEAST_VERBATIM)) return B200_E_INVAL;
    // A later asynchronous step may be in flight: it works in the other slot, and this call only reads the completed one.
    const uint32_t S = c->cfg.n_streams;
    Slot &sl = c->slot[c->cur];
    if (c->beast_slot != c->cur || c->beast_flags != flags) {        // encode every stream of this run once
        CU(c, cudaSetDevice(c->device));
        const bool mode_ac = (c->cfg.flags & B200_CFG_MODE_AC) != 0;
        const uint64_t records = (uint64_t)sl.run_frames + (mode_ac ? sl.h_ac_prefix[sl.nbuf] : 0);
        const uint64_t need = records * B200_BEAST_MAX_RECORD + 64;
        if (need > 0xffffffffull) return fail(c, B200_E_OVERFLOW, "Beast output of one run exceeds 4 GiB");
        if (!c->d_beast_meta) {
            CU(c, dev_alloc(&c->d_beast_meta, 2 * S + 1));
            CU(c, pin_alloc(&c->h_beast_meta, 2 * S + 1));
        }
        if (need > c->beast_cap) {
            cudaFree(c->d_beast); cudaFreeHost(c->h_beast); c->d_beast = nullptr; c->h_beast = nullptr; c->beast_cap = 0;
            const uint32_t cap2 = (uint32_t)std::min<uint64_t>(0xffffffffull, need + need / 2);
            if (dev_alloc(&c->d_beast, cap2) != cudaSuccess || pin_alloc(&c->h_beast, cap2) != cudaSuccess)
                return fail(c, B200_E_NOMEM, "cannot allocate %u bytes for the Beast output", cap2);
            c->beast_cap = cap2;
        }
        c->beast_slot = -1;
        cudaStream_t st = c->copy_stream;
        if (!sl.desc_on_device) { CU(c, cudaMemcpyAsync(sl.d_desc, sl.h_desc, sl.desc_bytes, cudaMemcpyHostToDevice, st)); sl.desc_on_device = true; }
        CU(c, cudaMemsetAsync(c->d_beast_meta, 0, (2 * (size_t)S + 1) * 4, st));
        BeastParams bp;
        bp.segs = sl.d_segs; bp.stream_seg_begin = sl.d_stream_seg_begin; bp.frames = sl.d_packed; bp.frame_span = sl.d_frame_span;
        bp.buf_out = sl.d_buf_out; bp.ac = mode_ac ? sl.d_ac_packed : nullptr; bp.ac_prefix = mode_ac ? sl.d_ac_prefix : nullptr;
        bp.out = c->d_beast; bp.stream_off = c->d_beast_meta; bp.stream_len = c->d_beast_meta + S; bp.total = c->d_beast_meta + 2 * S;
        bp.cap = c->beast_cap; bp.verbatim = (flags & B200_BEAST_VERBATIM) ? 1u : 0u;
        { int r = b200_launch_beast(&bp, S, st); if (r) return fail(c, B200_E_CUDA, "beast launch: %s", cudaGetErrorString((cudaError_t)r)); }
        CU(c, cudaMemcpyAsync(c->h_beast_meta, c->d_beast_meta, (2 * (size_t)S + 1) * 4, cudaMemcpyDeviceToHost, st));
        CU(c, cudaStreamSynchronize(st));
        const uint32_t total = c->h_beast_meta[2 * S];
        if (total > c->beast_cap) return fail(c, B200_E_OVERFLOW, "Beast output larger than its worst case (%u > %u)", total, c->beast_cap);
        if (total) {
            CU(c, cudaMemcpyAsync(c->h_beast, c->d_beast, total, cudaMemcpyDeviceToHost, st));
            CU(c, cudaStreamSynchronize(st));
        }
        c->beast_slot = c->cur; c->beast_flags = flags;
    }
    const uint32_t off = c->h_beast_meta[s], len = c->h_beast_meta[S + s];
    *nbytes = len;
    if (len > cap) return fail(c, B200_E_OVERFLOW, "stream %u has %u bytes of Beast output, buffer holds %u", s, len, cap);
    if (len) memcpy(out, c->h_beast + off, len);
    return B200_OK;
}

API int b200_demod_buffer_results(b200_demod_ctx *c, uint32_t s, b200_buffer_result *out, uint32_t cap, uint32_t *n) {
    if (!c || !n || s >= c->cfg.n_streams) return B200_E_INVAL;
    const Slot &sl = c->slot[c->cur];
    const uint32_t b0 = sl.stream_buf_begin[s], cnt = sl.stream_buf_begin[s + 1] - b0;
    *n = cnt;
    if (cnt > cap) return fail(c, B200_E_OVERFLOW, "stream %u has %u buffer results, output holds %u", s, cnt, cap);
    if (cnt) memcpy(out, sl.h_buf_out + b0, (size_t)cnt * sizeof(b200_buffer_result));
    return B200_OK;
}

API int b200_demod_get_stats(b200_demod_ctx *c, uint32_t s, b200_demod_stats *out) {
    if (!c || !out || s >= c->cfg.n_streams) return B200_E_INVAL;
    if (any_in_flight(c)) return fail(c, B200_E_STATE, "asynchronous steps are in flight: call b200_demod_wait first");
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaMemcpyAsync(out, &c->d_state[s].stats, sizeof(b200_demod_stats), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return B200_OK;
}

API int b200_demod_last_timing(b200_demod_ctx *c, float ms[5], uint32_t *launches) {
    if (!c) return B200_E_INVAL;
    if (ms) memcpy(ms, c->slot[c->cur].ms, sizeof(c->slot[c->cur].ms));
    if (launches) *launches = c->slot[c->cur].launches;
    return B200_OK;
}

// Instrumentation for tests: out[0] = tiles of the last run, [1] = sum of PosEntry counts, [2] = sum of Rec counts,
// [3] = RunCtl.rec_alloc, [4] = RunCtl.overflow, [5] = segments, [6] = buffers, [7] = frames.
API int b200_demod_debug_counters(b200_demod_ctx *c, uint64_t out[8]) {
    if (!c || !out) return B200_E_INVAL;
    CU(c, cudaSetDevice(c->device));
    const Slot &sl = c->slot[c->cur];
    std::vector<TileOut> t(sl.ntile);
    if (sl.ntile) CU(c, cudaMemcpy(t.data(), sl.d_tile_out, sl.ntile * sizeof(TileOut), cudaMemcpyDeviceToHost));
    uint64_t np = 0, nr = 0;
    for (auto &x : t) { np += x.n_pos; nr += x.n_rec; }
    out[0] = sl.ntile; out[1] = np; out[2] = nr; out[3] = sl.h_ctl->rec_alloc; out[4] = sl.h_ctl->overflow;
    out[5] = sl.nseg; out[6] = sl.nbuf; out[7] = sl.run_frames;
    return B200_OK;
}

#ifdef B200_SOLO_CLOCKS
API int b200_demod_debug_ctl(b200_demod_ctx *c, uint32_t out[8]) { memcpy(out, c->slot[c->cur].h_ctl, 32); return B200_OK; }
#endif

// ---- ICAO filter control -------------------------------------------------------------------------
static int icao_op(b200_demod_ctx *c, uint32_t s, int op, uint32_t addr, int *result) {
    if (!c || s >= c->cfg.n_streams) return B200_E_INVAL;
    if (any_in_flight(c)) return fail(c, B200_E_STATE, "asynchronous steps are in flight: call b200_demod_wait first");
    CU(c, cudaSetDevice(c->device));
    int r = b200_launch_icao_op(c->d_state, s, op, addr & 0xffffffu, c->d_result, c->stream);
    if (r) return fail(c, B200_E_CUDA, "icao op launch: %s", cudaGetErrorString((cudaError_t)r));
    int host = 0;
    CU(c, cudaMemcpyAsync(&host, c->d_result, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    if (op == 0 && host < 0) {               // the generation would pass half of its slots: larger tables, then once more
        int rc = grow_icao_tables(c);
        if (rc != B200_OK) return rc;
        r = b200_launch_icao_op(c->d_state, s, op, addr & 0xffffffu, c->d_result, c->stream);
        if (r) return fail(c, B200_E_CUDA, "icao op launch: %s", cudaGetErrorString((cudaError_t)r));
        CU(c, cudaMemcpyAsync(&host, c->d_result, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
        if (host < 0) return fail(c, B200_E_OVERFLOW, "ICAO filter could not be grown");
    }
    if (result) *result = host;
    return B200_OK;
}
API int b200_demod_icao_add(b200_demod_ctx *c, uint32_t s, uint32_t addr) { return icao_op(c, s, 0, addr, nullptr); }
API int b200_demod_icao_test(b200_demod_ctx *c, uint32_t s, uint32_t addr, int *present) { return icao_op(c, s, 1, addr, present); }
API int b200_demod_icao_expire(b200_demod_ctx *c, uint32_t s) { return icao_op(c, s, 2, 0, nullptr); }
API int b200_demod_icao_reset(b200_demod_ctx *c, uint32_t s) { return icao_op(c, s, 3, 0, nullptr); }
