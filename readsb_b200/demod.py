"""Host-side mirror of the reference interface for the demodulator path, over the C ABI.

`Demodulator` is a thin ctypes front end of include/b200_demod.h: `submit_iq` stands where a
readsb frontend calls its converter and publishes a mag_buf (sdr_ifile.c:241-259), `submit_mag`
+ `run` + `frames` stand where the decode thread calls demodulate2400(buf) (readsb.c:871) and the
frames reach netUseMessage().  There is no CPU implementation behind this class: if the CUDA
library is missing or no H100-class (sm_90) device is present, construction raises.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from .abi import BUFRES_DTYPE, CFG_MODE_AC, CFG_NO_TIMING, FRAME_DTYPE, MODEAC_DTYPE, RX_STEP_DTYPE, Config, Stats

_LIB = None
LIB_PATH = Path(__file__).resolve().parent / "libb200demod.so"


RAW_MLAT, RAW_VERBATIM, RAW_STDOUT = 0x1, 0x2, 0x4     # b200_demod_fetch_raw flags (include/b200_demod.h)


class DemodError(RuntimeError):
    pass


def lib():
    """Loads the in-tree CUDA library.  Never builds silently on a GPU box: the .so travels with the tree."""
    global _LIB
    if _LIB is None:
        import os
        path = Path(os.environ.get("B200_DEMOD_LIB") or LIB_PATH)     # another build of the same C ABI (the test suite's emulated kernels)
        if not path.exists():
            raise DemodError(f"{path} is missing: run `python -m readsb_b200.build` (nvcc, sm_90a). "
                             "There is no CPU fallback for the demodulator.")
        L = C.CDLL(str(path))
        vp, u32, i64, u64 = C.c_void_p, C.c_uint32, C.c_int64, C.c_uint64
        L.b200_demod_abi_version.restype = C.c_int
        L.b200_demod_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
        L.b200_demod_destroy.argtypes = [vp]
        L.b200_demod_last_error.restype = C.c_char_p
        L.b200_demod_last_error.argtypes = [vp]
        L.b200_demod_host_alloc.restype = vp
        L.b200_demod_host_alloc.argtypes = [C.c_size_t]
        L.b200_demod_host_free.argtypes = [vp]
        L.b200_demod_host_register.argtypes = [vp, C.c_size_t]
        L.b200_demod_host_unregister.argtypes = [vp]
        L.b200_demod_submit_iq_uc8.argtypes = [vp, u32, vp, u32, i64]
        L.b200_demod_submit_mag_u16.argtypes = [vp, u32, vp, u32, i64]
        L.b200_demod_submit_mag_u16_levels.argtypes = [vp, u32, vp, u32, i64, C.c_double, C.c_double]
        L.b200_demod_set_preamble_threshold.argtypes = [vp, C.c_int32]
        L.b200_demod_submit_iq_uc8_strided.argtypes = [vp, u32, u32, vp, u64, u32, u32, i64]
        L.b200_demod_set_stream.argtypes = [vp, vp]
        L.b200_demod_run.argtypes = [vp]
        L.b200_demod_run_device_uc8.argtypes = [vp, vp, u64, u32, u32, C.c_int, i64]
        L.b200_demod_run_device_uc8_async.argtypes = [vp, vp, u64, u32, u32, C.c_int, i64]
        L.b200_demod_run_host_uc8_async.argtypes = [vp, vp, u64, u32, u32, C.c_int, i64]
        L.b200_demod_run_device_sc16.argtypes = [vp, vp, u64, u32, u32, C.c_int, i64, C.c_int]
        L.b200_demod_run_device_sc16_async.argtypes = [vp, vp, u64, u32, u32, C.c_int, i64, C.c_int]
        L.b200_demod_run_host_sc16_async.argtypes = [vp, vp, u64, u32, u32, C.c_int, i64, C.c_int]
        L.b200_demod_run_device_rx.argtypes = [vp, C.c_int, vp, u64, u32, vp]
        L.b200_demod_run_device_rx_async.argtypes = [vp, C.c_int, vp, u64, u32, vp]
        L.b200_demod_run_host_rx_async.argtypes = [vp, C.c_int, vp, u64, u32, vp]
        L.b200_demod_restart_stream.argtypes = [vp, u32]
        L.b200_demod_wait.argtypes = [vp]
        L.b200_demod_frame_count.argtypes = [vp, u32, C.POINTER(u32)]
        L.b200_demod_fetch.argtypes = [vp, u32, vp, u32, C.POINTER(u32)]
        L.b200_demod_fetch_modeac.argtypes = [vp, u32, vp, u32, C.POINTER(u32)]
        L.b200_demod_submit_iq_sc16.argtypes = [vp, u32, vp, u32, C.c_int64, C.c_int]
        L.b200_demod_fetch_beast.argtypes = [vp, u32, u32, vp, u32, C.POINTER(u32)]
        L.b200_demod_fetch_raw.argtypes = [vp, u32, u32, vp, u32, C.POINTER(u32)]
        L.b200_demod_buffer_results.argtypes = [vp, u32, vp, u32, C.POINTER(u32)]
        L.b200_demod_total_frames.argtypes = [vp, C.POINTER(u64)]
        L.b200_demod_get_stats.argtypes = [vp, u32, C.POINTER(Stats)]
        L.b200_demod_icao_add.argtypes = [vp, u32, u32]
        L.b200_demod_icao_test.argtypes = [vp, u32, u32, C.POINTER(C.c_int)]
        L.b200_demod_icao_expire.argtypes = [vp, u32]
        L.b200_demod_icao_reset.argtypes = [vp, u32]
        L.b200_demod_last_timing.argtypes = [vp, C.POINTER(C.c_float * 5), C.POINTER(u32)]
        L.b200_demod_uc8_lut.argtypes = [vp]
        L.b200_demod_debug_counters.argtypes = [vp, C.POINTER(u64 * 8)]
        _LIB = L
    return _LIB


EXPORTED_SYMBOLS = [
    "b200_demod_abi_version", "b200_demod_create", "b200_demod_destroy", "b200_demod_last_error",
    "b200_demod_host_alloc", "b200_demod_host_free", "b200_demod_host_register", "b200_demod_host_unregister", "b200_demod_submit_iq_uc8", "b200_demod_submit_mag_u16",
    "b200_demod_run", "b200_demod_run_device_uc8", "b200_demod_frame_count", "b200_demod_fetch",
    "b200_demod_buffer_results", "b200_demod_total_frames", "b200_demod_get_stats", "b200_demod_icao_add",
    "b200_demod_fetch_beast", "b200_demod_submit_iq_sc16", "b200_demod_icao_test", "b200_demod_icao_expire", "b200_demod_icao_reset", "b200_demod_last_timing",
    "b200_demod_uc8_lut", "b200_demod_debug_counters", "b200_demod_submit_iq_uc8_strided", "b200_demod_set_stream",
    "b200_demod_run_device_uc8_async", "b200_demod_wait", "b200_demod_fetch_modeac", "b200_demod_run_host_uc8_async",
    "b200_demod_submit_mag_u16_levels", "b200_demod_set_preamble_threshold",
    "b200_demod_run_device_sc16", "b200_demod_run_device_sc16_async", "b200_demod_run_host_sc16_async",
    "b200_demod_run_device_rx", "b200_demod_run_device_rx_async", "b200_demod_run_host_rx_async", "b200_demod_restart_stream",
    "b200_demod_fetch_raw",
]


class PinnedBuffer:
    """Page-locked host memory from the library (cudaHostAlloc), exposed as a numpy uint8 array."""

    def __init__(self, nbytes: int):
        self._L = lib()
        self.ptr = self._L.b200_demod_host_alloc(nbytes)
        if not self.ptr:
            raise MemoryError(f"cannot pin {nbytes} bytes")
        self.array = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self.ptr))

    def free(self):
        if self.ptr:
            self.array = None
            self._L.b200_demod_host_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Demodulator:
    def __init__(self, n_streams: int = 1, buf_samples: int = 131072, max_buffers_per_run: int = 1,
                 preamble_threshold: int = 58, nfix_crc: int = 1, fix_df: int = 1, icao_ttl_ms: int = 60000,
                 device: int = -1, mode_ac: bool = False, no_timing: bool = False):
        self.L = lib()
        self.cfg = Config(C.sizeof(Config), device, n_streams, buf_samples, max_buffers_per_run,
                          preamble_threshold, nfix_crc, fix_df, icao_ttl_ms, (CFG_MODE_AC if mode_ac else 0) | (CFG_NO_TIMING if no_timing else 0))
        self.n_streams, self.buf_samples, self.max_buffers_per_run = n_streams, buf_samples, max_buffers_per_run
        h = C.c_void_p()
        rc = self.L.b200_demod_create(C.byref(self.cfg), C.byref(h))
        if rc != 0:
            raise DemodError(f"b200_demod_create failed ({rc}): {self.L.b200_demod_last_error(None).decode()}")
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.b200_demod_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            raise DemodError(f"error {rc}: {self.L.b200_demod_last_error(self.h).decode()}")

    # -- host-buffer path ----------------------------------------------------------------------
    def submit_iq(self, stream: int, iq: np.ndarray, sample_timestamp: int):
        """iq: uint8 array of interleaved I,Q; one reference buffer (<= buf_samples samples)."""
        assert iq.dtype == np.uint8 and iq.flags.c_contiguous and iq.size % 2 == 0
        self._check(self.L.b200_demod_submit_iq_uc8(self.h, stream, iq.ctypes.data, iq.size // 2, sample_timestamp))

    def submit_iq_ptr(self, stream: int, ptr: int, nsamples: int, sample_timestamp: int):
        self._check(self.L.b200_demod_submit_iq_uc8(self.h, stream, ptr, nsamples, sample_timestamp))

    def submit_mag(self, stream: int, data: np.ndarray, length: int, sample_timestamp: int, mean_level: float | None = None,
                   mean_power: float | None = None):
        """data: uint16 mag_buf.data = 326 halo magnitudes followed by `length` new ones; mean_level / mean_power: the
        mag_buf's own (Mode A/C noise floor for frontends whose converter is not the uc8 one)."""
        assert data.dtype == np.uint16 and data.flags.c_contiguous and data.size >= length + 326
        if mean_level is None:
            self._check(self.L.b200_demod_submit_mag_u16(self.h, stream, data.ctypes.data, length, sample_timestamp))
        else:
            self._check(self.L.b200_demod_submit_mag_u16_levels(self.h, stream, data.ctypes.data, length, sample_timestamp, mean_level, mean_power))

    def set_preamble_threshold(self, thr: int):
        """Modes.preambleThreshold for the runs that follow (demod_2400.c:334-338)."""
        self._check(self.L.b200_demod_set_preamble_threshold(self.h, thr))

    def submit_iq_sc16(self, stream: int, iq16: np.ndarray, sample_timestamp: int, q11: bool = False):
        """int16 I,Q pairs (convert_sc16_nodc, or convert_sc16q11_nodc with q11)."""
        iq16 = np.ascontiguousarray(iq16, dtype=np.int16)
        self._check(self.L.b200_demod_submit_iq_sc16(self.h, stream, iq16.ctypes.data, iq16.size // 2, sample_timestamp, 1 if q11 else 0))

    def submit_iq_strided(self, first_stream: int, n_streams: int, ptr: int, host_stride_bytes: int, n_buffers: int,
                          buf_len: int, first_sample_timestamp: int):
        self._check(self.L.b200_demod_submit_iq_uc8_strided(self.h, first_stream, n_streams, ptr, host_stride_bytes,
                                                            n_buffers, buf_len, first_sample_timestamp))

    def set_stream(self, cuda_stream: int | None):
        self._check(self.L.b200_demod_set_stream(self.h, cuda_stream))

    def run(self):
        self._check(self.L.b200_demod_run(self.h))

    # -- device-resident path --------------------------------------------------------------------
    def run_device(self, d_ptr: int, stream_stride_bytes: int, n_buffers: int, buf_len: int, continues: bool,
                   first_sample_timestamp: int):
        self._check(self.L.b200_demod_run_device_uc8(self.h, d_ptr, stream_stride_bytes, n_buffers, buf_len,
                                                     1 if continues else 0, first_sample_timestamp))

    def run_device_async(self, d_ptr: int, stream_stride_bytes: int, n_buffers: int, buf_len: int, continues: bool,
                         first_sample_timestamp: int):
        self._check(self.L.b200_demod_run_device_uc8_async(self.h, d_ptr, stream_stride_bytes, n_buffers, buf_len,
                                                           1 if continues else 0, first_sample_timestamp))

    def run_host_async(self, h_ptr: int, host_stride_bytes: int, n_buffers: int, buf_len: int, continues: bool,
                       first_sample_timestamp: int):
        """Pipelined host-buffer step (reader thread / decode thread overlap of the reference, readsb.c:871 +
        sdr_ifile.c:194-259): the host slab is copied on a stream of its own while the previous step's kernels run."""
        self._check(self.L.b200_demod_run_host_uc8_async(self.h, h_ptr, host_stride_bytes, n_buffers, buf_len,
                                                         1 if continues else 0, first_sample_timestamp))

    def run_device_sc16(self, d_ptr: int, stream_stride_bytes: int, n_buffers: int, buf_len: int, continues: bool,
                        first_sample_timestamp: int, q11: bool = False):
        """run_device for int16 I,Q input (convert_sc16_nodc, or convert_sc16q11_nodc with q11): 4 bytes per sample."""
        self._check(self.L.b200_demod_run_device_sc16(self.h, d_ptr, stream_stride_bytes, n_buffers, buf_len,
                                                      1 if continues else 0, first_sample_timestamp, 1 if q11 else 0))

    def run_device_sc16_async(self, d_ptr: int, stream_stride_bytes: int, n_buffers: int, buf_len: int, continues: bool,
                              first_sample_timestamp: int, q11: bool = False):
        self._check(self.L.b200_demod_run_device_sc16_async(self.h, d_ptr, stream_stride_bytes, n_buffers, buf_len,
                                                            1 if continues else 0, first_sample_timestamp, 1 if q11 else 0))

    def run_host_sc16_async(self, h_ptr: int, host_stride_bytes: int, n_buffers: int, buf_len: int, continues: bool,
                            first_sample_timestamp: int, q11: bool = False):
        self._check(self.L.b200_demod_run_host_sc16_async(self.h, h_ptr, host_stride_bytes, n_buffers, buf_len,
                                                          1 if continues else 0, first_sample_timestamp, 1 if q11 else 0))

    # -- independent receivers: one b200_rx_step per receiver (abi.RX_STEP_DTYPE), format abi.FORMAT_* ---------------------
    def _rx(self, rx: np.ndarray):
        rx = np.ascontiguousarray(rx, dtype=RX_STEP_DTYPE)
        assert rx.shape == (self.n_streams,), "one descriptor per receiver of the context"
        return rx

    def run_device_rx(self, fmt: int, d_ptr: int, stream_stride_bytes: int, buf_len: int, rx: np.ndarray):
        rx = self._rx(rx)
        self._check(self.L.b200_demod_run_device_rx(self.h, fmt, d_ptr, stream_stride_bytes, buf_len, rx.ctypes.data))

    def run_device_rx_async(self, fmt: int, d_ptr: int, stream_stride_bytes: int, buf_len: int, rx: np.ndarray):
        rx = self._rx(rx)
        self._check(self.L.b200_demod_run_device_rx_async(self.h, fmt, d_ptr, stream_stride_bytes, buf_len, rx.ctypes.data))

    def run_host_rx_async(self, fmt: int, h_ptr: int, host_stride_bytes: int, buf_len: int, rx: np.ndarray):
        rx = self._rx(rx)
        self._check(self.L.b200_demod_run_host_rx_async(self.h, fmt, h_ptr, host_stride_bytes, buf_len, rx.ctypes.data))

    def restart_stream(self, stream: int):
        """The receiver's next submit_iq* buffer starts with a zero halo (a block was dropped in front of it)."""
        self._check(self.L.b200_demod_restart_stream(self.h, stream))

    def wait(self):
        self._check(self.L.b200_demod_wait(self.h))

    # -- results -----------------------------------------------------------------------------------
    def frames(self, stream: int) -> np.ndarray:
        n = C.c_uint32()
        self._check(self.L.b200_demod_frame_count(self.h, stream, C.byref(n)))
        out = np.zeros(n.value, dtype=FRAME_DTYPE)
        self._check(self.L.b200_demod_fetch(self.h, stream, out.ctypes.data, n.value, C.byref(n)))
        return out

    def modeac(self, stream: int) -> np.ndarray:
        """Mode A/C replies of the last run (needs mode_ac=True), in order."""
        out = np.zeros(self.max_buffers_per_run * (self.buf_samples // 70 + 2), dtype=MODEAC_DTYPE)
        n = C.c_uint32()
        self._check(self.L.b200_demod_fetch_modeac(self.h, stream, out.ctypes.data, out.size, C.byref(n)))
        return out[: n.value].copy()

    def total_frames(self) -> int:
        n = C.c_uint64()
        self._check(self.L.b200_demod_total_frames(self.h, C.byref(n)))
        return n.value

    def buffer_results(self, stream: int) -> np.ndarray:
        out = np.zeros(self.max_buffers_per_run, dtype=BUFRES_DTYPE)
        n = C.c_uint32()
        self._check(self.L.b200_demod_buffer_results(self.h, stream, out.ctypes.data, out.size, C.byref(n)))
        return out[: n.value].copy()

    def beast(self, stream: int, verbatim: bool = False) -> bytes:
        """Beast binary records of the last run's frames (+ Mode A/C replies) of one stream (net_io.c:1655-1714)."""
        n = C.c_uint32()
        flags = 1 if verbatim else 0
        rc = self.L.b200_demod_fetch_beast(self.h, stream, flags, None, 0, C.byref(n))
        if n.value == 0:
            self._check(rc)
            return b""
        buf = (C.c_uint8 * n.value)()
        self._check(self.L.b200_demod_fetch_beast(self.h, stream, flags, buf, n.value, C.byref(n)))
        return bytes(buf)

    def raw(self, stream: int, mlat: bool = False, verbatim: bool = False, stdout: bool = False) -> bytes:
        """Raw / AVR text records of the last run's frames (+ Mode A/C replies) of one stream: the network record of
        modesSendRawOutput (net_io.c:1837-1863), or with stdout=True the --raw line of displayModesMessage (mode_s.c:1835-1841).
        mlat: '@' + 12 MHz timestamp instead of '*' (--mlat); verbatim: bytes as received (--net-verbatim, network form only)."""
        n = C.c_uint32()
        flags = (RAW_MLAT if mlat else 0) | (RAW_VERBATIM if verbatim else 0) | (RAW_STDOUT if stdout else 0)
        rc = self.L.b200_demod_fetch_raw(self.h, stream, flags, None, 0, C.byref(n))
        if n.value == 0:
            self._check(rc)
            return b""
        buf = (C.c_uint8 * n.value)()
        self._check(self.L.b200_demod_fetch_raw(self.h, stream, flags, buf, n.value, C.byref(n)))
        return bytes(buf)

    def stats(self, stream: int) -> dict:
        s = Stats()
        self._check(self.L.b200_demod_get_stats(self.h, stream, C.byref(s)))
        return s.as_dict()

    def timing(self):
        ms = (C.c_float * 5)()
        n = C.c_uint32()
        self._check(self.L.b200_demod_last_timing(self.h, C.byref(ms), C.byref(n)))
        return {"run_ms": ms[0], "scan_ms": ms[1], "resolve_ms": ms[2], "modeac_ms": ms[3], "d2h_ms": ms[4], "launches": n.value}

    def debug_counters(self) -> dict:
        out = (C.c_uint64 * 8)()
        self._check(self.L.b200_demod_debug_counters(self.h, C.byref(out)))
        return dict(zip(("tiles", "positions", "records", "rec_alloc", "overflow", "segments", "buffers", "frames"), list(out)))

    # -- ICAO filter -------------------------------------------------------------------------------
    def icao_add(self, stream: int, addr: int):
        self._check(self.L.b200_demod_icao_add(self.h, stream, addr))

    def icao_test(self, stream: int, addr: int) -> bool:
        r = C.c_int()
        self._check(self.L.b200_demod_icao_test(self.h, stream, addr, C.byref(r)))
        return bool(r.value)

    def icao_expire(self, stream: int):
        self._check(self.L.b200_demod_icao_expire(self.h, stream))

    def icao_reset(self, stream: int):
        self._check(self.L.b200_demod_icao_reset(self.h, stream))

    # -- convenience: replay a whole capture like `--device-type ifile` --------------------------------
    def replay(self, iq: np.ndarray, first_ts: int = 0, stream: int = 0, want_modeac: bool = False):
        """Feeds a uc8 capture as consecutive buffers of buf_samples (last one partial), max_buffers_per_run
        at a time; returns (frames, buffer_results[, modeac]) concatenated in order."""
        nsamples = iq.size // 2
        frames, bufres, acs = [], [], []
        nbuf_done = 0
        off = 0
        while off < nsamples:
            for _ in range(self.max_buffers_per_run):
                if off >= nsamples:
                    break
                n = min(self.buf_samples, nsamples - off)
                self.submit_iq(stream, iq[2 * off: 2 * (off + n)], first_ts + off * 5)
                off += n
            self.run()
            frames.append(self.frames(stream))
            bufres.append(self.buffer_results(stream))
            if want_modeac:
                a = self.modeac(stream)
                a["buffer_idx"] += nbuf_done          # make the per-run buffer index a running one
                acs.append(a)
            nbuf_done += len(bufres[-1])
        f = np.concatenate(frames) if frames else np.zeros(0, FRAME_DTYPE)
        b = np.concatenate(bufres) if bufres else np.zeros(0, BUFRES_DTYPE)
        if want_modeac:
            return f, b, (np.concatenate(acs) if acs else np.zeros(0, MODEAC_DTYPE))
        return f, b


def uc8_lut() -> np.ndarray:
    out = np.empty(65536, dtype=np.uint16)
    rc = lib().b200_demod_uc8_lut(out.ctypes.data)
    if rc != 0:
        raise DemodError("b200_demod_uc8_lut failed")
    return out
