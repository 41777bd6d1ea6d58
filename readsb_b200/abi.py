"""ctypes mirror of include/b200_demod.h (plain structs shared by product, oracle and tests)."""
from __future__ import annotations

import ctypes as C

import numpy as np

TRAILING_SAMPLES = 326


class Frame(C.Structure):
    _fields_ = [("timestamp", C.c_int64), ("sigpow_sum", C.c_uint64), ("j", C.c_uint32), ("crc", C.c_uint32),
                ("addr", C.c_uint32), ("score", C.c_int32), ("buffer_seq", C.c_uint32),
                ("signal_len", C.c_uint16), ("phase", C.c_uint8), ("msgtype", C.c_uint8), ("msgbits", C.c_uint8),
                ("correctedbits", C.c_uint8), ("fix_bit", C.c_int8), ("flags", C.c_uint8),
                ("msg", C.c_uint8 * 14), ("pad_", C.c_uint8 * 6)]


class BufferResult(C.Structure):
    _fields_ = [("sample_timestamp", C.c_int64), ("sum_level", C.c_uint64), ("sum_power", C.c_uint64),
                ("sum_signal_power", C.c_uint64), ("length", C.c_uint32), ("n_frames", C.c_uint32),
                ("buffer_seq", C.c_uint32), ("icao_flipped", C.c_uint32),
                ("demod_preambles", C.c_uint32), ("demod_rejected_bad", C.c_uint32), ("demod_rejected_unknown_icao", C.c_uint32),
                ("demod_accepted", C.c_uint32 * 2), ("demod_preamblePhase", C.c_uint32 * 5), ("demod_bestPhase", C.c_uint32 * 5),
                ("pad_", C.c_uint32)]


class Stats(C.Structure):
    _fields_ = [("samples_processed", C.c_uint64), ("demod_preambles", C.c_uint64),
                ("demod_rejected_bad", C.c_uint64), ("demod_rejected_unknown_icao", C.c_uint64),
                ("demod_accepted", C.c_uint64 * 2), ("demod_preamblePhase", C.c_uint64 * 5),
                ("demod_bestPhase", C.c_uint64 * 5), ("signal_power_count", C.c_uint64),
                ("sum_signal_power", C.c_uint64), ("strong_signal_count", C.c_uint64),
                ("peak_signal_power", C.c_double), ("demod_modeac", C.c_uint64), ("buffers", C.c_uint64),
                ("icao_flips", C.c_uint64)]

    def as_dict(self):
        d = {}
        for name, typ in self._fields_:
            v = getattr(self, name)
            d[name] = list(v) if hasattr(v, "__len__") else (float(v) if isinstance(v, float) else int(v))
        return d


class Config(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("device", C.c_int32), ("n_streams", C.c_uint32),
                ("buf_samples", C.c_uint32), ("max_buffers_per_run", C.c_uint32),
                ("preamble_threshold", C.c_int32), ("nfix_crc", C.c_int32), ("fix_df", C.c_int32),
                ("icao_ttl_ms", C.c_int32), ("flags", C.c_uint32)]


MODEAC_DTYPE = np.dtype([("timestamp", "<i8"), ("f1_sample", "<u4"), ("modeac", "<u2"), ("buffer_idx", "<u2")])
CFG_MODE_AC = 0x1
CFG_NO_TIMING = 0x2

assert C.sizeof(Frame) == 64 and C.sizeof(BufferResult) == 112 and MODEAC_DTYPE.itemsize == 16

FRAME_DTYPE = np.dtype([("timestamp", "<i8"), ("sigpow_sum", "<u8"), ("j", "<u4"), ("crc", "<u4"), ("addr", "<u4"),
                        ("score", "<i4"), ("buffer_seq", "<u4"), ("signal_len", "<u2"), ("phase", "u1"),
                        ("msgtype", "u1"), ("msgbits", "u1"), ("correctedbits", "u1"), ("fix_bit", "i1"),
                        ("flags", "u1"), ("msg", "u1", (14,)), ("pad_", "u1", (6,))])
BUFRES_DTYPE = np.dtype([("sample_timestamp", "<i8"), ("sum_level", "<u8"), ("sum_power", "<u8"),
                         ("sum_signal_power", "<u8"), ("length", "<u4"), ("n_frames", "<u4"),
                         ("buffer_seq", "<u4"), ("icao_flipped", "<u4"),
                         ("demod_preambles", "<u4"), ("demod_rejected_bad", "<u4"), ("demod_rejected_unknown_icao", "<u4"),
                         ("demod_accepted", "<u4", (2,)), ("demod_preamblePhase", "<u4", (5,)), ("demod_bestPhase", "<u4", (5,)),
                         ("pad_", "<u4")])
assert FRAME_DTYPE.itemsize == 64 and BUFRES_DTYPE.itemsize == 112

# b200_rx_step: one receiver's part of a step of the _rx calls (include/b200_demod.h)
RX_STEP_DTYPE = np.dtype([("first_sample_timestamp", "<i8"), ("n_buffers", "<u4"), ("flags", "<u4"), ("preamble_threshold", "<i4"),
                          ("reserved_", "<u4")])
assert RX_STEP_DTYPE.itemsize == 24
RX_CONTINUES = 0x1
FORMAT_UC8, FORMAT_SC16, FORMAT_SC16Q11 = 0, 1, 2

# fields of a frame that the reference itself defines (flags is this library's own annotation)
FRAME_PARITY_FIELDS = ("timestamp", "sigpow_sum", "j", "crc", "addr", "score", "buffer_seq", "signal_len",
                       "phase", "msgtype", "msgbits", "correctedbits", "fix_bit", "msg")


def frames_equal(a: np.ndarray, b: np.ndarray, fields=FRAME_PARITY_FIELDS) -> bool:
    if a.shape != b.shape:
        return False
    return all(np.array_equal(a[f], b[f]) for f in fields)


def frame_hex(fr) -> str:
    return bytes(fr["msg"][: int(fr["msgbits"]) // 8]).hex()
