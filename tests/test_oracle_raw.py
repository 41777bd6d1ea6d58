"""The CPU model of raw / AVR output (tests/rawlib.py) against the reference program's own network output and against the C library's
printf, which is what the reference formats the timestamp with."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest

from oraclelib import Oracle
from rawlib import raw_record, raw_records
from readsb_b200.abi import FRAME_DTYPE, MODEAC_DTYPE

GOLDEN = Path(__file__).parent / "golden"


@pytest.mark.parametrize("mlat", [False, True])
def test_oracle_raw_matches_reference_network_output(mlat):
    """tests/golden/raw/raw_stream.npz (tests/golden/make_raw_golden.py: --net-verbatim --modeac, a raw_out client) == the
    oracle's frames and replies of the same capture through rawlib.raw_records."""
    z = np.load(GOLDEN / "beast_stream.npz")
    meta = json.loads(bytes(z["meta"]).decode())
    iq = np.concatenate([np.full(2 * meta["silence_samples"], 127, np.uint8), z["traffic"]])
    frames, _ = Oracle().run_stream(iq, 131072)
    modeac = Oracle().run_stream_ac(iq, 131072)
    want = bytes(np.load(GOLDEN / "raw" / "raw_stream.npz")["raw_mlat" if mlat else "raw"])
    assert raw_records(frames, modeac, mlat=mlat, verbatim=True) == want
    assert want.count(b"\n") == meta["n_records"] == len(frames) + len(modeac)
    assert raw_records(frames, modeac, mlat=mlat) != want       # repaired frames: the corrected bytes differ


def _reference_network_record(msg: bytes, ts: int) -> bytes:
    """modesSendRawOutput's steps with --mlat, done with the C library: sprintf "@%012lX" into the record, p += 13, the frame hex
    (which overwrites whatever the sprintf wrote past 13 bytes), ';', '\\n'."""
    libc = C.CDLL(None)
    buf = C.create_string_buffer(64)
    libc.snprintf(buf, C.c_size_t(64), b"@%012lX", C.c_int64(ts))
    raw = bytearray(buf.raw)
    p = 13
    tail = msg.hex().upper().encode() + b";\n"
    raw[p: p + len(tail)] = tail
    return bytes(raw[: p + len(tail)])


@pytest.mark.parametrize("ts", [1, 0xFFFFFFFFFFFF, 1 << 48, (1 << 48) + 0xABC, 0x7FFFFFFFFFFFFFFF, -1, -12345])
def test_raw_timestamp_digits(ts):
    """Network: the first 12 hex digits of any timestamp; stdout: every digit (PRIX64 of the unsigned value); 0: '*'."""
    libc = C.CDLL(None)
    buf = C.create_string_buffer(64)
    for msg in (bytes.fromhex("8D4840D6202CC371C32CE0576098"), bytes.fromhex("1234")):
        assert raw_record(msg, ts, mlat=True) == _reference_network_record(msg, ts)
        libc.snprintf(buf, C.c_size_t(64), b"@%012lX", C.c_int64(ts))
        assert raw_record(msg, ts, mlat=True, stdout=True) == buf.value + msg.hex().encode() + b";\n"
        assert raw_record(msg, 0, mlat=True) == b"*" + msg.hex().upper().encode() + b";\n"
        assert raw_record(msg, ts) == b"*" + msg.hex().upper().encode() + b";\n"
        assert raw_record(msg, 0, mlat=True, stdout=True) == b"*" + msg.hex().encode() + b";\n"


def test_raw_order_and_verbatim():
    """Per buffer the Mode S frames, then the Mode A/C replies; verbatim flips the repaired bit back."""
    f = np.zeros(2, FRAME_DTYPE)
    f["timestamp"] = [10, 30]; f["buffer_seq"] = [0, 1]; f["msgbits"] = [56, 56]; f["fix_bit"] = [-1, 9]
    f["msg"][:, :7] = [0x5D, 0x48, 0x40, 0xD6, 0x11, 0x22, 0x33]
    a = np.zeros(1, MODEAC_DTYPE)
    a["timestamp"] = 20; a["modeac"] = 0x0A7F; a["buffer_idx"] = 0
    assert raw_records(f, a) == b"*5D4840D6112233;\n*0A7F;\n*5D4840D6112233;\n"
    assert raw_records(f, a, verbatim=True) == b"*5D4840D6112233;\n*0A7F;\n*5D0840D6112233;\n"
    assert raw_records(f, a, mlat=True, stdout=True) == b"@00000000000A5d4840d6112233;\n@0000000000140a7f;\n@00000000001E5d4840d6112233;\n"
