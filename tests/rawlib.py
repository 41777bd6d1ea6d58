"""The CPU model of readsb's raw / AVR output: the records modesSendRawOutput (net_io.c:1837-1863) writes to a raw_out client
and the --raw stdout line of displayModesMessage (mode_s.c:1835-1841), built from frames and Mode A/C replies of the oracle
(tests/oraclelib.py) or of the library.  TEST INFRASTRUCTURE — never imported by readsb_b200."""
from __future__ import annotations

import numpy as np


def raw_record(msg: bytes, timestamp: int, mlat: bool = False, stdout: bool = False) -> bytes:
    """One record as the reference writes it; `timestamp` is the int64 mm->timestamp."""
    if mlat and timestamp:
        digits = "%012X" % (timestamp & 0xFFFFFFFFFFFFFFFF)        # PRIX64 of the unsigned value
        # network: sprintf, then p += 13 - the frame hex overwrites whatever digits went past the first twelve
        prefix = "@" + (digits if stdout else digits[:12])
    else:
        prefix = "*"
    body = msg.hex() if stdout else msg.hex().upper()
    return (prefix + body + ";\n").encode()


def raw_records(frames: np.ndarray, modeac: np.ndarray = None, mlat: bool = False, verbatim: bool = False, stdout: bool = False) -> bytes:
    """Records of frames and Mode A/C replies in the reference's output order (as Oracle.beast): per buffer the Mode S frames,
    then the replies; frames["buffer_seq"] and modeac["buffer_idx"] must count buffers from the same origin.  The network form,
    or with stdout the --raw stdout form (always the corrected frame); verbatim: the bytes as received."""
    assert not (stdout and verbatim), "the stdout line always prints mm->msg"
    recs = []                                    # (buffer, 0 = Mode S / 1 = Mode A/C, index, record)
    for i, f in enumerate(frames):
        msg = bytearray(bytes(f["msg"])[: int(f["msgbits"]) // 8])
        fix = int(f["fix_bit"])
        if verbatim and fix >= 0:
            msg[fix >> 3] ^= 1 << (7 - (fix & 7))                   # mm->verbatim: the bit the CRC repair flipped
        recs.append((int(f["buffer_seq"]), 0, i, raw_record(bytes(msg), int(f["timestamp"]), mlat, stdout)))
    for i, a in enumerate(modeac if modeac is not None else ()):
        code = int(a["modeac"])
        recs.append((int(a["buffer_idx"]), 1, i, raw_record(bytes([(code >> 8) & 0xFF, code & 0xFF]), int(a["timestamp"]), mlat, stdout)))
    recs.sort(key=lambda r: r[:3])
    return b"".join(r[3] for r in recs)
