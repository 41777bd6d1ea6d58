"""Golden raw / AVR streams from the REFERENCE PROGRAM's own network output.

Runs oracle/_ref/readsb_cpu (the stock reference program, built by `make -C oracle readsb-pair`) on the capture already stored
in tests/golden/beast_stream.npz, behind the same silence, with
`--net --net-verbatim --net-connector 127.0.0.1,<port>,raw_out --modeac --throttle`, once with `--mlat` and once without, and
records every byte the program sends to that TCP client: that is modesSendRawOutput (net_io.c:1837-1863) at work.
--net-verbatim makes outputMessage (net_io.c:5846-5866) forward every accepted frame, 2-bit repairs included, as received.

The raw service's heartbeat is the line "*0000;\n" (net_io.c:110), sent after 60 s without output (checkFlushService); a
raw_out client gets no burst of heartbeats on connect (sendFiveHeartbeats is Beast only).  With --mlat every record of this
capture starts with '@' (no timestamp is 0), so "*0000;\n" lines there are heartbeats and are dropped; without --mlat a Mode A/C
reply 0000 is that same line, so the script checks that the count of such lines equals the count of 0000 replies of the MLAT
run, i.e. that no heartbeat was sent.

Only the two byte strings are stored, in tests/golden/raw/raw_stream.npz (a directory of its own: the *.npz files directly
under tests/golden/ are demodulator captures that the oracle and full-size tests replay).

    python tests/golden/make_raw_golden.py
"""
import json
import socket
import subprocess
import sys
import tempfile
import threading
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
HEARTBEAT = b"*0000;\n"


def capture():
    """The uc8 capture of beast_stream.npz: its silence, then its traffic."""
    z = np.load(HERE / "beast_stream.npz")
    meta = json.loads(bytes(z["meta"]).decode())
    return np.concatenate([np.full(2 * meta["silence_samples"], 127, np.uint8), z["traffic"]])


def run_reference(cap: np.ndarray, mlat: bool) -> bytes:
    srv = socket.socket(); srv.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1); srv.bind(("127.0.0.1", 0)); srv.listen(1)
    port = srv.getsockname()[1]
    data = bytearray()

    def reader():
        c, _ = srv.accept(); c.settimeout(10)
        try:
            while True:
                b = c.recv(65536)
                if not b:
                    break
                data.extend(b)
        except OSError:
            pass
    t = threading.Thread(target=reader); t.start()
    with tempfile.NamedTemporaryFile(suffix=".bin") as f:
        cap.tofile(f.name)
        subprocess.run([str(ROOT / "oracle" / "_ref" / "readsb_cpu"), "--device-type", "ifile", "--ifile", f.name, "--throttle", "--quiet",
                        "--modeac", "--net", "--net-verbatim", "--net-connector", f"127.0.0.1,{port},raw_out"] + (["--mlat"] if mlat else []),
                       check=True, timeout=120, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    t.join(timeout=15)
    srv.close()
    return bytes(data)


def lines(data: bytes):
    out = [l + b"\n" for l in data.split(b"\n")[:-1]]
    assert b"".join(out) == data and all(l.endswith(b";\n") for l in out), "raw output does not end in a complete record"
    return out


def main():
    cap = capture()
    mlat = [l for l in lines(run_reference(cap, True)) if l != HEARTBEAT]
    plain = lines(run_reference(cap, False))
    assert all(l.startswith(b"@") for l in mlat)
    n_zero_replies = sum(1 for l in mlat if len(l) == 1 + 12 + 4 + 2 and l.endswith(b"0000;\n"))
    assert plain.count(HEARTBEAT) == n_zero_replies, "a heartbeat reached the plain run's client"
    assert len(plain) == len(mlat) and all(a[13:] == b[1:] for a, b in zip(mlat, plain))
    raw_mlat, raw = b"".join(mlat), b"".join(plain)
    print(len(mlat), "records;", len(raw_mlat), "bytes with --mlat,", len(raw), "without;",
          sum(1 for l in plain if len(l) == 7), "Mode A/C replies")
    (HERE / "raw").mkdir(exist_ok=True)
    np.savez_compressed(HERE / "raw" / "raw_stream.npz", raw_mlat=np.frombuffer(raw_mlat, np.uint8), raw=np.frombuffer(raw, np.uint8))


if __name__ == "__main__":
    main()
