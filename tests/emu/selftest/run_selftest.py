"""TEST INFRASTRUCTURE: builds tests/emu/selftest/selftest.cu with the emulator's rewrite and checks every primitive against
what the CUDA / PTX definitions say (computed here in numpy)."""
import ctypes
import subprocess
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
import build_emu  # noqa: E402


def build() -> Path:
    out = build_emu.BUILD / "libemu_selftest.so"
    gen = build_emu.BUILD / "selftest_src"
    gen.mkdir(parents=True, exist_ok=True)
    (gen / "selftest.cpp").write_text(build_emu.transform((HERE / "selftest.cu").read_text()))
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-ffp-contract=off", "-fno-strict-aliasing", "-fvisibility=hidden", "-w",
           "-include", str(HERE.parent / "cuda_runtime.h"), "-I", str(HERE.parent), str(gen / "selftest.cpp"), str(HERE.parent / "emu_rt.cpp"),
           "-o", str(out), "-lpthread"]
    subprocess.run(cmd, check=True)
    return out


def s8(x):
    return ((x & 0xff) ^ 0x80) - 0x80


NB, NT = 3, 96


def make_input():
    rng = np.random.default_rng(1)
    inp = rng.integers(0, 1 << 32, size=NB * NT, dtype=np.uint64).astype(np.uint32)
    inp[5] = 0; inp[6] = 0xffffffff
    return inp


def build_sm90a() -> Path:
    """The same source as real CUDA (for the gpu-marked test that pins the emulator's definitions against the hardware)."""
    out = build_emu.BUILD / "libemu_selftest_sm90a.so"
    build_emu.BUILD.mkdir(parents=True, exist_ok=True)
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-shared", "-Xcompiler", "-fPIC", "-cudart", "shared",
                    str(HERE / "selftest.cu"), "-o", str(out)], check=True)
    return out


def check(inp, ow, ob, cnt):
    """inp, ow (32 x 16), ob (NB x NT), cnt (1): numpy uint32 arrays as the two kernels left them."""
    v = [int(x) for x in inp[:32]]
    M = 0xffffffff
    ballot = sum(((v[l] >> 3) & 1) << l for l in range(32))
    red = sum(x & 0xffff for x in v) & M
    for l in range(32):
        o = [int(x) for x in ow[l * 16:(l + 1) * 16]]
        x = v[l]
        nx = ~x & M
        assert o[0] == v[(l * 7 + 3) & 31], "shfl"
        assert o[1] == (v[l - 3] if l >= 3 else x), "shfl_up"
        assert o[2] == (v[l + 5] if l + 5 < 32 else x), "shfl_down"
        assert o[3] == v[l ^ 9], "shfl_xor"
        assert o[4] == ballot and o[5] == red, "ballot / reduce"
        ffs = (x & -x).bit_length() if x else 0
        clz = 32 - x.bit_length()
        assert o[6] == (bin(x).count("1") | (ffs << 8) | (clz << 16)), "popc / ffs / clz"
        assert o[7] == int(f"{x:032b}"[::-1], 2), "brev"
        wide = (nx << 32) | x
        assert o[8] == (wide >> (l & 31)) & M, "funnelshift_r"
        assert o[9] == ((wide << (l & 31)) >> 32) & M, "funnelshift_l"
        by = [(x >> (8 * i)) & 0xff for i in range(4)] + [(nx >> (8 * i)) & 0xff for i in range(4)]
        sel = 0x5410 + (l & 3) + ((l & 4) << 2) + ((l & 24) << 5)
        assert o[10] == sum(by[(sel >> (4 * i)) & 7] << (8 * i) for i in range(4)), "byte_perm"
        assert o[11] == sum((0xff if by[i] & 0x80 else 0) << (8 * i) for i in range(4)), "prmt sign replication"
        lo, hi = x & 0xffff, x >> 16
        assert o[12] == (-7 + lo * s8(0xee) + hi * s8(0x0f)) & M, "dp2a.lo"
        assert o[13] == (11 + lo * s8(0x14) + hi * s8(0xff)) & M, "dp2a.hi"
        src = 31 - l
        assert o[14] == sum(i + src for i in range(src & 3)), "reconvergence"
        w = 5 + x * x
        assert o[15] == ((w >> 32) ^ w) & M, "mad.wide"
    total_all = 0
    for b in range(NB):
        blk = [int(t) for t in inp[b * NT:(b + 1) * NT]]
        total = sum(t & 0xff for t in blk)
        total_all += total
        for t in range(NT):
            assert int(ob[b * NT + t]) == (blk[NT - 1 - t] + total) & M, "block kernel"
    assert int(cnt[0]) == total_all


def main():
    L = ctypes.CDLL(str(build()))
    inp = make_input()
    ow = np.zeros(32 * 16, np.uint32); ob = np.zeros(NB * NT, np.uint32); cnt = np.zeros(1, np.uint32)
    rc = L.b200_emu_selftest(inp.ctypes.data, ow.ctypes.data, ob.ctypes.data, cnt.ctypes.data, NB, NT)
    assert rc == 0
    check(inp, ow, ob, cnt)
    print("emulator self-test ok")


if __name__ == "__main__":
    main()
