"""TEST INFRASTRUCTURE: builds tests/emu/_build/libb200demod_emu.so — the repository's own .cu sources (kernels + C ABI),
rewritten mechanically and compiled by g++ against tests/emu/cuda_runtime.h, so the kernels' logic runs on the CPU under
the SIMT emulator (see that header).  Never used by the product; loaded only by tests/test_emu_kernels.py.

The rewrite touches three constructs and nothing else (anything it does not recognise is a build error, not a guess):
  * kernel<<<grid, block, smem, stream>>>(args);     ->  EMU_LAUNCH(grid, block, smem, kernel(args));
  * extern __shared__ [__align__(n)] T name[];       ->  T *name = reinterpret_cast<T *>(emu_smem);
  * asm [volatile]("op ..." : outs : ins : clobbers);->  emu_asm_<op>(outs..., ins..., immediates...);
"""
from __future__ import annotations

import re
import shutil
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
CSRC = ROOT / "readsb_b200" / "csrc"
BUILD = HERE / "_build"
LIB = BUILD / "libb200demod_emu.so"


def _balanced(src: str, i: int) -> int:
    """src[i] == '(' -> index just past the matching ')', string literals respected."""
    depth, j, n = 0, i, len(src)
    while j < n:
        c = src[j]
        if c == '"':
            j += 1
            while src[j] != '"':
                j += 2 if src[j] == "\\" else 1
        elif c == "(":
            depth += 1
        elif c == ")":
            depth -= 1
            if depth == 0:
                return j + 1
        j += 1
    raise ValueError("unbalanced parentheses")


def _split_top(s: str, sep: str) -> list[str]:
    out, depth, cur, j = [], 0, [], 0
    while j < len(s):
        c = s[j]
        if c == '"':
            k = j + 1
            while s[k] != '"':
                k += 2 if s[k] == "\\" else 1
            cur.append(s[j:k + 1]); j = k + 1
            continue
        if c in "([{":
            depth += 1
        elif c in ")]}":
            depth -= 1
        if c == sep and depth == 0:
            out.append("".join(cur)); cur = []
        else:
            cur.append(c)
        j += 1
    out.append("".join(cur))
    return out


def _operands(section: str) -> list[str]:
    exprs = []
    for item in _split_top(section, ","):
        item = item.strip()
        if not item:
            continue
        m = re.match(r'"[^"]*"\s*\(', item)
        if not m:
            raise ValueError(f"asm operand not understood: {item!r}")
        exprs.append(item[m.end():item.rindex(")")].strip())
    return exprs


def rewrite_asm(src: str) -> str:
    out, i = [], 0
    for m in re.finditer(r"\basm\s*(volatile\s*)?\(", src):
        if m.start() < i:
            continue
        end = _balanced(src, m.end() - 1)
        body = src[m.end():end - 1]
        parts = _split_top(body, ":")
        # "a::b" inside the template is protected by the string handling; "::" between sections gives an empty part
        template = "".join(re.findall(r'"((?:[^"\\]|\\.)*)"', parts[0]))
        outs = _operands(parts[1]) if len(parts) > 1 else []
        ins = _operands(parts[2]) if len(parts) > 2 else []
        stmts = [s.strip() for s in template.split(";") if s.strip()]
        if len(stmts) != 1:
            raise ValueError(f"asm with {len(stmts)} instructions is not supported: {template!r}")
        toks = stmts[0].split(None, 1)
        op = re.sub(r"[^A-Za-z0-9]", "_", toks[0])
        imms = []
        if len(toks) > 1:
            for t in re.split(r"[,\s]+", toks[1]):
                if re.fullmatch(r"-?\d+", t):
                    imms.append(t)
        call = f"emu_asm_{op}({', '.join(outs + ins + imms)})"
        tail = src[end:]
        out.append(src[i:m.start()]); out.append(call)
        i = end
        if not tail.lstrip().startswith(";"):
            raise ValueError("asm statement not followed by ';'")
    out.append(src[i:])
    return "".join(out)


def rewrite_launches(src: str) -> str:
    out, i = [], 0
    for m in re.finditer(r"([A-Za-z_]\w*(?:<[^<>;(){}]*>)?)\s*<<<", src):
        if m.start() < i:
            continue
        close = src.index(">>>", m.end())
        cfg = _split_top(src[m.end():close], ",")
        if len(cfg) not in (2, 3, 4):
            raise ValueError(f"launch configuration not understood: {src[m.end():close]!r}")
        cfg += ["0"] * (4 - len(cfg))
        j = close + 3
        while src[j].isspace():
            j += 1
        if src[j] != "(":
            raise ValueError("kernel launch without an argument list")
        end = _balanced(src, j)
        args = src[j:end]
        out.append(src[i:m.start()])
        out.append(f"EMU_LAUNCH({cfg[0].strip()}, {cfg[1].strip()}, {cfg[2].strip()}, {m.group(1)}{args})")
        i = end
    out.append(src[i:])
    return "".join(out)


def rewrite_dynamic_smem(src: str) -> str:
    pat = re.compile(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?([\w\s]+?)\s+(\w+)\s*\[\s*\]\s*;")
    return pat.sub(lambda m: f"{m.group(1)} *{m.group(2)} = reinterpret_cast<{m.group(1)} *>(emu_smem);", src)


def transform(text: str) -> str:
    text = rewrite_dynamic_smem(text)
    text = rewrite_launches(text)
    text = rewrite_asm(text)
    text = re.sub(r"\b__noinline__\b", "EMU_NOINLINE", text)      # libstdc++ spells __attribute__((__noinline__)): no macro of that name
    for leftover in ("<<<", "asm(", "asm volatile", "extern __shared__"):
        if leftover in re.sub(r"//[^\n]*", "", text):
            raise ValueError(f"construct left after the rewrite: {leftover}")
    return text


def sanitizer_runtime(sanitize: str) -> str:
    """The sanitizer's shared runtime, to LD_PRELOAD into the (uninstrumented) python that loads the library."""
    cxx = shutil.which("g++") or "g++"
    name = {"address": "libasan.so", "undefined": "libubsan.so"}[sanitize]
    return subprocess.run([cxx, f"-print-file-name={name}"], capture_output=True, text=True, check=True).stdout.strip()


def build(force: bool = False, verbose: bool = False, sanitize: str | None = None) -> Path:
    """sanitize = "address": heap "device" buffers get redzones, so a kernel reading or writing past a pool, an arena or a
    result array is reported with the source line; "undefined": oversized shifts, signed overflow, misaligned vector loads —
    the places where C++ on the CPU and the GPU's semantics could differ."""
    srcs = sorted(CSRC.glob("*.cu")) + sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h"))
    deps = srcs + [HERE / "cuda_runtime.h", HERE / "emu_rt.cpp", Path(__file__), ROOT / "include" / "b200_demod.h"]
    LIB = BUILD / ("libb200demod_emu.so" if not sanitize else f"libb200demod_emu_{sanitize}.so")
    if not force and LIB.exists() and all(d.stat().st_mtime <= LIB.stat().st_mtime for d in deps):
        return LIB
    gen = BUILD / ("src" if not sanitize else f"src_{sanitize}")
    if gen.exists():
        shutil.rmtree(gen)
    gen.mkdir(parents=True)
    cpp = []
    for s in srcs:
        text = transform(s.read_text())
        name = s.name.replace(".cu", ".cpp") if s.suffix == ".cu" else s.name
        (gen / name).write_text(f"// generated from readsb_b200/csrc/{s.name} by tests/emu/build_emu.py — do not edit\n" + text)
        if s.suffix == ".cu":
            cpp.append(gen / name)
    cxx = shutil.which("g++") or "g++"
    # -ffp-contract=off mirrors nvcc --fmad=false; -O1 keeps frames small and the build quick; -fno-strict-aliasing because the
    # kernels reinterpret shared memory freely (nvcc does not do type-based alias analysis on it either)
    san = [f"-fsanitize={sanitize}", "-fno-omit-frame-pointer"] if sanitize else []
    cmd = [cxx, "-std=c++17", "-O1", "-g", "-fPIC", "-shared", *san, "-ffp-contract=off", "-fno-strict-aliasing", "-fvisibility=hidden",
           "-Wall", "-Wno-unused-function", "-Wno-unknown-pragmas", "-Wno-unused-variable", "-Wno-unused-but-set-variable",
           "-include", str(HERE / "cuda_runtime.h"), "-I", str(HERE), "-I", str(gen), "-I", str(ROOT / "include"),
           *map(str, cpp), str(HERE / "emu_rt.cpp"), "-o", str(LIB), "-lpthread"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("emulator build failed:\n" + res.stdout + res.stderr[-8000:])
    if verbose and res.stderr:
        print(res.stderr[-4000:])
    return LIB


if __name__ == "__main__":
    san = next((a.split("=", 1)[1] for a in sys.argv if a.startswith("--sanitize=")), None)
    print(build(force="--force" in sys.argv, verbose=True, sanitize=san))
