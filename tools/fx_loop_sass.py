"""Instruction histogram of the fixed-point sample loop of the headline expansion kernel.

Compiles csrc/mplx_fxn.cu for sm_90a with the library's flags (or takes an object file built already),
finds the headline instantiation expand_fxn_kernel<3, 2, 4, 4, false, false, false, false, true> (3-D ACC,
UNR 4, unchecked loop, staged outputs) and prints the SASS of its sample loop by opcode, with the
instructions per sample.  The sample loop is the loop (backward branch) that holds the most 32-bit global
loads, one voxel word per sample; instructions per sample = loop length / those loads.  Needs nvcc and
cuobjdump, no GPU.

  python tools/fx_loop_sass.py                  # compile into a temporary directory
  python tools/fx_loop_sass.py --obj motion_primitive_library_b200/lib/obj/mplx_fxn.o
  python tools/fx_loop_sass.py --obj OLD.o --function _ZN4mplx17expand_fxn_kernelILi3ELi2ELi4ELi4ELb0ELb0ELb0ELb1E
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "motion_primitive_library_b200" / "csrc"
HEADLINE = "_ZN4mplx17expand_fxn_kernelILi3ELi2ELi4ELi4ELb0ELb0ELb0ELb0ELb1E"
CUDA = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda"))
LINE = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)\s*([^;]*);")


def compile_obj(out_dir: Path) -> Path:
    obj = out_dir / "mplx_fxn.cubin"
    cmd = [str(CUDA / "bin" / "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
           "-fmad=false", "-cubin", "-o", str(obj), str(CSRC / "mplx_fxn.cu")]
    subprocess.check_call(cmd, cwd=CSRC)
    return obj


def function_sass(obj: Path, prefix: str) -> tuple[str, list[tuple[int, str, str]]]:
    sass = subprocess.run([str(CUDA / "bin" / "cuobjdump"), "-sass", str(obj)], check=True, capture_output=True,
                          text=True).stdout
    name, body = None, []
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name is not None:
                break
            if m.group(1).startswith(prefix):
                name = m.group(1)
            continue
        if name is None:
            continue
        m = LINE.search(line)
        if m:
            body.append((int(m.group(1), 16), m.group(3), m.group(4).strip()))
    if name is None:
        sys.exit(f"no function {prefix}* in {obj}")
    return name, body


def is_word_load(op: str) -> bool:
    parts = op.split(".")
    return parts[0] == "LDG" and not any(p in ("64", "128", "U8", "S8", "U16", "S16") for p in parts[1:])


def sample_loop(body):
    addr = {a: i for i, (a, _, _) in enumerate(body)}
    best = None
    for i, (a, op, args) in enumerate(body):
        if not op.startswith("BRA"):
            continue
        m = re.search(r"0x([0-9a-f]+)\s*$", args)
        if not m or int(m.group(1), 16) >= a or int(m.group(1), 16) not in addr:
            continue
        lo = addr[int(m.group(1), 16)]
        loads = sum(is_word_load(o) for _, o, _ in body[lo:i + 1])
        key = (loads, -(i + 1 - lo))
        if loads and (best is None or key > best[0]):
            best = (key, lo, i)
    if best is None:
        sys.exit("no loop with 32-bit global loads")
    return body[best[1]:best[2] + 1]


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--obj", type=Path, help="object or cubin holding the kernel (default: compile mplx_fxn.cu)")
    ap.add_argument("--function", default=HEADLINE, help="mangled-name prefix of the kernel")
    ap.add_argument("--json", action="store_true", help="one JSON line instead of the table")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        obj = args.obj if args.obj else compile_obj(Path(tmp))
        name, body = function_sass(obj, args.function)
    loop = sample_loop(body)
    samples = sum(is_word_load(op) for _, op, _ in loop)
    hist = collections.Counter(op.split(".")[0] for _, op, _ in loop)
    const_reads = sum("c[0x" in args for _, _, args in loop)
    res = {"function": name, "loop_instructions": len(loop), "samples": samples,
           "per_sample": round(len(loop) / samples, 2), "ldc": hist.get("LDC", 0),
           "constant_bank_operands": const_reads, "histogram": dict(hist.most_common())}
    if args.json:
        print(json.dumps(res))
        return
    print(f"{name}\nsample loop: {len(loop)} instructions, {samples} voxel-word loads, "
          f"{res['per_sample']} instructions per sample; LDC {res['ldc']}, constant-bank operands {const_reads}")
    for op, n in hist.most_common():
        print(f"  {op:10s} {n:4d}  {n / samples:6.2f} per sample")


if __name__ == "__main__":
    main()
