"""The CTA-span copy-out of the fixed-point kernel without a GPU: the lead / head / body / tail / trail split of
csrc/mplx_span.cuh against a literal byte-by-byte statement for every element size, base offset and span
length the kernel uses (tests/fxn_span_host.cpp)."""
import subprocess
from pathlib import Path

HERE = Path(__file__).resolve().parent


def test_span_copy_split(tmp_path):
    exe = tmp_path / "fxn_span_host"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", str(exe), str(HERE / "fxn_span_host.cpp")])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    print(out.stdout[-2000:])
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert "fxn_span_host fails 0" in out.stdout
