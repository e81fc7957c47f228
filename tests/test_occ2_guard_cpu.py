"""The guard-banded occ2 buffer without a GPU: the padded pack, the padded and separable cell addresses and the
sample loop's reach bound of csrc/mplx_pack.cuh against a literal per-cell statement on odd 2-D and 3-D dims
(tests/occ2_guard_host.cpp)."""
import subprocess
from pathlib import Path

HERE = Path(__file__).resolve().parent


def test_guard_band_layout_address_and_reach(tmp_path):
    exe = tmp_path / "occ2_guard_host"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", str(exe), str(HERE / "occ2_guard_host.cpp")])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    print(out.stdout[-2000:])
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert "occ2_guard_host fails 0" in out.stdout
