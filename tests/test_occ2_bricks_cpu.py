"""The occ2 brick layout without a GPU: the addressing and the full pack of csrc/mplx_pack.cuh against a
literal per-voxel statement on odd 2-D and 3-D dims (tests/occ2_bricks_host.cpp)."""
import subprocess
from pathlib import Path

HERE = Path(__file__).resolve().parent


def test_brick_addressing_and_pack(tmp_path):
    exe = tmp_path / "occ2_bricks_host"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", str(exe), str(HERE / "occ2_bricks_host.cpp")])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    print(out.stdout[-2000:])
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert "occ2_bricks_host fails 0" in out.stdout
