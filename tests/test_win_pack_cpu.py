"""The packed fp64 slab entry of the column-windowed SpMV (csrc/win_pack.h) round-trips bit for bit -- CPU only.

tests/win_pack_probe.cu runs the encoder and the very __host__ __device__ decode functions spmv_win_kernel calls on
3.6 million random bit patterns (every exponent field, windows at both ends of the range), on +-0, subnormals, +-Inf
and NaNs with payloads, on both edges of the 14-binade window and on the columns 0, 127, 128 and 32767."""
import os
import shutil
import subprocess

import pytest


def test_packed_slab_entry_round_trips_bit_exactly(tmp_path):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("no nvcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "win_pack_probe")
    subprocess.run([nvcc, "-std=c++17", "-I", os.path.join(root, "cosmo.jl_b200", "csrc"), "-gencode", "arch=compute_90a,code=sm_90a",
                    "-o", exe, os.path.join(root, "tests", "win_pack_probe.cu")], check=True, cwd=str(tmp_path))
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "bad 0" in out.stdout, out.stdout + out.stderr
