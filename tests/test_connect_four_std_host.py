"""CPU: connect_four's default-board rule core (sizes known at compile time) against the general one, compiled for the host from
the product header (tests/connect_four_std_host.cc): identical keys, status, legal masks, observations and action handling
along random games, and no other board accepted."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"


@pytest.mark.skipif(shutil.which("g++") is None or not os.path.isdir(CUDA_INC), reason="needs g++ and the CUDA headers")
def test_default_board_core_equals_general_core(tmp_path):
    exe = tmp_path / "c4_std"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", ROOT, "-I", CUDA_INC, "-o", str(exe),
                           os.path.join(ROOT, "tests", "connect_four_std_host.cc")])
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("ok:"), r.stdout
