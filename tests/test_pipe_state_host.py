"""The ring position of the tensor-core kernels' TMA rings (PipeState in csrc/pipe_state.cuh), on the host.

tests/pipe_state_host.cpp compiles the header as plain C++ and checks, for rings of 1 to 4 buffers over 5000 positions, that advance()
and at(n) agree, that both equal the slot and parity arithmetic the kernels used before the ring existed (n % N with (n / N) & 1, the
wrapped counters, i & 1 with (i >> 1) & 1, and it & 1 with (it - 1) & 1), and that a model of mbarrier phases driven by the producer and
consumer parities, under random interleavings of one producer and 1, 2, 4 or 8 releasers, never refills a slot before all its releases,
never lets a consumer read a slot before it holds that position, and never deadlocks.
"""
import shutil
import subprocess

import pytest

from conftest import ROOT


def test_pipe_state_matches_the_ring_protocol(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = tmp_path / "pipe_state_host"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-I", str(ROOT / "k-diffusion_b200" / "csrc"),
                    str(ROOT / "tests" / "pipe_state_host.cpp"), "-o", str(exe)], check=True)
    run = subprocess.run([str(exe)], capture_output=True, text=True)
    assert run.returncode == 0 and run.stdout.strip() == "ok", run.stdout
