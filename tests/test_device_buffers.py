"""The library's owning buffers (tempestsdr_b200/csrc/devbuf.h) when an allocation fails, checked on the CPU.

tests/c_host/devbuf_check.cpp is built with the host compiler against a stub of the CUDA runtime calls the header uses (no
CUDA library is linked, so nothing else can sneak in).  The stub fails the k-th allocation, for every k over a fixed sequence
of assign / reserve calls.  A failure must leave each buffer as it was or empty, never a freed pointer or a capacity it does
not have; reserve must keep the elements it was asked to keep; and every allocation must be freed exactly once.
"""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def test_buffers_survive_every_failed_allocation(tmp_path):
    exe = tmp_path / "devbuf_check"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(CUDA_HOME, "include"), os.path.join(ROOT, "tests", "c_host", "devbuf_check.cpp"),
                    "-o", str(exe)], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    runs = int(r.stdout.split()[1])
    assert runs >= 12                     # no failure, then each of the sequence's allocations failing in turn
