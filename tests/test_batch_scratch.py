"""CPU: unit test of the scratch carver (redisearch_b200/csrc/batch_scratch.h) that lays out a batch's regions in one device
buffer.  Compiled with g++ and run as a plain host program over random region lists."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_batch_scratch_regions_are_aligned_disjoint_and_sized(tmp_path):
    exe = tmp_path / "batch_scratch_test"
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", os.path.join(ROOT, "tests", "cpp", "batch_scratch_test.cpp"), "-o", str(exe)],
                   check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "batch_scratch: ok" in r.stdout, r.stdout
