"""Builds tests/cpp/dropin_example.cpp against the replacement headers (include/ouster/core) and
libouster_b200.so with plain g++, then runs it on the GPU: source-level drop-in proof.  The binary goes
to a temporary directory, so the tests also run from a read-only checkout."""
import os
import subprocess

import pytest

import __graft_entry__ as graft

ROOT = graft.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "dropin_example.cpp")


def build_example(out_dir):
    graft.build()
    lib_dir = os.path.join(ROOT, "ouster-sdk_b200", "lib")
    exe = os.path.join(str(out_dir), "dropin_example")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), SRC,
           "-L", lib_dir, "-louster_b200", f"-Wl,-rpath,{lib_dir}", "-o", exe]
    subprocess.check_call(cmd)
    return exe


def test_dropin_example_compiles(tmp_path):
    """CPU: the reference-style user code compiles and links against the replacement headers."""
    assert os.path.exists(build_example(tmp_path))


@pytest.mark.gpu
def test_dropin_example_runs_on_gpu(tmp_path):
    exe = build_example(tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "DROPIN OK" in out.stdout
