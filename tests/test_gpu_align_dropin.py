"""The cloud-alignment drop-in header: tests/cpp/align_dropin_example.cpp builds with plain g++ against
include/ouster/algorithm/align_clouds.h and runs on the GPU; the new ABI structs compile as C99."""
import os
import subprocess

import pytest

import __graft_entry__ as graft

ROOT = graft.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "align_dropin_example.cpp")


def build_example(out_dir):
    graft.build()
    lib_dir = os.path.join(ROOT, "ouster-sdk_b200", "lib")
    exe = os.path.join(str(out_dir), "align_dropin_example")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), SRC,
                           "-L", lib_dir, "-louster_b200", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    return exe


def test_align_structs_are_plain_c99(tmp_path):
    graft.build()
    src = tmp_path / "align.c"
    src.write_text('#include "ouster_b200.h"\n'
                   "int main(void) { ob_cloud_align_io a = {0}; ob_cloud_nearest_io n = {0}; (void)a; (void)n;\n"
                   "  return ob_abi_sizeof(\"ob_cloud_align_io\") == sizeof(ob_cloud_align_io) &&\n"
                   "         ob_abi_sizeof(\"ob_cloud_nearest_io\") == sizeof(ob_cloud_nearest_io) ? 0 : 1; }\n")
    lib_dir = os.path.join(ROOT, "ouster-sdk_b200", "lib")
    exe = tmp_path / "align"
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I",
                           os.path.join(ROOT, "include"), str(src), "-L", lib_dir, "-louster_b200",
                           f"-Wl,-rpath,{lib_dir}", "-o", str(exe)])
    assert subprocess.run([str(exe)]).returncode == 0


def test_align_dropin_example_compiles(tmp_path):
    assert os.path.exists(build_example(tmp_path))


@pytest.mark.gpu
def test_align_dropin_example_runs_on_gpu(tmp_path):
    out = subprocess.run([build_example(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "ALIGN DROPIN OK" in out.stdout
