"""The voxel-downsampling ABI struct and drop-in headers: the ctypes mirror of ob_voxel_io has the C size, the
struct compiles as C99, and tests/cpp/voxel_dropin_example.cpp builds with plain g++ against
include/ouster/core/voxel_hash_map.h + include/ouster/algorithm/voxel_downsample.h and runs on the GPU."""
import ctypes
import os
import subprocess

import pytest

import __graft_entry__ as graft

ROOT = graft.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "voxel_dropin_example.cpp")


def build_example(out_dir):
    graft.build()
    lib_dir = os.path.join(ROOT, "ouster-sdk_b200", "lib")
    exe = os.path.join(str(out_dir), "voxel_dropin_example")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), SRC,
                           "-L", lib_dir, "-louster_b200", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    return exe


def test_voxel_io_layout_matches_the_c_abi():
    graft.build()
    capi = graft.load_package()._capi
    assert capi.lib.ob_abi_sizeof(b"ob_voxel_io") == ctypes.sizeof(capi.VoxelIO)


def test_voxel_io_is_plain_c99(tmp_path):
    graft.build()
    src = tmp_path / "voxel.c"
    src.write_text('#include "ouster_b200.h"\n'
                   "int main(void) { ob_voxel_io io = {0}; io.mode = OB_VOXEL_POINT_NORMAL; (void)io;\n"
                   "  return ob_abi_sizeof(\"ob_voxel_io\") == sizeof(ob_voxel_io) ? 0 : 1; }\n")
    lib_dir = os.path.join(ROOT, "ouster-sdk_b200", "lib")
    exe = tmp_path / "voxel"
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I",
                           os.path.join(ROOT, "include"), str(src), "-L", lib_dir, "-louster_b200",
                           f"-Wl,-rpath,{lib_dir}", "-o", str(exe)])
    assert subprocess.run([str(exe)]).returncode == 0


def test_voxel_dropin_example_compiles(tmp_path):
    assert os.path.exists(build_example(tmp_path))


@pytest.mark.gpu
def test_voxel_dropin_example_runs_on_gpu(tmp_path):
    out = subprocess.run([build_example(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "VOXEL DROPIN OK" in out.stdout
