"""The zone drop-in headers: tests/cpp/zone_dropin_example.cpp builds with plain g++ against
include/ouster/core/zone.h (mesh.h, beam_config.h, zrb.h, zone_state.h) and runs on the GPU; its rendered ZRB
equals the oracle's on the same LUT.  The new ABI structs compile as C99."""
import os
import subprocess

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import zone as oz
from tests.test_oracle_zone import ZDIR, s2b_z1, sensor_meta, stl_tris

ROOT = graft.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "zone_dropin_example.cpp")
LIB_DIR = os.path.join(ROOT, "ouster-sdk_b200", "lib")


def build_example(out_dir):
    graft.build()
    exe = os.path.join(str(out_dir), "zone_dropin_example")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "include"),
                           SRC, "-L", LIB_DIR, "-louster_b200", f"-Wl,-rpath,{LIB_DIR}", "-o", exe])
    return exe


def test_zone_structs_are_plain_c99(tmp_path):
    graft.build()
    src = tmp_path / "zone.c"
    src.write_text('#include "ouster_b200.h"\n'
                   "int main(void) { ob_zone_desc d = {0}; ob_zone_render_io r = {0}; ob_zone_live l = {0};\n"
                   "  ob_zone_state s = {0}; (void)d; (void)r; (void)l; (void)s;\n"
                   "  return sizeof(ob_zone_state) == 37 && ob_abi_sizeof(\"ob_zone_render_io\") == sizeof(r) &&\n"
                   "         ob_abi_sizeof(\"ob_zone_live\") == sizeof(l) && ob_abi_sizeof(\"ob_zone_desc\") == sizeof(d)"
                   " ? 0 : 1; }\n")
    exe = tmp_path / "zone"
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I",
                           os.path.join(ROOT, "include"), str(src), "-L", LIB_DIR, "-louster_b200",
                           f"-Wl,-rpath,{LIB_DIR}", "-o", str(exe)])
    assert subprocess.run([str(exe)]).returncode == 0


def test_zone_dropin_example_compiles(tmp_path):
    assert os.path.exists(build_example(tmp_path))


@pytest.mark.gpu
def test_zone_dropin_example_runs_on_gpu(tmp_path):
    ob = graft.load_package()
    meta = sensor_meta("785.json")
    h, w = meta["h"], meta["w"]
    beams = tmp_path / "beams.txt"
    with open(beams, "w") as f:
        f.write(f"{h} {w}\n")
        for key in ("beam_altitude_angles", "beam_azimuth_angles"):
            f.write(" ".join(repr(float(v)) for v in meta[key]) + "\n")
        for key in ("beam_to_lidar_transform", "lidar_to_sensor_transform"):
            f.write(" ".join(repr(float(v)) for v in np.asarray(meta[key]).reshape(16)) + "\n")
    out_bin = tmp_path / "zrb.bin"
    out = subprocess.run([build_example(tmp_path), ZDIR, str(beams), str(out_bin)], capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "ZONE DROPIN OK" in out.stdout
    got = np.fromfile(out_bin, np.uint32).reshape(2, h, w)
    # the oracle on the LUT the package builds for the same beams
    s2b = s2b_z1()
    s2b[:3, 3] *= 1000
    lut = ob.XYZLutT.from_intrinsics(w, h, 0.001, meta["beam_to_lidar_transform"],
                                     s2b @ meta["lidar_to_sensor_transform"], meta["beam_azimuth_angles"],
                                     meta["beam_altitude_angles"])
    near, far, px = oz.render(stl_tris("0.stl"), lut.direction, lut.offset, h, w)
    assert np.array_equal(got[0], near) and np.array_equal(got[1], far)
    assert f"({px} pixels hit)" in out.stdout and np.count_nonzero(near < far) == 12096
