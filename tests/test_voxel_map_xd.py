"""CPU checks of the voxel map with per-point attributes (VoxelHashMapXd, DESIGN f-11): the plain-Python statement
the GPU tests compare against (tests/voxel_map_xd_reference.py) agrees with the registration oracle on x, y, z, the
reference's known answers, and the C ABI's constructor checks, refusals and struct layouts without a device."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import icp as oi
from tests import voxel_map_xd_reference as xr

ROOT = graft.ROOT


def _cycles(seed, n_cycles=25):
    rs = np.random.default_rng(seed)
    for cycle in range(n_cycles):
        centre = np.array([np.cos(cycle / 9.0), np.sin(cycle / 7.0), 0.1 * cycle]) * 8.0
        pts = centre + rs.normal(0, 3.0, (int(rs.integers(0, 400)), 3))
        if cycle % 5 == 3:
            pts[: len(pts) // 2] = centre + rs.random((len(pts) // 2, 3)) * 0.49
        if cycle % 7 == 5 and len(pts) > 4:
            pts[0, 0], pts[1, 1], pts[2] = np.nan, 1e300, [-1e300, np.nan, 1e300]
        yield cycle, centre, pts


@pytest.mark.parametrize("max_pts", [1, 20])
def test_reference_without_attributes_is_the_oracle(max_pts):
    """num_attributes = 0: the Python statement and oracle/orc_icp.c give the same map, extracts and neighbours."""
    xm, om = xr.VoxelHashMapXd(0.5, 6.0, max_pts), oi.VoxelHashMap3d(0.5, 6.0, max_pts)
    for cycle, centre, pts in _cycles(max_pts):
        xm.add_points(pts)
        om.add_points(pts)
        if cycle % 3 == 0:
            assert np.array_equal(xm.extract_voxels_far_from_location(centre),
                                  om.extract_voxels_far_from_location(centre), equal_nan=True)
        elif cycle % 3 == 1:
            xm.remove_voxels_far_from_location(centre)
            om.remove_voxels_far_from_location(centre)
        assert xm.size() == om.size()
        assert np.array_equal(xm.point_cloud(), om.point_cloud(), equal_nan=True)
    q = centre + np.random.default_rng(1).normal(0, 2.0, (200, 3))
    for bound in (xr.DBL_MAX, 0.3):
        nb, d2 = xm.get_closest_neighbors(q, bound)
        wnb, wd2 = om.get_closest_neighbors(q, bound)
        assert np.array_equal(nb, wnb) and np.array_equal(d2, wd2)


def test_attributes_ride_along_and_the_gate_ignores_them():
    rs = np.random.default_rng(4)
    xyz = rs.normal(0, 3.0, (600, 3))
    xyz[300:] = xyz[:300]                          # every point twice: the second copy is always refused
    attrs = rs.normal(0, 1.0, (600, 2))
    xm = xr.VoxelHashMapXd(0.5, 100.0, 4, num_attributes=2)
    om = oi.VoxelHashMap3d(0.5, 100.0, 4)
    xm.add_points(np.hstack([xyz, attrs]))
    om.add_points(xyz)
    pc = xm.point_cloud()
    assert pc.shape[1] == 5 and np.array_equal(pc[:, :3], om.point_cloud())
    # an admitted row keeps its own attributes; the refused duplicates' attributes are dropped
    first = {tuple(p): a for p, a in zip(xyz[:300], attrs[:300])}
    assert all(np.array_equal(r[3:], first[tuple(r[:3])]) for r in pc)
    # extract rows carry the attributes
    ext = xm.extract_voxels_far_from_location(np.array([1000.0, 0.0, 0.0, 7.0, 7.0]))
    assert np.array_equal(ext, pc) and xm.empty
    # closest neighbour: the whole row; zeros and the bound when nothing qualifies
    xm.add_points(np.array([[0.1, 0.1, 0.1, 5.0, 6.0]]))
    nb, d2 = xm.get_closest_neighbor(np.array([0.1, 0.1, 0.2]))
    assert np.array_equal(nb, [0.1, 0.1, 0.1, 5.0, 6.0]) and d2 == pytest.approx(0.01)
    nb, d2 = xm.get_closest_neighbor(np.array([9.0, 9.0, 9.0]), 2.0)
    assert np.array_equal(nb, np.zeros(5)) and d2 == 2.0
    with pytest.raises(ValueError, match="unexpected point dimension"):
        xm.add_points(np.zeros((2, 3)))


def test_registration_with_an_attribute_map_known_answer():
    """python/tests/test_registration.py:49-70: ICP reads the map's x, y, z; on the oracle that is the 3-d map."""
    map_points = np.array([[0.0, 0.0, 0.0, 10.0], [1.0, 0.0, 0.0, 20.0], [0.0, 1.0, 0.0, 30.0], [0.0, 0.0, 1.0, 40.0]])
    xm = xr.VoxelHashMapXd(voxel_size=0.5, max_distance=10.0, num_attributes=1)
    xm.add_points(map_points)
    om = oi.VoxelHashMap3d(0.5, 10.0)
    om.add_points(xm.point_cloud()[:, :3])
    shifted = map_points[:, :3] + np.array([0.05, 0.02, -0.01])
    t, _ = oi.align_points_to_map(shifted, om, 0.5, 0.1, 20)
    assert t.shape == (4, 4)
    np.testing.assert_allclose((t[:3, :3] @ shifted.T).T + t[:3, 3], map_points[:, :3], atol=0.05)


@pytest.mark.parametrize("types", [("uint8", "float16"), ("uint16", "float32"), ("uint32", "float32"),
                                   ("int64", "uint64"), ("int8", "uint8", "float16"), ("float16", "float64")])
def test_widening_each_value_is_the_exporters_concatenate_then_astype(types):
    """The device widens every field value to double on its own; the exporter concatenates the fields first (numpy's
    common type) and then converts: the two agree for every mix of pixel types."""
    rs = np.random.default_rng(len(types))
    cols = []
    for t in types:
        dt = np.dtype(t)
        if dt.kind == "f":
            v = (rs.normal(0, 1e3, 500)).astype(dt)
        else:
            info = np.iinfo(dt)
            v = rs.integers(info.min, info.max, 500, dtype=dt, endpoint=True)
        cols.append(v.reshape(-1, 1))
    want = np.concatenate([np.zeros((500, 3)), np.concatenate(cols, axis=1)], axis=1).astype(np.float64)[:, 3:]
    got = np.hstack([c.astype(np.float64) for c in cols])
    assert np.array_equal(got, want, equal_nan=True)


def test_constructor_checks_and_refusals_through_the_abi():
    """voxel_hashmap_test.cpp:178-184: attributes are accepted for the Xd map (no argument error; without a GPU the
    device check answers), and the reference's texts come in its order."""
    ob = graft.load_package()
    lib = ob._capi.lib
    h = ctypes.c_void_p()
    assert lib.ob_voxel_map_create_xd(1.0, 100.0, 0, 1, 5, 0, ctypes.byref(h)) == ob._capi.OB_INVALID_ARGUMENT
    assert lib.ob_last_error() == b"max_points_per_voxel must be greater than 0"
    assert lib.ob_voxel_map_create_xd(0.0, -1.0, 20, 1, 5, 0, ctypes.byref(h)) == ob._capi.OB_INVALID_ARGUMENT
    assert lib.ob_last_error() == b"voxel_size must be greater than 0"
    assert lib.ob_voxel_map_create_xd(1.0, 0.0, 20, 1, 5, 0, ctypes.byref(h)) == ob._capi.OB_INVALID_ARGUMENT
    assert lib.ob_last_error() == b"max_distance must be greater than 0"
    rc = lib.ob_voxel_map_create_xd(1.0, 100.0, 20, 1, 5, 0, ctypes.byref(h))
    if ob.device_count() == 0:
        assert rc == ob._capi.OB_NO_DEVICE
    else:
        assert rc == ob._capi.OB_OK
        lib.ob_voxel_map_destroy(h)
    assert lib.ob_frames_to_map_rows(None, 0, None, 3, 0, None, None) == ob._capi.OB_INVALID_ARGUMENT


def test_new_struct_layouts_match_the_c_abi():
    ob = graft.load_package()
    capi = ob._capi
    for name, cls in {"ob_map_rows": capi.MapRows, "ob_map_field": capi.MapField,
                      "ob_map_rows_item": capi.MapRowsItem}.items():
        assert capi.lib.ob_abi_sizeof(name.encode()) == ctypes.sizeof(cls), name


def test_cpp_constructors_follow_the_reference(tmp_path):
    """voxel_hashmap_test.cpp:178-184 against the C++ drop-in header: VoxelHashMap3d refuses attributes with the
    reference's text; VoxelHashMapXd accepts them (it gets as far as the device)."""
    graft.build()
    src = tmp_path / "ctor.cpp"
    src.write_text(r'''
#include <cstdio>
#include <stdexcept>
#include <string>
#include "ouster/core/voxel_hash_map.h"
using namespace ouster::sdk::core;
int main() {
    try {
        VoxelHashMap3d m(1.0, 100.0, 20, 1, 5);
        return 1;
    } catch (const std::invalid_argument& e) {
        if (std::string(e.what()) != "num_attributes must be 0 for a fixed-size PointType") return 2;
    }
    try {
        VoxelHashMapXd m(1.0, 100.0, 20, 1, 5);
        if (m.point_cols() != 8) return 3;
    } catch (const std::invalid_argument&) {
        return 4;
    } catch (const std::exception& e) {
        std::printf("%s\n", e.what());   // no device here
    }
    std::printf("CTOR OK\n");
    return 0;
}
''')
    lib_dir = os.path.join(ROOT, "ouster-sdk_b200", "lib")
    exe = tmp_path / "ctor"
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), str(src),
                           "-L", lib_dir, "-louster_b200", f"-Wl,-rpath,{lib_dir}", "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "CTOR OK" in out.stdout, (out.returncode, out.stdout, out.stderr)


def test_map_rows_field_types_are_stated_for_signed_device_storage():
    """Device scans keep uint16 / uint32 / uint64 fields in signed tensors of the same width, so map_rows takes the
    type from the caller for those tensors and refuses to guess; numpy arrays carry their own type."""
    import torch
    core = graft.load_package().core
    assert core._field_tag(np.zeros((2, 2), np.uint16), None) == 2
    assert core._field_tag(np.zeros((2, 2), np.float16), None) == 12
    assert core._field_tag(torch.zeros((2, 2), dtype=torch.int16), np.uint16) == 2
    assert core._field_tag(torch.zeros((2, 2), dtype=torch.int32), "uint32") == 3
    assert core._field_tag(torch.zeros((2, 2), dtype=torch.int32), 7) == 7
    assert core._field_tag(torch.zeros((2, 2), dtype=torch.float32), None) == 9
    for t in (torch.int16, torch.int32, torch.int64):
        with pytest.raises(ValueError, match="must state its type"):
            core._field_tag(torch.zeros((2, 2), dtype=t), None)
    with pytest.raises(ValueError, match="width of its elements"):
        core._field_tag(torch.zeros((2, 2), dtype=torch.int16), np.uint32)
    with pytest.raises(ValueError, match="at least one item"):
        core.map_rows([None])
