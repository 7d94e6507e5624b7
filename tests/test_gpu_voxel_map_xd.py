"""GPU tests of the voxel map with per-point attributes (VoxelHashMapXd, ob_voxel_map.cu) and of the frame -> map-row
ingest (ob_map_rows.cu, DESIGN f-11) against their plain-Python statement (tests/voxel_map_xd_reference.py) and the
oracle: the map, extracts and neighbours bit for bit including order and attributes, ICP on an attribute map
bit-identical to ICP on the 3-d map with the same x, y, z, the ingest bit-exact, and the device chain."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import icp as oi
from oracle import voxel as orv
from tests import voxel_map_xd_reference as xr
from tests.test_oracle_normals import room_scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


def rot(axis_angle):
    from scipy.spatial.transform import Rotation
    return Rotation.from_rotvec(axis_angle).as_matrix()


def same_map(gm, xm):
    assert gm.size() == xm.size()
    assert np.array_equal(gm.point_cloud(), xm.point_cloud(), equal_nan=True)


@pytest.mark.parametrize("max_pts", [1, 20])
@pytest.mark.parametrize("na", [0, 1, 3, 5])
def test_map_add_remove_extract_bit_exact_over_many_cycles(ob, na, max_pts):
    rs = np.random.default_rng(10 * na + max_pts)
    vs, md = 0.5, 6.0
    gm = ob.VoxelMap(vs, md, max_pts, num_attributes=na)
    xm = xr.VoxelHashMapXd(vs, md, max_pts, num_attributes=na)
    assert gm.cols == 3 + na
    for cycle in range(40):
        centre = np.array([np.cos(cycle / 9.0), np.sin(cycle / 7.0), 0.1 * cycle]) * 8.0
        n = 6000 if cycle == 7 else int(rs.integers(0, 1500))      # cycle 7 grows the table
        pts = centre + rs.normal(0, 3.0 if cycle != 7 else 30.0, (n, 3))
        if cycle % 10 == 3:                                          # one dense voxel
            pts[: n // 2] = centre + rs.random((n // 2, 3)) * 0.49
        if cycle % 17 == 5 and n > 4:                                # rows in the INT32_MIN voxel
            pts[0, 0], pts[1, 1], pts[2] = np.nan, 1e300, [-1e300, np.nan, 1e300]
        rows = np.hstack([pts, rs.normal(0, 100.0, (n, na))])
        if cycle % 4 == 1 and n > 10:                                # duplicates with other attributes
            rows[n // 2:n // 2 + 5, :3] = rows[:5, :3]
        if na == 0 and cycle % 2:
            gm.add_rows(rows)                                        # the rows call works for the 3-d map too
        else:
            gm.add_points(rows)
        xm.add_points(rows)
        if cycle % 3 == 0:
            origin = np.concatenate([centre, np.full(na, 7.0)])
            assert np.array_equal(gm.remove_far(origin, extract=True), xm.extract_voxels_far_from_location(centre),
                                  equal_nan=True), cycle
        elif cycle % 3 == 1:
            gm.remove_far(centre)
            xm.remove_voxels_far_from_location(centre)
        same_map(gm, xm)
    q = centre + rs.normal(0, 3.0, (500, 3))
    for bound in (xr.DBL_MAX, 0.1):
        nb, d2 = gm.closest_neighbors(q, bound)
        wnb, wd2 = xm.get_closest_neighbors(q, bound)
        assert nb.shape == (500, 3 + na)
        assert np.array_equal(nb, wnb) and np.array_equal(d2, wd2), bound
    gm.clear()
    xm.clear()
    same_map(gm, xm)


def test_row_width_and_rows_refused(ob):
    gm = ob.VoxelMap(0.5, 10.0, 20, num_attributes=2)
    with pytest.raises(ValueError, match="VoxelHashMap::add_points received unexpected point dimension"):
        gm.add_rows(np.zeros((4, 4)))
    r, keep = ob.core._point_rows(np.zeros((4, 3)))
    with pytest.raises(ValueError, match="VoxelHashMap::add_points received unexpected point dimension"):
        ob._capi.check(ob._capi.lib.ob_voxel_map_add_points(gm._h, C.byref(r), ob.core._stream(None).h))
    cols = C.c_size_t(0)
    ob._capi.check(ob._capi.lib.ob_voxel_map_cols(gm._h, C.byref(cols)))
    assert cols.value == 5
    assert gm.size() == (0, 0)


def test_closest_neighbors_return_attributes_with_and_without_bound(ob):
    _, rng, d = room_scene(64, 1024)
    pts = (d * rng[..., None] * 0.001).reshape(-1, 3)
    rs = np.random.default_rng(5)
    rows = np.hstack([pts, rs.normal(0, 1.0, (len(pts), 3))])
    gm, xm = ob.VoxelMap(0.5, 100.0, 20, num_attributes=3), xr.VoxelHashMapXd(0.5, 100.0, 20, num_attributes=3)
    gm.add_points(rows)
    xm.add_points(rows)
    q = pts[rs.integers(0, len(pts), 2000)] + rs.normal(0, 0.4, (2000, 3))
    for bound in (xr.DBL_MAX, 0.25, 1e-4):
        nb, d2 = gm.closest_neighbors(q, bound)
        wnb, wd2 = xm.get_closest_neighbors(q, bound)
        assert np.array_equal(nb, wnb) and np.array_equal(d2, wd2), bound
    assert np.any(np.all(nb == 0, axis=1))        # the tight bound leaves some queries with zeros


def _scene_cloud(h=128, w=2048, seed=0):
    rs = np.random.default_rng(seed)
    _, rng, d = room_scene(h, w)
    rng = (rng.astype(np.int64) + rs.integers(-40, 41, rng.shape)).astype(np.float64)
    return (d * rng[..., None] * 0.001).reshape(-1, 3)


@pytest.mark.parametrize("iters", [1, 50])
def test_icp_on_attribute_map_is_the_3d_result(ob, iters):
    cloud = _scene_cloud()
    f1, _ = orv.voxel_downsample(cloud, 0.5)
    src, _ = orv.voxel_downsample(f1, 1.5)
    truth = np.eye(4)
    truth[:3, :3] = rot(np.radians([0.4, -0.7, 1.2]))
    truth[:3, 3] = [0.03, -0.02, 0.015]
    moved = (np.linalg.inv(truth)[:3, :3] @ src.T).T + np.linalg.inv(truth)[:3, 3]
    attrs = np.random.default_rng(2).normal(0, 1.0, (len(f1), 4))
    gx, g3, om = ob.VoxelMap(0.5, 100.0, 20, num_attributes=4), ob.VoxelMap(0.5, 100.0, 20), oi.VoxelHashMap3d(0.5)
    gx.add_points(np.hstack([f1, attrs]))
    g3.add_points(f1)
    om.add_points(f1)
    px, itx = ob.icp_align(gx, moved, 1.0, 0.3, iters)
    p3, it3 = ob.icp_align(g3, moved, 1.0, 0.3, iters)
    wp, wit = oi.align_points_to_map(moved, om, 1.0, 0.3, iters)
    assert itx == it3 and np.array_equal(px, p3)
    assert itx == wit and np.abs(px - wp).max() <= 1e-12
    # the Python front end takes either map
    api = ob.pyapi
    m = api.VoxelHashMapXd(voxel_size=0.5, max_distance=10.0, num_attributes=1)
    map_points = np.array([[0.0, 0.0, 0.0, 10.0], [1.0, 0.0, 0.0, 20.0], [0.0, 1.0, 0.0, 30.0], [0.0, 0.0, 1.0, 40.0]])
    m.add_points(map_points)
    shifted = map_points[:, :3] + np.array([0.05, 0.02, -0.01])
    t = api.ICPRegistration(max_num_iterations=20).align_points_to_map(shifted, m, max_distance=0.5, kernel_scale=0.1)
    assert t.shape == (4, 4)
    np.testing.assert_allclose((t[:3, :3] @ shifted.T).T + t[:3, 3], map_points[:, :3], atol=0.05)


def test_python_api_names_defaults_and_errors(ob):
    api = ob.pyapi
    m = api.VoxelHashMapXd()
    assert m.empty and m.max_points_per_voxel() == 20 and m.min_pts_threshold() == 1
    with pytest.raises(ValueError, match=r"add_points expects at least Nx\(3\+num_attributes\) columns"):
        m.add_points(np.zeros((4, 2)))
    with pytest.raises(ValueError, match="VoxelHashMap::add_points received unexpected point dimension"):
        m.add_points(np.zeros((4, 4)))
    with pytest.raises(ValueError, match=r"VoxelHashMap method expects a \(3\+attributes\)-element point"):
        m.get_closest_neighbor(np.zeros(2))
    m = api.VoxelHashMapXd(voxel_size=0.5, max_distance=10.0, num_attributes=2)
    pts = np.array([[0.0, 0, 0, 1, 2], [1, 0, 0, 3, 4], [0, 1, 0, 5, 6], [0, 0, 1, 7, 8]])
    m.add_points(pts)
    nb, d2 = m.get_closest_neighbor(np.array([0.9, 0.0, 0.0, 99.0, 99.0]))
    assert nb.shape == (5,) and np.array_equal(nb, [1, 0, 0, 3, 4]) and d2 == pytest.approx(0.01)
    nb, d2 = m.get_closest_neighbor(np.array([9.0, 9.0, 9.0]), 1.0)
    assert np.array_equal(nb, np.zeros(5)) and d2 == 1.0
    assert np.array_equal(m.point_cloud(), pts)
    ext = m.extract_voxels_far_from_location(np.array([100.0, 0, 0]))
    assert np.array_equal(ext, pts) and m.empty


def _lut_and_frames(h, w, n_returns, seed):
    rs = np.random.default_rng(seed)
    _, rng, d = room_scene(h, w)
    off = rs.normal(0, 0.01, (h * w, 3))
    lut_d = np.ascontiguousarray(d.reshape(-1, 3)) * 0.001     # range in mm, XYZ in metres
    step = np.eye(4)
    step[:3, :3] = rot(np.radians([0.1, -0.2, 0.8]))
    step[:3, 3] = [0.04, 0.01, 0.002]
    poses = np.stack([np.linalg.matrix_power(step, 1 + c % 7) for c in range(w)])
    poses[:, :3, 3] += rs.normal(0, 0.01, (w, 3))
    items = []
    for r in range(n_returns):
        rg = (rng.astype(np.int64) + rs.integers(-30, 31, rng.shape)).astype(np.uint32)
        rg[rs.random(rng.shape) < 0.15] = 0
        fields = [rs.integers(0, 65535, (h, w)).astype(np.uint16),
                  rs.integers(0, 1 << 32, (h, w), dtype=np.uint64).astype(np.uint32),
                  rs.normal(0, 100.0, (h, w)).astype(np.float32),
                  rs.normal(0, 1.0, (h, w, 3)).astype(np.float16),
                  rs.normal(0, 1.0, (h, w, 3)),
                  rs.integers(-128, 127, (h, w)).astype(np.int8)]
        items.append({"range": rg, "poses": poses, "fields": fields, "direction": lut_d, "offset": off})
    return lut_d, off, items


@pytest.mark.parametrize("n_returns,h,w,repeat", [
    pytest.param(1, 64, 1024, 1, id="1"), pytest.param(2, 64, 1024, 1, id="2"),
    # 12 items of 256 CTAs: a look-back chain of 3072 CTAs, more than an H100 holds at once
    pytest.param(2, 128, 2048, 6, id="2-x6-128x2048")])
@pytest.mark.parametrize("fields", [slice(0, 0), slice(0, 1), slice(3, 4), slice(0, 6)])
def test_map_rows_bit_exact_against_the_exporter_step(ob, n_returns, h, w, repeat, fields):
    lut_d, off, items = _lut_and_frames(h, w, n_returns, 7 + n_returns)
    lut = ob.XYZLutT.from_arrays(lut_d, off, h, w)
    items = [dict(it, range=np.roll(it["range"], 37 * k, axis=1)) for k in range(repeat) for it in items]
    its = [dict(it, fields=it["fields"][fields]) for it in items]
    want = xr.map_rows(its)
    got = ob.map_rows([dict(it, lut=lut) for it in its])
    assert got.shape == want.shape and got.dtype == np.float64
    assert np.array_equal(got, want, equal_nan=True)
    # the XYZ is the K1-with-poses result: cartesian then dewarp
    xyz = ob.dewarp(ob.cartesian(lut, its[0]["range"]).reshape(h, w, 3), its[0]["poses"])
    assert np.array_equal(got[: int(np.count_nonzero(its[0]["range"])), :3], xyz[its[0]["range"] > 0])


_SIGNED = {np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}


def _as_device_scan_stores(f, dev):
    """A field on the device the way DeviceLidarScan keeps it: unsigned 16/32/64-bit pixels in the signed torch type
    of the same width (same bits), with the reference type stated beside it."""
    import torch
    if f.dtype in _SIGNED:
        return torch.from_numpy(f.view(_SIGNED[f.dtype])).to(dev), f.dtype
    return torch.from_numpy(f).to(dev)


def test_map_rows_capacity_cut_and_device_count(ob):
    """Every field type on the device, unsigned fields in signed tensors as device scans hold them, with uint16 values
    >= 32768 and uint32 values >= 2^31: the rows equal the exporter's step bit for bit, including the capacity cut."""
    import torch
    h, w = 64, 1024
    lut_d, off, items = _lut_and_frames(h, w, 2, 3)
    for it in items:                                   # uint16, uint32, float32, float16 x 3, float64 x 3, int8
        assert it["fields"][0].max() >= 1 << 15 and it["fields"][1].max() >= 1 << 31
    lut = ob.XYZLutT.from_arrays(lut_d, off, h, w)
    want = xr.map_rows(items)
    assert want[:, 3].max() >= 1 << 15 and want[:, 4].max() >= 1 << 31
    host = [dict(it, lut=lut) for it in items]
    with pytest.raises(ValueError, match="output capacity too small"):
        ob.map_rows(host, capacity=len(want) - 1)
    dev = torch.device("cuda", 0)
    ditems = [{"lut": lut, "range": torch.from_numpy(it["range"].view(np.int32)).to(dev),
               "poses": torch.from_numpy(it["poses"]).to(dev),
               "fields": [_as_device_scan_stores(f, dev) for f in it["fields"]]} for it in items]
    for cap in (len(want), len(want) - 1000, 10):
        rows, n = ob.map_rows(ditems, capacity=cap)
        torch.cuda.synchronize()
        assert int(n.item()) == len(want) and rows.shape == (cap, want.shape[1])
        assert np.array_equal(rows.cpu().numpy(), want[:cap], equal_nan=True)
    # a signed 16/32/64-bit tensor without its type is refused rather than read as signed; a stated type must fit
    bare = [dict(it, fields=list(it["fields"])) for it in ditems]
    bare[0]["fields"][0] = bare[0]["fields"][0][0]
    with pytest.raises(ValueError, match="must state its type"):
        ob.map_rows(bare)
    bad = [dict(it, fields=list(it["fields"])) for it in ditems]
    bad[0]["fields"][0] = (bad[0]["fields"][0][0], np.uint32)
    with pytest.raises(ValueError, match="width of its elements"):
        ob.map_rows(bad)
    with pytest.raises(ValueError, match="at least one item"):
        ob.map_rows([None, None])


def test_device_chain_matches_the_host_path_and_replays_in_a_graph(ob):
    """DeviceScanBatcher (packets decoded on the device) -> map_rows on both returns with NEAR_IR (uint16, kept in an
    int16 tensor; values >= 32768 set here) and REFLECTIVITY -> add_points (device count) -> align on the map ->
    extract, over 3 poses of the recorded frame, against the host path on the oracle's decode of the same packets
    (the exporter's step, then the same map calls with host counts); then align on the built map inside a CUDA
    graph."""
    import torch
    from oracle import oracle as orc
    from tests.helpers import load_fixture, oracle_pf
    api = ob.pyapi
    dev = torch.device("cuda", 0)
    meta, packets = load_fixture("OS-1-128_767798045_1024x10_20230712_120049")
    info = api.SensorInfo.from_meta(meta)
    h, w = info.h, info.w
    lut = api.XYZLut(info)
    batcher = api.DeviceScanBatcher(info)
    scan = batcher.new_scan()
    if not [batcher(p, 77, scan) for p in packets][-1]:   # the fixture ends inside the frame
        batcher.flush(scan)
    pf = oracle_pf(meta)
    oframe = orc.Frame(pf)
    obat = orc.Batcher(pf, init_id=meta["init_id"], column_window=meta["column_window"])
    for p in packets:
        obat.batch(p, 77, oframe)
    nir = oframe.field("NEAR_IR") | np.uint16(0x8000)          # saturated ambient: the sign bit of an int16
    scan.field("NEAR_IR").bitwise_or_(torch.tensor(-0x8000, dtype=torch.int16, device=dev))
    assert scan.field("NEAR_IR").dtype == torch.int16 and scan.field_dtype("NEAR_IR") == np.uint16
    assert np.array_equal(scan.field("NEAR_IR").cpu().numpy().view(np.uint16), nir)
    d, o = lut._lut.direction, lut._lut.offset
    vs, md = 0.5, 30.0
    gm = ob.VoxelMap(vs, md, 20, num_attributes=2)
    hm = ob.VoxelMap(vs, md, 20, num_attributes=2)
    st = ob.Stream(0, cuda_stream=torch.cuda.current_stream(dev).cuda_stream)
    step = np.eye(4)
    step[:3, :3] = rot(np.radians([0.0, 0.0, 1.5]))
    step[:3, 3] = [0.2, 0.05, 0.0]
    for k in range(3):
        poses = np.repeat(np.linalg.matrix_power(step, k)[None], w, 0)
        poses[:, 0, 3] += np.linspace(0.0, 0.02, w)
        pt = torch.from_numpy(poses).to(dev)
        ditems, hitems = [], []
        for r, (rn, fl) in enumerate((("RANGE", "REFLECTIVITY"), ("RANGE2", "REFLECTIVITY2"))):
            ditems.append({"lut": lut, "range": scan.field(rn), "poses": pt,
                           "fields": [(scan.field("NEAR_IR"), scan.field_dtype("NEAR_IR")), scan.field(fl)]})
            hitems.append({"range": oframe.field(rn), "poses": poses, "direction": d, "offset": o,
                           "fields": [nir, oframe.field(fl)]})
        rows, n = ob.map_rows(ditems, stream=st)
        pose, it_ = ob.icp_align(gm, rows[:, :3].contiguous(), 3.0, 1.0, 20, n=n, stream=st)
        gm.add_points(rows, n=n, stream=st)
        ext = gm.remove_far(pose[:3, 3].contiguous(), extract=True, stream=st)
        # host path: the exporter's step on the oracle's decode, then the same map calls with host counts
        hrows = xr.map_rows(hitems)
        assert hrows[:, 3].max() >= 1 << 15
        assert int(n.item()) == len(hrows)
        assert np.array_equal(rows[: len(hrows)].cpu().numpy(), hrows)
        assert np.array_equal(ob.map_rows([dict(x, lut=lut) for x in hitems]), hrows)
        hp, hit = ob.icp_align(hm, np.ascontiguousarray(hrows[:, :3]), 3.0, 1.0, 20)
        hm.add_points(hrows)
        hext = hm.remove_far(hp[:3, 3], extract=True)
        assert np.array_equal(pose.cpu().numpy(), hp) and int(it_.item()) == hit
        assert np.array_equal(ext, hext)
    assert gm.size() == hm.size()
    assert np.array_equal(gm.point_cloud(), hm.point_cloud())
    src = torch.from_numpy(np.ascontiguousarray(hrows[::7, :3])).to(dev)
    ref_pose, ref_it = ob.icp_align(gm, src, 3.0, 1.0, 50)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    cs = torch.cuda.Stream()
    st_cs = ob.Stream(0, cuda_stream=cs.cuda_stream)
    with torch.cuda.stream(cs):
        ob.icp_align(gm, src, 3.0, 1.0, 50, stream=st_cs)
        cs.synchronize()
        with torch.cuda.graph(g, stream=cs, capture_error_mode="thread_local"):
            gp, git = ob.icp_align(gm, src, 3.0, 1.0, 50, stream=st_cs)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(gp, ref_pose) and torch.equal(git, ref_it)
    assert ob.kernel_launch_count("voxel_map") > 0


def test_dropin_example_runs_on_gpu(tmp_path):
    """tests/cpp/voxel_map_xd_dropin_example.cpp built with plain g++ against the drop-in headers."""
    graft.build()
    root = graft.ROOT
    lib_dir = os.path.join(root, "ouster-sdk_b200", "lib")
    exe = os.path.join(str(tmp_path), "xd_example")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(root, "include"),
                           os.path.join(root, "tests", "cpp", "voxel_map_xd_dropin_example.cpp"), "-L", lib_dir,
                           "-louster_b200", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "XD DROPIN OK" in out.stdout
