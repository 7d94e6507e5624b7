"""Every kernel launch is counted in exactly one family: one call of each C-ABI entry point grows the total by the
launches that call always made, grows only the family of the kernels it runs ("decode" together with its
sub-family "decode_pipe"), and the families' growth, "decode_pipe" left out, adds up to the total's."""
import numpy as np
import pytest

import __graft_entry__ as graft
from tests.helpers import random_lut, random_range

pytestmark = pytest.mark.gpu

FAMILIES = ("decode_pipe", "decode", "cloud", "normals", "voxel", "voxel_map", "icp", "align", "zone", "image",
            "frame_ops", "pose", "dewarp", "destagger", "lut", "encode")
H, W = 32, 512
ICP_ITERS = 5
ALIGN_ITERS = 10   # kMaxIterations of ob_align.cu: the cloud alignment launches every iteration


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


def _counts(ob):
    return ob.kernel_launch_count(), {f: ob.kernel_launch_count(f) for f in FAMILIES}


# ---- one call of each entry point: name -> (family, launches, setup(ob) -> the call) ----------------------------
def _cloud_inputs(ob, poses=False):
    d, o = random_lut(H * W, 1, np.float32)
    lut = ob.XYZLutT.from_arrays(d, o, H, W)
    rng = random_range(H, W, 2)[None, None]
    shifts = np.arange(H, dtype=np.int32) % 7
    xyz, rd = np.empty((1, 1, H * W, 3), np.float32), np.empty((1, 1, H, W), np.uint32)
    kw = {"poses": np.tile(np.eye(4, dtype=np.float32), (1, W, 1, 1))} if poses else {}
    return lambda: ob.scan_to_cloud(lut, shifts, rng, xyz=xyz, range_destaggered=rd, **kw)


def _cartesian(ob):
    d, o = random_lut(H * W, 1, np.float64)
    lut, rng = ob.XYZLutT.from_arrays(d, o, H, W), random_range(H, W, 3)
    return lambda: ob.cartesian(lut, rng)


def _dewarp(ob):
    pts = np.random.default_rng(4).normal(size=(H, W, 3))
    poses = np.tile(np.eye(4), (W, 1, 1))
    return lambda: ob.dewarp(pts, poses)


def _dewarp_frame_args(ob, seed):
    d, o = random_lut(H * W, seed, np.float64)
    return {"lut": ob.XYZLutT.from_arrays(d, o, H, W), "range": random_range(H, W, seed, max_range=60000),
            "poses": np.tile(np.eye(4), (W, 1, 1)), "status": np.ones(W, np.uint32)}


def _dewarp_frame(ob):
    a = _dewarp_frame_args(ob, 5)
    return lambda: ob.dewarp_frame(a["lut"], a["range"], a["poses"], a["status"], None, 0.5, 50.0)


def _dewarp_frames(ob):
    frames = [_dewarp_frame_args(ob, 6), None, _dewarp_frame_args(ob, 7)]
    return lambda: ob.dewarp_frames(frames, 0.5, 50.0)


def _destagger(ob):
    img = random_range(H, W, 8)
    shifts = np.arange(H, dtype=np.int32) % 5
    return lambda: ob.destagger(img, shifts)


def _lut(dtype):
    def setup(ob):
        az = np.linspace(-3.0, 3.0, H)
        alt = np.linspace(-20.0, 20.0, H)
        return lambda: ob.XYZLutT.from_intrinsics(W, H, 0.001, np.eye(4), np.eye(4), az, alt, dtype=dtype)
    return setup


def _decode(case):
    def setup(ob):
        from tests.test_gpu_decode_entry_points import _case, _outputs, _run
        from tests.helpers import decoder_desc_from_oracle
        pf, refs, packets, shifts, _ = _case(case)
        dec = ob.Decoder(*decoder_desc_from_oracle(pf, refs[0]))
        d, o = random_lut(dec.h_px * dec.w_px, 3, np.float32)
        lut = ob.XYZLutT.from_arrays(d, o, dec.h_px, dec.w_px)
        n_ret = sum(1 for f in dec.fields if f.get("range_return", -1) >= 0)
        out = _outputs(dec, len(refs), np.float32, n_ret, n_ret, False)
        return lambda: _run(ob, "decode", dec, packets, out, lut=lut, shifts=shifts)
    return setup


def _encode(ob):
    si = ob.SensorInfo("RNG19_RFL8_SIG16_NIR16_DUAL", 16, 256, fw_rev="v3.2.1")
    scan = ob.LidarScan(si)
    scan.measurement_id[:] = np.arange(256)
    scan.status[:] = 1
    return lambda: ob.frame_to_packets(scan, si, device=True)


def _normals(ob):
    d, o = random_lut(H * W, 9, np.float64)
    rng = random_range(H, W, 9, p_zero=0.1, max_range=50000)
    xyz = ob.cartesian(ob.XYZLutT.from_arrays(d, o, H, W), rng).reshape(H, W, 3)
    return lambda: ob.normals(xyz, rng, sensor_origins_xyz=np.zeros((W, 3)))


def _cloud(seed, n=3000):
    return np.random.default_rng(seed).normal(0, 5.0, (n, 3))


def _voxel_downsample(ob):
    pts = _cloud(10)
    return lambda: ob.voxel_downsample(pts, 0.5)


def _voxel_map(ob):
    m = ob.VoxelMap(0.5, 100.0, 3)
    m.add_points(_cloud(11))
    return m


def _map_add_points(ob):
    m, pts = _voxel_map(ob), _cloud(12)
    return lambda: m.add_points(pts)


def _map_add_rows(ob):
    m = ob.VoxelMap(0.5, 100.0, 3, num_attributes=1)
    m.add_rows(np.hstack([_cloud(13), np.ones((3000, 1))]))
    rows = np.hstack([_cloud(14), np.ones((3000, 1))])
    return lambda: m.add_rows(rows)


def _map_remove_far(ob):
    m = _voxel_map(ob)
    return lambda: m.remove_far(np.array([95.0, 0.0, 0.0]))


def _map_point_cloud(ob):
    m = _voxel_map(ob)
    return lambda: m.point_cloud()


def _map_closest(ob):
    m, q = _voxel_map(ob), _cloud(15, 500)
    return lambda: m.closest_neighbors(q)


def _icp_align(ob):
    m, src = _voxel_map(ob), _cloud(11)[:1000] + 0.01
    return lambda: ob.icp_align(m, src, 1.0, 0.5, max_num_iterations=ICP_ITERS, convergence_criterion=0.0)


def _icp_linear_system(ob):
    src = _cloud(16, 1000)
    return lambda: ob.icp_linear_system(src, src + 0.01, 1.0)


def _cloud_align(ob):
    tgt = _cloud(17)
    return lambda: ob.cloud_align(tgt + 0.01, tgt, max_corr_dist=0.5)


def _cloud_nearest(ob):
    tgt, q = _cloud(18), _cloud(19, 500)
    return lambda: ob.cloud_nearest(tgt, q, 0.5, 0.25)


def _zone_lut():
    rs = np.random.default_rng(20)
    d = np.column_stack([np.ones(H * W), rs.uniform(-0.5, 0.5, H * W), rs.uniform(-0.5, 0.5, H * W)])
    return d, np.zeros((H * W, 3))


def _zone_render(ob):
    tris = np.array([[5, -10, -10, 5, 10, -10, 5, 0, 10]], np.float32)
    lut = _zone_lut()
    return lambda: ob.zone_render([{"triangles": tris, "coordinate_frame": 2}], H, W, lut)


def _zone_live():
    near = np.full((H, W), 1000, np.uint32)
    return [{"id": 1, "mode": 1, "point_count": 1, "frame_count": 1, "near_mm": near, "far_mm": near * 4}]


def _zone_monitor_create(ob):
    return lambda: ob.ZoneMonitor(_zone_live(), H, W)


def _zone_monitor_update(ob):
    zm, rng = ob.ZoneMonitor(_zone_live(), H, W), random_range(H, W, 21, max_range=5000)
    return lambda: zm.update(rng)


def _image(kind, shape):
    def setup(ob):
        p = ob.ImageProcessor(kind)
        img = np.random.default_rng(22).uniform(1, 5, shape).astype(np.float32)
        return lambda: p.update(img)
    return setup


def _frame(ob):
    si = ob.SensorInfo("RNG19_RFL8_SIG16_NIR16", H, W, 16)
    fr = ob.LidarScan(si)
    fr.field("RANGE")[...] = random_range(H, W, 23)
    return fr


def _frame_mask(ob):
    fr = _frame(ob)
    return lambda: ob.frame_ops.clip(fr, ["RANGE"], 100, 30000)


def _frame_rows(ob):
    fr = _frame(ob)
    return lambda: ob.frame_ops.reduce_by_factor(fr, 2)


def _interp_pose(ob):
    rs = np.random.default_rng(24)
    knots = np.array([0.0, 1.0, 2.0])
    poses = np.tile(np.eye(4), (3, 1, 1))
    poses[:, :3, 3] = rs.normal(size=(3, 3))
    x = np.sort(rs.uniform(0, 2, 2048))
    return lambda: ob.core.interp_pose(x, knots, poses)


def _frames_interp_pose(ob):
    ts = (10**18 + np.arange(W, dtype=np.uint64) * np.uint64(48828)).astype(np.uint64)
    frames = [(ts, np.ones(W, np.uint32), np.zeros((W, 4, 4)))]
    x0, x1 = np.eye(4), np.eye(4)
    x1[0, 3] = 1.0
    return lambda: ob.core.frames_interp_pose(frames, 1e9 - 0.1, x0, 1e9, x1)


def _map_rows(ob):
    d, o = random_lut(H * W, 25, np.float64)
    item = {"lut": ob.XYZLutT.from_arrays(d, o, H, W), "range": random_range(H, W, 25),
            "poses": np.tile(np.eye(4), (W, 1, 1)), "fields": [np.ones((H, W), np.uint16)]}
    return lambda: ob.map_rows([item])


CALLS = {
    "scan_to_cloud": ("cloud", 1, _cloud_inputs),
    "scan_to_cloud_poses": ("cloud", 2, lambda ob: _cloud_inputs(ob, poses=True)),
    "cartesian": ("cloud", 1, _cartesian),
    "dewarp": ("dewarp", 1, _dewarp),
    "dewarp_frame": ("dewarp", 1, _dewarp_frame),
    "dewarp_frames": ("dewarp", 1, _dewarp_frames),
    "destagger": ("destagger", 1, _destagger),
    "lut_from_intrinsics_f64": ("lut", 1, _lut(np.float64)),
    "lut_from_intrinsics_f32": ("lut", 3, _lut(np.float32)),
    "decode_pipelined": ("decode_pipe", 1, _decode("dual_128x1024")),
    "decode_kernel": ("decode", 1, _decode("unaligned_8x64")),
    "encode": ("encode", 1, _encode),
    "normals": ("normals", 2, _normals),
    "voxel_downsample": ("voxel", 8, _voxel_downsample),
    "voxel_map_add_points": ("voxel_map", 5, _map_add_points),
    "voxel_map_add_rows": ("voxel_map", 5, _map_add_rows),
    "voxel_map_remove_far": ("voxel_map", 1, _map_remove_far),
    "voxel_map_point_cloud": ("voxel_map", 3, _map_point_cloud),
    "voxel_map_closest_neighbors": ("voxel_map", 1, _map_closest),
    "icp_align": ("icp", 2 + 4 * ICP_ITERS, _icp_align),
    "icp_linear_system": ("icp", 2, _icp_linear_system),
    "cloud_align": ("align", 3 + 2 + 6 * ALIGN_ITERS, _cloud_align),
    "cloud_nearest": ("align", 4, _cloud_nearest),
    "zone_render": ("zone", 1, _zone_render),
    "zone_monitor_create": ("zone", 2, _zone_monitor_create),
    "zone_monitor_update": ("zone", 2, _zone_monitor_update),
    "auto_exposure": ("image", 2, _image("auto_exposure", (H, W))),
    "beam_uniformity": ("image", 4, _image("beam_uniformity", (H, W))),
    "local_tone_map": ("image", 4, _image("local_tone_map", (H, W, 3))),
    "frame_mask": ("frame_ops", 1, _frame_mask),
    "frame_select_rows": ("frame_ops", 1, _frame_rows),
    "interp_pose": ("pose", 3, _interp_pose),
    "frames_interp_pose": ("pose", 2, _frames_interp_pose),
    "map_rows": ("voxel_map", 1, _map_rows),
}


@pytest.mark.parametrize("name", list(CALLS))
def test_one_call_grows_its_family_by_its_launches(ob, name):
    import torch
    family, launches, setup = CALLS[name]
    call = setup(ob)
    torch.cuda.synchronize()
    total0, fam0 = _counts(ob)
    call()
    torch.cuda.synchronize()
    total1, fam1 = _counts(ob)
    grew = {f: fam1[f] - fam0[f] for f in FAMILIES if fam1[f] != fam0[f]}
    assert total1 - total0 == launches, (name, total1 - total0, grew)
    want = {"decode_pipe", "decode"} if family == "decode_pipe" else {family}
    assert set(grew) == want, (name, total1 - total0, grew)
    assert sum(v for f, v in grew.items() if f != "decode_pipe") == total1 - total0, (name, grew)
    if family == "decode_pipe":
        assert grew["decode_pipe"] == grew["decode"]
