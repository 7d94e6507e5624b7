#!/usr/bin/env python
"""Small end-to-end invocations of every kernel, checked against the oracle; meant to run under
    compute-sanitizer --tool memcheck|racecheck|synccheck python tools/sanitize_cases.py
(kept tiny: the sanitizer slows kernels down by orders of magnitude)."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft
from oracle import oracle as orc
from oracle import voxel as orv
from tests.helpers import (col_map_from_packets, decoder_desc_from_oracle, oracle_pf, random_frame,
                           random_lut, random_range)

ob = graft.load_package()
st = ob.Stream(0)
h, w = 16, 256
for dtype in (np.float32, np.float64):
    for R in (1, 2):
        for aligned in (True, False):
            rs = np.random.default_rng(3)
            rng = np.stack([np.stack([random_range(h, w, 10 * f + r) for r in range(R)]) for f in range(2)])
            d, o = random_lut(h * w, 1, dtype)
            sh = rs.integers(-20, 21, h).astype(np.int32)
            if aligned:
                sh = sh // 4 * 4
            lut = ob.XYZLutT.from_arrays(d, o, h, w)
            xyz = np.zeros((2, R, h * w, 3), dtype)
            rd = np.zeros((2, R, h, w), np.uint32)
            xd = np.zeros((2, R, h, w, 3), dtype)
            ob.scan_to_cloud(lut, sh, rng, xyz=xyz, range_destaggered=rd, xyz_destaggered=xd, stream=st)
            st.sync()
            for f in range(2):
                for r in range(R):
                    want = orc.cartesian(rng[f, r], d, o)
                    assert np.array_equal(xyz[f, r], want)
                    assert np.array_equal(rd[f, r], orc.destagger(rng[f, r], sh))
                    assert np.array_equal(xd[f, r], orc.destagger(want.reshape(h, w, 3), sh))
# K1 with fused per-column poses (streamed rows + resident pose planes) and K3 (count/scan/emit)
for dtype in (np.float32, np.float64):
    hh, ww = 40, 256
    rngp = np.stack([np.stack([random_range(hh, ww, 50 + 10 * f + r) for r in range(2)]) for f in range(2)])
    d, o = random_lut(hh * ww, 4, dtype)
    lut = ob.XYZLutT.from_arrays(d, o, hh, ww)
    poses = np.tile(np.eye(4, dtype=dtype), (ww, 1, 1))
    poses[:, :3, 3] = np.random.default_rng(2).random((ww, 3)).astype(dtype)
    poses[:, 0, 1] = 0.25
    sh = (np.arange(hh, dtype=np.int32) * 5) % 23
    xyz = np.zeros((2, 2, hh * ww, 3), dtype)
    xd = np.zeros((2, 2, hh, ww, 3), dtype)
    ob.scan_to_cloud(lut, sh, rngp, xyz=xyz, xyz_destaggered=xd, stream=st, poses=poses)
    st.sync()
    for f in range(2):
        for r in range(2):
            want = orc.dewarp(orc.cartesian(rngp[f, r], d, o).reshape(hh, ww, 3), poses)
            assert np.array_equal(xyz[f, r].reshape(hh, ww, 3), want)
            assert np.array_equal(xd[f, r], orc.destagger(want, sh))
    status = np.ones(ww, np.uint32)
    status[:5] = 0
    status[100] = 0
    ts = np.arange(ww, dtype=np.uint64)
    got = ob.dewarp_frame(lut, rngp[0, 0], poses.astype(np.float64), status, ts, 1.0, 300.0, provenance=True)
    want = orc.dewarp_frame(rngp[0, 0], d, o, poses.astype(np.float64), status, ts, 1.0, 300.0)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
print("K1 ok (plain, posed), K3 ok")
img = np.random.default_rng(1).integers(0, 255, (h, w), dtype=np.uint8)
sh = np.arange(h, dtype=np.int32) - 5
assert np.array_equal(ob.destagger(img, sh), orc.destagger(img, sh))
img64 = np.random.default_rng(1).random((9, 35))
assert np.array_equal(ob.destagger(img64, np.arange(9, dtype=np.int32)), orc.destagger(img64, np.arange(9)))
print("destagger ok")
ident = np.eye(4)
l = ob.XYZLutT.from_intrinsics(64, 8, 0.001, ident, ident, np.linspace(-3, 3, 8), np.linspace(-10, 10, 8))
assert np.all(np.isfinite(l.direction))
print("lut ok")
for profile, hh, ww in (("RNG19_RFL8_SIG16_NIR16_DUAL", 16, 128), ("LEGACY", 16, 64), ("RNG19_RFL8_SIG16_NIR16_RGB16", 8, 64)):
    pf = oracle_pf(profile, hh, ww)
    src = random_frame(pf, seed=4)
    pk, ts = orc.frame_to_packets(src, pf)
    layout, fields = decoder_desc_from_oracle(pf, src)
    dec = ob.Decoder(layout, fields)
    d, o = random_lut(hh * ww, 2)
    lut = ob.XYZLutT.from_arrays(d, o, hh, ww)
    shifts = (np.arange(hh, dtype=np.int32) * 3) % 17
    for cmap in (None, "faulty"):
        pkk = pk.copy()
        col_src = None
        ref = src
        if cmap:
            pkk = np.delete(pkk, 1, axis=0)
            col_src = col_map_from_packets(pf, pkk)
            ref = orc.Frame(pf, with_window=True)
            b = orc.Batcher(pf)
            for p in pkk:
                b.batch(p, 5, ref)
            b.batch(orc.frame_to_packets(random_frame(pf, 9, frame_id=701), pf)[0][0], 5, ref)  # finalize
        outs = {f["name"]: np.zeros(ref.field(f["name"]).shape, ref.field(f["name"]).dtype) for f in fields}
        io = {"packets": np.ascontiguousarray(pkk), "n_slots": len(pkk), "packet_stride": pkk.shape[1],
              "col_src": col_src, "fields": outs, "timestamp": np.zeros(ww, np.uint64)}
        has_r = ref.has_field("RANGE")
        if has_r:
            io["xyz"] = [np.zeros((hh * ww, 3), np.float32)]
            io["range_destaggered"] = [np.zeros((hh, ww), np.uint32)]
        dec.decode([io], lut=lut if has_r else None, pixel_shift_by_row=shifts if has_r else None, stream=st)
        st.sync()
        for n, a in outs.items():
            assert np.array_equal(a, ref.field(n)), (profile, cmap, n)
        if has_r:
            assert np.array_equal(io["xyz"][0], orc.cartesian(ref.field("RANGE"), d, o))
            assert np.array_equal(io["range_destaggered"][0], orc.destagger(ref.field("RANGE"), shifts))
print("K2 ok")

# K2 through the runtime-plan phase A as well (the loop above took the compile-time layouts where
# one exists), then the pipelined host path: decode jobs, zero-copy bursts, frames in flight
ob.set_tunable("decode_runtime_plans", 1)
pf = oracle_pf("RNG19_RFL8_SIG16_NIR16_DUAL", 16, 128)
src = random_frame(pf, seed=6)
pk, ts = orc.frame_to_packets(src, pf)
layout, fields = decoder_desc_from_oracle(pf, src)
dec = ob.Decoder(layout, fields)
outs = {f["name"]: np.zeros(src.field(f["name"]).shape, src.field(f["name"]).dtype) for f in fields}
dec.decode([{"packets": np.ascontiguousarray(pk), "n_slots": len(pk), "packet_stride": pk.shape[1],
             "col_src": None, "fields": outs}], stream=st)
st.sync()
for n, a in outs.items():
    assert np.array_equal(a, src.field(n)), n
ob.set_tunable("decode_runtime_plans", 0)
print("K2 runtime plans ok")

si = ob.SensorInfo("RNG19_RFL8_SIG16_NIR16_DUAL", 16, 128, fw_rev="v3.2.1")
d, o = random_lut(16 * 128, 5)
lut = ob.XYZLutT.from_arrays(d, o, 16, 128)
shifts = (np.arange(16, dtype=np.int32) * 3) % 17
pipe = ob.FramePipeline(si, depth=2, lut=lut, pixel_shift_by_row=shifts)
buf = ob.pinned_empty(pk.shape, np.uint8)
want = []
got = []
for k in range(4):
    f = random_frame(pf, seed=30 + k, frame_id=900 + k)
    p, t = orc.frame_to_packets(f, pf)
    want.append(f)
    buf[...] = p
    used, slot = pipe.push_burst(buf, t)
    assert used == len(p)
    if slot is not None:
        got.append((slot.frame.field("RANGE").copy(), slot.xyz[0].copy(), slot.range_destaggered[1].copy()))
while (slot := pipe.drain()) is not None:
    got.append((slot.frame.field("RANGE").copy(), slot.xyz[0].copy(), slot.range_destaggered[1].copy()))
assert len(got) == 4
for f, (r, x, rd2) in zip(want, got):
    assert np.array_equal(r, f.field("RANGE"))
    assert np.array_equal(x, orc.cartesian(f.field("RANGE"), d, o))
    assert np.array_equal(rd2, orc.destagger(f.field("RANGE2"), shifts))
print("pipeline ok")
# ---- round 2 kernels: pipelined K2 with both LUT dtypes and the LUT-free mode, K4 encode, normals, batched K3 ----
from tests.helpers import default_os1_64
from tests.test_oracle_normals import room_scene
pf = oracle_pf("RNG19_RFL8_SIG16_NIR16_DUAL", 64, 128)
src = random_frame(pf, seed=8)
pk, ts = orc.frame_to_packets(src, pf)
layout, fields = decoder_desc_from_oracle(pf, src)
dec = ob.Decoder(layout, fields)
shifts = (np.arange(64, dtype=np.int32) * 3) % 17
n0 = ob.kernel_launch_count("decode_pipe")
for dt in (np.float32, np.float64):
    d, o = random_lut(64 * 128, 7, dt)
    lut = ob.XYZLutT.from_arrays(d, o, 64, 128)
    io = {"packets": np.ascontiguousarray(pk), "n_slots": len(pk), "packet_stride": pk.shape[1], "col_src": None,
          "fields": {f["name"]: np.zeros(src.field(f["name"]).shape, src.field(f["name"]).dtype) for f in fields},
          "xyz": [np.zeros((64 * 128, 3), dt) for _ in range(2)],
          "range_destaggered": [np.zeros((64, 128), np.uint32) for _ in range(2)]}
    dec.decode([io], lut=lut, pixel_shift_by_row=shifts, stream=st)
    st.sync()
    for n, a in io["fields"].items():
        assert np.array_equal(a, src.field(n)), n
    for r, nm in enumerate(("RANGE", "RANGE2")):
        assert np.array_equal(io["xyz"][r], orc.cartesian(src.field(nm), d, o))
        assert np.array_equal(io["range_destaggered"][r], orc.destagger(src.field(nm), shifts))
assert ob.kernel_launch_count("decode_pipe") == n0 + 2, "the pipelined K2 did not run"
si64 = default_os1_64(1024)
al = ob.XYZLutT.from_intrinsics(128, 64, 0.001, si64["beam_to_lidar_transform"], si64["lidar_to_sensor_transform"],
                                si64["beam_azimuth_angles"], si64["beam_altitude_angles"], dtype=np.float32).set_analytic(True)
io = {"packets": np.ascontiguousarray(pk), "n_slots": len(pk), "packet_stride": pk.shape[1], "col_src": None,
      "fields": {}, "xyz": [np.zeros((64 * 128, 3), np.float32) for _ in range(2)]}
dec.decode([io], lut=al, pixel_shift_by_row=shifts, stream=st)
rngs = np.stack([np.stack([src.field("RANGE"), src.field("RANGE2")])])
xa = np.zeros((1, 2, 64 * 128, 3), np.float32)
ob.scan_to_cloud(al, shifts, rngs, xyz=xa, stream=st)
st.sync()
assert np.allclose(xa[0, 0], io["xyz"][0], rtol=1e-5, atol=1e-4)
print("K2 pipelined (f32, f64, LUT-free) ok")
# the pipelined kernel's other launch shapes: 3 CTAs per SM (32-row sensor), phase-A helper warps, store-warp tensor
# copies for XYZ (batched launch), each against the oracle
pf32 = oracle_pf("RNG19_RFL8_SIG16_NIR16_DUAL", 32, 128)
src32 = random_frame(pf32, seed=9)
pk32, _ = orc.frame_to_packets(src32, pf32)
layout32, fields32 = decoder_desc_from_oracle(pf32, src32)
dec32 = ob.Decoder(layout32, fields32)
sh32 = (np.arange(32, dtype=np.int32) * 5) % 23
d32, o32 = random_lut(32 * 128, 11, np.float32)
lut32 = ob.XYZLutT.from_arrays(d32, o32, 32, 128)
for tun in ({"decode_pipe_ctas": 3}, {"decode_pipe_ctas": 1, "decode_pipe_helpers": 5}, {"decode_pipe_ctas": 1, "decode_pipe_tma_xyz": 1}):
    for k, v in tun.items():
        ob.set_tunable(k, v)
    n1 = ob.kernel_launch_count("decode_pipe")
    io = {"packets": np.ascontiguousarray(pk32), "n_slots": len(pk32), "packet_stride": pk32.shape[1], "col_src": None,
          "fields": {f["name"]: np.zeros(src32.field(f["name"]).shape, src32.field(f["name"]).dtype) for f in fields32},
          "xyz": [np.zeros((32 * 128, 3), np.float32) for _ in range(2)],
          "range_destaggered": [np.zeros((32, 128), np.uint32) for _ in range(2)]}
    if "decode_pipe_tma_xyz" in tun:   # the store warp needs a uniformly strided batch: the batch entry point
        import torch
        dev0 = torch.device("cuda", 0)
        F = 3
        t_pk = torch.from_numpy(np.stack([pk32] * F)).to(dev0)
        tf = {f["name"]: torch.zeros((F, 32, 128), dtype={1: torch.uint8, 2: torch.int16, 4: torch.int32}[f["elem_size"]], device=dev0)
              for f in dec32.fields}
        tx = [torch.zeros((F, 32 * 128, 3), dtype=torch.float32, device=dev0) for _ in range(2)]
        trd = [torch.zeros((F, 32, 128), dtype=torch.int32, device=dev0) for _ in range(2)]
        dec32.decode_batch(F, t_pk, pk32.shape[0], pk32.shape[1], pk32.shape[0] * pk32.shape[1], tf, lut=lut32,
                           pixel_shift_by_row=sh32, xyz=tx, range_destaggered=trd, stream=st)
        st.sync()
        for r, nm in enumerate(("RANGE", "RANGE2")):
            assert np.array_equal(tx[r][F - 1].cpu().numpy(), orc.cartesian(src32.field(nm), d32, o32))
            assert np.array_equal(trd[r][F - 1].cpu().numpy().view(np.uint32), orc.destagger(src32.field(nm), sh32))
    else:
        dec32.decode([io], lut=lut32, pixel_shift_by_row=sh32, stream=st)
        st.sync()
        for n, a in io["fields"].items():
            assert np.array_equal(a, src32.field(n)), n
        for r, nm in enumerate(("RANGE", "RANGE2")):
            assert np.array_equal(io["xyz"][r], orc.cartesian(src32.field(nm), d32, o32))
            assert np.array_equal(io["range_destaggered"][r], orc.destagger(src32.field(nm), sh32))
    assert ob.kernel_launch_count("decode_pipe") > n1, "the pipelined K2 did not run"
    for k in tun:
        ob.set_tunable(k, 0)
print("K2 pipelined: 3 CTAs/SM, helper warps, store-warp XYZ ok")
sih = ob.SensorInfo("RNG19_RFL8_SIG16_NIR16_DUAL", 16, 128, fw_rev="v3.2.1")
fr = ob.LidarFrame(sih)
rs = np.random.default_rng(12)
for name in fr.fields:
    a = fr.field(name)
    a[...] = rs.integers(0, 200, size=a.shape).astype(a.dtype)
fr.status[:] = 1
fr.status[3] = 0
fr.timestamp[:] = 5 + np.arange(128)
fr.packet_timestamp[:] = 1 + np.arange(8)
fr.frame_id = 77
hp, _ = ob.frame_to_packets(fr, sih, 3, 9)
dp, _ = ob.frame_to_packets(fr, sih, 3, 9, device=True)
assert np.array_equal(hp, dp)
print("K4 encode ok")
xyz, rngd, dirs = room_scene(24, 96)
org = np.zeros((96, 3))
nn, sub = ob.normals(xyz, rngd, org, 2, return_subtent=True)
assert np.array_equal(nn, orc.normals(xyz, rngd, sensor_origins_xyz=org, pixel_search_range=2, vertical_subtent=sub))
n1, n2 = ob.normals(xyz, rngd, xyz * 1.1, rngd, org)
print("normals ok")
frames = []
want = []
for i, (hh, ww) in enumerate(((16, 64), (24, 96))):
    rg = random_range(hh, ww, 80 + i, p_zero=0.3, max_range=50000)
    d, o = random_lut(hh * ww, 9 + i)
    poses = np.tile(np.eye(4), (ww, 1, 1))
    poses[:, :3, 3] = np.random.default_rng(i).random((ww, 3))
    stt = np.ones(ww, np.uint32)
    stt[:3] = 0
    tsn = np.arange(ww, dtype=np.uint64)
    frames.append({"lut": ob.XYZLutT.from_arrays(d, o, hh, ww), "range": rg, "poses": poses, "status": stt, "timestamps": tsn})
    want.append(orc.dewarp_frame(rg, d, o, poses, stt, tsn, 0.5, 40.0)[0])
assert np.array_equal(ob.dewarp_frames(frames, 0.5, 40.0), np.concatenate(want))
print("batched K3 ok")
# K3 with later turns of the slab loop (1000 rows), more than 48 KB of shared memory (6160 rows), and a look-back
# chain of 3072 CTAs (48 frames of 64 CTAs) with long runs of CTAs that emit nothing
for dt in (np.float32, np.float64):
    for hh, ww in ((1000, 33), (6160, 33)):
        rg = random_range(hh, ww, 90, p_zero=0.3, max_range=50000)
        d, o = random_lut(hh * ww, 91, dt)
        poses = np.tile(np.eye(4), (ww, 1, 1))
        poses[:, :3, 3] = np.random.default_rng(92).random((ww, 3))
        stt = np.ones(ww, np.uint32)
        tsn = np.arange(ww, dtype=np.uint64)
        got = ob.dewarp_frame(ob.XYZLutT.from_arrays(d, o, hh, ww), rg, poses, stt, tsn, 0.5, 40.0, provenance=True)
        for a, b in zip(got, orc.dewarp_frame(rg, d, o, poses, stt, tsn, 0.5, 40.0)):
            assert np.array_equal(a, b), (hh, ww)
hh, ww = 16, 2048
d, o = random_lut(hh * ww, 93)
lut = ob.XYZLutT.from_arrays(d, o, hh, ww)
frames, want = [], []
for i in range(48):
    rg = random_range(hh, ww, 200 + i, p_zero=0.3, max_range=50000)
    rg[:, (173 * i) % 1500:(173 * i) % 1500 + 400] = 0
    poses = np.tile(np.eye(4), (ww, 1, 1))
    poses[:, :3, 3] = np.random.default_rng(i).random((ww, 3))
    stt = np.ones(ww, np.uint32)
    frames.append({"lut": lut, "range": rg, "poses": poses, "status": stt})
    want.append(orc.dewarp_frame(rg, d, o, poses, stt, np.zeros(ww, np.uint64), 0.5, 40.0)[0])
assert np.array_equal(ob.dewarp_frames(frames, 0.5, 40.0), np.concatenate(want))
print("K3 tall frames and 3072 CTAs ok")
vp = np.random.default_rng(12).random((3000, 4)) * 3
for code, name in ((orv.FIRST_N_POINT, "first_n"), (orv.AVERAGE_POINT, "average"), (orv.RANDOM, "random")):
    got, gi = ob.voxel_downsample(vp, 0.5, name, max_points_per_voxel=3, min_pts_threshold=2)
    want, wi = orv.voxel_downsample_xd(vp, 0.5, 3, 2, code, with_indices=True)
    assert np.array_equal(got, want) and np.array_equal(gi, wi), name
got, gi = ob.voxel_downsample(vp[:, :3].copy(), 0.5)
assert np.array_equal(gi, orv.voxel_downsample(vp[:, :3], 0.5)[1])
vn = vp[:, 1:] - 1.5
gp, gn, _ = ob.voxel_downsample(vp[:, :3].copy(), 0.5, "point_normal", normals=vn)
wp, wn = orv.voxel_downsample_with_normals(vp[:, :3], vn, 0.5)
assert np.array_equal(gp, wp) and np.array_equal(gn, wn)
print("voxel ok")
# voxel map + ICP: add (f32 and f64), cull with extraction, point cloud, closest neighbours, linear system, align
from oracle import icp as oi
rs = np.random.default_rng(11)
gm, om = ob.VoxelMap(0.5, 3.0, 3), oi.VoxelHashMap3d(0.5, 3.0, 3)
for k in range(3):
    vm_pts = rs.normal(k, 2.0, (600, 3))
    gm.add_points(vm_pts.astype(np.float32) if k % 2 else vm_pts)
    om.add_points(vm_pts.astype(np.float32).astype(np.float64) if k % 2 else vm_pts)
    assert np.array_equal(gm.remove_far([k, 0, 0], extract=True), om.extract_voxels_far_from_location([k, 0, 0]))
assert np.array_equal(gm.point_cloud(), om.point_cloud())
vq = rs.normal(0, 2.0, (300, 3))
assert all(np.array_equal(a, b) for a, b in zip(gm.closest_neighbors(vq, 1.0), om.get_closest_neighbors(vq, 1.0)))
assert all(np.array_equal(a, b) for a, b in zip(ob.icp_linear_system(vq, vq + 0.01, 0.5),
                                                  oi.build_linear_system(vq, vq + 0.01, 0.5)))
vp, vit = ob.icp_align(gm, om.point_cloud() + 0.02, 1.0, 0.5, 10)
wp, wit = oi.align_points_to_map(om.point_cloud() + 0.02, om, 1.0, 0.5, 10)
assert vit == wit and np.abs(vp - wp).max() <= 1e-12
print("voxel map / icp ok")
# voxel map with attributes (growth, cull with extraction, neighbours with attributes) and the frame -> map-row ingest
from tests import voxel_map_xd_reference as xr
gx, xx = ob.VoxelMap(0.5, 3.0, 3, num_attributes=2), xr.VoxelHashMapXd(0.5, 3.0, 3, num_attributes=2)
for k in range(3):
    xrows = np.hstack([rs.normal(k, 2.0, (1500, 3)), rs.normal(0, 1.0, (1500, 2))])
    gx.add_points(xrows)
    xx.add_points(xrows)
    assert np.array_equal(gx.remove_far([k, 0, 0], extract=True), xx.extract_voxels_far_from_location([k, 0, 0]))
assert all(np.array_equal(a, b) for a, b in zip(gx.closest_neighbors(vq, 1.0), xx.get_closest_neighbors(vq, 1.0)))
mh, mw = 16, 64
mr = (rs.integers(0, 5000, (mh, mw)) * (rs.random((mh, mw)) > 0.2)).astype(np.uint32)
md = rs.normal(0, 1.0, (mh * mw, 3))
mlut = ob.XYZLutT.from_arrays(md, np.zeros_like(md), mh, mw)
mitem = {"range": mr, "poses": np.repeat(np.eye(4)[None], mw, 0), "direction": md, "offset": np.zeros_like(md),
         "fields": [rs.integers(0, 255, (mh, mw)).astype(np.uint8), rs.normal(0, 1, (mh, mw, 3)).astype(np.float16)]}
assert np.array_equal(ob.map_rows([dict(mitem, lut=mlut)] * 2), xr.map_rows([mitem] * 2))
print("voxel map xd / map rows ok")
# cloud-to-cloud ICP: nearest with NaN / 1e300 rows and bad normals, both aligns (f32 and f64)
from oracle import align as oa
rs = np.random.default_rng(12)
ct = np.round(rs.uniform(-2, 2, (800, 3)) / 0.1) * 0.1
ct[:5, 0] = [np.nan, np.inf, 1e300, -1e300, np.nan]
cn = rs.normal(size=ct.shape)
cn[5:15] = 0.0
cq = np.round(rs.uniform(-2, 2, (700, 3)) / 0.1) * 0.1
assert np.array_equal(ob.cloud_nearest(ct, cq, 0.3, 0.09, target_normals=cn), oa.cloud_nearest(ct, cq, 0.3, 0.09, cn))
cs = ct[5:] @ np.array([[1, -0.01, 0], [0.01, 1, 0], [0, 0, 1]]).T + [0.02, -0.01, 0.0]
for dt in (np.float64, np.float32):
    a, b, sn, tn = cs.astype(dt), ct[5:].astype(dt), cn[5:].astype(dt), cn[5:].astype(dt)
    gp, git = ob.cloud_align(a, b, max_corr_dist=0.5)
    wp, wit = oa.point_to_point_align(a, b, None, 0.5)
    assert git == wit and np.abs(gp - wp).max() <= 1e-12
    gp, git = ob.cloud_align(a, b, sn, tn, max_corr_dist=0.5, max_normal_angle_deg=180.0)
    wp, wit = oa.point_to_plane_align(a, b, sn, tn, None, 0.5, 180.0)
    assert git == wit and np.abs(gp - wp).max() <= 1e-12
print("cloud align ok")
# image post-processing: every kernel of AE (mono, rgb, f16), BUC (f32, f64; median with masked columns) and LTM
from oracle import image as oimg
ri = np.random.default_rng(13)
for dt in (np.float32, np.float64):
    for kind, shape in (("auto_exposure", (12, 96)), ("auto_exposure", (12, 96, 3)), ("beam_uniformity", (12, 96)),
                        ("local_tone_map", (12, 96, 3))):
        proc = ob.ImageProcessor(kind)
        ref = {"auto_exposure": oimg.AutoExposure, "beam_uniformity": oimg.BeamUniformityCorrector,
               "local_tone_map": oimg.LocalToneMapper}[kind]()
        for f in range(3):
            a = ri.uniform(0, 2, shape).astype(dt)
            a[..., ::7] = 0
            g, want = a.copy(), a.copy()
            proc.update(g)
            ref.update(want)
            assert np.array_equal(g, want, equal_nan=True), (kind, shape, f)
for kind, ref in (("auto_exposure", oimg.AutoExposure()), ("local_tone_map", oimg.LocalToneMapper())):
    proc = ob.ImageProcessor(kind)
    src = ri.uniform(0, 1, (12, 96, 3)).astype(np.float16)
    assert np.array_equal(proc.update(src), ref.update(src), equal_nan=True)
print("image ok")
# frame operations: every predicate of the masked write (aligned and ragged runs) and the row gather
import json
from oracle import frame_ops as ofo
FIX32 = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                     "OS-1-32-G_v2.1.1_1024x10.json")
rf = np.random.default_rng(17)
for h, w in ((3, 37), (4, 64)):
    si = ob.SensorInfo("RNG19_RFL8_SIG16_NIR16_DUAL", h, w, 1, pixel_shift_by_row=rf.integers(-5, 6, h))
    for op in ("clip", "filter_field", "u", "v", "mask"):
        fr = ob.LidarFrame(si)
        for n in fr.fields:
            fr.field(n)[...] = rf.integers(0, 200, fr.field(n).shape).astype(fr.field(n).dtype)
        o = ofo.Frame(h, w, si.pixel_shift_by_row)
        for n in fr.fields:
            o.add(n, fr.field(n).copy(), fr.field_tag(n))
        m = (rf.random((h, w)) < 0.5).astype(np.uint8)
        {"clip": lambda f, mod: mod.clip(f, [], 20, 150, 1),
         "filter_field": lambda f, mod: mod.filter_field(f, "RANGE", 20, 150),
         "u": lambda f, mod: mod.filter_uv(f, "u", 1, 2), "v": lambda f, mod: mod.filter_uv(f, "v", 3, 9),
         "mask": lambda f, mod: mod.mask(f, [], m)}[op](fr, ob.frame_ops)
        {"clip": lambda f: ofo.clip(f, [], 20, 150, 1), "filter_field": lambda f: ofo.filter_field(f, "RANGE", 20, 150),
         "u": lambda f: ofo.filter_uv(f, "u", 1, 2), "v": lambda f: ofo.filter_uv(f, "v", 3, 9),
         "mask": lambda f: ofo.mask(f, [], m)}[op](o)
        for n in fr.fields:
            assert np.array_equal(fr.field(n), o.field(n)), (op, n)
    sel = ob.frame_ops.select_by_index(fr, [h - 1, 0])
    assert np.array_equal(sel.field("RANGE"), fr.field("RANGE")[[h - 1, 0]])
si32 = ob.SensorInfo.from_meta(json.load(open(FIX32)))
lut = ob.pyapi.XYZLutFloat(si32)
fr32 = ob.LidarFrame(si32)
fr32.field("RANGE")[...] = rf.integers(0, 20000, fr32.field("RANGE").shape)
ob.frame_ops.filter_xyz(fr32, lut, 2, -0.2, 0.2, dewarp_points=True)
print("frame ops ok")
# pose interpolation (f-12): sorted, unsorted and NaN x, both dtypes, an error case, and the frame form
from oracle import pose as opose  # noqa: E402
rp = np.random.default_rng(23)
kp = np.cumsum(rp.random(7) + 0.1)
pkp = np.stack([opose.posev_exp(np.concatenate([rp.normal(size=3) * 0.3, rp.normal(size=3)])) for _ in kp])
for xs in (np.sort(rp.uniform(0, kp[-1] + 1, 300)), np.where(rp.random(300) < 0.1, np.nan,
                                                               np.sort(rp.uniform(0, 9, 300)))):
    assert np.allclose(ob.core.interp_pose(xs, kp, pkp), opose.interp_pose(xs, kp, pkp), atol=1e-9, equal_nan=True)
    ob.core.interp_pose(xs, kp, pkp.astype(np.float32))
xi = np.sort(rp.integers(0, 10**6, 200))
ob.core.interp_pose(xi, np.array([0, 10**6], np.int64), pkp[:2], two_pose=True)
try:
    ob.core.interp_pose(np.array([0.5, 0.2]), kp, pkp)
    raise AssertionError("descent not reported")
except ValueError:
    pass
tsp = (10**9 + np.arange(100) * 10**6).astype(np.uint64)
stp = (rp.random(100) < 0.7).astype(np.uint32)
psp = np.zeros((100, 4, 4))
ob.core.frames_interp_pose([(tsp, stp, psp), None], 1.0, pkp[0], 1.1, pkp[1])
ob.core.frames_interp_pose([(tsp, stp, psp)], 0.0, pkp[0])
print("pose ok")
# ground segmentation: two frames of different shapes in one set, with NORMALS given and with computed normals
from oracle import ground as og  # noqa: E402
from tests import test_gpu_ground as tg  # noqa: E402
ga, gb = tg._frame("box_rooftop", h=16, w=128, dual=True), tg._frame("room", h=8, w=64, seed=5)
dg = [tg._gpu_frame(f, normals=tg._normals32(f)) for f in (ga, gb)]
for f, d, got in zip((ga, gb), dg, ob.core.ground_mask([dg[0], None, dg[1]], model=True)[::2]):
    tg._assert_same(got, *tg._oracle(f, d), og.FINAL)
dg = [dict(tg._gpu_frame(f), sensor_to_body=f["sensor_to_body"]) for f in (ga, gb)]
for f, got in zip((ga, gb), ob.core.ground_mask(dg, model=True)):
    nrm = tg._oracle_normals(f, got["vertical_subtent"])
    tg._assert_same(got, *og.run(f["ranges"], f["status"], f["direction"], f["offset"], f["poses"], nrm), og.FINAL)
print("ground ok")
# zone monitoring: render of body- and sensor-frame zones, then monitor updates with a host and a device bitmask
import torch  # noqa: E402
from tests import test_gpu_zone as tz  # noqa: E402
tz.render_both(ob, tz.subsample(tz.sensor_meta("785.json"), 16, 128), [(tz.stl_tris("0.stl"), f) for f in (1, 2)],
               tz.s2b_z1())
tz.ZSD = ob.core.ZONE_STATE_DTYPE
zh, zw = 8, 64
zones = tz.random_zones(zh, zw, 3, 1)
mon = ob.ZoneMonitor([{"id": z[0], "mode": z[1], "point_count": z[2], "frame_count": z[3], "near_mm": z[4],
                       "far_mm": z[5]} for z in zones], zh, zw)
ref = tz.RefZoneMon(zones)
for f in range(4):
    r = tz.random_range(zones, zh, zw, f)
    want_bm = np.zeros((zh, zw), np.uint32)
    want = ref.calc(r, want_bm)
    if f % 2:
        bm = torch.zeros((zh, zw), dtype=torch.int32, device="cuda")
        mon.update(torch.from_numpy(r.view(np.int32)).cuda(), bm)
        bm = bm.cpu().numpy().view(np.uint32)
    else:
        bm = np.zeros((zh, zw), np.uint32)
        mon.update(r, bm)
    assert np.array_equal(mon.states(), want) and np.array_equal(bm, want_bm), f
print("zone ok")
print("SANITIZE CASES OK")
