"""The device chain pose interpolation was built for (DESIGN f-12): core.Decoder.decode on the recorded OS-1-128
packets writes RANGE and the column headers (TIMESTAMP in an int64 tensor, STATUS in an int32 tensor) to the
device; ob_frames_interp_pose poses the set from them with device x0 / x1 and a device error word; ob_dewarp_frames
projects it with a device count.  Bit-identical to the same calls on host inputs, within tolerance of the oracle's
decode -> oracle interpolation -> oracle dewarp, and bit-identical again when the pose step replays from a CUDA
graph.  Also: the C++ drop-in example against the Python results."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import oracle as orc
from oracle import pose as op
from tests.helpers import decoder_desc_from_oracle, load_fixture, oracle_pf

pytestmark = pytest.mark.gpu

ob = graft.load_package()
torch = pytest.importorskip("torch")
ROOT = graft.ROOT
FIXTURE = "OS-1-128_767798045_1024x10_20230712_120049"


def _pose(angle_z, t):
    c, s = np.cos(angle_z), np.sin(angle_z)
    p = np.eye(4)
    p[:2, :2] = [[c, -s], [s, c]]
    p[:3, 3] = t
    return p


def _dewarp_frames(lut, frames, cap, stream, device_count):
    """ob_dewarp_frames over [(range, poses, status) | None]; device_count: count and points stay on the device."""
    capi = ob._capi
    ios = (capi.DewarpFramesIO * len(frames))()
    for i, f in enumerate(frames):
        if f is None:
            continue
        ios[i].lut, ios[i].range, ios[i].poses, ios[i].status = lut._h, ob.core._ptr(f[0]), ob.core._ptr(f[1]), \
            ob.core._ptr(f[2])
    if device_count:
        pts = torch.zeros((cap, 3), dtype=torch.float64, device="cuda")
        n = torch.zeros(1, dtype=torch.int64, device="cuda")
        capi.check(capi.lib.ob_dewarp_frames(ios, len(frames), 0.0, 4294967.295, pts.data_ptr(), cap, None, None,
                                             None, None, C.cast(n.data_ptr(), C.POINTER(C.c_size_t)), stream.h))
        return pts, n
    pts = np.zeros((cap, 3))
    n = C.c_size_t(0)
    capi.check(capi.lib.ob_dewarp_frames(ios, len(frames), 0.0, 4294967.295, pts.ctypes.data, cap, None, None,
                                         None, None, C.byref(n), stream.h))
    return pts[:n.value]


def test_decode_interp_dewarp_chain_on_recorded_packets():
    meta, packets = load_fixture(FIXTURE)
    pf = oracle_pf(meta)
    oframe = orc.Frame(pf)
    obat = orc.Batcher(pf, init_id=meta["init_id"], column_window=meta["column_window"])
    for p in packets:
        obat.batch(p, 77, oframe)
    info = ob.pyapi.SensorInfo.from_meta(meta)
    lut = ob.pyapi.XYZLut(info)._lut
    h, w = lut.h, lut.w
    # the fixture holds 8 packets (columns 0..127): col_src maps each column to its packet column, -1 elsewhere
    cpp = pf.columns_per_packet
    col_src = np.full(w, -1, np.int32)
    col_src[oframe.measurement_id[: len(packets) * cpp]] = np.arange(len(packets) * cpp, dtype=np.int32)
    dec = ob.Decoder(*decoder_desc_from_oracle(pf, oframe))
    dev = torch.device("cuda", 0)
    cs = torch.cuda.Stream()
    st = ob.Stream(0, cuda_stream=cs.cuda_stream)
    slots = [0, 2]
    rng = {k: torch.zeros((h, w), dtype=torch.int32, device=dev) for k in slots}
    ts = {k: torch.zeros(w, dtype=torch.int64, device=dev) for k in slots}
    stt = {k: torch.zeros(w, dtype=torch.int32, device=dev) for k in slots}
    with torch.cuda.stream(cs):
        dec.decode([{"packets": packets, "n_slots": len(packets), "packet_stride": packets.shape[1],
                     "col_src": col_src, "fields": {"RANGE": rng[k]}, "timestamp": ts[k], "status": stt[k]}
                    for k in slots], stream=st)
        cs.synchronize()
    host_ts = oframe.timestamp.copy()
    host_st = oframe.status.copy()
    host_rng = oframe.field("RANGE").copy()
    for k in slots:
        assert np.array_equal(ts[k].cpu().numpy().view(np.uint64), host_ts)
        assert np.array_equal(stt[k].cpu().numpy().view(np.uint32), host_st)
        assert np.array_equal(rng[k].cpu().numpy().view(np.uint32), host_rng)
    assert int((host_st & 1).sum()) == len(packets) * cpp
    t1 = float(host_ts[len(packets) * cpp - 1]) * 1e-9
    t0 = t1 - 0.1
    x0, x1 = _pose(0.0, [0.0, 0.0, 0.0]), _pose(0.05, [1.0, 0.2, 0.0])
    init = np.repeat(np.eye(4)[None], w, 0) * 3.0
    # device chain: device headers, device x0 / x1, device error word, device count
    dposes = {k: torch.from_numpy(init.copy()).to(dev) for k in slots}
    dx0, dx1 = torch.from_numpy(x0).to(dev), torch.from_numpy(x1).to(dev)
    err = torch.full((3,), -1, dtype=torch.int64, device=dev)
    cap = 2 * h * w
    with torch.cuda.stream(cs):
        ob.core.frames_interp_pose([(ts[0], stt[0], dposes[0]), None, (ts[2], stt[2], dposes[2])], t0, dx0, t1, dx1,
                                   error=err, stream=st)
        dpts, dn = _dewarp_frames(lut, [(rng[0], dposes[0], stt[0]), None, (rng[2], dposes[2], stt[2])], cap, st,
                                  True)
        cs.synchronize()
    assert err.cpu().tolist() == [0, 0, 0]
    # host chain: the same calls on host inputs
    hposes = {k: init.copy() for k in slots}
    ob.core.frames_interp_pose([(host_ts, host_st, hposes[0]), None, (host_ts, host_st, hposes[2])], t0, x0, t1, x1)
    hpts = _dewarp_frames(lut, [(host_rng, hposes[0], host_st), None, (host_rng, hposes[2], host_st)], cap, st, False)
    n = int(dn.item())
    assert n == len(hpts) > 0
    for k in slots:
        assert np.array_equal(dposes[k].cpu().numpy(), hposes[k])
    assert np.array_equal(dpts[:n].cpu().numpy(), hpts)
    # oracle: interpolation on the oracle's decode, then the oracle's single-frame dewarp of each frame
    oposes = init.copy()
    assert op.frames_interp_pose([(host_ts, host_st, oposes)], t0, x0, t1, x1)[0] == 0
    d = np.ascontiguousarray(lut.direction, np.float64)
    o = np.ascontiguousarray(lut.offset, np.float64)
    opts, _, _ = orc.dewarp_frame(host_rng, d, o, oposes, host_st, host_ts, 0.0, 4294967.295)
    want = np.concatenate([opts, opts])
    assert want.shape == hpts.shape
    np.testing.assert_allclose(hpts, want, rtol=0, atol=1e-9)
    np.testing.assert_allclose(hposes[0], oposes, rtol=0, atol=1e-12)
    # the pose step replayed from a CUDA graph gives the same bits, and the dewarp after it the same points
    # (ob_dewarp_frames stages its frame table from pageable host memory, so it runs outside the graph)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(cs):
        with torch.cuda.graph(g, stream=cs, capture_error_mode="thread_local"):
            ob.core.frames_interp_pose([(ts[0], stt[0], dposes[0]), None, (ts[2], stt[2], dposes[2])], t0, dx0, t1,
                                       dx1, error=err, stream=st)
        for _ in range(2):
            for k in slots:
                dposes[k].copy_(torch.from_numpy(init))
            err.fill_(-1)
            g.replay()
            gpts, gn = _dewarp_frames(lut, [(rng[0], dposes[0], stt[0]), None, (rng[2], dposes[2], stt[2])], cap,
                                      st, True)
            cs.synchronize()
            assert err.cpu().tolist() == [0, 0, 0] and int(gn.item()) == n
            for k in slots:
                assert np.array_equal(dposes[k].cpu().numpy(), hposes[k])
            assert np.array_equal(gpts[:n].cpu().numpy(), hpts)


def test_cpp_dropin_example_matches_python(tmp_path):
    graft.build()
    lib_dir = os.path.join(ROOT, "ouster-sdk_b200", "lib")
    exe = str(tmp_path / "pose_dropin_example")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "pose_dropin_example.cpp"), "-L", lib_dir,
                           "-louster_b200", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    out = subprocess.run([exe, "gpu"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "POSE DROPIN GPU OK" in out.stdout, (out.stdout, out.stderr)
    got = {}
    for line in out.stdout.splitlines():
        parts = line.split()
        if len(parts) == 18 and parts[0] == "POSE":
            got[parts[1]] = np.array([float(v) for v in parts[2:]]).reshape(4, 4)
    curr = np.array([[0.950564, -0.29552, -0.0953745, 5], [0.294044, 0.955336, -0.0295028, 3],
                     [0.0998334, 0, 0.995004, 2], [0, 0, 0, 1]])
    nxt = np.array([[0.879923, -0.389418, -0.272192, 0], [0.372026, 0.921061, -0.115081, 0],
                    [0.29552, 0, 0.955336, 0], [0, 0, 0, 1]])
    x = np.array([100000.0, 100500.0, 101000.0, 101500.0, 102000.0, 102500.0, 103000.0, 103500.0])
    k = np.array([101000.0, 102000.0, 103000.0])
    pk = np.stack([np.eye(4), curr, nxt])
    py = ob.pyapi.interp_pose(x, k, pk)
    py32 = ob.pyapi.interp_pose_float(x, k, pk.astype(np.float32))
    for i in range(8):
        assert np.array_equal(got[f"knot{i}"], py[i])
        assert np.array_equal(got[f"f32_{i}"], py32[i].astype(np.float64))
    xi = np.array([-500, 0, 250, 1000, 1500], np.int64)
    two = ob.core.interp_pose(xi, np.array([0, 1000], np.int64), np.stack([curr, nxt]), two_pose=True)
    for i in range(5):
        assert np.array_equal(got[f"two{i}"], two[i])
    # the deskew of the example's set, through the Python ConstantVelocityDeskewMethod's call
    w = 64
    for f in (0, 2):
        tsf = (1000000000 + f * 100000000 + np.arange(w) * 1000000).astype(np.uint64)
        stf = np.where(np.arange(w) % 3 == 2, 0, 1).astype(np.uint32)
        poses = np.zeros((w, 4, 4))
        ob.core.frames_interp_pose([(tsf, stf, poses)], 0.9, curr, 1.0, nxt)
        for c in range(0, w, 5):
            if stf[c]:
                assert np.array_equal(got[f"deskew{f}_{c}"], poses[c])
