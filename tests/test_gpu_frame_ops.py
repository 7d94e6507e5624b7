"""Frame operations on the GPU (ouster_sdk_b200.frame_ops) against the CPU oracle (oracle/frame_ops.py), bit for
bit: every operation and field type on host frames and DeviceLidarScan, special values and bounds, the second
return, poses, row selection and its metadata, batches, graph capture and a packets-to-XYZ chain."""
import json
import os

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import frame_ops as ofo
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
PROFILE = "RNG19_RFL8_SIG16_NIR16_DUAL"
SHAPES = [(128, 2048), (64, 1024), (32, 512), (7, 333), (1, 1667)]
EXTRA = {"I8": np.int8, "I16": np.int16, "I32": np.int32, "I64": np.int64, "U64": np.uint64, "F32": np.float32,
         "F64": np.float64}


@pytest.fixture(scope="module")
def ob():
    m = graft.load_package()
    if m.device_count() == 0:
        pytest.skip("no CUDA device")
    return m


def _info(ob, h, w, seed=0):
    rs = np.random.default_rng(seed)
    return ob.SensorInfo(PROFILE, h, w, 16 if w % 16 == 0 else 1,
                         pixel_shift_by_row=rs.integers(-30, 31, h).astype(np.int32))


def _fill(a, rs, name):
    if a.dtype.kind == "f":
        v = rs.uniform(-2e4, 3e4, a.shape).astype(a.dtype)
        flat = v.reshape(-1)
        flat[::97] = np.nan
        flat[1::89] = np.inf
        flat[2::83] = -np.inf
        flat[3::79] = -0.0
        a[...] = v
    elif a.dtype == np.uint64:
        v = rs.integers(0, 1 << 62, a.shape, dtype=np.uint64)
        v.reshape(-1)[::7] = np.uint64(2 ** 53 + 1)
        a[...] = v
    else:
        info = np.iinfo(a.dtype)
        a[...] = rs.integers(max(info.min, -40000), min(info.max, 40000), a.shape, endpoint=True).astype(a.dtype)


def _host_frame(ob, info, seed=0, f16=True):
    rs = np.random.default_rng(seed + 100)
    fr = ob.LidarFrame(info)
    for n, dt in EXTRA.items():
        fr.add_field(n, dt)
    if f16:
        fr.add_field("H", np.uint16, tag=12)
    for n in fr.fields:
        _fill(fr.field(n), rs, n)
    return fr


def _oracle_of(fr, info):
    o = ofo.Frame(fr.h, fr.w, info.pixel_shift_by_row)
    for n in fr.fields:
        o.add(n, fr.field(n).copy(), fr.field_tag(n))
    o.body_to_world = fr.body_to_world.copy()
    return o


def _assert_same(fr_fields, o):
    for n, a in fr_fields.items():
        b = o.field(n)
        assert a.shape == b.shape, n
        assert np.array_equal(np.ascontiguousarray(a).view(np.uint8), b.view(np.uint8)), n


def _host_fields(fr):
    return {n: fr.field(n) for n in fr.fields}


def _ops(ob):
    """(name, gpu call, oracle call) of every masked-write operation, with awkward arguments."""
    rs = np.random.default_rng(5)
    return [
        ("clip", lambda f: ob.frame_ops.clip(f, [], 100, 30000, 7), lambda o: ofo.clip(o, [], 100, 30000, 7)),
        ("clip_inf", lambda f: ob.frame_ops.clip(f, ["F32", "F64", "RANGE"], -np.inf, 5000.5, 3.7),
         lambda o: ofo.clip(o, ["F32", "F64", "RANGE"], -np.inf, 5000.5, 3.7)),
        ("clip_u64_edge", lambda f: ob.frame_ops.clip(f, ["U64"], 0, float(2 ** 53), 0),
         lambda o: ofo.clip(o, ["U64"], 0, float(2 ** 53), 0)),
        ("clip_empty", lambda f: ob.frame_ops.clip(f, [], 10, 5, 1), lambda o: ofo.clip(o, [], 10, 5, 1)),
        ("filter_field", lambda f: ob.frame_ops.filter_field(f, "RANGE", 5000, 200000, 1.7),
         lambda o: ofo.filter_field(o, "RANGE", 5000, 200000, 1.7)),
        ("filter_field_f32", lambda f: ob.frame_ops.filter_field(f, "F32", -1e4, 1e4, 2, ["F32", "SIGNAL", "NOPE"]),
         lambda o: ofo.filter_field(o, "F32", -1e4, 1e4, 2, ["F32", "SIGNAL"])),
        ("filter_uv_u", lambda f: ob.frame_ops.filter_uv(f, "u", 0, (f.h + 1) // 2, 5),
         lambda o: ofo.filter_uv(o, "u", 0, (o.h + 1) // 2, 5)),
        ("filter_uv_v", lambda f: ob.frame_ops.filter_uv(f, "v", f.w // 3, f.w - 1, 9),
         lambda o: ofo.filter_uv(o, "v", o.w // 3, o.w - 1, 9)),
        ("filter_uv_v_frac", lambda f: ob.frame_ops.filter_uv(f, "v", 0.25, float("inf")),
         lambda o: ofo.filter_uv(o, "v", int(o.w * 0.25), o.w)),
        ("mask", lambda f: ob.frame_ops.mask(f, [], _MASK[(f.h, f.w)]),
         lambda o: ofo.mask(o, [], _MASK[(o.h, o.w)])),
    ]


_MASK = {s: (np.random.default_rng(s[0] * 7 + s[1]).random(s) < 0.5).astype(np.uint8) for s in SHAPES}


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_host_frames_match_oracle(ob, shape):
    info = _info(ob, *shape)
    for name, g, r in _ops(ob):
        fr = _host_frame(ob, info, seed=len(name) * 31)
        o = _oracle_of(fr, info)
        g(fr)
        r(o)
        _assert_same(_host_fields(fr), o)


def _device_scan(ob, info, fr):
    import torch
    from ouster_sdk_b200 import pyapi
    sc = pyapi.DeviceLidarScan(info)
    for n in fr.fields:
        a = fr.field(n)
        sc._fields[n] = torch.from_numpy(a.view({1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[a.itemsize])
                                         .copy()).cuda()
        if n not in sc.host.fields:
            cls = fr.field_class(n)
            sc.host.add_field(n, a.dtype, ob.frame_ops._extra(a.shape, cls), tag=fr.field_tag(n), field_class=cls)
    sc.host.body_to_world[:] = fr.body_to_world
    sc.host.timestamp[:] = fr.timestamp
    sc.host.frame_id = fr.frame_id
    return sc


def _dev_fields(sc, fr):
    return {n: sc.field(n).cpu().numpy().view(fr.field(n).dtype) for n in sc.fields}


@pytest.mark.parametrize("shape", [(128, 2048), (7, 333)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_device_scans_match_oracle(ob, shape):
    import torch
    info = _info(ob, *shape)
    for name, g, r in _ops(ob):
        if name == "mask":
            g = lambda f: ob.frame_ops.mask(f, [], torch.as_tensor(_MASK[(f.h, f.w)]).cuda())  # noqa: E731
        fr = _host_frame(ob, info, seed=len(name) * 31)
        o = _oracle_of(fr, info)
        sc = _device_scan(ob, info, fr)
        g(sc)
        torch.cuda.synchronize()
        r(o)
        _assert_same(_dev_fields(sc, fr), o)


def test_refused_invalid_leaves_every_field_unchanged(ob):
    info = _info(ob, 16, 256)
    for inv in (float("nan"), float("inf"), -1, 2.0 ** 64, 300):
        fr = _host_frame(ob, info)
        before = {n: a.copy() for n, a in _host_fields(fr).items()}
        with pytest.raises(ValueError, match="invalid value cannot be represented"):
            ob.frame_ops.clip(fr, [], 0, 1, inv)
        for n, a in _host_fields(fr).items():
            assert np.array_equal(a.view(np.uint8), before[n].view(np.uint8)), (inv, n)


def test_errors(ob):
    info = _info(ob, 8, 64)
    fr = _host_frame(ob, info)
    fr.add_field("E", np.uint16, 3)
    with pytest.raises(ValueError, match=r"^Field: Eigen array conversion failed due to dimension mismatch\. "
                                         r"Underlying data has 3 dimensions but must have 2 dimensions\.$"):
        ob.frame_ops.clip(fr, [], 0, 1)
    with pytest.raises(ValueError, match=r"^filter_field requires a pixel field with shape \(h, w\) to build a mask$"):
        ob.frame_ops.filter_field(fr, "E", 0, 1)
    with pytest.raises(ValueError, match=r"^filter_field requires a pixel field with shape \(h, w\) to build a mask$"):
        ob.frame_ops.filter_field(fr, "H", 0, 1)
    with pytest.raises(ValueError, match=r"^lower == 0 and upper == 65 must be in the range \[0, 64\]$"):
        ob.frame_ops.filter_uv(fr, "v", 0, 65)
    with pytest.raises(ValueError, match=r"doesn't match frame size \(\{frame\.h\}, \{frame\.w\}$"):
        ob.frame_ops.mask(fr, [], np.ones((2, 2), np.uint8))


def _golden_info(ob, name="OS-1-128_767798045_1024x10_20230712_120049.json"):
    meta = json.load(open(os.path.join(GOLDEN, name)))
    return ob.SensorInfo.from_meta(meta)


@pytest.mark.parametrize("lut_kind", ["XYZLut", "XYZLutFloat"])
@pytest.mark.parametrize("dewarp", [False, True])
@pytest.mark.parametrize("device", [False, True])
def test_filter_xyz_fused_matches_oracle(ob, lut_kind, dewarp, device):
    import torch
    from ouster_sdk_b200 import pyapi
    info = _golden_info(ob)
    lut = getattr(pyapi, lut_kind)(info)
    dt = lut._lut.dtype
    d, off = lut._lut.direction, lut._lut.offset
    # single: a device scan without RANGE, so every field takes the second return's mask
    for single in ((False, True) if device else (False,)):
        fr = _host_frame(ob, info, seed=11, f16=False)
        rs = np.random.default_rng(3)
        fr.field("RANGE")[...] = rs.integers(0, 30000, (info.h, info.w), dtype=np.uint32)
        fr.field("RANGE").reshape(-1)[::13] = 0
        if single:   # only the second return: every field takes its mask
            fr.field("RANGE2")[...] = fr.field("RANGE")[::-1]
        ang = np.linspace(0, 1.0, info.w)
        fr.body_to_world[:, 0, 0] = np.cos(ang)
        fr.body_to_world[:, 0, 1] = -np.sin(ang)
        fr.body_to_world[:, 1, 0] = np.sin(ang)
        fr.body_to_world[:, 1, 1] = np.cos(ang)
        fr.body_to_world[:, 2, 3] = np.linspace(-1, 1, info.w)
        o = _oracle_of(fr, info)

        def pts(name):
            p = orc.cartesian(o.field(name), d, off).reshape(info.h, info.w, 3)
            return orc.dewarp(p, o.body_to_world.astype(dt)) if dewarp else p

        # bound at a projected coordinate (and its neighbours one ulp away)
        z = pts("RANGE")[..., 2].reshape(-1)
        bound = float(z[1000])
        lo = float(np.nextafter(np.array(bound, dt), np.array(-np.inf, dt)))
        hi = float(np.nextafter(np.array(bound, dt), np.array(np.inf, dt)))
        for lower, upper in ((bound, 1e9), (-1e9, bound), (lo, hi), (-0.5, 0.5)):
            fr2 = _host_frame(ob, info, seed=11, f16=False)
            for n in fr.fields:
                fr2.field(n)[...] = fr.field(n)
            fr2.body_to_world[:] = fr.body_to_world
            o2 = _oracle_of(fr2, info)
            if single:
                o2._f.pop("RANGE")
            target = _device_scan(ob, info, fr2) if device else fr2
            if single:
                del target._fields["RANGE"]
            ob.frame_ops.filter_xyz(target, lut, 2, lower, upper, 4, dewarp_points=dewarp)
            ofo.filter_xyz(o2, pts, 2, lower, upper, 4)
            if device:
                torch.cuda.synchronize()
                _assert_same(_dev_fields(target, fr2), o2)
            else:
                _assert_same(_host_fields(fr2), o2)


def test_batch_with_different_shift_tables_is_refused_and_leaves_frames_alone(ob):
    import torch
    a, b = _info(ob, 32, 512, seed=1), _info(ob, 32, 512, seed=2)
    assert not np.array_equal(a.pixel_shift_by_row, b.pixel_shift_by_row)
    fa, fb = _host_frame(ob, a, f16=False), _host_frame(ob, b, seed=3, f16=False)
    sa, sb = _device_scan(ob, a, fa), _device_scan(ob, b, fb)
    before = [{n: s.field(n).clone() for n in s.fields} for s in (sa, sb)]
    with pytest.raises(ValueError, match="must share pixel_shift_by_row"):
        ob.frame_ops.filter_uv([sa, sb], "v", 10, 300)
    for s, bf in zip((sa, sb), before):
        for n in s.fields:
            assert torch.equal(s.field(n), bf[n]), n
    # each frame on its own uses its own shifts and matches the oracle
    for s, f, info in ((sa, fa, a), (sb, fb, b)):
        o = _oracle_of(f, info)
        ob.frame_ops.filter_uv(s, "v", 10, 300)
        ofo.filter_uv(o, "v", 10, 300)
        torch.cuda.synchronize()
        _assert_same(_dev_fields(s, f), o)
    # frames that share a table still go in one launch and equal single calls
    fc = _host_frame(ob, a, seed=5, f16=False)
    sc1, sc2 = _device_scan(ob, a, fc), _device_scan(ob, a, fc)
    sd1, sd2 = _device_scan(ob, a, fa), _device_scan(ob, a, fa)
    n0 = ob.kernel_launch_count("frame_ops")
    ob.frame_ops.filter_uv([sc1, sd1], "v", 10, 300)
    assert ob.kernel_launch_count("frame_ops") - n0 == 1
    ob.frame_ops.filter_uv(sc2, "v", 10, 300)
    ob.frame_ops.filter_uv(sd2, "v", 10, 300)
    torch.cuda.synchronize()
    for x, y in ((sc1, sc2), (sd1, sd2)):
        for n in x.fields:
            assert torch.equal(x.field(n), y.field(n)), n


@pytest.mark.parametrize("device", [False, True])
def test_non_pixel_fields(ob, device):
    import torch
    info = _info(ob, 16, 256)
    fr = _host_frame(ob, info, f16=False)
    fr.add_field("IMU", np.float64, 3, field_class=2)        # COLUMN_FIELD, w x 3
    fr.add_field("PKT", np.uint32, field_class=3)            # PACKET_FIELD
    fr.field("IMU")[...] = np.arange(fr.w * 3).reshape(fr.w, 3)
    fr.field("PKT")[...] = 5
    assert fr.field("IMU").shape == (fr.w, 3) and fr.field_class("IMU") == 2
    src = _device_scan(ob, info, fr) if device else fr
    with pytest.raises(ValueError, match=r"^Only PIXEL_FIELD frame fields are supported here; requested non-pixel "
                                         r"fields: \[IMU, PKT\]$"):
        ob.frame_ops.clip(src, ["RANGE", "IMU", "PKT", "NOPE"], 0, 1)
    with pytest.raises(ValueError, match=r"requested non-pixel fields: \['IMU'\]$"):
        ob.frame_ops.filter_xyz(src, lambda r: np.zeros((fr.h, fr.w, 3)), 0, filtered_fields=["IMU"])
    with pytest.raises(IndexError, match=r"^Field 'NOPE' not found in LidarFrame\.$"):
        ob.frame_ops.filter_field(src, "NOPE", 0, 1)
    o = _oracle_of(fr, info)
    o._f["IMU"] = (o._f["IMU"][0], 10, ofo.COLUMN_FIELD)
    o._f["PKT"] = (o._f["PKT"][0], 3, ofo.PACKET_FIELD)
    ob.frame_ops.clip(src, [], 100, 30000, 7)          # every pixel field; the others are left alone
    ofo.clip(o, [], 100, 30000, 7)
    if device:
        torch.cuda.synchronize()
        _assert_same(_dev_fields(src, fr), o)
    else:
        _assert_same(_host_fields(fr), o)
    out = ob.frame_ops.select_by_index(src, [3, 1])
    get = (lambda n: out.field(n).cpu().numpy().view(o.field(n).dtype)) if device else out.field
    assert np.array_equal(get("IMU"), o.field("IMU")) and np.array_equal(get("PKT"), o.field("PKT"))
    assert np.array_equal(get("RANGE"), o.field("RANGE")[[3, 1]])


def test_second_return_mapping_and_callable_lut(ob):
    info = _info(ob, 16, 128)
    rs = np.random.default_rng(9)
    p1 = rs.uniform(-5, 5, (16, 128, 3)).astype(np.float32)
    p2 = rs.uniform(-5, 5, (16, 128, 3)).astype(np.float32)
    fr = _host_frame(ob, info, f16=False)
    o = _oracle_of(fr, info)

    def lut(rng):
        return p1 if rng is fr.field("RANGE") or np.shares_memory(rng, fr.field("RANGE")) else p2

    ob.frame_ops.filter_xyz(fr, lut, 0, -1.0, 1.3)
    ofo.filter_xyz(o, lambda n: p1 if n == "RANGE" else p2, 0, -1.0, 1.3)
    _assert_same(_host_fields(fr), o)
    m2 = (p2[..., 0] >= np.float32(-1.0)) & (p2[..., 0] <= np.float32(1.3))
    assert np.all(fr.field("SIGNAL2")[m2] == 0)


@pytest.mark.parametrize("device", [False, True])
def test_select_and_reduce(ob, device):
    import torch
    info = _golden_info(ob)
    fr = _host_frame(ob, info, seed=4)
    fr.add_field("E", np.uint16, 3)
    fr.field("E")[...] = np.arange(fr.field("E").size, dtype=np.uint16).reshape(fr.field("E").shape)
    fr.frame_id = 77
    fr.timestamp[:] = np.arange(info.w)
    idx = [5, 0, 127, 64]
    src = _device_scan(ob, info, fr) if device else fr
    out = ob.frame_ops.select_by_index(src, idx)
    outm = ob.frame_ops.select_by_index(src, idx, update_metadata=True)
    for n in fr.fields:
        got = out.field(n).cpu().numpy().view(fr.field(n).dtype) if device else out.field(n)
        assert np.array_equal(got.view(np.uint8), fr.field(n)[idx].view(np.uint8)), n
    host = out.host if device else out
    assert host.frame_id == 77 and np.array_equal(host.timestamp, fr.timestamp)
    if device:
        assert out.info is None and outm.info is not None
    else:
        assert out.sensor_info is None and outm.sensor_info is not None
        assert outm.sensor_info.prod_line == "OS-1-4"
    red = ob.frame_ops.reduce_by_factor(src, 128)
    got = red.field("RANGE").cpu().numpy().view(np.uint32) if device else red.field("RANGE")
    assert np.array_equal(got, fr.field("RANGE")[[64]])
    torch.cuda.synchronize()


@pytest.mark.parametrize("factor", [2, 4, 128])
def test_xyzlut_of_reduced_metadata(ob, factor):
    from ouster_sdk_b200 import pyapi
    info = _golden_info(ob)
    small = ob.frame_ops.reduce_by_factor_metadata(info, factor)
    idx = ob.frame_ops.reduce_factor_to_indices(factor, info.h)
    assert small.h == len(idx) and np.array_equal(small.pixel_shift_by_row, info.pixel_shift_by_row[idx])
    for kind in ("XYZLut", "XYZLutFloat"):
        big, red = getattr(pyapi, kind)(info), getattr(pyapi, kind)(small)
        rng = np.random.default_rng(1).integers(0, 50000, (info.h, info.w), dtype=np.uint32)
        a = big(rng)[idx]
        b = red(np.ascontiguousarray(rng[idx]))
        assert np.array_equal(a, b), kind


def test_batch_equals_single_calls_in_one_launch(ob):
    import torch
    info = _info(ob, 128, 2048)
    frames = [_host_frame(ob, info, seed=s, f16=False) for s in range(4)]
    scans = [_device_scan(ob, info, f) for f in frames]
    singles = [_device_scan(ob, info, f) for f in frames]
    n0 = ob.kernel_launch_count("frame_ops")
    ob.frame_ops.clip(scans, [], 100, 30000, 7)
    assert ob.kernel_launch_count("frame_ops") - n0 == 1
    for s in singles:
        ob.frame_ops.clip(s, [], 100, 30000, 7)
    n0 = ob.kernel_launch_count("frame_ops")
    ob.frame_ops.filter_uv(scans, "v", 10, 900)
    assert ob.kernel_launch_count("frame_ops") - n0 == 1
    for s in singles:
        ob.frame_ops.filter_uv(s, "v", 10, 900)
    torch.cuda.synchronize()
    for a, b, f in zip(scans, singles, frames):
        for n in f.fields:
            assert torch.equal(a.field(n), b.field(n)), n


def test_graph_capture_replay_is_bit_identical(ob):
    import torch
    info = _info(ob, 64, 1024)
    fr = _host_frame(ob, info, f16=False)
    base = _device_scan(ob, info, fr)
    work = _device_scan(ob, info, fr)
    ref = _device_scan(ob, info, fr)
    m = torch.as_tensor(_MASK[(64, 1024)]).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up outside capture
        ob.frame_ops.clip(ref, [], 100, 30000, 7)
        ob.frame_ops.filter_uv(ref, "v", 3, 500)
        ob.frame_ops.mask(ref, [], m)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        ob.frame_ops.clip(work, [], 100, 30000, 7)
        ob.frame_ops.filter_uv(work, "v", 3, 500)
        ob.frame_ops.mask(work, [], m)
    for _ in range(2):
        for n in fr.fields:
            work.field(n).copy_(base.field(n))
        g.replay()
        torch.cuda.synchronize()
        for n in fr.fields:
            assert torch.equal(work.field(n), ref.field(n)), n


def test_chain_packets_reduce_clip_filter_xyz(ob):
    import torch
    from ouster_sdk_b200 import pyapi
    info = _golden_info(ob)
    rs = np.random.default_rng(2)
    src = ob.LidarScan(info)
    masks = {f[0]: f[6] for f in info.fields()}
    for n in src.fields:
        a = src.field(n)
        a[...] = (rs.integers(0, 1 << 32, size=a.shape, dtype=np.uint64) & np.uint64(masks[n])).astype(a.dtype)
    for n in ("RANGE", "RANGE2"):
        src.field(n)[...] = rs.integers(0, 40000, (info.h, info.w), dtype=np.uint32) & np.uint32(masks[n])
    src.measurement_id[:] = np.arange(info.w)
    src.status[:] = 1
    src.packet_timestamp[:] = 1 + np.arange(src.n_packets)
    packets, ts = ob.frame_to_packets(src, info)
    batcher = pyapi.DeviceScanBatcher(info)
    scan = batcher.new_scan()
    for p, t in zip(packets, ts):
        batcher(p, int(t), scan)
    torch.cuda.synchronize()
    # oracle chain on the host copy of the source frame, compared after every stage
    o = ofo.Frame(info.h, info.w, info.pixel_shift_by_row)
    for n in src.fields:
        o.add(n, src.field(n).copy(), src.field_tag(n))

    def same(stage, scan_):
        for n in ["RANGE", "RANGE2"] + src.fields:
            got = scan_.field(n).cpu().numpy().view(o.field(n).dtype)
            assert np.array_equal(got, o.field(n)), (stage, n, int(np.count_nonzero(got != o.field(n))))

    same("decode", scan)
    small = ob.frame_ops.reduce_by_factor_metadata(info, 2)
    lut2 = pyapi.XYZLutFloat(small)
    d, off = lut2._lut.direction, lut2._lut.offset
    # the device chain, traced: no device-to-host copy may happen between the stages
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        red = ob.frame_ops.reduce_by_factor(scan, 2, update_metadata=True)
        ob.frame_ops.clip(red, ["RANGE"], 500, 30000)
        ob.frame_ops.filter_xyz(red, lut2, 2, -0.3, 0.3)
        xyz_dev = lut2(red.field("RANGE").view(torch.int32))
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert any("frame_mask_kernel" in n for n in names) and any("frame_rows_kernel" in n for n in names)
    d2h = [n for n in names if "DtoH" in n or "Device -> Pageable" in n or "Device -> Pinned" in n]
    assert not d2h, d2h
    o = ofo.select_rows(o, list(range(0, info.h, 2)))
    ofo.clip(o, ["RANGE"], 500, 30000)
    ofo.filter_xyz(o, lambda n: orc.cartesian(o.field(n), d, off).reshape(o.h, o.w, 3), 2, -0.3, 0.3)
    same("filter_xyz", red)
    xyz = xyz_dev.cpu().numpy()
    assert np.array_equal(xyz.reshape(-1, 3), orc.cartesian(o.field("RANGE"), d, off))
