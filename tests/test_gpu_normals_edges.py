"""GPU surface normals (ob_normals) beyond the room scene: real sensor frames, one scene per branch of
compute_unit_normals, the vertical-subtent search, dual returns whose first return has a subtent of 0,
degenerate shapes and search ranges, non-finite input and batched frames through the C ABI.

Every GPU result is compared bit for bit with the oracle given the subtent the GPU reports (the device
acos may differ from glibc's in the last bit), and, where the geometry gives one, with a float64
expectation (tests/test_oracle_normals.py builds the scenes and their checks)."""
import ctypes as C
from importlib import import_module

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import oracle as orc
from tests.helpers import load_fixture
from tests.test_gpu_normals import noisy_scene, ulp_close
from tests.test_oracle_normals import (BRANCH_CASES, SUBTENT_SEARCH_CASES, beams_of, dual_zero_subtent_scene,
                                       expected_subtent, room_scene, subtent_scene)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


def gpu_vs_oracle(ob, xyz, rng, *dual, org, equal_nan=False, **kw):
    """GPU normals, checked bit for bit against the oracle fed the GPU's subtent; returns (normals, subtent)."""
    got, sub = ob.normals(xyz, rng, *dual, sensor_origins_xyz=org, return_subtent=True, **kw)
    kw = dict(kw, vertical_subtent=kw.get("vertical_subtent") or sub)
    want = orc.normals(xyz, rng, *dual, sensor_origins_xyz=org, **kw)
    for g, r in zip(got, want) if dual else ((got, want),):
        assert np.array_equal(g, r, equal_nan=equal_nan)
    return got, sub


# ---- real sensor frames --------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sensor_frames():
    """RANGE / RANGE2 of two recorded frames decoded by the oracle batcher, projected through the
    oracle's LUT and destaggered: (xyz, range, xyz2, range2, per-column origins)."""
    out = {}
    for name in ("OS-1-128_767798045_1024x10_20230712_120049", "OS-0-32-U1_v2.2.0_1024x10"):
        meta, packets = load_fixture(name)
        pf = orc.PacketFormat(meta["profile"], meta["h"], meta["w"], meta["columns_per_packet"],
                              orc.HEADER_FUSA if meta["header_type"] == "FUSA" else orc.HEADER_STANDARD)
        frame = orc.Frame(pf, with_window=False)
        b = orc.Batcher(pf, init_id=meta["init_id"], column_window=meta["column_window"])
        for p in packets:
            b.batch(p, 1234, frame)
        h, w = meta["h"], meta["w"]
        shifts = np.asarray(meta["pixel_shift_by_row"], np.int32)
        d, o = orc.make_xyz_lut(w, h, 0.001, meta["beam_to_lidar_transform"], meta["lidar_to_sensor_transform"],
                                meta["beam_azimuth_angles"], meta["beam_altitude_angles"])
        rets = []
        for field in ("RANGE", "RANGE2"):
            rng = np.array(frame.field(field), np.uint32)
            xyz = orc.cartesian(rng, d, o).reshape(h, w, 3)
            rets += [orc.destagger(xyz, shifts), orc.destagger(rng, shifts)]
        assert np.count_nonzero(rets[1]) > 10000 and np.count_nonzero(rets[3]) > 100    # both hold a partial frame
        org = orc.destagger(o.reshape(h, w, 3), shifts).mean(axis=0)
        out[name] = (*rets, org)
    return out


@pytest.mark.parametrize("search", [1, 3])
@pytest.mark.parametrize("name", ["OS-1-128_767798045_1024x10_20230712_120049", "OS-0-32-U1_v2.2.0_1024x10"])
def test_sensor_frame_bit_exact(ob, sensor_frames, name, search):
    x1, r1, x2, r2, org = sensor_frames[name]
    n, sub = gpu_vs_oracle(ob, x1, r1, org=org, pixel_search_range=search)
    assert ulp_close(sub, orc.normals_vertical_subtent(x1, r1, org))
    assert np.count_nonzero(np.any(n != 0, axis=-1)) > 0.8 * np.count_nonzero(r1)
    (d1, d2), dsub = gpu_vs_oracle(ob, x1, r1, x2, r2, org=org, pixel_search_range=search)
    assert dsub == sub and np.array_equal(d2[r2 == 0], np.zeros_like(d2[r2 == 0]))


# ---- one scene per branch --------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(BRANCH_CASES))
def test_branch_scene(ob, name):
    c = BRANCH_CASES[name]()
    got, _ = gpu_vs_oracle(ob, c["xyz"], c["rng"], org=c["org"], **c["kw"])
    c["check"](got)


def test_thresholds_are_wired(ob):
    """A non-default target distance and angle of incidence change the answer, and an angle below 1e-6
    gives what 1e-6 gives."""
    xyz, rng, _, _ = noisy_scene(24, 96, 3)      # neighbours 1.4 m (vertical) and 2.6 m (horizontal) apart
    org = np.zeros((96, 3))
    base, _ = gpu_vs_oracle(ob, xyz, rng, org=org, pixel_search_range=3)
    for kw in (dict(target_distance_m=3.0), dict(min_angle_of_incidence_rad=np.deg2rad(45.0))):
        other, _ = gpu_vs_oracle(ob, xyz, rng, org=org, pixel_search_range=3, **kw)
        assert np.count_nonzero(np.any(other != base, axis=-1)) > 0.3 * np.count_nonzero(rng)
    tiny, _ = gpu_vs_oracle(ob, xyz, rng, org=org, pixel_search_range=3, min_angle_of_incidence_rad=1e-9)
    assert np.array_equal(tiny, ob.normals(xyz, rng, org, 3, min_angle_of_incidence_rad=1e-6))


# ---- the vertical-subtent search -------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SUBTENT_SEARCH_CASES))
def test_subtent_search(ob, name):
    w, cols, want_col = SUBTENT_SEARCH_CASES[name]
    xyz, rng, org = subtent_scene(13, w, cols)
    _, sub = gpu_vs_oracle(ob, xyz, rng, org=org)
    assert ulp_close(sub, expected_subtent(xyz, rng, org, want_col))
    assert ulp_close(sub, orc.normals_vertical_subtent(xyz, rng, org))


@pytest.mark.parametrize("h,valid", [(1, True), (2, False), (2, "one_row"), (5, False)])
def test_subtent_fallback(ob, h, valid):
    xyz, rng, _ = room_scene(h, 16)
    if valid is False:
        rng[:] = 0
    elif valid == "one_row":
        rng[1] = 0
    _, sub = gpu_vs_oracle(ob, xyz, rng, org=np.zeros((16, 3)))
    assert sub == (0.5 * np.pi) / max(1, h - 1)


# ---- dual returns whose first return has a vertical subtent of 0 --------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kind", ["parallel", "inf"])
def test_dual_zero_subtent_second_return_derives_its_own(ob, kind, dtype):
    x1, r1, x2, r2, org = dual_zero_subtent_scene(kind)
    x1, x2 = x1.astype(dtype), x2.astype(dtype)
    (n1, n2), sub = ob.normals(x1, r1, x2, r2, org, return_subtent=True)
    assert sub == 0.0
    # the reference's second pass is the swapped call's first pass (both derive the subtent of xyz2):
    # GPU against GPU, so the device acos is on both sides
    (m2, m1), sub2 = ob.normals(x2, r2, x1, r1, org, return_subtent=True)
    assert sub2 > 0
    assert np.array_equal(n2, m2)
    # the swapped call shares sub2 > 0, so the oracle fed it reproduces it bit for bit
    w2, w1 = orc.normals(x2.astype(np.float64), r2, x1.astype(np.float64), r1, org, vertical_subtent=sub2)
    assert np.array_equal(m2, w2.astype(dtype)) and np.array_equal(m1, w1.astype(dtype), equal_nan=True)
    # the first return is unchanged: its pass uses 0, which the oracle derives exactly as well
    r1_want, _ = orc.normals(x1.astype(np.float64), r1, x2.astype(np.float64), r2, org)
    assert np.array_equal(n1, r1_want.astype(dtype), equal_nan=True)


def test_dual_override_is_shared_by_both_returns(ob):
    x1, r1, x2, r2, org = dual_zero_subtent_scene("parallel")
    (n1, n2), sub = ob.normals(x1, r1, x2, r2, org, vertical_subtent=0.004, return_subtent=True)
    assert sub == 0.004
    w1, w2 = orc.normals(x1, r1, x2, r2, org, vertical_subtent=0.004)
    assert np.array_equal(n1, w1) and np.array_equal(n2, w2)


# ---- shapes and search ranges ----------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(1, 1), (1, 40), (24, 1), (2, 2), (8, 3), (37, 200)])
def test_shapes_and_search_ranges(ob, h, w):
    xyz, rng, xyz2, rng2 = noisy_scene(h, w, 31 + h + w, p_zero=0.1)
    org = np.random.default_rng(h * w).normal(0, 0.05, (w, 3))
    beam = beams_of(xyz, org)
    for search in sorted({0, 1, 3, h, h + 2, w + 1, 2 * w + 3}):
        n, sub = gpu_vs_oracle(ob, xyz, rng, org=org, pixel_search_range=search)
        assert ulp_close(sub, orc.normals_vertical_subtent(xyz, rng, org))
        if h == 1:
            assert sub == 0.5 * np.pi
        if search == 0:                                 # no neighbours at all: case A everywhere
            assert np.array_equal(n[rng > 0], -beam[rng > 0])
        gpu_vs_oracle(ob, xyz, rng, xyz2, rng2, org=org, pixel_search_range=search)


# ---- non-finite and inconsistent input -------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_non_finite_and_zero_xyz_with_a_range(ob, dtype):
    xyz, rng, xyz2, rng2 = noisy_scene(16, 40, 8, p_zero=0.05)
    for x, r in ((xyz, rng), (xyz2, rng2)):
        x[5, 7] = (np.nan, 1.0, 2.0)
        x[8, 20, 0] = np.inf
        x[3, 30, 2] = -np.inf
        x[10, 10] = 0.0                                 # zero beam
        x[12, 3] = (np.inf, -np.inf, np.nan)
        r[[5, 8, 3, 10, 12], [7, 20, 30, 10, 3]] = 5000
    org = np.zeros((40, 3))
    x1, x2 = xyz.astype(dtype), xyz2.astype(dtype)
    n, sub = ob.normals(x1, rng, org, return_subtent=True)
    assert sub > 0
    want = orc.normals(x1.astype(np.float64), rng, sensor_origins_xyz=org, vertical_subtent=sub)
    assert np.array_equal(n, want.astype(dtype), equal_nan=True)
    assert np.array_equal(n[10, 10], np.zeros(3, dtype))       # a valid pixel whose beam is zero
    assert np.all(np.isfinite(n[rng == 0])) and np.all(n[rng == 0] == 0)
    (d1, d2), dsub = ob.normals(x1, rng, x2, rng2, org, return_subtent=True)
    w1, w2 = orc.normals(x1.astype(np.float64), rng, x2.astype(np.float64), rng2, org, vertical_subtent=dsub)
    assert np.array_equal(d1, w1.astype(dtype), equal_nan=True)
    assert np.array_equal(d2, w2.astype(dtype), equal_nan=True)


# ---- batched frames through the C ABI --------------------------------------------------------------
def _frames(h, w):
    """Three different dual-return frames; the last has a first-return subtent of 0."""
    f0 = noisy_scene(h, w, 41)
    f1 = noisy_scene(h, w, 42, p_zero=0.4)
    x1, r1, x2, r2, _ = dual_zero_subtent_scene("inf", h, w, seed=9)
    return [f0, f1, (x1, r1, x2, r2)]


@pytest.mark.parametrize("per_frame_origins", [True, False])
@pytest.mark.parametrize("dtype,on_device", [(np.float32, False), (np.float64, False), (np.float32, True),
                                             (np.float64, True)])
def test_batched_frames_equal_single_frame_calls(ob, dtype, on_device, per_frame_origins):
    import torch
    capi = import_module(ob.__name__ + "._capi")
    h, w, F = 24, 64, 3
    n_px = h * w
    frames = _frames(h, w)
    rs = np.random.default_rng(5)
    orgs = rs.normal(0, 0.05, (F, w, 3)) if per_frame_origins else np.broadcast_to(rs.normal(0, 0.05, (w, 3)),
                                                                                    (F, w, 3))
    xfs, rfs, ofs = n_px * 3 + 5, n_px + 3, n_px * 3 + 7          # padded frame strides, in elements
    sentinel = -12345.0
    bx = [np.full(F * xfs, 7.0e30, dtype) for _ in range(2)]     # inputs: padding the kernel must not read
    br = [np.full(F * rfs, 0xDEADBEEF, np.uint32) for _ in range(2)]
    for f, fr in enumerate(frames):
        for k in range(2):
            bx[k][f * xfs: f * xfs + n_px * 3] = fr[2 * k].astype(dtype).ravel()
            br[k][f * rfs: f * rfs + n_px] = fr[2 * k + 1].ravel()
    bo = np.array(orgs if per_frame_origins else orgs[0]).ravel()
    bn = [np.full(F * ofs, sentinel, dtype) for _ in range(2)]
    bsub = np.full(F, sentinel)
    bufs = bx + br + [bo] + bn + [bsub]
    if on_device:
        bufs = [torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).cuda() for a in bufs]
        ptr = lambda a: a.data_ptr()
        st = ob.Stream(0, cuda_stream=torch.cuda.current_stream().cuda_stream)
    else:
        ptr = lambda a: a.ctypes.data
        st = ob.Stream(0)
    io = capi.NormalsIO()
    io.n_frames, io.h, io.w = F, h, w
    io.xyz, io.xyz2, io.range, io.range2 = (ptr(a) for a in bufs[:4])
    io.sensor_origins_xyz, io.n_origins, io.origins_frame_stride = ptr(bufs[4]), w, 3 * w if per_frame_origins else 0
    io.normals, io.normals2, io.vertical_subtent_out = (ptr(a) for a in bufs[5:])
    io.xyz_frame_stride, io.range_frame_stride, io.normals_frame_stride = xfs, rfs, ofs
    io.pixel_search_range, io.min_angle_of_incidence_rad, io.target_distance_m = 2, np.pi / 180.0, 0.025
    capi.check(capi.lib.ob_normals(capi.OB_F64 if dtype == np.float64 else capi.OB_F32, C.byref(io), st.h))
    if on_device:
        torch.cuda.synchronize()
        bn, bsub = [a.cpu().numpy() for a in bufs[5:7]], bufs[7].cpu().numpy()
    else:
        st.sync()
    for f, (x1, r1, x2, r2) in enumerate(frames):
        (s1, s2), sub = ob.normals(x1.astype(dtype), r1, x2.astype(dtype), r2, orgs[f], 2, return_subtent=True)
        assert bsub[f] == sub
        for k, single in enumerate((s1, s2)):
            got = bn[k][f * ofs: f * ofs + n_px * 3].reshape(h, w, 3)
            assert np.array_equal(got, single, equal_nan=True), (f, k)
            assert np.all(bn[k][f * ofs + n_px * 3: (f + 1) * ofs] == sentinel)      # padding untouched
    assert bsub[2] == 0.0 and np.all(bsub[:2] > 0)
