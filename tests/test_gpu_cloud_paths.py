"""K1 (ob_scan_to_cloud) down every path its host code can pick, driven through the C ABI so that strides and
pointer offsets are the test's, and compared element by element with the CPU oracle: launch geometries (tile width,
ring depth, compute threads, CTAs per SM, store lag, the wide single-return geometry), partial last tiles, row
shifts of every alignment that wrap past the last column, every subset of the outputs, padded / unaligned /
shared-range strides in host and device memory, the pose-fused path and its row blocks, extreme ranges and the
LUT-free projection.  Every output starts as a 0xA5 byte pattern: every pixel must be overwritten and every byte
between frames and returns must still hold the pattern afterwards.  A profiler test checks which kernel each kind of
case ran, so that a slip in the alignment rules cannot quietly send the matrix to the generic kernel."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import oracle as orc
from tests.helpers import default_os1_64, load_fixture, random_lut, random_range

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
TAIL_BYTES = 64          # sentinel bytes after the last block of every buffer
OUTS = ("xyz", "rd", "xd")
UINT = {4: np.uint32, 8: np.uint64}

# library defaults of the K1 tunables (OB_* environment variables override them at load, as in ob_api.cu)
K1_TUNABLES = {"cloud_tw": 512, "cloud_stages": 3, "cloud_threads": 128, "cloud_ctas_per_sm": 3,
               "cloud_store_lag": 1, "cloud_pose_tw": 256, "cloud_pose_stages": 4, "cloud_pose_ctas_per_sm": 5,
               "cloud_pose_threads": 64, "cloud_pose_rows": 16, "force_generic": 0}
AUTO_OFF_ENV = ("OB_CLOUD_TW", "OB_CLOUD_STAGES", "OB_CLOUD_CTAS_PER_SM", "OB_CLOUD_THREADS")


def _env_default(name, value):
    v = os.environ.get("OB_" + name.upper())
    return int(v) if v else value


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


@pytest.fixture
def tunables(ob):
    """set(**tunables) for one case; every K1 tunable and the automatic geometry are restored afterwards, since the
    other test files in the process run K1 with the defaults"""
    def set_(**kw):
        for k, v in kw.items():
            ob.set_tunable(k, v)
    try:
        yield set_
    finally:
        for k, v in K1_TUNABLES.items():
            ob.set_tunable(k, _env_default(k, v))
        ob.set_tunable("cloud_auto", 0 if any(os.environ.get(e) for e in AUTO_OFF_ENV) else 1)


# ------------------------------------------------------------------------------------------------------------------
# strided buffers and the call
# ------------------------------------------------------------------------------------------------------------------
class Strided:
    """[F][R][n] elements of `dtype` at ptr + f*fs + r*rs (+ offset elements into the buffer), in one flat byte
    buffer that starts as the sentinel: a numpy array, or a CUDA tensor when `device`."""

    def __init__(self, F, R, n, dtype, fs, rs, offset=0, device=False, data=None):
        self.F, self.R, self.n, self.fs, self.rs, self.off = F, R, n, fs, rs, offset
        self.dtype, self.device = np.dtype(dtype), device
        it = self.dtype.itemsize
        n_el = offset + (F - 1) * fs + (R - 1) * rs + n
        host = np.full(n_el * it + TAIL_BYTES, SENTINEL, np.uint8)
        if data is not None:
            typed = host[:n_el * it].view(self.dtype)
            for f in range(F):
                for r in range(R):
                    typed[self.start(f, r):self.start(f, r) + n] = data[f, r].reshape(-1)
        if device:
            import torch
            self.buf = torch.from_numpy(host).cuda()
        else:
            self.buf = host

    def start(self, f, r):
        return self.off + f * self.fs + r * self.rs

    @property
    def ptr(self):
        base = self.buf.data_ptr() if self.device else self.buf.ctypes.data
        return base + self.off * self.dtype.itemsize

    def host_bytes(self):
        return self.buf.cpu().numpy() if self.device else self.buf

    def blocks(self):
        """(values [F, R, n], number of bytes outside the blocks that lost the sentinel)"""
        b = self.host_bytes()
        it = self.dtype.itemsize
        n_el = (b.size - TAIL_BYTES) // it
        typed = b[:n_el * it].view(self.dtype)
        vals = np.stack([np.stack([typed[self.start(f, r):self.start(f, r) + self.n] for r in range(self.R)])
                         for f in range(self.F)])
        spans = sorted({(self.start(f, r) * it, (self.start(f, r) + self.n) * it)
                        for f in range(self.F) for r in range(self.R)})
        bad, pos = 0, 0
        for s, e in spans:
            if s > pos:
                bad += int(np.count_nonzero(b[pos:s] != SENTINEL))
            pos = max(pos, e)
        bad += int(np.count_nonzero(b[pos:] != SENTINEL))
        return vals, bad


def layout(kind, F, R, H, W, dtype):
    """name -> (frame stride, return stride, offset), in elements of the array's scalar type"""
    it = np.dtype(dtype).itemsize
    lay = {}
    for name, n, esz in (("range", H * W, 4), ("rd", H * W, 4), ("xyz", 3 * H * W, it), ("xd", 3 * H * W, it)):
        v = 16 // esz  # elements per 16 bytes
        if kind == "padded":      # gaps of 16 and 48 bytes: still 16-byte aligned slices, the TMA kernel
            rs = n + v
            lay[name] = (R * rs + 3 * v, rs, 0)
        elif kind == "odd":       # strides that are not a multiple of 16 bytes: the generic kernel
            rs = n + 1
            lay[name] = (R * rs + 2, rs, 0)
        else:
            lay[name] = (R * n, n, 0)
    if kind == "range_fs0":       # one range image (both returns) for every frame
        lay["range"] = (0, H * W, 0)
    if kind == "range_off1":      # a device range one element past a 16-byte boundary: the generic kernel
        lay["range"] = (R * H * W, H * W, 1)
    if kind == "xyz_off1":        # a device XYZ output one element past a 16-byte boundary: the generic kernel
        lay["xyz"] = (R * 3 * H * W, 3 * H * W, 1)
    return lay


def takes_tma(H, W, dtype, lay, outs, device, force_generic=False):
    """launch_cloud's choice between the TMA and the generic kernel (host-staged arrays are freshly allocated,
    hence aligned; device arrays are where the caller put them)"""
    if force_generic or W % 4 or H > 512:
        return False
    it = np.dtype(dtype).itemsize

    def ok(name, esz):
        fs, rs, off = lay[name]
        unit = 16 // esz
        return fs % unit == 0 and rs % unit == 0 and (not device or (off * esz) % 16 == 0)
    return ok("range", 4) and all(ok(o, 4 if o == "rd" else it) for o in outs)


def kernel_names(dtype, R, tma, pose, analytic):
    t = "float" if np.dtype(dtype) == np.float32 else "double"
    if not tma:
        return [f"cloud_generic_kernel<{t}>"]
    b = lambda x: "true" if x else "false"
    names = [f"cloud_tma_kernel<{t}, {R}, {b(pose)}, {b(analytic and not pose)}>"]
    return ([f"pose_planes_kernel<{t}>"] if pose else []) + names


def prepare(ob, lut, shifts, rng, outs, *, poses=None, kind="contiguous", device=False, force_generic=False):
    """ob_scan_to_cloud over rng [F, R, H, W] into sentinel-filled outputs `outs` of layout `kind`.
    Returns ({name: Strided}, the kernels it should launch, the call: runs it, waits, checks the launch count)."""
    F, R, H, W = rng.shape
    dtype = lut.dtype
    lay = layout(kind, F, R, H, W, dtype)
    if kind == "range_fs0":
        assert all(np.array_equal(rng[f], rng[0]) for f in range(F))
    n = {"rd": H * W, "xyz": 3 * H * W, "xd": 3 * H * W}
    src = Strided(F, R, H * W, np.uint32, *lay["range"][:2], offset=lay["range"][2], device=device, data=rng)
    arrs = {o: Strided(F, R, n[o], np.uint32 if o == "rd" else dtype, *lay[o][:2], offset=lay[o][2], device=device)
            for o in outs}
    io = ob._capi.CloudIO()
    io.n_frames, io.n_returns = F, R
    io.range, (io.range_frame_stride, io.range_return_stride) = src.ptr, lay["range"][:2]
    if "xyz" in arrs:
        io.xyz, io.xyz_frame_stride, io.xyz_return_stride = arrs["xyz"].ptr, arrs["xyz"].fs, arrs["xyz"].rs
    if "rd" in arrs:
        io.range_destaggered, io.rd_frame_stride, io.rd_return_stride = arrs["rd"].ptr, arrs["rd"].fs, arrs["rd"].rs
    if "xd" in arrs:
        io.xyz_destaggered, io.xd_frame_stride, io.xd_return_stride = arrs["xd"].ptr, arrs["xd"].fs, arrs["xd"].rs
    if poses is not None:
        poses = np.ascontiguousarray(poses, dtype)
        io.poses, io.poses_frame_stride = poses.ctypes.data, (W * 16 if poses.ndim == 4 else 0)
    sh = np.ascontiguousarray(shifts, np.int32)
    need_lut = "xyz" in outs or "xd" in outs
    tma = takes_tma(H, W, dtype, lay, outs, device, force_generic)
    want = kernel_names(dtype, R, tma, poses is not None and need_lut, lut.analytic and need_lut)
    def call():
        if device:
            import torch
            torch.cuda.synchronize()
        st = ob.Stream(0)
        before = ob.kernel_launch_count("cloud")
        ob._capi.check(ob._capi.lib.ob_scan_to_cloud(lut._h, sh.ctypes.data, sh.size, C.byref(io), st.h))
        st.sync()
        assert ob.kernel_launch_count("cloud") - before == len(want), want
    call._keep = (src, poses)  # the call structure holds raw pointers into these
    return arrs, want, call


def scan_to_cloud(ob, lut, shifts, rng, outs, **kw):
    """prepare() and run; returns ({name: Strided}, the kernels it launched)"""
    arrs, want, call = prepare(ob, lut, shifts, rng, outs, **kw)
    call()
    return arrs, want


def oracle_outputs(rng, d, o, shifts, poses=None):
    """{name: [F, R, n]} of the oracle: cartesianT (+ dewarp) and destagger of every frame and return"""
    F, R, H, W = rng.shape
    xyz, rd = orc.pool_k1(rng, shifts, d, o)
    if poses is not None:
        for f in range(F):
            pf = poses[f] if poses.ndim == 4 else poses
            for r in range(R):
                xyz[f, r] = orc.dewarp(xyz[f, r].reshape(H, W, 3), pf).reshape(-1, 3)
    xd = np.stack([np.stack([orc.destagger(xyz[f, r].reshape(H, W, 3), shifts) for r in range(R)])
                   for f in range(F)])
    return {"xyz": xyz.reshape(F, R, -1), "rd": rd.reshape(F, R, -1), "xd": xd.reshape(F, R, -1)}


def same_bits(got, want):
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    return np.array_equal(got.view(UINT[got.dtype.itemsize]), want.view(UINT[want.dtype.itemsize]))


def check_outputs(arrs, want):
    for name, a in arrs.items():
        vals, bad = a.blocks()
        assert bad == 0, f"{name}: {bad} bytes between or after the blocks lost the sentinel"
        w = want[name]
        if not same_bits(vals, w):
            diff = np.flatnonzero(vals.reshape(-1).view(UINT[vals.dtype.itemsize])
                                  != w.reshape(-1).view(UINT[w.dtype.itemsize]))
            raise AssertionError(f"{name}: {diff.size} elements differ, first at flat index {diff[0]}")


def run_and_check(ob, lut, d, o, shifts, rng, outs=OUTS, poses=None, **kw):
    arrs, names = scan_to_cloud(ob, lut, shifts, rng, outs, poses=poses, **kw)
    check_outputs(arrs, oracle_outputs(rng, d, o, shifts, poses))
    return names


def ranges(F, R, H, W, seed, p_zero=0.4):
    return np.stack([np.stack([random_range(H, W, seed + 7 * f + r, p_zero) for r in range(R)]) for f in range(F)])


def shifts_for(H, W, seed):
    """random shifts of every alignment; negative ones only on power-of-two widths (DESIGN §9)"""
    rs = np.random.default_rng(seed)
    lo = -2 * W if (W & (W - 1)) == 0 else 0
    return rs.integers(lo, 2 * W, size=H).astype(np.int32)


def lut_of(ob, H, W, dtype, seed=3):
    d, o = random_lut(H * W, seed, dtype)
    return ob.XYZLutT.from_arrays(d, o, H, W), d, o


def random_poses(n_cols, dtype, seed, frames=None):
    rs = np.random.default_rng(seed)
    n = n_cols * (frames or 1)
    ang = rs.random(n) * 2 * np.pi
    p = np.zeros((n, 4, 4))
    p[:, 0, 0], p[:, 0, 1], p[:, 1, 0], p[:, 1, 1] = np.cos(ang), -np.sin(ang), np.sin(ang), np.cos(ang)
    p[:, 2, 2] = p[:, 3, 3] = 1
    p[:, :3, 3] = rs.random((n, 3)) * 10 - 5
    p = p.astype(dtype)
    return p if frames is None else p.reshape(frames, n_cols, 4, 4)


DTYPES = [pytest.param(np.float32, id="f32"), pytest.param(np.float64, id="f64")]
RETURNS = [pytest.param(1, id="R1"), pytest.param(2, id="R2")]

# ------------------------------------------------------------------------------------------------------------------
# launch geometry
# ------------------------------------------------------------------------------------------------------------------
GEOMETRIES = {
    "default": {},
    "store_lag0": {"cloud_store_lag": 0},
    "threads32": {"cloud_threads": 32},
    "threads256": {"cloud_threads": 256},
    "stages2": {"cloud_stages": 2},
    "stages8": {"cloud_stages": 8},
    "tw64": {"cloud_tw": 64},
    "tw2048": {"cloud_tw": 2048},
    "ctas1": {"cloud_ctas_per_sm": 1},
}
# (H, W, frames): partial last tiles of 104..488 pixels (1000) and of 4 pixels (516, 1028), and full-size frames
GEOMETRY_SHAPES = [(64, 1000, 7), (16, 516, 3), (32, 1028, 8), (128, 2048, 8)]
GEOMETRY_CASES = [pytest.param(g, s, id=f"{g}-{s[0]}x{s[1]}x{s[2]}") for g in GEOMETRIES for s in GEOMETRY_SHAPES]
# one CTA per SM over 16 frames of 128x1024: every CTA runs tens of tiles, its ring's phase wraps many times
GEOMETRY_CASES.append(pytest.param("ctas1", (128, 1024, 16), id="ctas1-128x1024x16"))


@pytest.mark.parametrize("R", RETURNS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("geometry,shape", GEOMETRY_CASES)
def test_geometry(ob, tunables, geometry, shape, dtype, R):
    H, W, F = shape
    tunables(**GEOMETRIES[geometry])
    lut, d, o = lut_of(ob, H, W, dtype)
    rng = ranges(F, R, H, W, seed=H + W)
    names = run_and_check(ob, lut, d, o, shifts_for(H, W, W), rng)
    assert names == kernel_names(dtype, R, True, False, False)


def test_wide_geometry(ob, tunables):
    """8 single-return float frames of 128x2048, tunables in their automatic state: 1024-pixel tiles, 4 stages"""
    H, W, F = 128, 2048, 8
    tunables(cloud_auto=1)
    lut, d, o = lut_of(ob, H, W, np.float32)
    rng = ranges(F, 1, H, W, seed=17)
    run_and_check(ob, lut, d, o, shifts_for(H, W, 5), rng)


# ------------------------------------------------------------------------------------------------------------------
# row shifts
# ------------------------------------------------------------------------------------------------------------------
def edge_shifts(W):
    """each q = shift & 3 on rows whose destination wraps past column W (for q = 0 the two bulk stores of a split
    tile), shifts of whole rows and several rows; negative ones on power-of-two widths only"""
    s = []
    for q in range(4):
        s += [q, 4 + q, W // 2 + q, W - 8 + q, W - 4 + q, W - 132 + q]
    s += [W, 3 * W + 2, W + 1, 2 * W - 1]
    if (W & (W - 1)) == 0:
        s += [-W, W - 1, -(W + 1), -1, -3, -4, -W // 2 - 1]
    return np.array(s, np.int32)


@pytest.mark.parametrize("R", RETURNS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("W", [512, 2048, 1000, 516])
def test_row_shifts(ob, W, dtype, R):
    shifts = edge_shifts(W)
    H, F = shifts.size, 2
    lut, d, o = lut_of(ob, H, W, dtype)
    run_and_check(ob, lut, d, o, shifts, ranges(F, R, H, W, seed=W))


# ------------------------------------------------------------------------------------------------------------------
# output subsets
# ------------------------------------------------------------------------------------------------------------------
SUBSETS = [("xyz",), ("rd",), ("xd",), ("xyz", "rd"), ("xyz", "xd"), ("rd", "xd"), ("xyz", "rd", "xd")]
SUBSET_CASES = [pytest.param(s, p, id="+".join(s) + ("-poses" if p else "")) for s in SUBSETS for p in (False, True)
                if not (p and s == ("rd",))]


@pytest.mark.parametrize("R", RETURNS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("outs,with_poses", SUBSET_CASES)
def test_output_subsets(ob, outs, with_poses, dtype, R):
    H, W, F = 24, 1028, 3
    lut, d, o = lut_of(ob, H, W, dtype)
    poses = random_poses(W, dtype, 2) if with_poses else None
    names = run_and_check(ob, lut, d, o, shifts_for(H, W, 9), ranges(F, R, H, W, seed=4), outs, poses)
    assert names == kernel_names(dtype, R, True, with_poses, False)


# ------------------------------------------------------------------------------------------------------------------
# strides and pointer offsets
# ------------------------------------------------------------------------------------------------------------------
STRIDE_CASES = [pytest.param(k, dev, id=f"{k}-{'device' if dev else 'host'}")
                for k in ("contiguous", "padded", "odd", "range_fs0") for dev in (False, True)]
STRIDE_CASES += [pytest.param("range_off1", True, id="range_off1-device"),
                 pytest.param("xyz_off1", True, id="xyz_off1-device")]


@pytest.mark.parametrize("R", RETURNS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind,device", STRIDE_CASES)
def test_strides(ob, kind, device, dtype, R):
    if device:
        pytest.importorskip("torch")
    H, W, F = 32, 1024, 3
    lut, d, o = lut_of(ob, H, W, dtype)
    rng = ranges(F, R, H, W, seed=6)
    if kind == "range_fs0":
        rng[:] = rng[0]
    names = run_and_check(ob, lut, d, o, shifts_for(H, W, 3), rng, kind=kind, device=device)
    generic = kind in ("odd", "range_off1", "xyz_off1")
    assert names == kernel_names(dtype, R, not generic, False, False)


# ------------------------------------------------------------------------------------------------------------------
# pose-fused path
# ------------------------------------------------------------------------------------------------------------------
POSE_GEOMETRIES = {
    "default": {},
    "rows4": {"cloud_pose_rows": 4},
    "rows64": {"cloud_pose_rows": 64},
    "tw64": {"cloud_pose_tw": 64},
    "tw1024": {"cloud_pose_tw": 1024},
    "stages2": {"cloud_pose_stages": 2},
    "stages8": {"cloud_pose_stages": 8},
    "threads32": {"cloud_pose_threads": 32},
    "threads256": {"cloud_pose_threads": 256},
    "ctas1": {"cloud_pose_ctas_per_sm": 1},
}


@pytest.mark.parametrize("per_frame", [pytest.param(False, id="shared"), pytest.param(True, id="per_frame")])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H", [20, 70])
@pytest.mark.parametrize("geometry", list(POSE_GEOMETRIES))
def test_pose_geometry(ob, tunables, geometry, H, dtype, per_frame):
    """row blocks of 4 / 16 / 64 rows over 20 and 70 rows leave the last block short"""
    W, F, R = 1024, 6, 2
    tunables(**POSE_GEOMETRIES[geometry])
    lut, d, o = lut_of(ob, H, W, dtype)
    poses = random_poses(W, dtype, 8, F if per_frame else None)
    names = run_and_check(ob, lut, d, o, shifts_for(H, W, H), ranges(F, R, H, W, seed=H), poses=poses)
    assert names == kernel_names(dtype, R, True, True, False)


# ------------------------------------------------------------------------------------------------------------------
# range values
# ------------------------------------------------------------------------------------------------------------------
EXTREMES = np.array([(1 << 19) - 1, (1 << 24) - 1, 1 << 24, (1 << 24) + 1, (1 << 32) - 1, (1 << 32) - 2, 1, 0],
                    np.uint32)


def extreme_ranges(F, R, H, W, seed):
    """all-zero rows, rows without a zero, and rows of the values where uint32 -> float rounds (2^24 + 1, 2^32 - 1)"""
    rng = ranges(F, R, H, W, seed)
    rs = np.random.default_rng(seed)
    rng[:, :, 1] = rs.integers(1, 1 << 32, size=(F, R, W), dtype=np.uint64).astype(np.uint32)
    for k, v in enumerate(EXTREMES):
        rng[:, :, 2 + k] = v
    rng[:, :, 2 + EXTREMES.size] = np.resize(EXTREMES, W)
    rng[:, :, 0] = 0
    rng[:, :, H - 1] = 0
    return rng


@pytest.mark.parametrize("R", RETURNS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("W", [pytest.param(1024, id="tma"), pytest.param(1030, id="generic")])
def test_extreme_ranges(ob, W, dtype, R):
    H, F = 16, 2
    lut, d, o = lut_of(ob, H, W, dtype)
    rng = extreme_ranges(F, R, H, W, seed=W)
    names = run_and_check(ob, lut, d, o, shifts_for(H, W, 1), rng)
    assert names == kernel_names(dtype, R, W % 4 == 0, False, False)


# ------------------------------------------------------------------------------------------------------------------
# LUT-free projection
# ------------------------------------------------------------------------------------------------------------------
def intrinsics(source):
    if source.startswith("os1_64_"):
        m = default_os1_64(int(source.split("_")[-1]))
    else:
        m, _ = load_fixture(source)
    return m


ANALYTIC_SOURCES = ["os1_64_512", "os1_64_1024", "os1_64_2048", "OS-0-32-U1_v2.2.0_1024x10",
                    "OS-1-128_767798045_1024x10_20230712_120049"]
# norm-wise relative error of the LUT-free projection against the float64 restatement: float keeps the documented
# 1e-5; double is held to 1e-12, far above double rounding and far below what float-rounded tables would give
ANALYTIC_TOL = {np.dtype(np.float32): (1e-5, 1e-7), np.dtype(np.float64): (1e-12, 1e-12)}


def analytic_lut(ob, m, dtype):
    args = (m["w"], m["h"], 0.001, m["beam_to_lidar_transform"], m["lidar_to_sensor_transform"],
            m["beam_azimuth_angles"], m["beam_altitude_angles"])
    lut = ob.XYZLutT.from_intrinsics(*args, dtype=dtype)
    return lut, args


@pytest.mark.parametrize("R", RETURNS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("source", ANALYTIC_SOURCES)
def test_lut_free_against_float64(ob, source, dtype, R):
    m = intrinsics(source)
    H, W, F = m["h"], m["w"], 2
    lut, args = analytic_lut(ob, m, dtype)
    lut.set_analytic(True)
    shifts = np.asarray(m["pixel_shift_by_row"], np.int32)
    rng = ranges(F, R, H, W, seed=W + H)
    rng[:, :, :, :8] = (1 << 19) - 1
    rng[:, :, -1, :len(EXTREMES)] = EXTREMES
    arrs, names = scan_to_cloud(ob, lut, shifts, rng, OUTS)
    assert names == kernel_names(dtype, R, True, False, True)
    d64, o64 = orc.make_xyz_lut(*args)
    rel, ab = ANALYTIC_TOL[np.dtype(dtype)]
    got = {}
    for name, a in arrs.items():
        got[name], bad = a.blocks()
        assert bad == 0, name
    for f in range(F):
        for r in range(R):
            rv = rng[f, r].reshape(-1)
            ref = np.where(rv[:, None] == 0, 0.0, rv[:, None].astype(np.float64) * d64 + o64)
            xyz = got["xyz"][f, r].reshape(-1, 3)
            err = np.linalg.norm(xyz.astype(np.float64) - ref, axis=-1)
            lim = rel * np.linalg.norm(ref, axis=-1) + ab
            assert np.all(err <= lim), (f, r, float(np.max(err / np.maximum(lim, 1e-300))))
            zero = rv == 0
            assert not np.any(xyz[zero].view(UINT[xyz.itemsize])), "empty returns must stay +0.0"
            assert same_bits(got["xd"][f, r], orc.destagger(xyz.reshape(H, W, 3), shifts).reshape(-1))
            assert np.array_equal(got["rd"][f, r], orc.destagger(rng[f, r], shifts).reshape(-1))


def _generic_width_intrinsics():
    m = dict(default_os1_64(512))
    m["w"] = 130
    m["pixel_shift_by_row"] = np.arange(m["h"], dtype=np.int32) % 11
    return m


@pytest.mark.parametrize("R", RETURNS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", ["poses_shared", "poses_per_frame", "generic_w130"])
def test_lut_free_falls_back_bit_exact(ob, case, dtype, R):
    """where the LUT-free flag cannot apply (fused poses, the generic kernel) the result is the LUT path's, bit for
    bit"""
    m = _generic_width_intrinsics() if case == "generic_w130" else intrinsics("os1_64_1024")
    H, W, F = m["h"], m["w"], 3
    lut, _ = analytic_lut(ob, m, dtype)
    d, o = lut.direction, lut.offset        # the device-built tables the LUT path reads
    lut.set_analytic(True)
    poses = None
    if case != "generic_w130":
        poses = random_poses(W, dtype, 4, F if case == "poses_per_frame" else None)
    shifts = np.asarray(m["pixel_shift_by_row"], np.int32)
    names = run_and_check(ob, lut, d, o, shifts, ranges(F, R, H, W, seed=2), poses=poses)
    assert names == kernel_names(dtype, R, case != "generic_w130", poses is not None, True)


# ------------------------------------------------------------------------------------------------------------------
# which kernel ran
# ------------------------------------------------------------------------------------------------------------------
def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# one representative per table above: (id, tunables, call arguments); the grid / block of the K1 kernel where the
# geometry is the point of the row (block = compute threads + the copy warp)
PROFILED = [
    ("geometry_f32_R2", {}, dict(shape=(128, 2048, 8), dtype=np.float32, R=2), (3, 160)),
    ("geometry_f64_R1_threads256", {"cloud_threads": 256}, dict(shape=(64, 1000, 7), dtype=np.float64, R=1),
     (None, 288)),
    ("geometry_ctas1", {"cloud_ctas_per_sm": 1}, dict(shape=(128, 1024, 16), dtype=np.float32, R=2), (1, 160)),
    ("wide", {}, dict(shape=(128, 2048, 8), dtype=np.float32, R=1), (2, 160)),
    ("wide_pinned", {"cloud_tw": 512}, dict(shape=(128, 2048, 8), dtype=np.float32, R=1), (3, 160)),
    ("row_shifts", {}, dict(shape=(28, 516, 2), dtype=np.float64, R=2, shifts="edge"), None),
    ("subset_rd", {}, dict(shape=(24, 1028, 3), dtype=np.float32, R=1, outs=("rd",)), None),
    ("subset_xd_poses", {}, dict(shape=(24, 1028, 3), dtype=np.float64, R=2, outs=("xd",), poses=True), None),
    ("strides_padded_host", {}, dict(shape=(32, 1024, 3), dtype=np.float32, R=2, kind="padded"), None),
    ("strides_padded_device", {}, dict(shape=(32, 1024, 3), dtype=np.float64, R=2, kind="padded", device=True),
     None),
    ("strides_range_fs0", {}, dict(shape=(32, 1024, 3), dtype=np.float32, R=2, kind="range_fs0"), None),
    ("strides_odd", {}, dict(shape=(32, 1024, 3), dtype=np.float32, R=2, kind="odd"), None),
    ("strides_range_off1", {}, dict(shape=(32, 1024, 3), dtype=np.float64, R=1, kind="range_off1", device=True),
     None),
    ("strides_xyz_off1", {}, dict(shape=(32, 1024, 3), dtype=np.float32, R=2, kind="xyz_off1", device=True), None),
    ("pose_rows4", {"cloud_pose_rows": 4}, dict(shape=(70, 1024, 6), dtype=np.float64, R=2, poses=True), None),
    ("ranges_generic", {}, dict(shape=(16, 1030, 2), dtype=np.float32, R=2), None),
    ("force_generic", {"force_generic": 1}, dict(shape=(32, 1024, 2), dtype=np.float64, R=2, force_generic=True),
     None),
    ("lut_free", {}, dict(source="os1_64_1024", dtype=np.float32, R=2), None),
    ("lut_free_poses", {}, dict(source="os1_64_1024", dtype=np.float64, R=2, poses=True), None),
    ("lut_free_generic", {}, dict(source="w130", dtype=np.float32, R=1), None),
]


def _profiled_call(ob, shape=None, dtype=np.float32, R=2, outs=OUTS, poses=False, kind="contiguous", device=False,
                   shifts=None, source=None, force_generic=False):
    if source is not None:
        m = _generic_width_intrinsics() if source == "w130" else intrinsics(source)
        H, W, F = m["h"], m["w"], 2
        lut, _ = analytic_lut(ob, m, dtype)
        d, o = lut.direction, lut.offset
        lut.set_analytic(True)
        sh = np.asarray(m["pixel_shift_by_row"], np.int32)
    else:
        H, W, F = shape
        sh = edge_shifts(W)[:H] if shifts == "edge" else shifts_for(H, W, 1)
        lut, d, o = lut_of(ob, H, W, dtype)
    rng = ranges(F, R, H, W, seed=1)
    if kind == "range_fs0":
        rng[:] = rng[0]
    p = random_poses(W, dtype, 1) if poses else None
    return lambda: scan_to_cloud(ob, lut, sh, rng, outs, poses=p, kind=kind, device=device,
                                 force_generic=force_generic)


def test_kernels_that_ran(ob, tunables, tmp_path):
    """each representative case under torch.profiler: the K1 kernels it launched are the ones its row expects (TMA
    variant and template arguments, or the generic kernel), and where the row is about launch geometry, the grid
    and block say which geometry ran.  A case that should take the TMA kernel but falls to the generic one fails
    here."""
    torch = pytest.importorskip("torch")
    from torch.profiler import ProfilerActivity, profile
    sm = _sm_count()
    seen = {}
    for case_id, tun, kw, geom in PROFILED:
        for k, v in K1_TUNABLES.items():
            ob.set_tunable(k, _env_default(k, v))
        ob.set_tunable("cloud_auto", 1)
        tunables(**tun)
        call = _profiled_call(ob, **kw)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _, want = call()
            torch.cuda.synchronize()
        trace = tmp_path / f"{case_id}.json"
        prof.export_chrome_trace(str(trace))
        events = json.load(open(trace))["traceEvents"]
        ran = [e for e in events if e.get("cat") == "kernel" and ("cloud_" in e["name"] or "pose_planes" in e["name"])]
        names = [e["name"] for e in ran]
        seen[case_id] = names
        assert len(ran) == len(want), (case_id, names, want)
        for w, e in zip(want, ran):
            assert w in e["name"], (case_id, names, want)
        if geom is not None:
            ctas, block = geom
            k1 = ran[-1]["args"]
            if ctas is not None:
                assert k1["grid"][0] == ctas * sm, (case_id, k1)
            assert k1["block"][0] == block, (case_id, k1)
    print(json.dumps(seen, indent=1))


# ------------------------------------------------------------------------------------------------------------------
# errors
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,device", [pytest.param("contiguous", False, id="host"),
                                         pytest.param("padded", False, id="host_padded"),
                                         pytest.param("contiguous", True, id="device")])
def test_shared_memory_that_does_not_fit(ob, tunables, kind, device):
    """f64, 2 returns, 2048-pixel tiles (4096 requested), 8 stages over 8 frames of 128x2048: enough tiles that the
    small-launch loop keeps the width, and a ring larger than shared memory.  The call fails and writes nothing."""
    if device:
        pytest.importorskip("torch")
    H, W, F, R = 128, 2048, 8, 2
    tunables(cloud_tw=4096, cloud_stages=8)
    lut, _, _ = lut_of(ob, H, W, np.float64)
    arrs, _, call = prepare(ob, lut, shifts_for(H, W, 2), ranges(F, R, H, W, seed=3), OUTS, kind=kind,
                            device=device)
    before = ob.kernel_launch_count("cloud")
    with pytest.raises(RuntimeError, match="scan_to_cloud launch"):
        call()
    assert ob.kernel_launch_count("cloud") == before
    for name, a in arrs.items():
        b = a.host_bytes()
        assert np.all(b == SENTINEL), f"{name}: a failed call wrote {np.count_nonzero(b != SENTINEL)} bytes"
