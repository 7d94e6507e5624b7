"""GPU tests of the C ABI's two shared argument rules:

- results whose length the GPU decides (rows plus a count, each in host or device memory): ob_voxel_downsample,
  ob_frames_to_map_rows, ob_voxel_map_point_cloud, ob_voxel_map_remove_far with extraction, ob_dewarp_frame and
  ob_dewarp_frames.  Every memory combination gives the same rows and count; the count reads 0 after an empty input
  and after a refused call; a device count with a host array is refused before anything is launched; a host count
  with too small a capacity fails with the count 0 and the host rows untouched; a device count with a small
  capacity cuts the rows and reports the true total; rows past the count keep what the buffer held; and each valid
  call launches the kernels it always did.
- input row counts (n on the host, or a device word clamped to `capacity`) of every call that reads one."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as graft

pytestmark = pytest.mark.gpu

SENT_COUNT = 0x5A5A5A5A5A
SENT = {np.float32: -7.5, np.float64: -7.5, np.uint32: 0xDEADBEEF, np.uint64: 0xDEADBEEFDEADBEEF}
SIGNED = {np.float32: np.float32, np.float64: np.float64, np.uint32: np.int32, np.uint64: np.int64}
MIXED = "a device-side count needs device outputs"
MIXED_DEWARP = "a device-side count needs device outputs and no per-frame counts"
SIZE_P = C.POINTER(C.c_size_t)


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


@pytest.fixture(scope="module")
def capi(ob):
    from ouster_sdk_b200 import _capi
    return _capi


@pytest.fixture(scope="module")
def st(ob):
    return ob.core.Stream(0)


def _alloc(spec, rows, dev):
    cols, dt = spec
    a = np.full((max(rows, 1),) if cols is None else (max(rows, 1), cols), SENT[dt], dt)
    if not dev:
        return a
    import torch
    return torch.from_numpy(a.view(SIGNED[dt])).cuda()


def _host(a, dt):
    return a if isinstance(a, np.ndarray) else a.cpu().numpy().view(dt)


class Count:
    """A sentinel-filled size_t count in host or device memory."""

    def __init__(self, dev):
        import torch
        self.dev = dev
        if dev:
            self.t = torch.full((1,), SENT_COUNT, dtype=torch.int64, device="cuda")
            self.ptr = self.t.data_ptr()
        else:
            self.c = C.c_size_t(SENT_COUNT)
            self.ptr = C.addressof(self.c)

    def value(self):
        return int(self.t.item()) if self.dev else self.c.value


def run(ob, capi, st, case, cap, rows_dev, count_dev):
    """One call of `case` with sentinel-filled outputs: (status, message, host copies of the arrays, count,
    kernels launched)."""
    outs = [_alloc(s, cap, rows_dev) for s in case.specs]
    cnt = Count(count_dev)
    if hasattr(case, "prepare"):
        case.prepare()
    before = ob.kernel_launch_count()
    status = case.call([ob.core._ptr(a) for a in outs], cap, cnt.ptr)
    launches = ob.kernel_launch_count() - before
    msg = capi.lib.ob_last_error().decode() if status else ""
    st.sync()
    return status, msg, [_host(a, s[1]) for a, s in zip(outs, case.specs)], cnt.value(), launches


# ---- the counted entry points ----

class VoxelCase:
    """ob_voxel_downsample, POINT_NORMAL with normals_out and indices_out: outputs hold the input's rows, so there
    is no capacity to exceed."""
    launches = 5
    has_capacity = False

    def __init__(self, ob, capi, st, empty=False):
        rs = np.random.default_rng(3)
        n = 0 if empty else 4000
        self.pts = rs.normal(0, 4.0, (max(n, 1), 3))
        nrm = rs.normal(0, 1.0, (max(n, 1), 3))
        self.nrm = nrm / np.linalg.norm(nrm, axis=1, keepdims=True)
        self.n, self.capi, self.st = n, capi, st
        self.specs = [(3, np.float64), (3, np.float64), (None, np.uint32)]
        self.rows = n

    def call(self, ptrs, cap, n_ptr):
        io = self.capi.VoxelIO()
        io.mode, io.dtype = self.capi.OB_VOXEL_POINT_NORMAL, self.capi.OB_F64
        io.points, io.cols, io.normals, io.n = self.pts.ctypes.data, 3, self.nrm.ctypes.data, self.n
        io.voxel_size = 0.5
        io.points_out, io.normals_out, io.indices_out, io.n_out = ptrs[0], ptrs[1], ptrs[2], n_ptr
        return self.capi.lib.ob_voxel_downsample(C.byref(io), self.st.h)


class MapRowsCase:
    launches = 1
    has_capacity = True

    def __init__(self, ob, capi, st, empty=False):
        from tests.helpers import random_lut, random_range
        h, w = 32, 512
        d, o = random_lut(h * w, 5, np.float64)
        self.lut = ob.XYZLutT.from_arrays(d, o, h, w)
        self.rng = random_range(h, w, 6, p_zero=0.4) * (0 if empty else 1)
        self.poses = np.tile(np.eye(4), (w, 1, 1))
        self.sig = np.arange(h * w, dtype=np.uint16).reshape(h, w)
        self.tab = (capi.MapField * 1)()
        self.tab[0].data, self.tab[0].type, self.tab[0].channels = self.sig.ctypes.data, 2, 1
        self.items = (capi.MapRowsItem * 1)()
        self.items[0].lut, self.items[0].range, self.items[0].poses = self.lut._h, self.rng.ctypes.data, \
            self.poses.ctypes.data
        self.items[0].fields, self.items[0].n_fields = self.tab, 1
        self.capi, self.st = capi, st
        self.specs = [(4, np.float64)]
        self.rows = h * w

    def call(self, ptrs, cap, n_ptr):
        return self.capi.lib.ob_frames_to_map_rows(self.items, 1, ptrs[0], 4, cap, n_ptr, self.st.h)


def _filled_map(ob, empty=False):
    rs = np.random.default_rng(8)
    m = ob.VoxelMap(0.5, 100.0, 3, num_attributes=1)
    if not empty:
        m.add_rows(np.hstack([rs.normal(0, 6.0, (3000, 3)), rs.normal(0, 1.0, (3000, 1))]))
    return m


class PointCloudCase:
    launches = 3
    has_capacity = True

    def __init__(self, ob, capi, st, empty=False):
        self.m = _filled_map(ob, empty)
        self.capi, self.st = capi, st
        self.specs = [(4, np.float64)]
        self.rows = self.m.size()[1]

    def call(self, ptrs, cap, n_ptr):
        return self.capi.lib.ob_voxel_map_point_cloud(self.m._h, ptrs[0], cap, n_ptr, self.st.h)


class RemoveFarCase:
    """ob_voxel_map_remove_far with extraction on a fresh map per call; the origin leaves about half the voxels."""
    launches = 4
    has_capacity = True

    def __init__(self, ob, capi, st, empty=False):
        self.ob, self.capi, self.st, self.empty = ob, capi, st, empty
        self.origin = np.array([0.0, 0.0, 0.0]) if empty else np.array([95.0, 0.0, 0.0])
        self.specs = [(4, np.float64)]
        self.rows = _filled_map(ob).size()[1]
        self.sizes = []

    def prepare(self):
        self.m = _filled_map(self.ob)

    def call(self, ptrs, cap, n_ptr):
        m = self.m
        io = self.capi.VoxelMapCullIO()
        io.origin, io.extracted, io.capacity, io.n_extracted = self.origin.ctypes.data, ptrs[0], cap, n_ptr
        before = m.size()
        status = self.capi.lib.ob_voxel_map_remove_far(m._h, C.byref(io), self.st.h)
        self.sizes.append((before, m.size()))
        return status


class DewarpFrameCase:
    launches = 1
    has_capacity = True

    def __init__(self, ob, capi, st, empty=False):
        from tests.helpers import random_lut, random_range
        h, w = 32, 1024
        d, o = random_lut(h * w, 2, np.float32)
        self.lut = ob.XYZLutT.from_arrays(d, o, h, w)
        self.rng = random_range(h, w, 4, p_zero=0.5, max_range=60000) * (0 if empty else 1)
        self.poses = np.tile(np.eye(4), (w, 1, 1))
        self.status = np.ones(w, np.uint32)
        self.ts = np.arange(w, dtype=np.uint64) * 7
        self.capi, self.st = capi, st
        self.specs = [(3, np.float32), (None, np.uint32), (None, np.uint64)]
        self.rows = h * w

    def call(self, ptrs, cap, n_ptr):
        io = self.capi.DewarpFrameIO()
        io.range, io.poses, io.status, io.timestamps = (self.rng.ctypes.data, self.poses.ctypes.data,
                                                        self.status.ctypes.data, self.ts.ctypes.data)
        io.min_range, io.max_range = 0.5, 50.0
        io.points, io.col_idx, io.timestamps_out, io.capacity = ptrs[0], ptrs[1], ptrs[2], cap
        return self.capi.lib.ob_dewarp_frame(self.lut._h, C.byref(io), C.cast(C.c_void_p(n_ptr), SIZE_P),
                                             self.st.h)


class DewarpFramesCase:
    """ob_dewarp_frames over two frames and an empty slot, with provenance; per-frame counts with a host count."""
    launches = 1
    has_capacity = True

    def __init__(self, ob, capi, st, empty=False):
        from tests.helpers import random_lut, random_range
        self.keep, self.capi, self.st = [], capi, st
        self.frames = (capi.DewarpFramesIO * 3)()
        for i, (h, w) in enumerate([(16, 512), (0, 0), (32, 256)]):
            if h == 0:                            # an empty slot of the set
                continue
            d, o = random_lut(h * w, 10 + i, np.float64)
            lut = ob.XYZLutT.from_arrays(d, o, h, w)
            rng = random_range(h, w, 20 + i, p_zero=0.5, max_range=60000) * (0 if empty else 1)
            poses, status = np.tile(np.eye(4), (w, 1, 1)), np.ones(w, np.uint32)
            ts = np.arange(w, dtype=np.uint64) + 1000 * i
            self.keep += [lut, rng, poses, status, ts]
            f = self.frames[i]
            f.lut, f.range, f.poses, f.status, f.timestamps = (lut._h, rng.ctypes.data, poses.ctypes.data,
                                                               status.ctypes.data, ts.ctypes.data)
        self.specs = [(3, np.float64), (None, np.uint32), (None, np.uint32), (None, np.uint64)]
        self.rows = 16 * 512 + 32 * 256
        self.counts = None

    def call(self, ptrs, cap, n_ptr, counts=None):
        self.counts = counts
        cp = counts.ctypes.data_as(SIZE_P) if counts is not None else None
        return self.capi.lib.ob_dewarp_frames(self.frames, 3, 0.5, 50.0, ptrs[0], cap, ptrs[1], ptrs[2], ptrs[3], cp,
                                              C.cast(C.c_void_p(n_ptr), SIZE_P), self.st.h)


CASES = {"voxel_downsample": VoxelCase, "frames_to_map_rows": MapRowsCase, "voxel_map_point_cloud": PointCloudCase,
         "voxel_map_remove_far": RemoveFarCase, "dewarp_frame": DewarpFrameCase, "dewarp_frames": DewarpFramesCase}


@pytest.mark.parametrize("name", list(CASES))
def test_counted_result_memory_combinations_agree(ob, capi, st, name):
    case = CASES[name](ob, capi, st)
    cap = case.rows
    s, msg, want, total, launches = run(ob, capi, st, case, cap, rows_dev=False, count_dev=False)
    assert s == 0, msg
    assert 0 < total <= cap and launches == case.launches
    for a, spec in zip(want, case.specs):
        assert not np.any(a[total:] != SENT[spec[1]]), "host rows past the count were written"
    for rows_dev, count_dev in ((True, False), (True, True)):
        s, msg, got, n, launches = run(ob, capi, st, case, cap, rows_dev, count_dev)
        assert s == 0, msg
        assert n == total and launches == case.launches, (rows_dev, count_dev)
        for a, b, spec in zip(got, want, case.specs):
            assert np.array_equal(a[:total], b[:total]), (rows_dev, count_dev)
            assert not np.any(a[total:] != SENT[spec[1]]), "device rows past the count were written"
    if name == "voxel_map_point_cloud":          # count only: never too small, with either count
        for count_dev in (False, True):
            cnt = Count(count_dev)
            assert capi.lib.ob_voxel_map_point_cloud(case.m._h, None, 0, cnt.ptr, st.h) == 0
            st.sync()
            assert cnt.value() == total
    if name == "dewarp_frames":                  # per-frame counts with a host count
        counts = np.full(3, SENT_COUNT, np.uint64)
        outs = [_alloc(sp, cap, False) for sp in case.specs]
        cnt = Count(False)
        assert case.call([ob.core._ptr(a) for a in outs], cap, cnt.ptr, counts) == 0
        assert cnt.value() == total and counts[1] == 0 and counts.sum() == total and counts.min() == 0
        assert counts[0] > 0 and counts[2] > 0


@pytest.mark.parametrize("name", list(CASES))
def test_counted_result_reads_zero_after_an_empty_input(ob, capi, st, name):
    case = CASES[name](ob, capi, st, empty=True)
    cap = max(case.rows, 1)
    for rows_dev, count_dev in ((False, False), (True, False), (True, True)):
        s, msg, got, n, _ = run(ob, capi, st, case, cap, rows_dev, count_dev)
        assert s == 0, msg
        assert n == 0, (rows_dev, count_dev)
        for a, spec in zip(got, case.specs):
            assert not np.any(a != SENT[spec[1]])


@pytest.mark.parametrize("name", list(CASES))
def test_device_count_with_host_rows_is_refused_before_any_launch(ob, capi, st, name):
    case = CASES[name](ob, capi, st)
    s, msg, got, n, launches = run(ob, capi, st, case, case.rows, rows_dev=False, count_dev=True)
    assert s == capi.OB_INVALID_ARGUMENT
    assert msg == (MIXED_DEWARP if name.startswith("dewarp") else MIXED)
    assert launches == 0 and n == 0
    for a, spec in zip(got, case.specs):
        assert not np.any(a != SENT[spec[1]])
    if name == "voxel_map_remove_far":           # the map is left as it was
        before, after = case.sizes[-1]
        assert before == after
    if name == "dewarp_frames":                  # per-frame counts need a host count
        outs = [_alloc(sp, case.rows, True) for sp in case.specs]
        cnt = Count(True)
        counts = np.zeros(3, np.uint64)
        before = ob.kernel_launch_count()
        s = case.call([ob.core._ptr(a) for a in outs], case.rows, cnt.ptr, counts)
        assert s == capi.OB_INVALID_ARGUMENT and capi.lib.ob_last_error().decode() == MIXED_DEWARP
        assert ob.kernel_launch_count() == before
        st.sync()
        assert cnt.value() == 0


@pytest.mark.parametrize("name", [k for k, v in CASES.items() if v.has_capacity])
def test_host_count_above_capacity_fails_and_leaves_the_rows(ob, capi, st, name):
    case = CASES[name](ob, capi, st)
    s, msg, _, total, _ = run(ob, capi, st, case, case.rows, rows_dev=False, count_dev=False)
    assert s == 0, msg
    for rows_dev in (False, True):
        s, msg, got, n, launches = run(ob, capi, st, case, total - 1, rows_dev, count_dev=False)
        assert s == capi.OB_INVALID_ARGUMENT and msg == "output capacity too small"
        assert n == 0 and launches == case.launches
        if not rows_dev:
            for a, spec in zip(got, case.specs):
                assert not np.any(a != SENT[spec[1]]), "host rows were written by a failed call"


@pytest.mark.parametrize("name", [k for k, v in CASES.items() if v.has_capacity])
def test_device_count_with_small_capacity_cuts_the_rows(ob, capi, st, name):
    case = CASES[name](ob, capi, st)
    s, msg, want, total, _ = run(ob, capi, st, case, case.rows, rows_dev=False, count_dev=False)
    assert s == 0, msg
    cap = total // 3
    s, msg, got, n, launches = run(ob, capi, st, case, cap, rows_dev=True, count_dev=True)
    assert s == 0, msg
    assert n == total and launches == case.launches
    for a, b, spec in zip(got, want, case.specs):
        assert np.array_equal(a[:cap], b[:cap])
        assert not np.any(a[cap:] != SENT[spec[1]])


# ---- input row counts ----

def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _dev_n(v):
    import torch
    return torch.tensor([v], dtype=torch.int64, device="cuda")


class Inputs:
    """Every call that reads an input row count, as f(n, n_device, capacity) -> (status, result)."""

    def __init__(self, ob, capi, st):
        rs = np.random.default_rng(12)
        self.ob, self.capi, self.st = ob, capi, st
        self.pts = _dev(rs.normal(0, 5.0, (2000, 3)))
        self.tgt = _dev(self.pts.cpu().numpy() + rs.normal(0, 0.01, (2000, 3)))
        self.rows4 = _dev(np.hstack([self.pts.cpu().numpy(), rs.normal(0, 1.0, (2000, 1))]))

    def add_points(self, n, n_device, cap):
        m = self.ob.VoxelMap(0.5, 100.0, 3)
        r = self.capi.PointRows()
        r.dtype, r.points, r.n, r.n_device, r.capacity = self.capi.OB_F64, self.pts.data_ptr(), n, n_device, cap
        s = self.capi.lib.ob_voxel_map_add_points(m._h, C.byref(r), self.st.h)
        return s, (m.point_cloud(stream=self.st) if s == 0 else None)

    def add_rows(self, n, n_device, cap):
        m = self.ob.VoxelMap(0.5, 100.0, 3, num_attributes=1)
        r = self.capi.MapRows()
        r.rows, r.cols, r.n, r.n_device, r.capacity = self.rows4.data_ptr(), 4, n, n_device, cap
        s = self.capi.lib.ob_voxel_map_add_rows(m._h, C.byref(r), self.st.h)
        return s, (m.point_cloud(stream=self.st) if s == 0 else None)

    def voxel_downsample(self, n, n_device, cap):
        import torch
        out = torch.zeros((2000, 3), dtype=torch.float64, device="cuda")
        cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        io = self.capi.VoxelIO()
        io.mode, io.dtype, io.points, io.cols = self.capi.OB_VOXEL_FIRST_N_POINT, self.capi.OB_F64, \
            self.pts.data_ptr(), 3
        io.n, io.n_device, io.capacity = n, n_device, cap
        io.voxel_size, io.max_points_per_voxel, io.min_pts_threshold = 0.5, 1, 1
        io.points_out, io.n_out = out.data_ptr(), cnt.data_ptr()
        s = self.capi.lib.ob_voxel_downsample(C.byref(io), self.st.h)
        self.st.sync()
        return s, (out[:int(cnt.item())].cpu().numpy() if s == 0 else None)

    def icp_linear_system(self, n, n_device, cap):
        import torch
        jtj = torch.zeros(36, dtype=torch.float64, device="cuda")
        jtr = torch.zeros(6, dtype=torch.float64, device="cuda")
        io = self.capi.IcpSystemIO()
        io.source, io.target, io.n, io.n_device, io.capacity = self.pts.data_ptr(), self.tgt.data_ptr(), n, \
            n_device, cap
        io.kernel_scale, io.jtj, io.jtr = 1.0, jtj.data_ptr(), jtr.data_ptr()
        s = self.capi.lib.ob_icp_linear_system(C.byref(io), self.st.h)
        self.st.sync()
        return s, (np.concatenate([jtj.cpu().numpy(), jtr.cpu().numpy()]) if s == 0 else None)

    def cloud_align(self, n, n_device, cap):
        pose = np.zeros(16)
        io = self.capi.CloudAlignIO()
        io.mode, io.max_corr_dist = self.capi.OB_ALIGN_POINT_TO_POINT, 0.5
        io.source.dtype, io.source.points, io.source.n = self.capi.OB_F64, self.tgt.data_ptr(), 2000
        io.target.dtype, io.target.points = self.capi.OB_F64, self.pts.data_ptr()
        io.target.n, io.target.n_device, io.target.capacity = n, n_device, cap
        io.pose = pose.ctypes.data
        s = self.capi.lib.ob_cloud_align(C.byref(io), self.st.h)
        return s, (pose if s == 0 else None)


ROW_INPUTS = ["add_points", "add_rows", "voxel_downsample", "icp_linear_system", "cloud_align"]


@pytest.mark.parametrize("name", ROW_INPUTS)
def test_input_row_count_rule(ob, capi, st, name):
    f = getattr(Inputs(ob, capi, st), name)
    too_many = "too many pairs in one call" if name == "icp_linear_system" else "too many points in one call"
    host_word = C.c_size_t(10)
    s, _ = f(0, C.addressof(host_word), 100)
    assert s == capi.OB_INVALID_ARGUMENT and capi.lib.ob_last_error().decode() == "n_device must be device memory"
    big = _dev_n(5)
    s, _ = f(0, big.data_ptr(), 1 << 31)
    assert s == capi.OB_INVALID_ARGUMENT and capi.lib.ob_last_error().decode() == too_many
    s, want = f(1500, None, 0)
    assert s == 0
    above = _dev_n(1 << 40)                       # clamped on the device to the capacity
    s, got = f(0, above.data_ptr(), 1500)
    assert s == 0 and np.array_equal(got, want)
