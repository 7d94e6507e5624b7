"""K3 (k3_fused_kernel: LUT projection, per-column pose, range filter and the order-preserving compaction with its
decoupled look-back, in one launch) down every path its host code can pick, driven through the C ABI so that every
pointer, placement and capacity is the test's, and compared byte for byte with the CPU oracle's dewarp_frame: frames
of a set concatenated in slot order with the slot index as frame_idx.  Cases: frames taller than the 8 slabs one CTA
covers in one turn (and than 48 KB of per-slab counts), sets of thousands of CTAs and of hundreds of tiny frames with
empty slots, pixels on both edges of the range window and windows the reference cannot convert, every subset of the
provenance outputs, both capacity rules, host / device placements, the refusals and the status words.  Every output
starts as a 0xA5 byte pattern: bytes past the count and around the output arrays must still hold it afterwards, and
each call checks how many K3 launches it made."""
import ctypes as C
import itertools
import math
import sys
from importlib import import_module

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import oracle as orc
from tests.helpers import random_lut, random_range

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
GAP = 64                                   # sentinel bytes before, between and after the output arrays
SENT_COUNT = 0xA5A5A5A5A5A5A5A5
SIZE_P = C.POINTER(C.c_size_t)
PROV = ("frame_idx", "col_idx", "timestamps")
ROW_BYTES = {"frame_idx": 4, "col_idx": 4, "timestamps": 8}
DTYPES = [pytest.param(np.float32, id="f32"), pytest.param(np.float64, id="f64")]
ENTRIES = [pytest.param(True, id="frame"), pytest.param(False, id="frames")]
MIXED = "a device-side count needs device outputs and no per-frame counts"
TOO_TALL = "dewarp supports at most 25600 rows per frame"
NO_TS = "timestamps_out requested without column timestamps"
MAX_ROWS = 25600


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


@pytest.fixture(scope="module")
def capi(ob):
    return import_module(ob.__name__ + "._capi")


@pytest.fixture(scope="module")
def st(ob):
    return ob.Stream(0)


def _torch_sync():
    """device inputs and outputs are written by torch on its own stream: done before the call's stream reads them"""
    torch = sys.modules.get("torch")
    if torch is not None and torch.cuda.is_initialized():
        torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------
# frames, outputs and the oracle
# ------------------------------------------------------------------------------------------------------------------
def random_poses(w, seed):
    """body_to_world per column: rotations about random axes (all nine entries non-zero) and translations"""
    rs = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rs.normal(size=(w, 3, 3)))
    q[np.linalg.det(q) < 0, :, 0] *= -1
    p = np.zeros((w, 4, 4))
    p[:, :3, :3] = q
    p[:, :3, 3] = rs.uniform(-20, 20, (w, 3))
    p[:, 3, 3] = 1
    return p


def default_status(w, rs):
    """invalid leading and trailing columns, holes, a non-zero word without the valid bit inside the span"""
    if w < 10:
        return rs.choice(np.array([0, 1, 1, 2, 3], np.uint32), w)
    s = np.ones(w, np.uint32)
    s[: w // 10] = 0
    s[rs.integers(w // 10, w, w // 8)] = 0
    s[w // 2] = 2
    s[-2:] = 0
    return s


class Frame:
    """one frame of a set: range image, LUT tables and handle, per-column poses, status and timestamps, with its
    inputs in host or device memory"""

    def __init__(self, ob, h, w, dtype, seed, *, rng=None, status=None, tables=None, lut=None, device=False):
        rs = np.random.default_rng(seed)
        self.h, self.w, self.dtype = h, w, np.dtype(dtype)
        self.rng = random_range(h, w, seed, p_zero=0.3, max_range=60000) if rng is None else rng
        self.d, self.o = random_lut(h * w, seed + 1, dtype) if tables is None else tables
        self.lut = lut if lut is not None else ob.XYZLutT.from_arrays(self.d, self.o, h, w)
        self.poses = random_poses(w, seed + 2)
        self.status = default_status(w, rs) if status is None else np.asarray(status, np.uint32)
        self.ts = (10 ** 12 + 1000 * seed + 17 * np.arange(w)).astype(np.uint64)
        self.device = device
        self._dev = None

    def ptrs(self):
        """(range, poses, status, timestamps)"""
        arrs = (self.rng.view(np.int32), self.poses, self.status.view(np.int32), self.ts.view(np.int64))
        if not self.device:
            return tuple(a.ctypes.data for a in arrs)
        if self._dev is None:
            import torch
            self._dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs]
        return tuple(t.data_ptr() for t in self._dev)

    def oracle(self, lo, hi):
        return orc.dewarp_frame(self.rng, self.d, self.o, self.poses, self.status, self.ts, lo, hi)


def expected(slots, lo, hi):
    """the oracle's set result as {output: bytes} and the points per slot"""
    parts = {k: [] for k in ("points",) + PROV}
    counts = []
    for i, fr in enumerate(slots):
        if fr is None:
            counts.append(0)
            continue
        p, c, t = fr.oracle(lo, hi)
        parts["points"].append(p)
        parts["frame_idx"].append(np.full(len(c), i, np.uint32))
        parts["col_idx"].append(c)
        parts["timestamps"].append(t)
        counts.append(len(c))
    want = {k: np.ascontiguousarray(np.concatenate(v)).reshape(-1).view(np.uint8) for k, v in parts.items()}
    return want, counts


class Outputs:
    """sentinel-filled arrays of `cap` rows in one flat buffer (numpy, or a CUDA tensor), GAP sentinel bytes around
    each one"""

    def __init__(self, names, cap, dtype, device=False):
        self.rb = {n: 3 * np.dtype(dtype).itemsize if n == "points" else ROW_BYTES[n] for n in names}
        self.off, pos = {}, GAP
        for n in names:
            self.off[n] = pos
            pos = (pos + cap * self.rb[n] + 255) // 256 * 256 + GAP
        host = np.full(pos, SENTINEL, np.uint8)
        self.device = device
        if device:
            import torch
            self.buf = torch.from_numpy(host).cuda()
        else:
            self.buf = host

    def ptrs(self):
        base = self.buf.data_ptr() if self.device else self.buf.ctypes.data
        return {n: base + off for n, off in self.off.items()}

    def check(self, want, n):
        """the first n rows of every array equal `want` byte for byte and every other byte holds the sentinel"""
        b = self.buf.cpu().numpy() if self.device else self.buf
        pos = 0
        for name, off in sorted(self.off.items(), key=lambda kv: kv[1]):
            assert not np.any(b[pos:off] != SENTINEL), f"bytes before {name} (or past the count) were written"
            nb = n * self.rb[name]
            got, exp = b[off:off + nb], want[name][:nb]
            if not np.array_equal(got, exp):
                diff = np.flatnonzero(got != exp) if got.size == exp.size else [0]
                raise AssertionError(f"{name}: {len(diff)} bytes differ, first in row {diff[0] // self.rb[name]}")
            pos = off + nb
        assert not np.any(b[pos:] != SENTINEL), "bytes past the last array were written"

    def untouched(self):
        self.check({n: np.zeros(0, np.uint8) for n in self.off}, 0)


class Count:
    """n_points in host memory (a size_t holding a sentinel) or device memory (one int64)"""

    def __init__(self, device):
        self.device = device
        if device:
            import torch
            self.t = torch.full((1,), -0x5A5A5A5A5A5A5A5B, dtype=torch.int64, device="cuda")
            self.ptr = self.t.data_ptr()
        else:
            self.h = C.c_size_t(SENT_COUNT)
            self.ptr = C.addressof(self.h)

    def value(self):
        return int(self.t.item()) if self.device else self.h.value


def call(ob, capi, st, slots, lo, hi, ptrs, cap, count, *, single=False, counts=None, timestamps=True):
    """one ob_dewarp_frame (single: slots == [frame]) or ob_dewarp_frames call; (status, message, K3 launches)"""
    _torch_sync()
    before = ob.kernel_launch_count("dewarp")
    n_p = C.cast(C.c_void_p(count.ptr), SIZE_P)
    if single:
        fr = slots[0]
        io = capi.DewarpFrameIO()
        r, p, s, t = fr.ptrs()
        io.range, io.poses, io.status, io.timestamps = r, p, s, t if timestamps else None
        io.min_range, io.max_range = lo, hi
        io.points, io.col_idx, io.timestamps_out = ptrs.get("points"), ptrs.get("col_idx"), ptrs.get("timestamps")
        io.capacity = cap
        status = capi.lib.ob_dewarp_frame(fr.lut._h, C.byref(io), n_p, st.h)
    else:
        ios = (capi.DewarpFramesIO * max(len(slots), 1))()
        for i, fr in enumerate(slots):
            if fr is None:
                continue
            r, p, s, t = fr.ptrs()
            ios[i].lut, ios[i].range, ios[i].poses, ios[i].status = fr.lut._h, r, p, s
            ios[i].timestamps = t if timestamps else None
        cp = counts.ctypes.data_as(SIZE_P) if counts is not None else None
        status = capi.lib.ob_dewarp_frames(ios, len(slots), lo, hi, ptrs.get("points"), cap, ptrs.get("frame_idx"),
                                           ptrs.get("col_idx"), ptrs.get("timestamps"), cp, n_p, st.h)
    msg = capi.lib.ob_last_error().decode() if status else ""
    st.sync()
    return status, msg, ob.kernel_launch_count("dewarp") - before


def names_for(single, prov=PROV):
    return ("points",) + tuple(p for p in prov if not (single and p == "frame_idx"))


def window_launches(lo, hi):
    return 1 if math.ceil(lo * 1e3) <= math.floor(hi * 1e3) else 0


def dewarp_and_check(ob, capi, st, slots, lo, hi, *, single=False, prov=PROV, out_device=False, count_device=False,
                     cap=None, with_counts=None, launches=None):
    """one call into fresh sentinel outputs, checked against the oracle; returns the number of points"""
    live = [f for f in slots if f is not None]
    want, per_slot = expected(slots, lo, hi)
    n = sum(per_slot)
    cap = sum(f.h * f.w for f in live) if cap is None else cap
    out = Outputs(names_for(single, prov), cap, live[0].dtype, out_device)
    count = Count(count_device)
    with_counts = (not single and not count_device) if with_counts is None else with_counts
    counts = np.full(len(slots), SENT_COUNT, np.uint64) if with_counts else None
    status, msg, ran = call(ob, capi, st, slots, lo, hi, out.ptrs(), cap, count, single=single, counts=counts)
    assert status == 0, msg
    assert ran == (window_launches(lo, hi) if launches is None else launches)
    assert count.value() == n
    out.check(want, min(n, cap))
    if counts is not None:
        assert counts.tolist() == per_slot
    return n


# ------------------------------------------------------------------------------------------------------------------
# tall frames: the slab loop's later turns, more than 48 KB of shared memory, the row limit
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("w", [33, 64])
@pytest.mark.parametrize("h", [129, 257, 1000])
def test_tall_frames(ob, capi, st, h, w, dtype):
    """8 warps take 16-row slabs k, k + 8, ...: 129 rows give warp 0 a ninth slab of one row, 257 a seventeenth,
    1000 rows 63 slabs with a partial last one"""
    fr = Frame(ob, h, w, dtype, h + w)
    for single in (True, False):
        assert dewarp_and_check(ob, capi, st, [fr], 0.5, 45.0, single=single) > 0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("h,w", [(6160, 33), (MAX_ROWS, 1)])
def test_frames_past_48kb_of_shared_memory(ob, capi, st, h, w, dtype):
    """385 slabs need the opt-in above 48 KB of dynamic shared memory, set per template instance; 25600 rows are
    the 200 KB limit itself"""
    fr = Frame(ob, h, w, dtype, 3 + w, status=np.ones(w, np.uint32))
    for single in (True, False):
        assert dewarp_and_check(ob, capi, st, [fr, None], 0.5, 45.0, single=single) > 0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("single", ENTRIES)
def test_too_tall_frame_is_refused_before_staging(ob, capi, st, single, dtype):
    tall = Frame(ob, MAX_ROWS + 16, 1, dtype, 5, status=np.ones(1, np.uint32))
    small = Frame(ob, 20, 40, dtype, 6)
    slots = [tall] if single else [small, tall]
    out = Outputs(names_for(single), tall.h + small.h * small.w, dtype)
    count = Count(False)
    counts = None if single else np.full(2, SENT_COUNT, np.uint64)
    status, msg, ran = call(ob, capi, st, slots, 0.5, 45.0, out.ptrs(), tall.h, count, single=single, counts=counts)
    assert status == capi.OB_INVALID_ARGUMENT and msg == TOO_TALL
    assert ran == 0 and count.value() == 0
    out.untouched()
    if counts is not None:
        assert not counts.any()
    # the stream is still usable
    assert dewarp_and_check(ob, capi, st, [small], 0.5, 45.0, single=single) > 0
    with pytest.raises(ValueError, match="at most 25600 rows"):
        ob.dewarp_frame(tall.lut, tall.rng, tall.poses, tall.status)


# ------------------------------------------------------------------------------------------------------------------
# scale: look-back chains past co-residency, hundreds of tiny frames
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_48_frames_of_3072_ctas(ob, capi, st, dtype):
    """48 frames of 128 x 2048 (64 CTAs each, 3072 in all: more than an H100 holds at once) whose CTAs wait on
    predecessors that were not yet resident; long zero runs make many CTAs publish zero aggregates, one frame is all
    zeros and one has no valid column.  Twice, since the CTAs are scheduled in a different order each time."""
    h, w, F = 128, 2048, 48
    tables = random_lut(h * w, 8, dtype)
    lut = ob.XYZLutT.from_arrays(*tables, h, w)
    slots = []
    for f in range(F):
        rng = random_range(h, w, 100 + f, p_zero=0.3, max_range=60000)
        a = (173 * f) % 1500
        rng[:, a:a + 300 + (91 * f) % 500] = 0
        if f == 7:
            rng[:] = 0
        status = np.zeros(w, np.uint32) if f == 20 else None
        slots.append(Frame(ob, h, w, dtype, 100 + f, rng=rng, status=status, tables=tables, lut=lut))
    n = sum(len(fr.oracle(0.2, 55.0)[1]) for fr in slots)
    for _ in range(2):
        assert dewarp_and_check(ob, capi, st, slots, 0.2, 55.0, cap=n + 7) == n


@pytest.mark.parametrize("dtype", DTYPES)
def test_hundreds_of_tiny_frames_with_empty_slots(ob, capi, st, dtype):
    """300 slots of 1-3 rows x 1-40 columns (one or two CTAs each), every seventh slot empty: the frame lookup,
    slot-indexed frame_idx and counts[]"""
    rs = np.random.default_rng(17)
    slots = []
    for i in range(300):
        if i % 7 == 3:
            slots.append(None)
            continue
        h, w = int(rs.integers(1, 4)), int(rs.integers(1, 41))
        rng = random_range(h, w, 500 + i, p_zero=0.2, max_range=60000)
        slots.append(Frame(ob, h, w, dtype, 500 + i, rng=rng))
    for _ in range(2):
        assert dewarp_and_check(ob, capi, st, slots, 0.5, 45.0) > 0


@pytest.mark.parametrize("count_device", [pytest.param(False, id="host_count"), pytest.param(True, id="device_count")])
def test_sets_without_a_live_frame(ob, capi, st, count_device):
    """no slot, or only empty ones: nothing launched, the count 0, counts[] zeroed"""
    for n_slots in (0, 3):
        out = Outputs(names_for(False), 100, np.float32, count_device)
        count = Count(count_device)
        counts = None if count_device else np.full(max(n_slots, 1), SENT_COUNT, np.uint64)
        status, msg, ran = call(ob, capi, st, [None] * n_slots, 0.5, 45.0, out.ptrs(), 100, count, counts=counts)
        assert status == 0 and ran == 0 and count.value() == 0, msg
        out.untouched()
        if counts is not None:
            assert counts.tolist() == ([0] * n_slots if n_slots else [SENT_COUNT])


# ------------------------------------------------------------------------------------------------------------------
# range windows
# ------------------------------------------------------------------------------------------------------------------
def edge_frame(ob, lo, hi, dtype, seed=9, h=64, w=100):
    """pixels at ceil(lo * 1e3) - 1, + 0, + 1 and floor(hi * 1e3) - 1, + 0, + 1 millimetres, 0 and 2^32 - 1"""
    lo_mm, hi_mm = math.ceil(lo * 1e3), math.floor(hi * 1e3)
    edges = [v for v in (lo_mm - 1, lo_mm, lo_mm + 1, hi_mm - 1, hi_mm, hi_mm + 1, 0, (1 << 32) - 1)
             if 0 <= v < (1 << 32)]
    rs = np.random.default_rng(seed)
    rng = random_range(h, w, seed, p_zero=0.1, max_range=60000)
    pick = rs.random((h, w)) < 0.5
    rng[pick] = rs.choice(np.array(edges, np.uint32), int(pick.sum()))
    return Frame(ob, h, w, dtype, seed, rng=rng)


# (min_range, max_range) in metres: whole millimetres, bounds between millimetres (0.2995 -> 300; 1.001 * 1e3 is
# 1000.999..., whose floor is 1000; 1.005 * 1e3 is 1004.999..., whose ceil is 1005), 0 m (zero ranges pass, at the
# column translation), ceil(-0.4) = -0.0, the largest window, single-millimetre windows and an empty one
WINDOWS = [(0.5, 30.0), (0.1, 30.0004), (0.2995, 1.001), (1.005, 33.0001), (0.0, 30.0), (-0.0004, 30.0),
           (-0.0, -0.0), (0.0, 4294967.295), (4294967.295, 4294967.295), (10.0, 10.0), (50.0, 40.0)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("single", ENTRIES)
@pytest.mark.parametrize("lo,hi", WINDOWS)
def test_range_window_edges(ob, capi, st, lo, hi, single, dtype):
    fr = edge_frame(ob, lo, hi, dtype)
    slots = [fr] if single else [fr, None, edge_frame(ob, lo, hi, dtype, seed=10, h=7, w=33)]
    n = dewarp_and_check(ob, capi, st, slots, lo, hi, single=single)
    assert (n > 0) == (window_launches(lo, hi) == 1)


# windows whose conversion to uint32 millimetres is undefined in the reference (gcc on x86 keeps the low 32 bits of
# a 64-bit truncation: -1 m selects nothing there, NaN a zero minimum, +inf and 1e300 a zero maximum)
REFUSED = [(-1.0, 30.0), (float("nan"), 30.0), (0.0, float("inf")), (0.0, 1e300), (0.0, float("nan")), (0.0, 5e6),
           (-float("inf"), 30.0), (0.0, -0.002), (4294967.296, 4294967.296)]


@pytest.mark.parametrize("count_device", [pytest.param(False, id="host_count"), pytest.param(True, id="device_count")])
@pytest.mark.parametrize("single", ENTRIES)
@pytest.mark.parametrize("lo,hi", REFUSED)
def test_unconvertible_range_window_is_refused(ob, capi, st, lo, hi, single, count_device):
    fr = Frame(ob, 16, 64, np.float32, 4)
    slots = [fr] if single else [fr, None, Frame(ob, 8, 40, np.float32, 5)]
    out = Outputs(names_for(single), 16 * 64 + 8 * 40, np.float32, count_device)
    count = Count(count_device)
    counts = None if single or count_device else np.full(3, SENT_COUNT, np.uint64)
    status, msg, ran = call(ob, capi, st, slots, lo, hi, out.ptrs(), 16 * 64 + 8 * 40, count, single=single,
                            counts=counts)
    assert status == capi.OB_INVALID_ARGUMENT and msg.startswith("range window outside [0, 4294967.295] m"), msg
    assert ran == 0 and count.value() == 0
    out.untouched()
    if counts is not None:
        assert not counts.any()


def test_python_wrappers_refuse_the_window_and_map_an_infinite_maximum(ob):
    fr = edge_frame(ob, 0.0, 4294967.295, np.float64)
    with pytest.raises(ValueError, match="range window"):
        ob.dewarp_frame(fr.lut, fr.rng, fr.poses, fr.status, None, -1.0, 30.0)
    with pytest.raises(ValueError, match="range window"):
        ob.dewarp_frames([{"lut": fr.lut, "range": fr.rng, "poses": fr.poses, "status": fr.status}], 0.0, 5e6)
    want = fr.oracle(0.0, 4294967.295)[0]
    assert np.array_equal(ob.dewarp_frame(fr.lut, fr.rng, fr.poses, fr.status), want)
    frames = [{"lut": fr.lut, "range": fr.rng, "poses": fr.poses, "status": fr.status}]
    assert np.array_equal(ob.dewarp_frames(frames), want)


# ------------------------------------------------------------------------------------------------------------------
# provenance, capacity, placements
# ------------------------------------------------------------------------------------------------------------------
def _subsets(items):
    return [pytest.param(s, id="+".join(s) or "none") for k in range(len(items) + 1)
            for s in itertools.combinations(items, k)]


def small_set(ob, dtype, device=(False, False)):
    return [Frame(ob, 20, 70, dtype, 31, device=device[0]), None, Frame(ob, 9, 40, dtype, 32, device=device[1])]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("prov", _subsets(PROV))
def test_provenance_subsets_of_a_set(ob, capi, st, prov, dtype):
    assert dewarp_and_check(ob, capi, st, small_set(ob, dtype), 0.5, 45.0, prov=prov) > 0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("prov", _subsets(("col_idx", "timestamps")))
def test_provenance_subsets_of_a_frame(ob, capi, st, prov, dtype):
    fr = Frame(ob, 20, 70, dtype, 33)
    assert dewarp_and_check(ob, capi, st, [fr], 0.5, 45.0, single=True, prov=prov) > 0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("single", ENTRIES)
def test_host_count_capacity(ob, capi, st, single, dtype):
    """one point too few: "output capacity too small", the count 0, every output byte and counts[] untouched;
    exactly enough: the result"""
    slots = small_set(ob, dtype)[:1] if single else small_set(ob, dtype)
    want, per_slot = expected(slots, 0.5, 45.0)
    n = sum(per_slot)
    out = Outputs(names_for(single), n - 1, dtype)
    count = Count(False)
    counts = None if single else np.full(len(slots), SENT_COUNT, np.uint64)
    status, msg, ran = call(ob, capi, st, slots, 0.5, 45.0, out.ptrs(), n - 1, count, single=single, counts=counts)
    assert status == capi.OB_INVALID_ARGUMENT and msg == "output capacity too small"
    assert ran == 1 and count.value() == 0
    out.untouched()
    if counts is not None:
        assert not counts.any(), counts
    assert dewarp_and_check(ob, capi, st, slots, 0.5, 45.0, single=single, cap=n) == n


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("single", ENTRIES)
def test_device_count_capacity_cuts_the_rows(ob, capi, st, single, dtype):
    slots = small_set(ob, dtype)[:1] if single else small_set(ob, dtype)
    n = sum(expected(slots, 0.5, 45.0)[1])
    for cap in (n - 1, 10, 0):
        dewarp_and_check(ob, capi, st, slots, 0.5, 45.0, single=single, out_device=True, count_device=True, cap=cap)


# id -> (frame inputs on the device, outputs on the device, count on the device)
PLACEMENTS = {
    "host_in_device_out_host_count": ((False, False), True, False),
    "device_in_host_out": ((True, True), False, False),
    "mixed_in_host_out": ((True, False), False, False),
    "mixed_in_device_out_device_count": ((False, True), True, True),
}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("placement,single", [
    pytest.param(p, single, id=f"{p}-{'frame' if single else 'frames'}") for p in PLACEMENTS for single in (True, False)
    if not (single and p.startswith("mixed"))])
def test_placements(ob, capi, st, placement, single, dtype):
    dev_in, out_dev, count_dev = PLACEMENTS[placement]
    slots = small_set(ob, dtype, dev_in)
    assert dewarp_and_check(ob, capi, st, slots[:1] if single else slots, 0.5, 45.0, single=single,
                            out_device=out_dev, count_device=count_dev) > 0


# ------------------------------------------------------------------------------------------------------------------
# refusals, all before anything is staged or launched
# ------------------------------------------------------------------------------------------------------------------
def refused(ob, capi, st, slots, outs, count, msg, *, single=False, counts=None, timestamps=True):
    ptrs = {}
    for o in outs:
        ptrs.update(o.ptrs())
    status, got, ran = call(ob, capi, st, slots, 0.5, 45.0, ptrs, 2000, count, single=single, counts=counts,
                            timestamps=timestamps)
    assert status == capi.OB_INVALID_ARGUMENT and got == msg
    assert ran == 0 and count.value() == 0
    for o in outs:
        o.untouched()


@pytest.mark.parametrize("single", ENTRIES)
def test_device_count_with_a_host_output_is_refused(ob, capi, st, single):
    slots = small_set(ob, np.float32)[:1] if single else small_set(ob, np.float32)
    names = names_for(single)
    for host_name in names:
        dev = Outputs([n for n in names if n != host_name], 2000, np.float32, device=True)
        host = Outputs([host_name], 2000, np.float32)
        refused(ob, capi, st, slots, [dev, host], Count(True), MIXED, single=single)


def test_device_count_with_counts_is_refused(ob, capi, st):
    out = Outputs(names_for(False), 2000, np.float32, device=True)
    counts = np.full(3, SENT_COUNT, np.uint64)
    refused(ob, capi, st, small_set(ob, np.float32), [out], Count(True), MIXED, counts=counts)


def test_luts_of_two_dtypes_are_refused(ob, capi, st):
    slots = [Frame(ob, 20, 70, np.float32, 41), None, Frame(ob, 9, 40, np.float64, 42)]
    out = Outputs(names_for(False), 2000, np.float64)
    counts = np.full(3, SENT_COUNT, np.uint64)
    refused(ob, capi, st, slots, [out], Count(False), "the luts of a set must share one dtype", counts=counts)
    assert not counts.any()


@pytest.mark.parametrize("single", ENTRIES)
def test_timestamps_out_without_timestamps_is_refused(ob, capi, st, single):
    slots = small_set(ob, np.float32)[:1] if single else small_set(ob, np.float32)
    out = Outputs(names_for(single), 2000, np.float32)
    refused(ob, capi, st, slots, [out], Count(False), NO_TS, single=single, timestamps=False)
    # without timestamps_out the column timestamps are not needed
    ok = Outputs(names_for(single, ("frame_idx", "col_idx")), 2000, np.float32)
    status, msg, ran = call(ob, capi, st, slots, 0.5, 45.0, ok.ptrs(), 2000, Count(False), single=single,
                            timestamps=False)
    assert status == 0 and ran == 1, msg


# ------------------------------------------------------------------------------------------------------------------
# status words
# ------------------------------------------------------------------------------------------------------------------
def _status(kind, w):
    s = np.zeros(w, np.uint32)
    if kind == "valid_at_the_two_ends":       # inside: skipped zeros and visited words without the valid bit
        s[1:-1] = np.resize(np.array([0, 2, 0xFFFFFFFE, 4, 0], np.uint32), w - 2)
        s[0] = s[-1] = 1
    elif kind == "one_valid_column":          # the span is that column; the 2s around it are not visited
        s[:] = 2
        s[w // 2 + 7] = 0x80000001
    elif kind == "2_outside_the_span":
        s[:] = 2
        s[5:w - 9] = 1
        s[40:45] = 0
    elif kind == "no_valid_column":           # the kernel runs and finds nothing
        s[:] = 2
    return s


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("single", ENTRIES)
@pytest.mark.parametrize("kind", ["valid_at_the_two_ends", "one_valid_column", "2_outside_the_span",
                                  "no_valid_column"])
def test_status_words(ob, capi, st, kind, single, dtype):
    """100 columns: four CTAs, the last one partial, each finding the frame's first and last valid column"""
    fr = Frame(ob, 20, 100, dtype, 51, status=_status(kind, 100))
    slots = [fr] if single else [Frame(ob, 9, 40, dtype, 52), fr, None]
    n = dewarp_and_check(ob, capi, st, slots, 0.5, 45.0, single=single, launches=1)
    assert (n == 0) == (single and kind == "no_valid_column")
