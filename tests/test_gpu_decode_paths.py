"""K2 (the fused packet decode: decode_pipe_kernel and its fallback decode_kernel) down every path its host code can
pick, driven through the C ABI so that strides and pointer offsets are the test's, and compared byte for byte with
the CPU oracle's FrameBatcher, cartesian and destagger: launch shapes (CTAs per SM, packets per tile, columns per
packet, widths, LUT dtypes), row shifts of every alignment that wrap past the last column, padded / odd / unaligned
packet buffers, strided, interleaved and pooled batch outputs in host and device memory, extreme ranges and the
LUT-free projection.  Every output starts as a 0xA5 byte pattern: every pixel and header entry must be overwritten
and every byte between frames and outputs must still hold the pattern afterwards.  Every case checks which K2 kernel
ran, and a profiler test checks the template instance, grid and block of one case of each kind."""
import ctypes as C
import functools
import json
import os
from importlib import import_module

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import oracle as orc
from tests.helpers import (decoder_desc_from_oracle, default_os1_64, load_fixture, oracle_pf, random_frame,
                           random_lut)

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
TAIL_BYTES = 64          # sentinel bytes after the last block of every buffer
PATHS = ("decode", "batch", "job")
PIPE, GENERIC = "decode_pipe", "decode"
DUAL, SINGLE, LOW, LEGACY = ("RNG19_RFL8_SIG16_NIR16_DUAL", "RNG19_RFL8_SIG16_NIR16", "RNG15_RFL8_NIR8", "LEGACY")

# library defaults of the K2 tunables (OB_* environment variables override them at load, as in ob_api.cu)
K2_TUNABLES = {"decode_stages": 1, "decode_threads": 384, "decode_ctas_per_sm": 3, "decode_tile_packets": 0,
               "decode_prefetch": 0, "decode_runtime_plans": 0, "decode_pipe": 1, "decode_pipe_warps": 24,
               "decode_pipe_dyn_rows": 3, "decode_pipe_tma_xyz": 0, "decode_pipe_ctas": 0, "decode_pipe_helpers": 0,
               "decode_pipe_lane_arrive": 1, "decode_pipe_pk_split": 1, "decode_pipe_lut_split": 1,
               "decode_pipe_prefetch": 0}


def _env_default(name, value):
    v = os.environ.get("OB_" + name.upper())
    return int(v) if v else value


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


def _reset(ob):
    for k, v in K2_TUNABLES.items():
        ob.set_tunable(k, _env_default(k, v))


@pytest.fixture(autouse=True)
def tunables(ob):
    """set(**tunables) for one case; every decode_* tunable is back at its default after each case of the module,
    since the other test files in the process run K2 with the defaults"""
    def set_(**kw):
        for k, v in kw.items():
            ob.set_tunable(k, v)
    try:
        yield set_
    finally:
        _reset(ob)


def _capi(ob):
    capi = import_module(ob.__name__ + "._capi")
    lib = capi.lib
    lib.ob_decode_job_create.restype = C.c_int
    lib.ob_decode_job_create.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_void_p)]
    lib.ob_decode_job_upload.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t]
    lib.ob_decode_job_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    for f in ("ob_decode_job_uploads_done", "ob_decode_job_wait", "ob_decode_job_destroy"):
        getattr(lib, f).argtypes = [C.c_void_p]
    return capi


# ------------------------------------------------------------------------------------------------------------------
# frames, packets and the oracle
# ------------------------------------------------------------------------------------------------------------------
class Frames:
    """F random frames of one packet format: their packets [F, slots, packet_size] and the oracle's batched frames"""

    def __init__(self, pf, srcs):
        self.pf, self.F = pf, len(srcs)
        self.h, self.w = pf.pixels_per_column, pf.columns_per_frame
        self.packets = np.ascontiguousarray(np.stack([orc.frame_to_packets(s, pf)[0] for s in srcs]))
        self.refs = []
        for f, src in enumerate(srcs):
            ref = orc.Frame(pf, with_window=src.has_field("WINDOW"))
            b = orc.Batcher(pf)
            for p in self.packets[f]:
                b.batch(p, 3, ref)
            self.refs.append(ref)
        self.layout, self.fields = decoder_desc_from_oracle(pf, srcs[0])
        self.range_names = {f["range_return"]: f["name"] for f in self.fields if f["range_return"] >= 0}

    def ranges(self, f, r):
        return self.refs[f].field(self.range_names[r])


@functools.lru_cache(maxsize=None)
def frames_of(profile, h, w, cpp=16, F=2, seed=0, extremes=False):
    pf = oracle_pf(profile, h, w, cpp)
    srcs = [random_frame(pf, seed=seed + 31 * f, frame_id=700 + f) for f in range(F)]
    if extremes:   # ranges 0 and 2^19 - 1 (the top of every profile's range field) on whole rows and columns
        for s in srcs:
            for name in ("RANGE", "RANGE2"):
                if s.has_field(name):
                    a = s.field(name)
                    top = pf.value_mask(name)
                    a[0], a[h - 1], a[:, 0] = 0, top, top
                    a[1::7, 3::5] = 0
                    a[2::5, 1::3] = top
    return Frames(pf, srcs)


# the values where uint32 -> float rounds, in a custom layout whose range field is a whole 32-bit word
EXTREMES_32 = np.array([(1 << 24) - 1, 1 << 24, (1 << 24) + 1, (1 << 32) - 1, (1 << 32) - 2, (1 << 19) - 1, 1, 0],
                       np.uint32)


@functools.lru_cache(maxsize=None)
def frames_32bit_range(h=32, w=1024, F=2):
    pf = oracle_pf(SINGLE, h, w)
    pf.set_fields([("RANGE", orc.UINT32, 0, 0xffffffff, 0), ("SIGNAL", orc.UINT16, 4, 0xffff, 0)], 8)
    srcs = []
    for f in range(F):
        s = random_frame(pf, seed=90 + f, with_window=False, frame_id=700 + f)
        a = s.field("RANGE")
        for k, v in enumerate(EXTREMES_32):
            a[3 + k] = v
        a[3 + EXTREMES_32.size] = np.resize(EXTREMES_32, w)
        a[:, 5] = (1 << 32) - 1
        srcs.append(s)
    return Frames(pf, srcs)


def oracle_bytes(fr, d=None, o=None, shifts=None, returns=(0, 1)):
    """{output name: [F] byte rows} of the oracle: fields, column headers, XYZ and destaggered range"""
    raw = lambda a: np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8)
    want = {}
    for f in fr.fields:
        want["field " + f["name"]] = [raw(r.field(f["name"])) for r in fr.refs]
    for k in ("timestamp", "measurement_id", "status"):
        want[k] = [raw(getattr(r, k)) for r in fr.refs]
    for r in fr.range_names:
        if r not in returns:
            continue
        if d is not None:
            want[f"xyz{r}"] = [raw(orc.cartesian(fr.ranges(f, r), d, o)) for f in range(fr.F)]
        if shifts is not None:
            want[f"rd{r}"] = [raw(orc.destagger(fr.ranges(f, r), shifts)) for f in range(fr.F)]
    return want


# ------------------------------------------------------------------------------------------------------------------
# outputs in one allocation, packets with strides and offsets
# ------------------------------------------------------------------------------------------------------------------
def block_sizes(fr, lut_dtype, n_xyz, n_rd):
    """{output name: (bytes per frame, element size)}"""
    n_px, esz = fr.h * fr.w, np.dtype(lut_dtype).itemsize
    out = {"field " + f["name"]: (n_px * f["elem_size"], f["elem_size"]) for f in fr.fields}
    out.update({"timestamp": (fr.w * 8, 8), "measurement_id": (fr.w * 2, 2), "status": (fr.w * 4, 4)})
    out.update({f"xyz{r}": (n_px * 3 * esz, esz) for r in range(n_xyz)})
    out.update({f"rd{r}": (n_px * 4, 4) for r in range(n_rd)})
    return out


def output_layout(kind, blocks, F):
    """{name: (offset, frame stride)} in bytes of one allocation.
    dense: every output its own F-block region; padded: 64 bytes between frames; odd: 3 elements between frames
    (not a multiple of 16 bytes); xyz_odd: dense, XYZ as in odd; interleaved: XYZ and destaggered range as K1's
    [F, R, ...] arrays (return 1 right after return 0, frame stride two blocks); pool: all outputs of a frame
    back to back, 16-byte aligned, frame after frame"""
    lay, pos = {}, 0
    up = lambda n, a: (n + a - 1) // a * a
    if kind == "pool":
        for name, (b, _) in blocks.items():
            lay[name] = pos
            pos = up(pos + b, 16)
        return {name: (off, pos) for name, off in lay.items()}
    for name, (b, es) in blocks.items():
        if kind == "interleaved" and name[:-1] in ("xyz", "rd") and name[-1] == "1":
            continue
        fs = b
        if kind == "padded":
            fs = b + 64
        elif kind == "odd" or (kind == "xyz_odd" and name.startswith("xyz")):
            fs = b + 3 * es
        pair = kind == "interleaved" and name[:-1] in ("xyz", "rd") and name[:-1] + "1" in blocks
        if pair:
            fs = 2 * b
            lay[name[:-1] + "1"] = (pos + b, fs)
        lay[name] = (pos, fs)
        pos = up(pos + (F - 1) * fs + (2 * b if pair else b), 256) + 256   # a sentinel gap between regions
    return lay


class Outputs:
    """sentinel-filled outputs of F frames at (offset, frame stride) in one flat buffer: numpy, or a CUDA tensor"""

    def __init__(self, blocks, lay, F, device):
        self.blocks, self.lay, self.F, self.device = blocks, lay, F, device
        size = max(off + (F - 1) * fs + blocks[n][0] for n, (off, fs) in lay.items()) + TAIL_BYTES
        host = np.full(size, SENTINEL, np.uint8)
        if device:
            import torch
            self.buf = torch.from_numpy(host).cuda()
        else:
            self.buf = host

    def ptr(self, name, f=0):
        if name not in self.lay:
            return None
        base = self.buf.data_ptr() if self.device else self.buf.ctypes.data
        off, fs = self.lay[name]
        return base + off + f * fs

    def stride(self, name):
        return self.lay[name][1] if name in self.lay else 0

    def check(self, want, approx=None):
        """every block equals `want` byte for byte (outputs in `approx` are left to the caller) and no byte outside
        the blocks lost the sentinel; returns {name: [F] byte rows}"""
        b = self.buf.cpu().numpy() if self.device else self.buf
        covered = np.zeros(b.size, bool)
        got = {}
        for name, (off, fs) in self.lay.items():
            n = self.blocks[name][0]
            got[name] = [b[off + f * fs: off + f * fs + n] for f in range(self.F)]
            for f in range(self.F):
                covered[off + f * fs: off + f * fs + n] = True
        bad = np.count_nonzero(b[~covered] != SENTINEL)
        assert bad == 0, f"{bad} bytes between or after the output blocks lost the sentinel"
        assert sorted(got) == sorted(want), (sorted(got), sorted(want))
        for name in want:
            if approx and name in approx:
                continue
            for f in range(self.F):
                if not np.array_equal(got[name][f], want[name][f]):
                    diff = np.flatnonzero(got[name][f] != want[name][f])
                    raise AssertionError(f"{name} frame {f}: {diff.size} bytes differ, first at byte {diff[0]}")
        return got


class Packets:
    """packets [F, slots, size] at base + offset + f * frame stride + k * packet stride, in host or device memory"""

    def __init__(self, packets, stride=None, frame_stride=None, offset=0, device=False):
        F, n, size = packets.shape
        self.n_slots, self.size = n, size
        self.stride = stride or size
        self.frame_stride = frame_stride or n * self.stride
        self.off = offset
        host = np.full(offset + (F - 1) * self.frame_stride + (n - 1) * self.stride + size + TAIL_BYTES, 0x5A,
                       np.uint8)
        for f in range(F):
            for k in range(n):
                s = offset + f * self.frame_stride + k * self.stride
                host[s:s + size] = packets[f, k]
        if device:
            import torch
            self.buf = torch.from_numpy(host).cuda()
        else:
            self.buf = host
        self.device = device

    def ptr(self, f=0):
        return (self.buf.data_ptr() if self.device else self.buf.ctypes.data) + self.off + f * self.frame_stride


def decoder(ob, fr):
    return ob.Decoder(fr.layout, fr.fields)


def run(ob, path, dec, fr, pk, out, lut=None, frame_luts=None, shifts=None, want=PIPE):
    """one decode of fr.F frames through one entry point; checks that it launched the `want` K2 kernel"""
    capi = _capi(ob)
    lib, check = capi.lib, capi.check
    F = fr.F
    sh = None if shifts is None else np.ascontiguousarray(shifts, np.int32)
    sh_ptr, n_sh = (None, 0) if sh is None else (sh.ctypes.data, sh.size)
    lut_h = lut._h if lut is not None else None
    names_r = lambda prefix: [f"{prefix}{r}" for r in range(2)]
    if out.device or pk.device:
        import torch
        torch.cuda.synchronize()
    st = ob.Stream(0)
    before = {k: ob.kernel_launch_count(k) for k in (PIPE, GENERIC)}

    def fill_io(io, f):
        for i, fd in enumerate(fr.fields):
            io.fields[i] = out.ptr("field " + fd["name"], f)
        io.timestamp, io.measurement_id = out.ptr("timestamp", f), out.ptr("measurement_id", f)
        io.status = out.ptr("status", f)
        for r, (x, d) in enumerate(zip(names_r("xyz"), names_r("rd"))):
            io.xyz[r], io.range_destaggered[r] = out.ptr(x, f), out.ptr(d, f)
        if frame_luts:
            io.lut = frame_luts[f]._h

    if path == "batch":
        b = capi.DecodeBatch()
        b.n_frames, b.packets, b.n_slots = F, pk.ptr(), pk.n_slots
        b.packet_stride, b.packets_frame_stride = pk.stride, pk.frame_stride
        for i, fd in enumerate(fr.fields):
            b.fields[i] = out.ptr("field " + fd["name"])
            b.field_frame_stride[i] = out.stride("field " + fd["name"])
        b.timestamp, b.timestamp_frame_stride = out.ptr("timestamp"), out.stride("timestamp")
        b.measurement_id, b.measurement_id_frame_stride = out.ptr("measurement_id"), out.stride("measurement_id")
        b.status, b.status_frame_stride = out.ptr("status"), out.stride("status")
        for r, (x, d) in enumerate(zip(names_r("xyz"), names_r("rd"))):
            b.xyz[r], b.range_destaggered[r] = out.ptr(x), out.ptr(d)
        b.xyz_frame_stride, b.rd_frame_stride = out.stride("xyz0"), out.stride("rd0")
        if frame_luts:
            handles = (C.c_void_p * F)(*[lt._h.value for lt in frame_luts])
            b.frame_luts = C.cast(handles, C.POINTER(C.c_void_p))
        check(lib.ob_decode_batch_run(dec._h, C.byref(b), lut_h, sh_ptr, n_sh, st.h))
    elif path == "decode":
        ios = (capi.DecodeIO * F)()
        for f in range(F):
            ios[f].packets, ios[f].n_slots, ios[f].packet_stride = pk.ptr(f), pk.n_slots, pk.stride
            fill_io(ios[f], f)
        check(lib.ob_decode_frames(dec._h, ios, F, lut_h, sh_ptr, n_sh, st.h))
    else:
        job = C.c_void_p()
        check(lib.ob_decode_job_create(dec._h, 0, st.h, C.byref(job)))
        try:
            for f in range(F):
                check(lib.ob_decode_job_upload(job, pk.ptr(f), pk.stride, 0, pk.n_slots))
                check(lib.ob_decode_job_uploads_done(job))
                io = capi.DecodeIO()
                io.n_slots = pk.n_slots
                fill_io(io, f)
                check(lib.ob_decode_job_submit(job, C.byref(io), lut_h, sh_ptr, n_sh))
                check(lib.ob_decode_job_wait(job))
        finally:
            check(lib.ob_decode_job_destroy(job))
    st.sync()
    launches = 1 if path == "batch" or path == "decode" else F
    grew = {k: ob.kernel_launch_count(k) - before[k] for k in before}
    assert grew == {PIPE: launches if want == PIPE else 0, GENERIC: launches}, (want, grew)


def decode_and_check(ob, fr, *, path="batch", dtype=np.float32, kind="dense", device=False, returns=None,
                     shifts=None, want=PIPE, pk=None, lut_seed=3):
    """decodes fr with a random table LUT and shifts into outputs of layout `kind`; everything byte-exact"""
    dec = decoder(ob, fr)
    n_ret = len(fr.range_names) if returns is None else returns
    d, o = random_lut(fr.h * fr.w, lut_seed, dtype)
    lut = ob.XYZLutT.from_arrays(d, o, fr.h, fr.w)
    if shifts is None:
        shifts = np.random.default_rng(fr.w + fr.h).integers(-fr.w, 2 * fr.w, fr.h).astype(np.int32)
        if fr.w & (fr.w - 1):
            shifts = np.abs(shifts)
    blocks = block_sizes(fr, dtype, n_ret, n_ret)
    out = Outputs(blocks, output_layout(kind, blocks, fr.F), fr.F, device)
    run(ob, path, dec, fr, pk or Packets(fr.packets), out, lut=lut, shifts=shifts, want=want)
    out.check(oracle_bytes(fr, d, o, shifts, returns=range(n_ret)))


DTYPES = [pytest.param(np.float32, id="f32"), pytest.param(np.float64, id="f64")]


# ------------------------------------------------------------------------------------------------------------------
# launch shapes
# ------------------------------------------------------------------------------------------------------------------
# id -> (profile, H, W, columns per packet, tunables, kernel).  From the packet sizes (32 + 32 bytes of packet header
# and footer, 16 columns of 12 + H * pixel bytes): the automatic shape gives 3 CTAs per SM to 32-row dual (8448-byte
# packets), 2 to 64-row LEGACY (12608) and 1 to 128-row dual (33024); one-packet tiles (16 columns) are below the
# pipelined kernel's 32-column minimum and a width that is not a multiple of 32 columns has no whole tiles.
SHAPES = {
    "auto3_32_dual": (DUAL, 32, 1024, 16, {}, PIPE),
    "auto3_32_single": (SINGLE, 32, 512, 16, {}, PIPE),
    "auto2_64_legacy": (LEGACY, 64, 1024, 16, {}, PIPE),
    "auto1_64_dual": (DUAL, 64, 1024, 16, {}, PIPE),
    "auto1_128_dual": (DUAL, 128, 1024, 16, {}, PIPE),
    "auto1_128_single": (SINGLE, 128, 2048, 16, {}, PIPE),
    "ctas1": (DUAL, 32, 1024, 16, {"decode_pipe_ctas": 1}, PIPE),
    "ctas2": (DUAL, 32, 1024, 16, {"decode_pipe_ctas": 2}, PIPE),
    "ctas3": (DUAL, 32, 1024, 16, {"decode_pipe_ctas": 3}, PIPE),
    "tile_packets2": (DUAL, 64, 1024, 16, {"decode_tile_packets": 2}, PIPE),
    "tile_packets4": (DUAL, 32, 1024, 16, {"decode_tile_packets": 4}, PIPE),
    "tile_packets1": (DUAL, 64, 1024, 16, {"decode_tile_packets": 1}, GENERIC),
    "cpp4_64": (SINGLE, 64, 1024, 4, {}, PIPE),
    "cpp8_64": (SINGLE, 64, 1024, 8, {}, PIPE),
    "cpp32_64": (SINGLE, 64, 1024, 32, {}, PIPE),
    "cpp4_128": (SINGLE, 128, 1024, 4, {}, PIPE),
    "cpp8_128": (SINGLE, 128, 1024, 8, {}, PIPE),
    "cpp32_128": (SINGLE, 128, 1024, 32, {}, PIPE),
    "w512": (DUAL, 64, 512, 16, {}, PIPE),
    "w2048": (DUAL, 64, 2048, 16, {}, PIPE),
    "w1008_partial_tile": (DUAL, 64, 1008, 16, {}, GENERIC),
    "pipe_off": (DUAL, 64, 1024, 16, {"decode_pipe": 0}, GENERIC),
}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_launch_shapes(ob, tunables, shape, dtype):
    profile, H, W, cpp, tun, want = SHAPES[shape]
    tunables(**tun)
    decode_and_check(ob, frames_of(profile, H, W, cpp, seed=H + W + cpp), dtype=dtype, want=want)


# ------------------------------------------------------------------------------------------------------------------
# row shifts
# ------------------------------------------------------------------------------------------------------------------
def edge_shifts(W):
    """each q = shift & 3 on rows whose destination wraps past column W, shifts that cross a 32- and a 64-column tile,
    shifts of whole rows and several rows; negative ones on power-of-two widths only (DESIGN §9)"""
    s = []
    for q in range(4):
        s += [q, 4 + q, 28 + q, 60 + q, W // 2 + q, W - 8 + q, W - 4 + q, W - 132 + q]
    s += [0, W, 3 * W + 2, W - 1, W + 1, 2 * W - 1]
    if (W & (W - 1)) == 0:
        s += [-W, -(W + 1), -1, -3, -4, -33, -65, -W // 2 - 1, -3 * W + 5]
    return np.array(s, np.int32)


SHIFT_CASES = [pytest.param(DUAL, 48, 512, id="dual_512"), pytest.param(SINGLE, 48, 1024, id="single_1024"),
               pytest.param(DUAL, 48, 1008, id="dual_1008"), pytest.param(LOW, 512, 1024, id="low_512rows")]


@pytest.mark.parametrize("kernel", [PIPE, GENERIC])
@pytest.mark.parametrize("profile,H,W", SHIFT_CASES)
def test_row_shifts(ob, tunables, profile, H, W, kernel):
    """the edge table repeated over H rows; W = 1008 has no whole 32-column tiles and always takes decode_kernel;
    512 rows is the fused destagger's limit"""
    if kernel == GENERIC:
        tunables(decode_pipe=0)
    want = GENERIC if W % 32 else kernel
    fr = frames_of(profile, H, W, seed=H * 3 + W)
    decode_and_check(ob, fr, shifts=np.resize(edge_shifts(W), H), want=want)


# ------------------------------------------------------------------------------------------------------------------
# packet layout
# ------------------------------------------------------------------------------------------------------------------
# id -> (extra bytes per packet slot, extra bytes per frame, base offset)
PACKET_LAYOUTS = {
    "dense": (0, 0, 0),
    "stride_pad64": (64, 0, 0),
    "stride_odd": (1, 0, 0),
    "frame_pad": (0, 48, 0),
    "frame_odd": (0, 5, 0),
    "base_off1": (0, 0, 1),
    "all_odd": (3, 7, 1),
}


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("device", [pytest.param(False, id="host"), pytest.param(True, id="device")])
@pytest.mark.parametrize("pk_layout", list(PACKET_LAYOUTS))
def test_packet_layout(ob, pk_layout, device, path):
    """packet strides and offsets that turn the producer's bulk copies off (the column gather path) must decode the
    same frames"""
    if device:
        pytest.importorskip("torch")
    fr = frames_of(DUAL, 32, 1024, seed=11, F=3)
    dp, df, off = PACKET_LAYOUTS[pk_layout]
    psize = fr.packets.shape[2]
    pk = Packets(fr.packets, psize + dp, fr.packets.shape[1] * (psize + dp) + df, off, device)
    decode_and_check(ob, fr, path=path, pk=pk)


# ------------------------------------------------------------------------------------------------------------------
# batch outputs
# ------------------------------------------------------------------------------------------------------------------
OUTPUT_KINDS = ("dense", "padded", "odd", "xyz_odd", "interleaved", "pool")


def batch_kernel(kind, device):
    """host outputs with a frame stride are staged densely; device XYZ whose frame stride is not a multiple of 16
    bytes leaves the pipelined kernel's aligned stores out"""
    return GENERIC if device and kind in ("odd", "xyz_odd") else PIPE


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("device", [pytest.param(False, id="host"), pytest.param(True, id="device")])
@pytest.mark.parametrize("kind", OUTPUT_KINDS)
def test_batch_outputs(ob, kind, device, dtype):
    if device:
        pytest.importorskip("torch")
    fr = frames_of(DUAL, 32, 512, seed=5, F=3)
    decode_and_check(ob, fr, dtype=dtype, kind=kind, device=device, want=batch_kernel(kind, device))


@pytest.mark.parametrize("path", ["decode", "job"])
@pytest.mark.parametrize("kind", ["padded", "interleaved", "pool"])
def test_per_frame_outputs_in_one_allocation(ob, kind, path):
    """the same layouts through the per-frame entry points, which stage one block per output"""
    fr = frames_of(DUAL, 32, 512, seed=5, F=3)
    decode_and_check(ob, fr, path=path, kind=kind)


@pytest.mark.parametrize("device", [pytest.param(False, id="host"), pytest.param(True, id="device")])
def test_batch_single_return_subset(ob, device):
    """a dual-return decoder asked for return 0's XYZ and destaggered range only, in the pool layout"""
    if device:
        pytest.importorskip("torch")
    fr = frames_of(DUAL, 32, 512, seed=5, F=3)
    decode_and_check(ob, fr, kind="pool", device=device, returns=1)


# ------------------------------------------------------------------------------------------------------------------
# range extremes
# ------------------------------------------------------------------------------------------------------------------
EXTREME_PROFILES = [DUAL, SINGLE, LOW, LEGACY, "RNG15_RFL8_NIR8_DUAL", "RNG15_RFL8_WIN8",
                    "RNG19_RFL8_SIG16_ZONE16_DUAL"]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("profile", EXTREME_PROFILES)
def test_range_extremes(ob, profile, dtype):
    """ranges 0 and the largest value of each profile's range field on whole rows and columns"""
    fr = frames_of(profile, 32, 512, seed=13, extremes=True)
    decode_and_check(ob, fr, dtype=dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kernel", [PIPE, GENERIC])
def test_32bit_range_extremes(ob, tunables, kernel, dtype):
    if kernel == GENERIC:
        tunables(decode_pipe=0)
    decode_and_check(ob, frames_32bit_range(), dtype=dtype, want=kernel)


# ------------------------------------------------------------------------------------------------------------------
# LUT-free projection
# ------------------------------------------------------------------------------------------------------------------
def intrinsics(source):
    if source.startswith("os1_64_"):
        return default_os1_64(int(source.split("_")[-1]))
    m, _ = load_fixture(source)
    return m


ANALYTIC_SOURCES = ["os1_64_512", "os1_64_1024", "os1_64_2048", "OS-0-32-U1_v2.2.0_1024x10",
                    "OS-1-128_767798045_1024x10_20230712_120049"]
# norm-wise relative and absolute error of the LUT-free projection against the float64 restatement (K1's bounds)
ANALYTIC_TOL = {np.dtype(np.float32): (1e-5, 1e-7), np.dtype(np.float64): (1e-12, 1e-12)}


def analytic_lut(ob, m, dtype):
    args = (m["w"], m["h"], 0.001, m["beam_to_lidar_transform"], m["lidar_to_sensor_transform"],
            m["beam_azimuth_angles"], m["beam_altitude_angles"])
    return ob.XYZLutT.from_intrinsics(*args, dtype=dtype), args


def check_lut_free(fr, got, returns, dtype, args_by_frame):
    """XYZ of the frames in args_by_frame ({frame: intrinsics}) within ANALYTIC_TOL of their float64 LUT, empty
    returns +0.0 by bit pattern"""
    rel, ab = ANALYTIC_TOL[np.dtype(dtype)]
    for f, args in args_by_frame.items():
        d64, o64 = orc.make_xyz_lut(*args)
        for r in returns:
            rv = fr.ranges(f, r).reshape(-1)
            xyz = got[f"xyz{r}"][f].view(dtype).reshape(-1, 3)
            ref = np.where(rv[:, None] == 0, 0.0, rv[:, None].astype(np.float64) * d64 + o64)
            err = np.linalg.norm(xyz.astype(np.float64) - ref, axis=-1)
            lim = rel * np.linalg.norm(ref, axis=-1) + ab
            assert np.all(err <= lim), (f, r, float(np.max(err / np.maximum(lim, 1e-300))))
            assert not np.any(xyz[rv == 0].view(np.uint64 if xyz.itemsize == 8 else np.uint32)), \
                "empty returns must be +0.0"


def profile_for(m, R):
    if R == 1:
        return LOW if m["h"] != 64 else SINGLE
    return DUAL


def lut_free_case(ob, source, R, dtype, F=2, seed=1):
    m = intrinsics(source)
    H, W = m["h"], m["w"]
    fr = frames_of(profile_for(m, R), H, W, seed=seed + H, F=F, extremes=True)
    lut, args = analytic_lut(ob, m, dtype)
    return fr, lut, args, np.asarray(m["pixel_shift_by_row"], np.int32)


LUT_FREE_CASES = [pytest.param(s, "batch", id=f"{s}-batch") for s in ANALYTIC_SOURCES]
LUT_FREE_CASES += [pytest.param("os1_64_1024", p, id=f"os1_64_1024-{p}") for p in ("decode", "job")]
LUT_FREE_CASES += [pytest.param("OS-0-32-U1_v2.2.0_1024x10", "job", id="OS-0-32-job")]


@pytest.mark.parametrize("R", [pytest.param(1, id="R1"), pytest.param(2, id="R2")])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("source,path", LUT_FREE_CASES)
def test_lut_free(ob, source, path, dtype, R):
    fr, lut, args, shifts = lut_free_case(ob, source, R, dtype)
    lut.set_analytic(True)
    dec = decoder(ob, fr)
    blocks = block_sizes(fr, dtype, R, R)
    out = Outputs(blocks, output_layout("dense", blocks, fr.F), fr.F, False)
    run(ob, path, dec, fr, Packets(fr.packets), out, lut=lut, shifts=shifts)
    xyz = {f"xyz{r}" for r in range(R)}   # checked against the float64 LUT below
    got = out.check({**oracle_bytes(fr, None, None, shifts), **dict.fromkeys(xyz)}, approx=xyz)
    check_lut_free(fr, got, range(R), dtype, dict.fromkeys(range(fr.F), args))


@pytest.mark.parametrize("path", ["batch", "decode"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_lut_free_mixed_with_table_luts(ob, path, dtype):
    """per-frame LUTs of one dtype in one launch: LUT-free ones (two sensors' intrinsics) next to table ones; the
    table frames stay bit-exact, the LUT-free ones within tolerance"""
    m0 = intrinsics("os1_64_1024")
    m1 = dict(m0)
    m1["beam_azimuth_angles"] = np.asarray(m0["beam_azimuth_angles"]) * 1.5
    m1["lidar_to_sensor_transform"] = np.array(m0["lidar_to_sensor_transform"]) @ np.diag([1.0, -1.0, -1.0, 1.0])
    H, W, F = m0["h"], m0["w"], 4
    fr = frames_of(DUAL, H, W, seed=23, F=F, extremes=True)
    free0, args0 = analytic_lut(ob, m0, dtype)
    free1, args1 = analytic_lut(ob, m1, dtype)
    tables = [random_lut(H * W, 50 + f, dtype) for f in range(F)]
    luts = [free0.set_analytic(True), ob.XYZLutT.from_arrays(*tables[1], H, W), free1.set_analytic(True),
            ob.XYZLutT.from_arrays(*tables[3], H, W)]
    shifts = np.asarray(m0["pixel_shift_by_row"], np.int32)
    dec = decoder(ob, fr)
    blocks = block_sizes(fr, dtype, 2, 2)
    out = Outputs(blocks, output_layout("dense", blocks, F), F, False)
    run(ob, path, dec, fr, Packets(fr.packets), out, frame_luts=luts, shifts=shifts)
    want = oracle_bytes(fr, None, None, shifts)
    got = out.check({**want, "xyz0": None, "xyz1": None}, approx={"xyz0", "xyz1"})
    for f in (1, 3):
        for r in range(2):
            assert np.array_equal(got[f"xyz{r}"][f].view(dtype).reshape(-1, 3),
                                  orc.cartesian(fr.ranges(f, r), *tables[f])), (f, r)
    check_lut_free(fr, got, range(2), dtype, {0: args0, 2: args1})


def _w1008_intrinsics():
    m = dict(default_os1_64(1024))
    m["w"] = 1008
    return m


FALLBACKS = {   # id -> (intrinsics, tunables, output layout, device outputs)
    "pipe_off": (lambda: intrinsics("os1_64_1024"), {"decode_pipe": 0}, "dense", False),
    "w1008": (_w1008_intrinsics, {}, "dense", False),
    "xyz_odd_device": (lambda: intrinsics("os1_64_1024"), {}, "xyz_odd", True),
}


@pytest.mark.parametrize("R", [pytest.param(1, id="R1"), pytest.param(2, id="R2")])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", list(FALLBACKS))
def test_lut_free_falls_back_bit_exact(ob, tunables, case, dtype, R):
    """decode_kernel has no LUT-free path: where the pipelined kernel declines, a LUT-free LUT gives its tables'
    result bit for bit"""
    mk, tun, kind, device = FALLBACKS[case]
    if device:
        pytest.importorskip("torch")
    tunables(**tun)
    m = mk()
    fr = frames_of(profile_for(m, R), m["h"], m["w"], seed=7, extremes=True)
    lut, _ = analytic_lut(ob, m, dtype)
    d, o = lut.direction, lut.offset        # the device-built tables the LUT path reads
    lut.set_analytic(True)
    shifts = np.asarray(m["pixel_shift_by_row"], np.int32)
    blocks = block_sizes(fr, dtype, R, R)
    out = Outputs(blocks, output_layout(kind, blocks, fr.F), fr.F, device)
    run(ob, "batch", decoder(ob, fr), fr, Packets(fr.packets), out, lut=lut, shifts=shifts, want=GENERIC)
    out.check(oracle_bytes(fr, d, o, shifts))


# ------------------------------------------------------------------------------------------------------------------
# which kernel ran
# ------------------------------------------------------------------------------------------------------------------
def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pipe(t, ctas, block, tc):
    """decode_pipe_kernel<T, build>: the 1024-thread build when CTAs share an SM, else the 864-thread one"""
    return (f"decode_pipe_kernel<{t}, {1024 if ctas > 1 else 864}>", ctas, block, tc)


# id -> (tunables, call, (kernel, CTAs per SM, block, tile columns) or the kernel name alone).  Block = compute
# warps + producer + store warp + one helper slot: 6 compute warps at 3 CTAs per SM, 12 at 2, 24 at 1.
PROFILED = [
    ("shape_auto3", {}, dict(shape="auto3_32_dual"), _pipe("float", 3, 288, 32)),
    ("shape_auto2", {}, dict(shape="auto2_64_legacy"), _pipe("float", 2, 480, 32)),
    ("shape_auto1", {}, dict(shape="auto1_128_dual", dtype=np.float64), _pipe("double", 1, 864, 32)),
    ("shape_ctas1", {"decode_pipe_ctas": 1}, dict(shape="ctas1"), _pipe("float", 1, 864, 64)),
    ("shape_ctas2", {"decode_pipe_ctas": 2}, dict(shape="ctas2"), _pipe("float", 2, 480, 32)),
    ("shape_tile_packets4", {"decode_tile_packets": 4}, dict(shape="tile_packets4"), _pipe("float", 1, 864, 64)),
    ("shape_cpp4", {}, dict(shape="cpp4_128"), "decode_pipe_kernel<float"),
    ("shape_tile_packets1", {"decode_tile_packets": 1}, dict(shape="tile_packets1"), "decode_kernel<float>"),
    ("shape_w1008", {}, dict(shape="w1008_partial_tile", dtype=np.float64), "decode_kernel<double>"),
    ("row_shifts", {}, dict(shifts=("low_512rows",)), "decode_pipe_kernel<float"),
    ("packet_all_odd", {}, dict(packets="all_odd"), "decode_pipe_kernel<float"),
    ("batch_pool_host", {}, dict(kind="pool"), "decode_pipe_kernel<float"),
    ("batch_odd_device", {}, dict(kind="odd", device=True), "decode_kernel<float>"),
    ("range_32bit", {}, dict(range32=True), "decode_pipe_kernel<float"),
    ("lut_free", {}, dict(lut_free="os1_64_1024"), "decode_pipe_kernel<float"),
    ("lut_free_fallback", {}, dict(lut_free="w1008"), "decode_kernel<float>"),
]


def _profiled_call(ob, shape=None, dtype=np.float32, shifts=None, packets=None, kind="dense", device=False,
                   range32=False, lut_free=None):
    """(call, frames in the launch, width): one case of the tables above"""
    if shape is not None:
        profile, H, W, cpp, _, want = SHAPES[shape]
        fr = frames_of(profile, H, W, cpp, seed=H + W + cpp)
        return (lambda: decode_and_check(ob, fr, dtype=dtype, want=want)), fr
    if shifts is not None:
        fr = frames_of(LOW, 512, 1024, seed=512 * 3 + 1024)
        return (lambda: decode_and_check(ob, fr, shifts=np.resize(edge_shifts(1024), 512))), fr
    if packets is not None:
        fr = frames_of(DUAL, 32, 1024, seed=11, F=3)
        dp, df, off = PACKET_LAYOUTS[packets]
        psize = fr.packets.shape[2]
        pk = Packets(fr.packets, psize + dp, fr.packets.shape[1] * (psize + dp) + df, off)
        return (lambda: decode_and_check(ob, fr, pk=pk)), fr
    if range32:
        fr = frames_32bit_range()
        return (lambda: decode_and_check(ob, fr)), fr
    if lut_free is not None:
        m = _w1008_intrinsics() if lut_free == "w1008" else intrinsics(lut_free)
        fr = frames_of(DUAL, m["h"], m["w"], seed=7, extremes=True)
        lut, _ = analytic_lut(ob, m, np.float32)
        lut.set_analytic(True)
        blocks = block_sizes(fr, np.float32, 2, 2)
        out = Outputs(blocks, output_layout("dense", blocks, fr.F), fr.F, False)
        want = GENERIC if lut_free == "w1008" else PIPE
        sh = np.asarray(m["pixel_shift_by_row"], np.int32)
        return (lambda: run(ob, "batch", decoder(ob, fr), fr, Packets(fr.packets), out, lut=lut, shifts=sh,
                            want=want)), fr
    fr = frames_of(DUAL, 32, 512, seed=5, F=3)
    return (lambda: decode_and_check(ob, fr, kind=kind, device=device, want=batch_kernel(kind, device))), fr


def test_kernels_that_ran(ob, tunables, tmp_path):
    """each representative case under torch.profiler: the K2 kernel it launched is the template instance its row
    expects, and where the row is about launch geometry, the grid and block say which geometry ran.  A case that
    should take the pipelined kernel but falls to decode_kernel fails here."""
    torch = pytest.importorskip("torch")
    from torch.profiler import ProfilerActivity, profile
    sm = _sm_count()
    seen = {}
    for case_id, tun, kw, want in PROFILED:
        _reset(ob)
        tunables(**tun)
        call, fr = _profiled_call(ob, **kw)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        trace = tmp_path / f"{case_id}.json"
        prof.export_chrome_trace(str(trace))
        events = json.load(open(trace))["traceEvents"]
        ran = [e for e in events if e.get("cat") == "kernel" and "decode" in e["name"] and "_kernel" in e["name"]]
        names = [e["name"] for e in ran]
        seen[case_id] = names
        assert len(ran) == 1, (case_id, names)
        name = want if isinstance(want, str) else want[0]
        assert name in names[0], (case_id, names, want)
        if not isinstance(want, str):
            _, ctas, block, tc = want
            args = ran[0]["args"]
            assert args["block"][0] == block, (case_id, args)
            assert args["grid"][0] == min(fr.F * fr.w // tc, ctas * sm), (case_id, args)
    print(json.dumps(seen, indent=1))
