"""The three decode entry points -- Decoder.decode (ob_decode_frames), Decoder.decode_batch (ob_decode_batch_run)
and the ob_decode_job_* C ABI -- build their launches through one set of argument rules.  The same frames come out
byte-identical through each of them and equal to the oracle, each path takes the same kernel, and every invalid
input is refused by each entry point that can receive it with one message, before any output is written."""
import ctypes as C
import functools
from importlib import import_module

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import oracle as orc
from tests.helpers import decoder_desc_from_oracle, oracle_pf, random_frame, random_lut

pytestmark = pytest.mark.gpu

PATHS = ("decode", "batch", "job")
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


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


def _ptr(a):
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


def _outputs(dec, n, lut_dtype, n_xyz, n_rd, device):
    """sentinel-filled outputs of n frames, one row of bytes per frame"""
    h, w = dec.h_px, dec.w_px
    esz = np.dtype(lut_dtype).itemsize

    def buf(nbytes):
        if device:
            import torch
            return torch.full((n, nbytes), SENTINEL, dtype=torch.uint8, device="cuda")
        return np.full((n, nbytes), SENTINEL, np.uint8)
    return {"fields": {f["name"]: buf(h * w * f["elem_size"]) for f in dec.fields},
            "timestamp": buf(w * 8), "measurement_id": buf(w * 2), "status": buf(w * 4),
            "xyz": [buf(h * w * 3 * esz) for _ in range(n_xyz)], "rd": [buf(h * w * 4) for _ in range(n_rd)]}


def _flat(out):
    d = {"field " + k: v for k, v in out["fields"].items()}
    d.update({k: out[k] for k in ("timestamp", "measurement_id", "status")})
    d.update({f"xyz{r}": a for r, a in enumerate(out["xyz"])})
    d.update({f"rd{r}": a for r, a in enumerate(out["rd"])})
    return {k: (v.cpu().numpy() if hasattr(v, "cpu") else v.copy()) for k, v in d.items()}


def _run(ob, path, dec, packets, out, lut=None, frame_luts=None, shifts=None, packet_stride=None, n_slots=None):
    """decodes packets[k] (one row of packet slots per frame) into row k of every output through one entry point"""
    st = ob.Stream()
    n = packets.shape[0]
    stride = packet_stride or packets.shape[2]
    n_slots = n_slots or packets.shape[1]
    if path == "decode":
        frames = [{"packets": packets[k], "n_slots": n_slots, "packet_stride": stride, "col_src": None,
                   "fields": {name: a[k] for name, a in out["fields"].items()},
                   "timestamp": out["timestamp"][k], "measurement_id": out["measurement_id"][k],
                   "status": out["status"][k], "xyz": [a[k] for a in out["xyz"]],
                   "range_destaggered": [a[k] for a in out["rd"]],
                   "lut": frame_luts[k] if frame_luts else None} for k in range(n)]
        dec.decode(frames, lut=lut, pixel_shift_by_row=shifts, stream=st)
    elif path == "batch":
        dec.decode_batch(n, packets, n_slots, stride, packets.shape[1] * packets.shape[2], out["fields"], lut=lut,
                         pixel_shift_by_row=shifts, xyz=out["xyz"], range_destaggered=out["rd"],
                         timestamp=out["timestamp"], measurement_id=out["measurement_id"], status=out["status"],
                         stream=st, frame_luts=frame_luts)
    else:
        capi = _capi(ob)
        lib, check = capi.lib, capi.check
        job = C.c_void_p()
        check(lib.ob_decode_job_create(dec._h, 0, st.h, C.byref(job)))
        try:
            for k in range(n):
                check(lib.ob_decode_job_upload(job, packets[k].ctypes.data, stride, 0, n_slots))
                check(lib.ob_decode_job_uploads_done(job))
                io = capi.DecodeIO()
                io.n_slots = n_slots
                for i, f in enumerate(dec.fields):
                    io.fields[i] = _ptr(out["fields"][f["name"]][k])
                io.timestamp, io.measurement_id = _ptr(out["timestamp"][k]), _ptr(out["measurement_id"][k])
                io.status = _ptr(out["status"][k])
                for r, a in enumerate(out["xyz"]):
                    io.xyz[r] = _ptr(a[k])
                for r, a in enumerate(out["rd"]):
                    io.range_destaggered[r] = _ptr(a[k])
                if frame_luts:
                    io.lut = frame_luts[k]._h
                check(lib.ob_decode_job_submit(job, C.byref(io), lut._h if lut is not None else None,
                                               shifts.ctypes.data if shifts is not None else None,
                                               0 if shifts is None else shifts.size))
                check(lib.ob_decode_job_wait(job))
        finally:
            check(lib.ob_decode_job_destroy(job))
    st.sync()


# ---- same frames, three entry points ------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _case(name):
    """(pf, oracle frames, packets [n, slots, bytes], shifts, kernel family) of three frames"""
    if name == "dual_128x1024":   # the pipelined kernel
        pf = oracle_pf("RNG19_RFL8_SIG16_NIR16_DUAL", 128, 1024)
        srcs = [random_frame(pf, seed=40 + k, frame_id=800 + k) for k in range(3)]
        kw = dict(with_window=True)
        shifts = np.tile(np.array([12, 8, 4, 0], np.int32), 32)
        family = "decode_pipe"
    else:                         # 7-byte pixels and a 64-bit field (test_gpu_edge_cases): decode_kernel
        pf = oracle_pf("RNG19_RFL8_SIG16_NIR16", 8, 64)
        pf.set_fields([("RANGE", orc.UINT32, 0, 0x7ffff, 0), ("SIGNAL", orc.UINT16, 3, 0xffff, 0),
                       ("FLAGS", orc.UINT8, 5, 0xf0, 4), ("WIDE", orc.UINT64, 0, 0x00ffffffffffffff, 0)], 7)
        kw = dict(with_window=False, extra_fields=[("WIDE", orc.UINT64)])
        srcs = []
        for k in range(3):
            src = orc.Frame(pf, **kw)
            src.field("WIDE")[...] = np.random.default_rng(5 + k).integers(0, 1 << 56, size=(8, 64), dtype=np.uint64)
            src.measurement_id[:] = np.arange(64)
            src.status[:] = 1
            src.packet_timestamp[:] = 7
            src.frame_id = 9 + k
            srcs.append(src)
        shifts = np.arange(8, dtype=np.int32)
        family = "decode"
    refs, packets = [], []
    for src in srcs:
        pk, _ = orc.frame_to_packets(src, pf)
        ref = orc.Frame(pf, **kw)
        b = orc.Batcher(pf)
        for p in pk:
            b.batch(p, 3, ref)
        refs.append(ref)
        packets.append(pk)
    return pf, refs, np.ascontiguousarray(np.stack(packets)), shifts, family


def _oracle(dec, refs, d, o, shifts):
    def rows(arrays):
        return np.stack([np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8) for a in arrays])
    want = {"field " + f["name"]: rows(r.field(f["name"]) for r in refs) for f in dec.fields}
    for k in ("timestamp", "measurement_id", "status"):
        want[k] = rows(getattr(r, k) for r in refs)
    for f in dec.fields:
        r = f.get("range_return", -1)
        if r >= 0:
            want[f"xyz{r}"] = rows(orc.cartesian(ref.field(f["name"]), d, o) for ref in refs)
            want[f"rd{r}"] = rows(orc.destagger(ref.field(f["name"]), shifts) for ref in refs)
    return want


@pytest.mark.parametrize("device_out", [False, True], ids=["host_out", "device_out"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", ["dual_128x1024", "unaligned_8x64"])
def test_entry_points_decode_the_same_frames_alike(ob, case, dtype, device_out):
    pf, refs, packets, shifts, family = _case(case)
    dec = ob.Decoder(*decoder_desc_from_oracle(pf, refs[0]))
    h, w = dec.h_px, dec.w_px
    d, o = random_lut(h * w, 3, dtype)
    lut = ob.XYZLutT.from_arrays(d, o, h, w)
    want = _oracle(dec, refs, d, o, shifts)
    n_ret = sum(1 for f in dec.fields if f.get("range_return", -1) >= 0)
    for path in PATHS:
        out = _outputs(dec, len(refs), dtype, n_ret, n_ret, device_out)
        before = {f: ob.kernel_launch_count(f) for f in ("decode_pipe", "decode")}
        _run(ob, path, dec, packets, out, lut=lut, shifts=shifts)
        grew = {f: ob.kernel_launch_count(f) - before[f] for f in before}
        assert grew["decode"] > 0 and (grew["decode_pipe"] > 0) == (family == "decode_pipe"), (path, grew)
        got = _flat(out)
        assert sorted(got) == sorted(want), path
        for k in want:   # byte for byte, so equal across the paths too
            assert np.array_equal(got[k], want[k]), (path, k)


# ---- one rule table -----------------------------------------------------------------------------------------------
def _small_decoder(ob, h=8, w=64, cpp=16):
    """4-byte pixels behind a 16-byte column header; zero packets are enough for inputs that must be refused"""
    col = 16 + 4 * h
    layout = {"packet_header_size": 16, "col_header_size": 16, "channel_data_size": 4, "col_size": col,
              "packet_size": 16 + cpp * col, "columns_per_packet": cpp, "pixels_per_column": h,
              "columns_per_frame": w, "col_timestamp": (0, (1 << 64) - 1, 0),
              "col_measurement_id": (8, 0xffff, 0), "col_status": (12, 0xffff, 0)}
    fields = [{"name": "RANGE", "offset": 0, "mask": 0x7ffff, "shift": 0, "elem_size": 4, "range_return": 0}]
    return ob.Decoder(layout, fields)


def _lut(ob, h, w, dtype=np.float32):
    d, o = random_lut(h * w, 1, dtype)
    return ob.XYZLutT.from_arrays(d, o, h, w)


# rule -> (message, entry points that can receive the input)
RULES = {
    "lut_shape": ("unexpected image dimensions", PATHS),
    "shift_length": ("image height does not match shifts size", PATHS),
    "over_512_rows": ("fused destagger supports at most 512 rows", PATHS),
    "xyz_without_lut": ("xyz output requested without a lut", PATHS),
    "rd_without_shifts": ("image height does not match shifts size", PATHS),
    "short_packet_stride": ("packet_stride smaller than the lidar packet size", PATHS),
    "frame_lut_dtype_vs_call_lut": ("per-frame lut dtype differs from the call-level lut", PATHS),
    "frame_lut_dtypes": ("per-frame lut dtype differs", ("decode", "batch")),  # a job decodes one frame
    "too_many_slots": ("too many packet slots", PATHS),
}


@pytest.mark.parametrize("rule,path", [(r, p) for r, (_, paths) in RULES.items() for p in paths])
def test_invalid_input_is_refused_alike_before_any_output(ob, rule, path):
    msg = RULES[rule][0]
    dec = _small_decoder(ob, h=600, cpp=1) if rule == "over_512_rows" else \
        _small_decoder(ob, h=1, w=4, cpp=1) if rule == "too_many_slots" else _small_decoder(ob)
    h, w, psize = dec.h_px, dec.w_px, dec.layout["packet_size"]
    # ob_decode_batch_run reads the whole strided packet buffer, so it is as long as the slots claimed
    n_slots = (1 << 20) + 1 if rule == "too_many_slots" else w // dec.layout["columns_per_packet"]
    packets = np.zeros((2, n_slots, psize), np.uint8)
    args = dict(lut=_lut(ob, h, w), shifts=np.zeros(h, np.int32))
    n_xyz = n_rd = 1
    if rule == "lut_shape":
        args["lut"] = _lut(ob, h, 2 * w)
    elif rule == "shift_length":
        args["shifts"] = np.zeros(h + 1, np.int32)
    elif rule == "xyz_without_lut":
        args["lut"], n_rd = None, 0
    elif rule == "rd_without_shifts":
        args["shifts"] = None
    elif rule == "short_packet_stride":
        args["packet_stride"] = psize - 1
    elif rule == "frame_lut_dtype_vs_call_lut":
        args["frame_luts"] = [_lut(ob, h, w, np.float64)] * 2
    elif rule == "frame_lut_dtypes":
        args["lut"], args["frame_luts"] = None, [_lut(ob, h, w), _lut(ob, h, w, np.float64)]
    out = _outputs(dec, 2, np.float64, n_xyz, n_rd, device=False)  # room for XYZ of either dtype
    with pytest.raises(ValueError) as e:
        _run(ob, path, dec, packets, out, **args)
    assert str(e.value) == msg
    for k, a in _flat(out).items():
        assert np.all(a == SENTINEL), k
