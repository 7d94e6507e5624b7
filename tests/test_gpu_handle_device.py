"""Every *_destroy frees the handle's memory on the handle's device and leaves the caller's current device as it was
(include/ouster_b200.h).  Python destroys handles from _Handle.__del__, so a destroy can run at any point of a
caller's program; on a machine with several GPUs, a destroy that left the handle's device current would move the
caller's next torch allocation there.

Each handle type is created on device 1 and used once, so that its growable buffers grow.  Device 0 is then made
current, as a caller's own code would, and the handle is destroyed: device 0 must still be current.  A second
round on device 1 must work as the first."""
import ctypes as C
from importlib import import_module

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import oracle as orc
from tests.helpers import decoder_desc_from_oracle, oracle_pf, random_frame, random_lut

pytestmark = pytest.mark.gpu

DEV = 1


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    if m.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    return m


def _cloud(ob, lut):
    """one scan_to_cloud through `lut` on its device"""
    st = ob.Stream(DEV)
    rng = np.random.default_rng(0).integers(0, 20000, (1, 1, lut.h, lut.w)).astype(np.uint32)
    xyz = np.zeros((1, 1, lut.h * lut.w, 3), lut.dtype)
    ob.scan_to_cloud(lut, np.zeros(lut.h, np.int32), rng, xyz=xyz, stream=st)
    st.sync()
    assert np.isfinite(xyz).all()


def _frame(ob):
    """(decoder on device 1, source frame, its packets)"""
    pf = oracle_pf("RNG19_RFL8_SIG16_NIR16_DUAL", 16, 128)
    src = random_frame(pf, seed=4)
    pk, _ = orc.frame_to_packets(src, pf)
    return ob.Decoder(*decoder_desc_from_oracle(pf, src), device=DEV), src, np.ascontiguousarray(pk)


def _fields(dec, src):
    return {f["name"]: np.zeros(src.field(f["name"]).shape, src.field(f["name"]).dtype) for f in dec.fields}


def _assert_decoded(outs, src):
    for n, a in outs.items():
        assert np.array_equal(a, src.field(n)), n


# each maker creates a handle on device 1, uses it once and returns (destroy, objects the handle needs until then)
def _lut_arrays(ob):
    d, o = random_lut(16 * 128, 1, np.float32)
    lut = ob.XYZLutT.from_arrays(d, o, 16, 128, device=DEV)
    _cloud(ob, lut)
    return lut.__del__, ()


def _lut_intrinsics(ob):
    lut = ob.XYZLutT.from_intrinsics(128, 16, 0.001, np.eye(4), np.eye(4), np.linspace(-3, 3, 16),
                                     np.linspace(-10, 10, 16), dtype=np.float32, device=DEV).set_analytic(True)
    assert lut.analytic
    _cloud(ob, lut)
    return lut.__del__, ()


def _stream(ob):
    dec, src, pk = _frame(ob)
    st = ob.Stream(DEV)
    outs = _fields(dec, src)
    # the frame table goes to the stream's device-resident table
    dec.decode([{"packets": pk, "n_slots": len(pk), "packet_stride": pk.shape[1], "col_src": None, "fields": outs}],
               stream=st)
    st.sync()
    _assert_decoded(outs, src)
    return st.__del__, (dec,)


def _decode_job(ob):
    capi = import_module(ob.__name__ + "._capi")
    lib = capi.lib
    lib.ob_decode_job_create.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_void_p)]
    lib.ob_decode_job_upload.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t]
    lib.ob_decode_job_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    for f in ("ob_decode_job_wait", "ob_decode_job_destroy"):
        getattr(lib, f).argtypes = [C.c_void_p]
    dec, src, pk = _frame(ob)
    st = ob.Stream(DEV)
    job = C.c_void_p()
    capi.check(lib.ob_decode_job_create(dec._h, 0, st.h, C.byref(job)))  # no slots yet: the upload grows them
    capi.check(lib.ob_decode_job_upload(job, pk.ctypes.data, pk.shape[1], 0, len(pk)))
    outs = _fields(dec, src)
    io = capi.DecodeIO()
    io.n_slots = len(pk)
    for i, f in enumerate(dec.fields):
        io.fields[i] = outs[f["name"]].ctypes.data  # host outputs: the job's output slab grows
    capi.check(lib.ob_decode_job_submit(job, C.byref(io), None, None, 0))
    capi.check(lib.ob_decode_job_wait(job))
    _assert_decoded(outs, src)
    return (lambda: capi.check(lib.ob_decode_job_destroy(job))), (dec, st)


def _voxel_map(ob):
    cells = np.stack(np.meshgrid(*[np.arange(20.0)] * 3, indexing="ij"), -1).reshape(-1, 3) + 0.5
    m = ob.VoxelMap(1.0, 1000.0, 3, device=DEV)
    m.add_points(cells[:100])  # the first table: 1024 slots
    m.add_points(cells[100:])  # 8000 voxels: rebuilt for 32768 slots
    assert m.size() == (8000, 8000)
    return m.__del__, ()


def _zone_monitor(ob):
    rs = np.random.default_rng(2)
    near = rs.integers(1, 4000, (8, 64)).astype(np.uint32)
    mon = ob.ZoneMonitor([{"id": 3, "mode": 1, "point_count": 5, "frame_count": 1, "near_mm": near,
                           "far_mm": near + 1000}], 8, 64, device=DEV)
    mon.update(rs.integers(0, 8000, (8, 64)).astype(np.uint32))
    mon.states()
    return mon.__del__, ()


def _image(kind, shape):
    def make(ob):
        proc = ob.ImageProcessor(kind, device=DEV)
        img = np.random.default_rng(3).uniform(0, 2, shape)
        proc.update(img)
        proc.state()
        assert np.isfinite(img).all()
        return proc.__del__, ()
    return make


MAKERS = {"lut_arrays": _lut_arrays, "lut_intrinsics": _lut_intrinsics, "stream": _stream, "decode_job": _decode_job,
          "voxel_map": _voxel_map, "zone_monitor": _zone_monitor,
          "auto_exposure": _image("auto_exposure", (12, 96)), "beam_uniformity": _image("beam_uniformity", (12, 96)),
          "local_tone_map": _image("local_tone_map", (12, 96, 3))}


@pytest.mark.parametrize("kind", list(MAKERS))
def test_destroy_leaves_the_callers_device_current(ob, kind):
    import torch
    for _ in range(2):
        destroy, keep = MAKERS[kind](ob)
        torch.cuda.set_device(0)  # every other entry point leaves the handle's device current
        destroy()
        assert torch.cuda.current_device() == 0, kind
        del keep
