"""GPU tests of the image post-processing (ouster-sdk_b200/csrc/ob_image.cu): AutoExposure, BeamUniformityCorrector
and LocalToneMapper bit for bit (NaN-aware) against the CPU oracle (oracle/orc_image.c) over frame sequences with
mixed update_state, the state read back after every update, the Python binding's call shapes, and a device chain
from packets replayed from a CUDA graph."""
import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import image as oi

pytestmark = pytest.mark.gpu

SHAPES = [(128, 2048), (64, 1024), (32, 1024), (16, 512), (1, 1667), (7, 333), (5, 64)]
UPDATE = [True, True, False, True, True, True, False, True, True, True, True, True]


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


def frame(r, shape, f, dtype, rgb=False):
    """frame f of a sequence: cycles through spread values, skewed values, a constant image, too few candidates and
    an all-zero image, with zeros sprinkled in.  Damped state keeps these sequences on the lo/hi branch; the other
    two branches are reached by test_every_affine_branch"""
    full = shape + (3,) if rgb else shape
    mode = f % 6
    if mode in (0, 5):
        a = r.uniform(10, 20, full) * (1 + 0.05 * f)
    elif mode == 1:
        a = r.random(full) ** 4
    elif mode == 2:
        a = np.full(full, 3.0)
    elif mode == 3:
        a = np.zeros(full)
        a.reshape(-1)[::97][:60] = 1.0        # well under 100 candidates
    else:
        a = np.zeros(full)
    if mode in (0, 1, 5):
        a[r.random(shape) < 0.2] = 0
    return a.astype(dtype)


def same(a, b):
    return np.array_equal(a, b, equal_nan=True)


def check_state(gs, os_, kind):
    if kind == "beam_uniformity":
        assert gs["counter"] == os_["counter"]
        assert same(gs["dark_count"], os_["dark_count"])
    else:
        for k in ("lo", "hi", "lo_state", "hi_state", "counter", "initialized"):
            assert gs[k] == os_[k] or (np.isnan(gs[k]) and np.isnan(os_[k])), k


def run_sequence(ob, kind, shape, dtype, layout, gpu_kw, orc_obj, n=12, seed=0):
    r = np.random.default_rng(seed)
    proc = ob.ImageProcessor(kind, **gpu_kw)
    for f in range(n):
        us = UPDATE[f % len(UPDATE)]
        if layout == "f16":
            src = (frame(r, shape, f, np.float32, rgb=True) / 25).astype(np.float16)
            got = proc.update(src, update_state=us)
            want = orc_obj.update(src, us)
        else:
            img = frame(r, shape, f, dtype, rgb=layout == "rgb")
            if kind == "local_tone_map":
                img = img / dtype(25)
            got, want = img.copy(), img.copy()
            proc.update(got, update_state=us)
            orc_obj.update(want, us)
        assert same(got, want), (kind, layout, shape, f)
        check_state(proc.state(), orc_obj.state(), kind)


AE_KW = dict(lo_percentile=0.1, hi_percentile=0.1, update_every=3, damping=0.9)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("layout", ["mono", "rgb"])
def test_auto_exposure(ob, shape, dtype, layout):
    run_sequence(ob, "auto_exposure", shape, dtype, layout, AE_KW, oi.AutoExposure(0.1, 0.1, 3, 0.9))


@pytest.mark.parametrize("shape", SHAPES)
def test_auto_exposure_f16(ob, shape):
    run_sequence(ob, "auto_exposure", shape, np.float32, "f16", AE_KW, oi.AutoExposure(0.1, 0.1, 3, 0.9))


@pytest.mark.parametrize("params", [(0.05, 0.1, 1), (0.0, 0.0, 2), (0.3, 0.3, 1), (0.6, 0.39, 1)])
def test_auto_exposure_percentiles(ob, params):
    lo, hi, ue = params
    run_sequence(ob, "auto_exposure", (64, 1024), np.float32, "mono",
                 dict(lo_percentile=lo, hi_percentile=hi, update_every=ue, damping=0.5),
                 oi.AutoExposure(lo, hi, ue, 0.5))


def test_auto_exposure_early_returns(ob):
    """fewer than 100 candidates before and after initialisation, and an all-zero image: untouched, counter kept"""
    proc, o = ob.ImageProcessor("auto_exposure", **AE_KW), oi.AutoExposure(0.1, 0.1, 3, 0.9)
    few = np.zeros((32, 64), np.float32)
    few.reshape(-1)[::4][:99] = 2.0
    r = np.random.default_rng(5)
    for img in (few, np.zeros((32, 64), np.float32), r.uniform(1, 2, (32, 64)).astype(np.float32), few, few):
        g, w = img.copy(), img.copy()
        proc.update(g)
        o.update(w)
        assert same(g, w)
        check_state(proc.state(), o.state(), "auto_exposure")


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_beam_uniformity(ob, shape, dtype):
    run_sequence(ob, "beam_uniformity", shape, dtype, "mono", {}, oi.BeamUniformityCorrector(), n=20)


def test_beam_uniformity_reset_and_masks(ob):
    """a new height resets the dark count; all columns masked; odd and even n_cols"""
    proc, o = ob.ImageProcessor("beam_uniformity"), oi.BeamUniformityCorrector()
    r = np.random.default_rng(9)
    imgs = []
    for h, w in ((16, 64), (16, 64), (24, 64), (24, 65), (8, 64), (8, 64)):
        a = (r.random((h, w)) + np.linspace(0, 0.5, h)[:, None]).astype(np.float32)
        imgs.append(a)
    imgs[3][:, ::2] = 0                 # 32 live columns of 65
    imgs[4][:] = 0                      # every column masked
    imgs[5][:, 1::3] = 0                # odd count of live columns
    for f, img in enumerate(imgs):
        g, w = img.copy(), img.copy()
        proc.update(g, update_state=f != 1)
        o.update(w, f != 1)
        assert same(g, w), f
        check_state(proc.state(), o.state(), "beam_uniformity")


LTM_CASES = [(0.0, 0.2, 1, 0.3, 0.2, True), (0.0, 0.2, 1, 0.3, 0.0, True), (0.1, 0.1, 2, 0.5, 5.0, False),
             (0.0, 0.2, 1, 0.3, 100.0, True)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_local_tone_mapper(ob, shape, dtype):
    run_sequence(ob, "local_tone_map", shape, dtype, "rgb",
                 dict(lo_percentile=0.0, hi_percentile=0.2, update_every=1, damping=0.3, compress_dr_max_lum=0.2,
                      color_correct=True), oi.LocalToneMapper())


@pytest.mark.parametrize("case", LTM_CASES)
@pytest.mark.parametrize("layout", ["rgb", "f16"])
def test_local_tone_mapper_options(ob, case, layout):
    """compression on and off, colour correction off, and a high hi_state (colour_factor 0.75) / low (0)"""
    lo, hi, ue, d, c, cc = case
    run_sequence(ob, "local_tone_map", (32, 512), np.float32, layout,
                 dict(lo_percentile=lo, hi_percentile=hi, update_every=ue, damping=d, compress_dr_max_lum=c,
                      color_correct=cc), oi.LocalToneMapper(lo, hi, ue, d, c, cc))


def test_local_tone_mapper_color_factor_zero(ob):
    """hi_state <= 0.5 makes color_factor 0, which takes the plain branch even with color_correct"""
    proc = ob.ImageProcessor("local_tone_map", lo_percentile=0.0, hi_percentile=0.2, update_every=1, damping=0.3,
                             compress_dr_max_lum=0.2, color_correct=True)
    o = oi.LocalToneMapper()
    img = (np.random.default_rng(2).random((32, 256, 3)) * 0.3).astype(np.float32)
    g, w = img.copy(), img.copy()
    proc.update(g)
    o.update(w)
    assert o.state()["hi_state"] < 0.5 and same(g, w)


def test_pyapi_call_shapes(ob):
    """python/tests/test_ndarray_convert.py:195-260 through pyapi"""
    api = ob.pyapi
    for dtype in (np.float32, np.float64):
        image = np.outer(np.linspace(0.2, 1.0, 32, dtype=dtype), np.linspace(0.3, 1.0, 32, dtype=dtype))
        original = image.copy()
        ae = api.AutoExposure()
        assert ae.update(image) is None
        assert not np.allclose(image, original)
        for bad in (np.uint16, np.uint32):
            with pytest.raises(TypeError, match="incompatible function arguments"):
                ae.update(image.astype(bad))
        rng = np.random.default_rng(0)
        image = rng.random((32, 32), dtype=dtype)
        image += np.linspace(0.0, 0.4, 32, dtype=dtype)[:, np.newaxis]
        original = image.copy()
        buc = api.BeamUniformityCorrector()
        assert buc.update(image) is None
        assert not np.allclose(image, original)
        with pytest.raises(TypeError, match="incompatible function arguments"):
            buc.update(image.astype(np.uint16))
        mono = np.linspace(0.2, 1.0, 32 * 32, dtype=dtype).reshape(32, 32)
        image = np.stack([mono, mono * 0.9, mono * 0.8], axis=-1)
        original = image.copy()
        assert api.AutoExposure().update(image) is None
        assert not np.allclose(image, original)
    result = api.AutoExposure().update(np.random.rand(8, 16, 3).astype(np.float16))
    assert result is not None and result.dtype == np.float32 and result.shape == (8, 16, 3)
    with pytest.raises(TypeError):
        api.AutoExposure().update(np.asfortranarray(np.random.rand(8, 16).astype(np.float32)))
    with pytest.raises(ValueError, match="H x W x 3"):
        api.AutoExposure().update(np.random.rand(8, 16, 4).astype(np.float32))
    ltm = api.LocalToneMapper(0.0, 0.2, 1, 0.3, True, True)
    out = ltm.update(np.random.rand(16, 32, 3).astype(np.float16))
    assert out.dtype == np.float32 and out.shape == (16, 32, 3)
    with pytest.raises(TypeError):
        ltm.update(np.random.rand(16, 32, 3).astype(np.float32))


def test_torch_in_place_and_launch_family(ob):
    import torch
    img = np.random.default_rng(4).uniform(1, 5, (64, 1024)).astype(np.float32)
    t = torch.from_numpy(img.copy()).cuda()
    before = ob.kernel_launch_count("image")
    ae = ob.pyapi.AutoExposure()
    assert ae.update(t) is None
    torch.cuda.synchronize()
    assert ob.kernel_launch_count("image") > before
    want = img.copy()
    oi.AutoExposure().update(want)
    assert same(t.cpu().numpy(), want)


def test_device_chain_from_packets_in_cuda_graph(ob):
    """K2's device NEAR_IR -> .float() -> BeamUniformityCorrector -> AutoExposure on the torch stream, the update
    pair captured once in a CUDA graph and replayed over frames; the bits equal the host path"""
    import torch
    from tests.helpers import load_fixture
    api = ob.pyapi
    meta, packets = load_fixture("OS-1-32-G_v2.1.1_1024x10")
    info = api.SensorInfo.from_meta(meta)
    batcher = api.DeviceScanBatcher(info)
    scan = batcher.new_scan()
    done = [batcher(p, 77, scan) for p in packets]
    if not done[-1]:
        batcher.flush(scan)
    nir = scan.field("NEAR_IR")
    assert nir.is_cuda
    nir_host = nir.cpu().numpy().astype(np.float32)
    buc, ae = api.BeamUniformityCorrector(), api.AutoExposure(0.1, 0.1, 2)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    outs = []
    with torch.cuda.stream(side):
        x = nir.float()
        buc.update(x)       # first call: sizes the dark count, outside the capture
        ae.update(x)
        outs.append(x.clone())
        g = torch.cuda.CUDAGraph()
        static = torch.empty_like(x)
        with torch.cuda.graph(g, stream=side):
            static.copy_(nir.float())
            buc.update(static)
            ae.update(static)
    torch.cuda.current_stream().wait_stream(side)
    for _ in range(10):
        g.replay()
        outs.append(static.clone())
    torch.cuda.synchronize()
    hb, ha = oi.BeamUniformityCorrector(), oi.AutoExposure(0.1, 0.1, 2)
    for f, o in enumerate(outs):
        want = nir_host.copy()
        hb.update(want)
        ha.update(want)
        assert same(o.cpu().numpy(), want), f


def branch_of(state, lo_p, hi_p):
    """the affine branch an applied update took, from its damped state: 0 inf/nan scale, 1 lo/hi map, 2 hi only"""
    with np.errstate(divide="ignore", invalid="ignore"):
        scale = np.float64(1.0 - (lo_p + hi_p)) / np.float64(state["hi_state"] - state["lo_state"])
    if np.isinf(scale) or np.isnan(scale):
        return 0
    return 1 if scale * (0.0 - state["lo_state"]) + lo_p <= 0.0 else 2


BRANCH_RUNS = [("auto_exposure", "mono", np.float32), ("auto_exposure", "mono", np.float64),
               ("auto_exposure", "rgb", np.float32), ("auto_exposure", "rgb", np.float64),
               ("auto_exposure", "f16", np.float32), ("local_tone_map", "rgb", np.float32),
               ("local_tone_map", "rgb", np.float64), ("local_tone_map", "f16", np.float32)]


@pytest.mark.parametrize("want", [0, 2])
@pytest.mark.parametrize("run", BRANCH_RUNS, ids=lambda r: f"{r[0]}-{r[1]}-{np.dtype(r[2]).name}")
def test_every_affine_branch(ob, run, want):
    """a fresh processor whose first frames are constant takes the inf scale (hi_state == lo_state); frames of
    r ** 8 take the hi-only branch (lo_state far below hi_state / 9); both asserted, bits equal to the oracle"""
    kind, layout, dtype = run
    lo, hi, ue, d = 0.1, 0.1, 1, 0.5
    proc = ob.ImageProcessor(kind, lo_percentile=lo, hi_percentile=hi, update_every=ue, damping=d,
                             compress_dr_max_lum=0.2, color_correct=True)
    orc_obj = (oi.AutoExposure(lo, hi, ue, d) if kind == "auto_exposure" else
               oi.LocalToneMapper(lo, hi, ue, d, 0.2, True))
    r = np.random.default_rng(want)
    shape = (32, 256, 3) if layout != "mono" else (32, 256)
    for f in range(4):
        a = np.full(shape, 0.4) if want == 0 else r.random(shape) ** 8
        if layout == "f16":
            src = a.astype(np.float16)
            got, exp = proc.update(src), orc_obj.update(src)
        else:
            got, exp = a.astype(dtype), a.astype(dtype)
            proc.update(got)
            orc_obj.update(exp)
        assert same(got, exp), f
        s = proc.state()
        check_state(s, orc_obj.state(), kind)
        assert branch_of(s, lo, hi) == want, (f, s)


def test_local_tone_mapper_inf_input(ob):
    """inf pixels reach Reinhard as inf / (1 + inf) = NaN: the NaN luminance counts in CLAHE bin 0 on both sides.
    Without colour correction the NaN survives the final min(x, 1) (the colour stage's max(0, .) would make it 0)"""
    for layout in ("rgb", "f16"):
        proc = ob.ImageProcessor("local_tone_map", color_correct=False)
        o = oi.LocalToneMapper(0.0, 0.2, 1, 0.3, 0.2, False)
        r = np.random.default_rng(8)
        for f in range(3):
            a = r.random((32, 256, 3)).astype(np.float32)
            a.reshape(-1, 3)[5::97] = np.inf
            if layout == "f16":
                src = a.astype(np.float16)          # inf is 0x7c00, which the bit trick maps to 65536
                src.reshape(-1, 3)[7::89] = np.float16(np.nan)
                got, want = proc.update(src), o.update(src)
            else:
                got, want = a.copy(), a.copy()
                proc.update(got)
                o.update(want)
            assert same(got, want), (layout, f)
            if layout == "rgb":
                assert np.isnan(got).any()
