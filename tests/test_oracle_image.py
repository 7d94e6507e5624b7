"""CPU tests of the image post-processing oracle (oracle/orc_image.c): it equals an independent numpy restatement of
AutoExposure, BeamUniformityCorrector and the CLAHE LUTs (ouster_core/src/image_processing.cpp), its FullPivLU "fit"
reduces to the closed form through the two pivot rows, and the behaviour the reference's
tests/integration/ouster_autoexposure_test.py asserts holds on generated data and on a decoded sensor frame."""
import numpy as np
import pytest

from oracle import image as oi
from oracle import oracle as orc
from tests.helpers import load_fixture

AE_PARAMS = [(0.1, 0.1, 1), (0.05, 0.1, 1), (0.1, 0.02, 1), (0.0, 0.0, 1), (0.3, 0.3, 1)]


def np_ae(img, lo_p, hi_p, damping=0.9, state=None):
    """numpy restatement of one AutoExposure update of a float64 mono image with update_state (counter 0)"""
    flat = img.reshape(-1)
    cand = flat[::4][flat[::4] > 0]
    n = cand.size
    if n < 100:
        return state
    k_lo = int(n * lo_p)
    k_hi = int(n * hi_p)
    lo = np.partition(cand, k_lo)[k_lo]
    hi = np.partition(cand, n - k_hi - 1)[n - k_hi - 1]
    ls, hs = (lo, hi) if state is None else state
    ls = damping * ls + (1.0 - damping) * lo
    hs = damping * hs + (1.0 - damping) * hi
    with np.errstate(divide="ignore", invalid="ignore"):
        scale = (1.0 - (lo_p + hi_p)) / (hs - ls)
    if np.isinf(scale) or np.isnan(scale):
        flat *= 0.5 / hs
    elif scale * (0.0 - ls) + lo_p <= 0.0:
        flat -= ls
        flat *= scale
        flat += lo_p
    else:
        flat *= (1.0 - hi_p) / hs
    np.copyto(flat, np.minimum(np.maximum(flat, 0), 1))
    return ls, hs


@pytest.mark.parametrize("case", ["affine", "hi_only", "inf"])
def test_ae_branches_match_numpy(case):
    r = np.random.default_rng(3)
    if case == "affine":
        img = r.uniform(10, 20, (32, 64))
    elif case == "hi_only":
        img = r.uniform(0.0, 1.0, (32, 64))  # lo near 0: the lo/hi map would send 0 above 0
    else:
        img = np.full((32, 64), 5.0)          # hi == lo: the scale is inf
    ae = oi.AutoExposure(0.1, 0.1, 1)
    st = None
    for f in range(4):
        frame = (img * (1 + 0.1 * f)).copy()
        expect = frame.copy()
        st = np_ae(expect, 0.1, 0.1, state=st)
        ae.update(frame)
        assert np.array_equal(frame, expect), (case, f)
    assert ae.state()["initialized"]


def test_ae_too_few_candidates_keeps_image_and_counter():
    img = np.zeros((20, 20))
    img.reshape(-1)[::4][:99] = 1.0          # 99 candidates
    ae = oi.AutoExposure(0.1, 0.1, 3)
    before = img.copy()
    ae.update(img)
    assert np.array_equal(img, before) and ae.state()["counter"] == 0 and not ae.state()["initialized"]
    img.reshape(-1)[::4][:200] = 2.0
    ae.update(img)
    assert ae.state()["counter"] == 1 and ae.state()["initialized"]


def test_f16_trick():
    bits = np.array([0, 0x7e00, 0x0001, 0x03ff, 0x3c00, 0x7c00, 0xfc00, 0xbc00, 0x8000, 0x7e01, 0xffff], np.uint16)
    got = oi.f16_to_f32(bits).view(np.uint32)
    expect = np.array([0 if b in (0, 0x7e00) else ((int(b) + 0x1C000) << 13) & 0xffffffff for b in bits], np.uint32)
    assert np.array_equal(got, expect)
    # positive normals convert as IEEE does; +inf, negatives and denormals do not (the sign bit is shifted out)
    assert oi.f16_to_f32(np.array([0x3c00, 0x7c00, 0xbc00], np.uint16)).tolist() == [1.0, 65536.0, 2.0 ** 32]
    assert oi.f16_to_f32(np.array([0x0001], np.uint16))[0] != np.float32(np.float16(6e-8))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("h", [2, 3, 7, 32, 128])
def test_fullpivlu_fit_is_two_point_line(dtype, h):
    r = np.random.default_rng(h)
    dc = np.concatenate([[0.0], np.cumsum(r.normal(0, 1, h - 1))]).astype(dtype)
    x = oi.fullpivlu_fit(dc)
    assert x[0] == 0
    assert x[1] == dtype(dc[h - 1] / dtype(h - 1))
    if h > 2:
        ls = np.polyfit(np.arange(h), dc.astype(np.float64), 1)
        assert not np.allclose([x[1], x[0]], ls, rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape", [(32, 64), (16, 33), (5, 8), (1, 20)])
def test_dark_count_matches_numpy(dtype, shape):
    h, w = shape
    r = np.random.default_rng(w)
    img = (r.random(shape) + np.linspace(0, 0.4, h)[:, None]).astype(dtype)
    img[:, ::5] = 0                       # masked columns
    mask = (img != 0).any(axis=0)
    n = int(mask.sum())
    dc = np.zeros(h, dtype)
    for i in range(1, h):
        d = (img[i, mask] - img[i - 1, mask]).astype(dtype)
        dc[i] = dtype(dc[i - 1] + np.partition(d, n // 2)[n // 2])
    if h > 1:
        slope = dtype(dc[h - 1] / dtype(h - 1))
        dc = (dc - (dtype(1) * dtype(0) + np.arange(h).astype(dtype) * slope)).astype(dtype)
    dc = (dc - dc.min()).astype(dtype)
    assert np.array_equal(oi.dark_count(img), dc)


def test_dark_count_all_columns_masked():
    assert np.array_equal(oi.dark_count(np.zeros((8, 16))), np.zeros(8))


def test_buc_state_machine():
    r = np.random.default_rng(1)
    buc = oi.BeamUniformityCorrector()
    img = r.random((16, 32))
    buc.update(img.copy(), update_state=False)   # first call computes without damping even without update_state
    s = buc.state()
    assert s["counter"] == 1 and np.array_equal(s["dark_count"], oi.dark_count(img))
    for _ in range(7):
        buc.update(r.random((16, 32)))
    assert buc.state()["counter"] == 0
    img2 = r.random((16, 32))
    prev = buc.state()["dark_count"]
    buc.update(img2.copy())
    assert np.array_equal(buc.state()["dark_count"], prev * 0.92 + oi.dark_count(img2) * (1.0 - 0.92))
    buc.update(r.random((8, 32)), update_state=False)  # a new height resets
    assert buc.state()["dark_count"].size == 8


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape", [(64, 128), (16, 40), (5, 64)])
@pytest.mark.parametrize("nan", [False, True])
def test_clahe_luts_match_numpy(dtype, shape, nan):
    h, w = shape
    lum = np.random.default_rng(h).random(shape).astype(dtype)
    if nan:
        lum.reshape(-1)[::7] = np.nan           # a NaN luminance counts in bin 0
    got = oi.clahe_luts(lum)
    scaled = lum.astype(np.float32) * np.float32(1024)
    bins = np.minimum(np.where(np.isnan(scaled), 0, scaled).astype(np.int32), 1023)
    for ty in range(8):
        for tx in range(8):
            y0, y1, x0, x1 = ty * h // 8, (ty + 1) * h // 8, tx * w // 8, (tx + 1) * w // 8
            tp = (y1 - y0) * (x1 - x0)
            hist = np.bincount(bins[y0:y1, x0:x1].ravel(), minlength=1024).astype(np.float32)
            clip = np.float32(np.float32(tp) / np.float32(1024))
            excess = np.float32(0)
            for b in range(1024):
                if hist[b] > clip:
                    excess = np.float32(excess + np.float32(hist[b] - clip))
                    hist[b] = clip
            red = np.float32(excess / np.float32(1024))
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = np.float32(np.float32(1) / np.float32(tp))
                cdf = np.float32(0)
                lut = np.empty(1024, np.float32)
                for b in range(1024):
                    cdf = np.float32(cdf + np.float32(hist[b] + red))
                    v = np.float32(cdf * inv)
                    lut[b] = v if not (np.float32(1) < v) else np.float32(1)
            assert np.array_equal(got[ty * 8 + tx], lut, equal_nan=True), (ty, tx)


def golden_fields():
    meta, packets = load_fixture("OS-1-32-G_v2.1.1_1024x10")
    pf = orc.PacketFormat(meta["profile"], meta["h"], meta["w"], meta["columns_per_packet"],
                          orc.HEADER_FUSA if meta["header_type"] == "FUSA" else orc.HEADER_STANDARD)
    frame = orc.Frame(pf, with_window=False)
    b = orc.Batcher(pf, init_id=meta["init_id"], column_window=meta["column_window"])
    for p in packets:
        b.batch(p, 1234, frame)
    return frame.field("NEAR_IR").astype(float), frame.field("RANGE").astype(float)


def outlierized(r, mean, std, rows, cols):
    a = r.normal(mean, std, (rows, cols))
    idx = r.integers(0, rows * cols, 100)
    a.reshape(-1)[idx[::2]] = mean - std * 10
    a.reshape(-1)[idx[1::2]] = mean + std * 10
    return a


@pytest.mark.parametrize("params", AE_PARAMS, ids=lambda p: "-".join(map(str, p)))
def test_autoexposure_integration_behaviour(params):
    r = np.random.default_rng(0)
    nir, rng = golden_fields()
    line = np.arange(0.0, 500, 0.3).reshape(1, -1)
    ae = oi.AutoExposure(*params)
    for key in (r.normal(100, 5, (128, 512)), outlierized(r, 25, 2, 64, 1024), line.copy(), nir.copy()):
        ae.update(key)
        assert np.all(key >= 0.0) and np.all(key <= 1.0)
    ae = oi.AutoExposure(*params)
    for key in (outlierized(r, 25, 2, 64, 1024), line.copy(), rng.copy()):
        zeros = key <= 0.0
        if not zeros.any():
            continue
        ae.update(key)
        assert np.all(key[zeros] == 0.0)
    ae = oi.AutoExposure(*params)
    ones = np.ones((50, 100))
    ae.update(ones)
    assert np.all(ones == ones[0, 0])
    ae = oi.AutoExposure(*params)
    line = np.arange(0.0, 500, 0.3).reshape(1, -1)
    ae.update(line)
    mx = np.max(line)
    assert 1 - params[1] <= mx <= 1.0
    # The reference's "one minimum at 0 / one max" checks count the True entries of `isclose(...) == 1`, so they
    # only ask that some value is 0 and some is the maximum.  "Exactly one 0" does not hold: the values below the
    # lo order statistic (and the input 0, which is no candidate) all clamp to 0.  What does hold: the ramp stays
    # nondecreasing from 0, and it is a straight line between the clamps.
    assert line.min() == 0.0 and np.count_nonzero(line == 0.0) >= 1
    assert np.all(np.diff(line) >= 0)
    inner = line[(line > 0) & (line < mx)]
    assert inner.size > 2 and np.allclose(np.diff(inner), np.diff(inner)[0], rtol=1e-6, atol=1e-12)


def test_abi_structs_match_ctypes_mirror():
    import ctypes
    import __graft_entry__ as graft
    capi = graft.load_package()._capi
    for name, cls in (("ob_image_params", capi.ImageParams), ("ob_image_state", capi.ImageState)):
        assert capi.lib.ob_abi_sizeof(name.encode()) == ctypes.sizeof(cls), name
    assert ctypes.sizeof(oi.State) == ctypes.sizeof(capi.ImageState)
    assert ctypes.sizeof(oi.Params) == ctypes.sizeof(capi.ImageParams)
