"""GPU tests of the product FrameBatcher / LidarScan path (host state machine + fused GPU decode)
through the host C ABI: the reference's md5 digests and snapshot hashes on its pcap fixtures,
step-by-step equality with the CPU oracle on multi-frame streams with injected faults, and the
fused XYZ / destaggered-range outputs."""
import hashlib

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import oracle as orc
from tests.helpers import PCAP_FIXTURES, load_fixture, oracle_pf, random_frame

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


def md5(a):
    return hashlib.md5(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("name", PCAP_FIXTURES)
def test_pcap_digests_through_product_batcher(ob, name):
    """python/tests/test_core.py:272-279 equivalent: batch the pcap, compare md5 of every field."""
    meta, packets = load_fixture(name)
    si = ob.SensorInfo.from_meta(meta)
    b = ob.FrameBatcher(si)
    fr = ob.LidarFrame(si)
    rets = [b.batch(p, 1234, fr) for p in packets]
    if len(packets) == 64:
        assert rets[-1] and not any(rets[:-1])
    else:
        b.flush(fr)      # the 8-packet FUSA capture never completes a 64-packet frame
    dg, snap = meta["md5_digests"], meta["snapshot_hashes"]
    if dg:
        assert str(fr.frame_id) == dg["FRAME_ID"]
        assert md5(fr.timestamp.astype(np.uint64)) == dg["TIMESTAMP"]
        assert md5(fr.status.astype(np.uint64)) == dg["STATUS"]
        assert md5(fr.measurement_id.astype(np.uint16)) == dg["MEASUREMENT_ID"]
        for k, v in dg.items():
            if k in ("FRAME_ID", "TIMESTAMP", "STATUS", "MEASUREMENT_ID", "ENCODER_COUNT"):
                continue
            assert md5(fr.field(k)) == v, k
    if snap:   # tests/frame_batcher_test.cpp:548-611
        for k, v in snap.items():
            assert orc.snapshot_hash(fr.field(k)) == int(v), k
    assert b.gpu_launches == 1


def _compare(fr, of):
    assert fr.frame_id == of.frame_id
    for n in of.field_names:
        assert np.array_equal(fr.field(n), of.field(n)), n
    assert np.array_equal(fr.timestamp, of.timestamp)
    assert np.array_equal(fr.measurement_id, of.measurement_id)
    assert np.array_equal(fr.status, of.status)
    assert np.array_equal(fr.packet_timestamp, of.packet_timestamp)
    assert np.array_equal(fr.alert_flags, of.alert_flags)


def _stream(opf, n_frames, first_id=700, seed=5):
    pk, ts = [], []
    for k in range(n_frames):
        f = random_frame(opf, seed=seed + k, frame_id=(first_id + k) & opf.max_frame_id)
        p, t = orc.frame_to_packets(f, opf, prod_sn=77)
        pk += list(p)
        ts += list(t)
    return pk, ts


@pytest.mark.parametrize("profile,header,h,w", [
    ("RNG19_RFL8_SIG16_NIR16_DUAL", "STANDARD", 128, 1024), ("RNG19_RFL8_SIG16_NIR16", "STANDARD", 64, 512),
    ("LEGACY", "STANDARD", 64, 512), ("FUSA_RNG15_RFL8_NIR8_DUAL", "FUSA", 32, 512),
    ("RNG19_RFL8_SIG16_NIR16_RGB16", "STANDARD", 16, 256)])
def test_multi_frame_stream_with_faults_matches_oracle(ob, profile, header, h, w):
    opf = oracle_pf(profile, h, w, 16, header)
    si = ob.SensorInfo(profile, h, w, header_type=header, fw_rev="v3.2.1")
    pk, ts = _stream(opf, 5)
    n = w // 16
    pk, ts = [p.copy() for p in pk], list(ts)
    pk[3], pk[4] = pk[4], pk[3]
    ts[3], ts[4] = ts[4], ts[3]
    del pk[n + 7], ts[n + 7]                           # dropped packet in frame 1
    pk.insert(2 * n + 5, pk[2 * n + 4].copy()); ts.insert(2 * n + 5, ts[2 * n + 4])   # duplicate
    b = ob.FrameBatcher(si)
    fr = ob.LidarFrame(si)                             # the SAME frame object is reused
    ob_b = orc.Batcher(opf)
    of = orc.Frame(opf, with_window=True)
    done = 0
    for p, t in zip(pk, ts):
        r1 = b.batch(p, int(t), fr)
        r2 = ob_b.batch(p, int(t), of)
        assert r1 == r2
        if r1:
            done += 1
            _compare(fr, of)
    assert done >= 4
    assert b.dropped_packets == ob_b.dropped_packets


def test_custom_field_untouched_and_missing_profile_field(ob):
    # fields outside the profile are never touched; profile fields absent from the frame are skipped
    # (tests/frame_batcher_test.cpp:292-297)
    profile, h, w = "RNG19_RFL8_SIG16_NIR16", 32, 512
    opf = oracle_pf(profile, h, w)
    si = ob.SensorInfo(profile, h, w, fw_rev="v2.5.0")
    fr = ob.LidarFrame(si)
    assert "WINDOW" not in fr.fields
    fr.add_field("CUSTOM", np.uint32)
    fr.field("CUSTOM")[...] = 0xC0FFEE
    fr.add_field("RAW32_WORD1", np.uint32)            # optional profile field added by the user
    src = random_frame(opf, seed=3)
    pk, ts = orc.frame_to_packets(src, opf)
    b = ob.FrameBatcher(si)
    assert [b.batch(p, int(t), fr) for p, t in zip(pk, ts)][-1]
    assert np.all(fr.field("CUSTOM") == 0xC0FFEE)
    for n in ("RANGE", "SIGNAL", "REFLECTIVITY", "NEAR_IR", "FLAGS"):
        assert np.array_equal(fr.field(n), src.field(n)), n
    raw = np.zeros((h, w), np.uint32)
    for slot, p in enumerate(pk):
        orc.lib().orc_block_field(__import__("ctypes").byref(opf.c), b"RAW32_WORD1", 4,
                                  raw.ctypes.data, w, np.concatenate([p, np.zeros(8, np.uint8)]).ctypes.data, 16)
    assert np.array_equal(fr.field("RAW32_WORD1"), raw)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_fused_cloud_outputs(ob, dtype):
    name = "OS-0-32-U1_v2.2.0_1024x10"
    meta, packets = load_fixture(name)
    si = ob.SensorInfo.from_meta(meta)
    lut = ob.XYZLutT.from_sensor_info(
        {"w": meta["w"], "h": meta["h"], "beam_to_lidar_transform": meta["beam_to_lidar_transform"],
         "lidar_to_sensor_transform": meta["lidar_to_sensor_transform"],
         "beam_azimuth_angles": meta["beam_azimuth_angles"],
         "beam_altitude_angles": meta["beam_altitude_angles"]}, dtype=dtype)
    b = ob.FrameBatcher(si)
    b.set_fused_cloud(lut, meta["pixel_shift_by_row"])
    fr = ob.LidarFrame(si)
    assert [b.batch(p, 99, fr) for p in packets][-1]
    d, o = lut.direction, lut.offset
    for r, fname in enumerate(["RANGE", "RANGE2"]):
        xyz, rd = b.fused_outputs(r)
        assert np.array_equal(xyz, orc.cartesian(fr.field(fname), d, o))
        assert np.array_equal(rd, orc.destagger(fr.field(fname), meta["pixel_shift_by_row"]))
        # and the stand-alone entry points agree with the fused pass
        assert np.array_equal(lut(fr.field(fname)), xyz)
        assert np.array_equal(ob.destagger(fr.field(fname), meta["pixel_shift_by_row"]), rd)


def test_custom_profile_through_batcher(ob):
    # tests/frame_batcher_test.cpp:694-747: an alternative (widening) table decodes identically
    name = "OS-2-128-U1_v2.3.0_1024x10"
    meta, packets = load_fixture(name)
    si = ob.SensorInfo.from_meta(meta)
    fr = ob.LidarFrame(si)
    b = ob.FrameBatcher(si)
    assert [b.batch(p, 5, fr) for p in packets][-1]
    alt = ob.SensorInfo.from_meta(meta)
    alt.set_custom_fields([("RANGE", 3, 0, 0x0007ffff, 0), ("FLAGS", 1, 2, 0b11111000, 3),
                           ("REFLECTIVITY", 1, 3, 0xff00, 8), ("SIGNAL", 2, 6, 0, 0),
                           ("NEAR_IR", 2, 8, 0, 0), ("WINDOW", 1, 11, 0, 0)], 12)
    fr2 = ob.LidarFrame(alt)
    b2 = ob.FrameBatcher(alt)
    assert [b2.batch(p, 5, fr2) for p in packets][-1]
    for n in ("RANGE", "FLAGS", "REFLECTIVITY", "SIGNAL", "NEAR_IR"):
        assert np.array_equal(fr.field(n), fr2.field(n)), n


# the named fields FIVE_WORD_PIXEL's RAW32_WORD1..5 cover (tests/golden/profile_tables.json)
FIVE_WORD_NAMED_FIELDS = {"FLAGS": np.uint8, "FLAGS2": np.uint8, "NEAR_IR": np.uint16, "RANGE": np.uint32,
                          "RANGE2": np.uint32, "REFLECTIVITY": np.uint8, "REFLECTIVITY2": np.uint8,
                          "SIGNAL": np.uint16, "SIGNAL2": np.uint16}


@pytest.mark.parametrize("profile,header,h,w", [
    ("RNG19_RFL8_SIG16_NIR16_DUAL", "STANDARD", 128, 1024), ("RNG19_RFL8_SIG16_NIR16", "STANDARD", 64, 512),
    ("RNG15_RFL8_NIR8", "STANDARD", 32, 512), ("LEGACY", "STANDARD", 32, 512),
    ("FUSA_RNG15_RFL8_NIR8_DUAL", "FUSA", 32, 512), ("RNG19_RFL8_SIG16_NIR16_RGB16", "STANDARD", 32, 512),
    ("FIVE_WORD_PIXEL", "STANDARD", 32, 512), ("RNG15_RFL8_NIR8_DUAL", "STANDARD", 64, 512),
    ("RNG15_RFL8_WIN8", "STANDARD", 32, 512), ("RNG19_RFL8_SIG16_NIR16_ZONE16", "STANDARD", 32, 512),
    ("RNG15_RFL8_NIR8_ZONE16", "STANDARD", 32, 512), ("RNG19_RFL8_SIG16_ZONE16_DUAL", "STANDARD", 32, 512),
    ("RNG19_RFL8_SIG16_NIR16_RGB16_DUAL", "STANDARD", 32, 512),
])
def test_gpu_frame_to_packets_is_byte_identical(ob, profile, header, h, w):
    """K4 (ob_encode_frames): set_block of every field + column headers + CRC64 on the device ==
    the host encoder == the oracle's frame_to_packets (impl/lidar_frame_impl.h:435-531), byte for
    byte, including invalid columns (no pixel data) and packets that are not emitted at all.
    FIVE_WORD_PIXEL's frame also carries the named fields its RAW32 words cover, each drawn on its
    own: where masks overlap, the field set last (PacketFormat order) decides the bits."""
    si = ob.SensorInfo(profile, h, w, 16, header_type=header, fw_rev="v3.2.1")
    masks = {f[0]: f[6] for f in si.fields()}
    rs = np.random.default_rng(99)
    src = ob.LidarFrame(si)
    if profile == "FIVE_WORD_PIXEL":
        for name, dt in FIVE_WORD_NAMED_FIELDS.items():
            src.add_field(name, dt)
    for name in src.fields:
        a = src.field(name)
        a[...] = (rs.integers(0, 1 << 32, size=a.shape, dtype=np.uint64) & np.uint64(masks.get(name, 0xffff))).astype(a.dtype)
    src.measurement_id[:] = np.arange(w)
    src.timestamp[:] = 1000 + np.arange(w)
    src.status[:] = 1
    src.status[5::7] = 0                      # invalid columns: headers only
    src.status[32:48] = 0                     # a whole packet without valid columns ...
    src.packet_timestamp[:] = 10 + np.arange(w // 16)
    src.packet_timestamp[2] = 0               # ... and no host timestamp: not emitted
    src.alert_flags[:] = rs.integers(0, 256, w // 16)
    src.frame_id = 1234
    host_pk, host_ts = ob.frame_to_packets(src, si, init_id=77, prod_sn=991)
    dev_pk, dev_ts = ob.frame_to_packets(src, si, init_id=77, prod_sn=991, device=True)
    assert host_pk.shape == dev_pk.shape == (w // 16 - 1, si.lidar_packet_size)
    assert np.array_equal(host_ts, dev_ts)
    assert np.array_equal(host_pk, dev_pk)
    if profile != "LEGACY" and header == "STANDARD":   # the CRC the sensor would have computed
        for p in dev_pk:
            crc = int(p[-8:].view(np.uint64)[0])
            assert crc == si.calculate_crc(p) == orc.crc64(p[:-8])
    if profile == "FIVE_WORD_PIXEL":   # the overlaps really disagree, and the oracle agrees on the outcome
        opf = oracle_pf(profile, h, w, 16, header)
        of = orc.Frame(opf, with_window=False,
                       extra_fields=[(n, orc.NP_TYPE[np.dtype(dt)]) for n, dt in FIVE_WORD_NAMED_FIELDS.items()])
        assert set(opf.field_names) <= set(src.fields) and set(opf.field_names) <= set(of.field_names)
        for name in opf.field_names:
            of.field(name)[...] = src.field(name)
        of.timestamp[:], of.status[:] = src.timestamp, src.status
        of.packet_timestamp[:], of.alert_flags[:] = src.packet_timestamp, src.alert_flags
        of.frame_id = src.frame_id
        opk, _ = orc.frame_to_packets(of, opf, init_id=77, prod_sn=991)
        assert np.array_equal(opk, dev_pk)
        assert np.any(src.field("RANGE") != (src.field("RAW32_WORD1") & np.uint32(0x7ffff)))
