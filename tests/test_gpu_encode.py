"""GPU tests of K4 (ob_encode_frames: frame fields -> lidar packets + CRC64) driven through the C ABI and
checked byte for byte against the CPU oracle's frame_to_packets (impl::frame_to_packets + set_block +
CRC64): every profile, custom layouts whose masks overlap, launch shapes (columns per packet, several
frames, strides, NULL inputs, host and device buffers), CRC64 over many packet lengths, the round trip
K4 -> K2 on the device, and the argument errors."""
import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import oracle as orc
from tests.helpers import decoder_desc_from_oracle, oracle_pf, random_frame, random_lut
from tests.test_gpu_decode import PROFILE_CASES

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


# the named fields FIVE_WORD_PIXEL's RAW32_WORD1..5 cover (tests/golden/profile_tables.json)
FIVE_WORD_NAMED = [("FLAGS", orc.UINT8), ("FLAGS2", orc.UINT8), ("NEAR_IR", orc.UINT16), ("RANGE", orc.UINT32),
                   ("RANGE2", orc.UINT32), ("REFLECTIVITY", orc.UINT8), ("REFLECTIVITY2", orc.UINT8),
                   ("SIGNAL", orc.UINT16), ("SIGNAL2", orc.UINT16)]
SENTINEL = 0xA5


def _ptr(a):
    if a is None:
        return None
    if type(a).__module__.startswith("torch"):
        assert a.is_contiguous()
        return a.data_ptr()
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data


def encode(ob, dec, frames, with_crc, stream=None):
    """ob_encode_frames over `frames`: dicts {fields: [array or None, decoder order], timestamp, status,
    headers, header_bytes, packets, stride}; waits for the stream."""
    capi = ob._capi
    ios = (capi.EncodeIO * len(frames))()
    for io, fr in zip(ios, frames):
        for k, a in enumerate(fr["fields"]):
            io.fields[k] = _ptr(a)
        io.timestamp, io.status = _ptr(fr.get("timestamp")), _ptr(fr.get("status"))
        io.packet_headers, io.packet_header_bytes = _ptr(fr.get("headers")), fr.get("header_bytes", 0)
        io.packets, io.packet_stride = _ptr(fr["packets"]), fr["stride"]
    st = stream if stream is not None else ob.Stream(0)
    capi.check(capi.lib.ob_encode_frames(dec._h, ios, len(frames), int(with_crc), st.h))
    st.sync()


def is_legacy(pf):
    return pf.profile == orc.PROFILES["LEGACY"]


def oracle_packets(pf, frame, init_id=5, prod_sn=1234):
    """The oracle's packets of `frame`, one row per packet slot (zeros where frame_to_packets emits
    nothing), which slots it emits, and the header template K4 gets: the first packet_header_size bytes
    of every packet -- for LEGACY, whose frame-level words live in the column headers, the whole packet
    with every channel-data block zeroed, so the template cannot supply pixel bytes."""
    pk, _ = orc.frame_to_packets(frame, pf, init_id=init_id, prod_sn=prod_sn)
    cpp, n = pf.columns_per_packet, frame.c.n_packets
    emitted = ((frame.status.reshape(n, cpp) & 1).any(axis=1)) | (frame.packet_timestamp != 0)
    assert len(pk) == emitted.sum()
    refs = np.zeros((n, pf.lidar_packet_size), np.uint8)
    refs[emitted] = pk
    if is_legacy(pf):
        headers = refs.copy()
        for c in range(cpp):
            base = pf.packet_header_size + c * pf.col_size + pf.col_header_size
            headers[:, base:base + pf.pixels_per_column * pf.channel_data_size] = 0
    else:
        headers = np.ascontiguousarray(refs[:, :pf.packet_header_size])
    return refs, emitted, headers


def with_crc_of(pf):
    return not is_legacy(pf) and pf.header_type == orc.HEADER_STANDARD


def frame_io(frame, fields, headers, packets, stride):
    return {"fields": [frame.field(f["name"]) for f in fields], "timestamp": frame.timestamp,
            "status": frame.status, "headers": headers, "header_bytes": 0 if headers is None else headers.shape[1],
            "packets": packets, "stride": stride}


def invalidate_some_columns(frame, cpp):
    frame.status[5::7] = 0                       # invalid columns: headers only
    frame.status[2 * cpp:3 * cpp] = 0            # a packet without a valid column, still emitted
    frame.status[4 * cpp:5 * cpp] = 0            # ... and one that is not emitted at all
    frame.packet_timestamp[4] = 0


def check_against_oracle(ob, pf, frame, stride=None):
    """encode `frame` with K4 into a sentinel-filled host buffer; the emitted packets must equal the
    oracle's, the bytes between packets must keep the sentinel, and every CRC must check."""
    layout, fields = decoder_desc_from_oracle(pf, frame)
    dec = ob.Decoder(layout, fields)
    refs, emitted, headers = oracle_packets(pf, frame)
    n, psz = refs.shape
    stride = stride or psz
    buf = np.full(n * stride, SENTINEL, np.uint8)
    encode(ob, dec, [frame_io(frame, fields, headers, buf, stride)], with_crc_of(pf))
    got = np.stack([buf[k * stride:k * stride + psz] for k in range(n)])
    assert np.array_equal(got[emitted], refs[emitted])
    for k in range(n):
        assert np.all(buf[k * stride + psz:(k + 1) * stride] == SENTINEL), k
    if with_crc_of(pf):
        for p in got:
            assert int(p[-8:].view(np.uint64)[0]) == orc.crc64(p[:-8])
    return got, refs, emitted


ENCODE_CASES = [(p, hd, h, w, ()) for p, hd, h, w in PROFILE_CASES] + [
    ("FIVE_WORD_PIXEL", "STANDARD", 32, 1024, tuple(FIVE_WORD_NAMED))]


@pytest.mark.parametrize("profile,header,h,w,extra", ENCODE_CASES,
                         ids=[f"{p}-{hd}-{h}-{w}" + ("-named_fields" if e else "") for p, hd, h, w, e in ENCODE_CASES])
def test_every_profile_matches_oracle(ob, profile, header, h, w, extra):
    """Every profile, with invalid columns, a packet with no valid column and one not emitted.  The
    FIVE_WORD_PIXEL case carries the RAW32 words and the named fields they overlap, every field drawn on
    its own, so the overlapping bits disagree and only set's clear-then-OR in field order gets them right."""
    pf = oracle_pf(profile, h, w, 16, header)
    src = random_frame(pf, seed=31 + h + w, extra_fields=extra)
    invalidate_some_columns(src, 16)
    got, refs, emitted = check_against_oracle(ob, pf, src)
    assert emitted.sum() == w // 16 - 1
    if extra:   # the named fields really disagree with the RAW32 words under them
        assert np.any(src.field("RANGE") != (src.field("RAW32_WORD1") & np.uint32(0x7ffff)))


def wide_layout(pf, wide_name):
    """the 7-byte pixel of test_decode_unaligned_wire_layout_and_wide_fields: a 56-bit field under three
    narrower ones (nothing word aligned)"""
    pf.set_fields([("RANGE", orc.UINT32, 0, 0x7ffff, 0), ("SIGNAL", orc.UINT16, 3, 0xffff, 0),
                   ("FLAGS", orc.UINT8, 5, 0xf0, 4), (wide_name, orc.UINT64, 0, 0x00ffffffffffffff, 0)], 7)


@pytest.mark.parametrize("wide_name", ["WIDE", "A_WIDE"])   # encoded last / first (PacketFormat order)
def test_overlapping_wide_field_layout(ob, wide_name):
    pf = oracle_pf("RNG19_RFL8_SIG16_NIR16", 8, 128)
    wide_layout(pf, wide_name)
    src = random_frame(pf, seed=5, with_window=False, extra_fields=[(wide_name, orc.UINT64)])
    src.field(wide_name)[:, ::3] = 0              # zeros must clear what an earlier field set
    invalidate_some_columns(src, 16)
    assert pf.channel_data_size == 7 and pf.lidar_packet_size % 4 == 0
    check_against_oracle(ob, pf, src)


# masks overlapping each other with positive and negative shifts, in one 8-byte pixel; names give the
# order A..E in which set_block writes them
SHIFT_LAYOUT = [("A", orc.UINT32, 0, 0x00ffff00, 8), ("B", orc.UINT16, 1, 0x0ff0, 4), ("C", orc.UINT8, 2, 0x3c, -2),
                ("D", orc.UINT64, 0, 0x0000ffffffff0000, 16), ("E", orc.UINT16, 3, 0x0ff0, -4)]


@pytest.mark.parametrize("zero_last", [False, True])
def test_overlapping_shifted_masks(ob, zero_last):
    """zero_last: E is 0 everywhere, so its bits must come out clear although D (written before it) set
    them -- an OR into a zeroed buffer would keep D's bits."""
    pf = oracle_pf("RNG19_RFL8_SIG16_NIR16", 16, 128)
    pf.set_fields(SHIFT_LAYOUT, 8)
    src = random_frame(pf, seed=17, with_window=False, extra_fields=[(f[0], f[1]) for f in SHIFT_LAYOUT])
    for f in SHIFT_LAYOUT:
        assert np.any(src.field(f[0]) != 0)
    if zero_last:
        src.field("E")[...] = 0
    got, refs, emitted = check_against_oracle(ob, pf, src)
    if zero_last:   # column 0 of packet 0: D, written before E, set bits under E's mask; they come out clear
        e_bits = np.uint64(0x0ff0 << 24)             # E's mask in the pixel's 8-byte window
        d_bits = (src.field("D")[:, 0].astype(np.uint64) << np.uint64(16)) & np.uint64(0x0000ffffffff0000)
        assert np.any(d_bits & e_bits)
        base = pf.packet_header_size + pf.col_header_size
        px = got[0, base:base + 16 * 8].copy().view(np.uint64)
        assert np.all(px & e_bits == 0)


def test_mask_past_the_pixel_is_refused(ob):
    """a mask reaching into the next pixel's bytes: the reference's result then depends on the order it
    writes pixels in, which the one-thread-per-pixel encoder does not reproduce, so the call is refused"""
    pf = oracle_pf("RNG19_RFL8_SIG16_NIR16", 8, 64)
    pf.set_fields([("RANGE", orc.UINT32, 0, 0x7ffff, 0), ("SIGNAL", orc.UINT32, 2, 0xffffff, 0)], 4)
    src = random_frame(pf, seed=1, with_window=False)
    layout, fields = decoder_desc_from_oracle(pf, src)
    dec = ob.Decoder(layout, fields)
    _, _, headers = oracle_packets(pf, src)
    buf = np.full(4 * pf.lidar_packet_size, SENTINEL, np.uint8)
    with pytest.raises(ValueError, match="field mask reaches past the pixel's channel data"):
        encode(ob, dec, [frame_io(src, fields, headers, buf, pf.lidar_packet_size)], True)
    assert np.all(buf == SENTINEL)


@pytest.mark.parametrize("cpp", [4, 8, 16, 32])
def test_columns_per_packet(ob, cpp):
    pf = oracle_pf("RNG19_RFL8_SIG16_NIR16_DUAL", 32, 512, cpp)
    src = random_frame(pf, seed=40 + cpp)
    invalidate_some_columns(src, cpp)
    got, refs, emitted = check_against_oracle(ob, pf, src)
    assert len(got) == 512 // cpp and emitted.sum() == 512 // cpp - 1


def test_several_frames_in_one_launch(ob):
    """five frames, each its own values, frame id, invalid columns and stride, in one ob_encode_frames call"""
    pf = oracle_pf("RNG15_RFL8_NIR8_DUAL", 32, 256)
    psz = pf.lidar_packet_size
    srcs = [random_frame(pf, seed=60 + i, frame_id=900 + i) for i in range(5)]
    for i, s in enumerate(srcs):
        s.status[(3 + i)::(5 + i)] = 0
        s.timestamp[:] = 77 * i + np.arange(256)
    layout, fields = decoder_desc_from_oracle(pf, srcs[0])
    dec = ob.Decoder(layout, fields)
    cases, ios = [], []
    for i, s in enumerate(srcs):
        refs, emitted, headers = oracle_packets(pf, s)
        stride = psz + 16 * i
        buf = np.full(len(refs) * stride, SENTINEL, np.uint8)
        cases.append((refs, emitted, buf, stride))
        ios.append(frame_io(s, fields, headers, buf, stride))
    encode(ob, dec, ios, True)
    for i, (refs, emitted, buf, stride) in enumerate(cases):
        got = np.stack([buf[k * stride:k * stride + psz] for k in range(len(refs))])
        assert np.array_equal(got[emitted], refs[emitted]), i
        for k in range(len(refs)):
            assert np.all(buf[k * stride + psz:(k + 1) * stride] == SENTINEL), (i, k)
    assert not np.array_equal(cases[0][0], cases[1][0])


@pytest.mark.parametrize("extra,offset", [(0, 0), (64, 0), (1, 1)])
def test_packet_stride(ob, extra, offset):
    """packet_stride = packet_size, + 64, and odd with an odd base address (K4's byte-store path); the
    bytes between packets are not written"""
    pf = oracle_pf("RNG19_RFL8_SIG16_NIR16", 16, 256)
    src = random_frame(pf, seed=70 + extra)
    invalidate_some_columns(src, 16)
    layout, fields = decoder_desc_from_oracle(pf, src)
    dec = ob.Decoder(layout, fields)
    refs, emitted, headers = oracle_packets(pf, src)
    n, psz = refs.shape
    stride = psz + extra
    raw = np.full(n * stride + offset, SENTINEL, np.uint8)
    buf = raw[offset:]
    encode(ob, dec, [frame_io(src, fields, headers, buf, stride)], True)
    assert raw[:offset].tolist() == [SENTINEL] * offset
    for k in range(n):
        if emitted[k]:
            assert np.array_equal(buf[k * stride:k * stride + psz], refs[k]), k
        assert np.all(buf[k * stride + psz:(k + 1) * stride] == SENTINEL), k


def test_null_fields_and_headers(ob):
    """NULL entries of fields[] leave their bits zero; NULL packet_headers leaves the header bytes zero;
    NULL timestamps leave the column timestamps zero.  The CRC covers what was written."""
    pf = oracle_pf("RNG19_RFL8_SIG16_NIR16_DUAL", 32, 512)
    src = random_frame(pf, seed=80)
    invalidate_some_columns(src, 16)
    layout, fields = decoder_desc_from_oracle(pf, src)
    dec = ob.Decoder(layout, fields)
    skip = {"SIGNAL", "RANGE2", "WINDOW"}
    ref_frame = random_frame(pf, seed=80)
    invalidate_some_columns(ref_frame, 16)
    for name in skip:
        ref_frame.field(name)[...] = 0
    ref_frame.timestamp[:] = 0
    refs, emitted, _ = oracle_packets(pf, ref_frame)
    refs[:, :pf.packet_header_size] = 0
    for p in refs:
        p[-8:] = np.frombuffer(np.uint64(orc.crc64(p[:-8])).tobytes(), np.uint8)
    n, psz = refs.shape
    buf = np.full(n * psz, SENTINEL, np.uint8)
    io = frame_io(src, fields, None, buf, psz)
    io["fields"] = [None if f["name"] in skip else a for f, a in zip(fields, io["fields"])]
    io["timestamp"] = None
    encode(ob, dec, [io], True)
    got = buf.reshape(n, psz)
    assert np.array_equal(got[emitted], refs[emitted])
    assert np.all(got[:, :pf.packet_header_size] == 0)


def test_device_buffers_on_a_torch_stream(ob):
    """fields, status, timestamps, headers and packets as CUDA tensors on a side torch stream == the same
    call from host buffers == the oracle, byte for byte, gaps between packets untouched in both"""
    torch = pytest.importorskip("torch")
    pf = oracle_pf("RNG19_RFL8_SIG16_NIR16_RGB16_DUAL", 32, 512)
    src = random_frame(pf, seed=90)
    invalidate_some_columns(src, 16)
    layout, fields = decoder_desc_from_oracle(pf, src)
    dec = ob.Decoder(layout, fields)
    refs, emitted, headers = oracle_packets(pf, src)
    n, psz = refs.shape
    stride = psz + 64
    host_io = frame_io(src, fields, headers, np.full(n * stride, SENTINEL, np.uint8), stride)
    encode(ob, dec, [host_io], True)
    signed = {1: np.uint8, 2: np.int16, 4: np.int32, 8: np.int64}
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        def dev(a):
            return torch.from_numpy(np.ascontiguousarray(a).view(signed[a.dtype.itemsize])).to("cuda")
        dev_io = dict(host_io, fields=[dev(a) for a in host_io["fields"]], timestamp=dev(src.timestamp),
                      status=dev(src.status), headers=dev(headers),
                      packets=torch.full((n * stride,), SENTINEL, dtype=torch.uint8, device="cuda"))
        encode(ob, dec, [dev_io], True, stream=ob.Stream(0, cuda_stream=side.cuda_stream))
    torch.cuda.synchronize()
    dev_buf = dev_io["packets"].cpu().numpy()
    assert np.array_equal(dev_buf, host_io["packets"])
    got = np.stack([dev_buf[k * stride:k * stride + psz] for k in range(n)])
    assert np.array_equal(got[emitted], refs[emitted])
    assert np.all(dev_buf.reshape(n, stride)[:, psz:] == SENTINEL)


def crc_lengths():
    """multiples of 4 from 16 to 65532: every length up to 1100, then lengths where crc_len = packet_size - 8
    fills 256 chunks exactly (no padding) and their neighbours, lengths whose chunk gets the odd-word-count
    adjustment, and a sparse sweep to the top"""
    out = set(range(16, 1100, 4))
    for cb in range(4, 264, 8):        # cb / 4 odd: no adjustment, exact fit at crc_len = 256 * cb
        for d in (-4, 0, 4):
            out.add(256 * cb + 8 + d)
    for cb in range(8, 264, 8):        # cb / 4 even: rounded up to cb + 4, padding 1024 bytes
        out.add(256 * cb + 8)
        out.add(256 * (cb - 4) + 12)
    out.update(range(1100, 65536, 1996))
    out.add(65532)
    return sorted(p for p in out if 16 <= p <= 65532 and p % 4 == 0)


def test_crc_over_packet_lengths(ob):
    """CRC64 of K4 at many packet lengths, all in one process so the (device, crc_len) table cache serves
    several lengths and is met again: a one-packet layout whose header template is the whole packet of
    random bytes, so the CRC runs over data everywhere; crc64(p[:-8]) == p[-8:], the rest is the template"""
    rs = np.random.default_rng(123)
    lengths = crc_lengths()
    assert len(lengths) > 400
    st = ob.Stream(0)
    decs = {}
    for rep in range(2):
        for psz in (lengths if rep == 0 else lengths[::7]):
            if psz not in decs:
                layout = {"packet_header_size": 0, "col_header_size": 0, "channel_data_size": 4, "col_size": 4,
                          "packet_size": psz, "columns_per_packet": 1, "pixels_per_column": 1,
                          "columns_per_frame": 1, "col_timestamp": (0, 0, 0), "col_measurement_id": (0, 0, 0),
                          "col_status": (0, 0, 0)}
                decs[psz] = ob.Decoder(layout, [])
            tmpl = rs.integers(0, 256, size=(1, psz), dtype=np.uint8)
            buf = np.full(psz, SENTINEL, np.uint8)
            encode(ob, decs[psz], [{"fields": [], "headers": tmpl, "header_bytes": psz, "packets": buf,
                                    "stride": psz}], True, stream=st)
            assert np.array_equal(buf[:-8], tmpl[0, :-8]), psz
            assert int(buf[-8:].view(np.uint64)[0]) == orc.crc64(tmpl[0, :-8]), psz


@pytest.mark.parametrize("profile,header,h,w", PROFILE_CASES)
def test_device_round_trip_through_k2(ob, profile, header, h, w):
    """K4 then K2 (Decoder.decode_batch) on the same device packet buffer: fields, column headers, fused XYZ
    and destaggered range equal the source frame and the oracle's cartesian / destagger"""
    torch = pytest.importorskip("torch")
    pf = oracle_pf(profile, h, w, 16, header)
    src = random_frame(pf, seed=0x5eed + h)
    layout, fields = decoder_desc_from_oracle(pf, src)
    dec = ob.Decoder(layout, fields)
    refs, emitted, headers = oracle_packets(pf, src)
    n, psz = refs.shape
    t_pk = torch.empty((n, psz), dtype=torch.uint8, device="cuda")
    st = ob.Stream(0, cuda_stream=torch.cuda.current_stream().cuda_stream)
    encode(ob, dec, [frame_io(src, fields, headers, t_pk, psz)], with_crc_of(pf), stream=st)
    assert np.array_equal(t_pk.cpu().numpy(), refs)
    tdt = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
    outs = {}
    for f in fields:
        a = src.field(f["name"])
        outs[f["name"]] = torch.empty((1,) + a.shape, dtype=tdt[a.dtype.itemsize], device="cuda")
    n_ret = int(src.has_field("RANGE")) + int(src.has_field("RANGE2"))
    d, o = random_lut(h * w, 7)
    lut = ob.XYZLutT.from_arrays(d, o, h, w) if n_ret else None
    shifts = np.random.default_rng(3).integers(-24, 25, h).astype(np.int32)
    xyz = [torch.empty((1, h * w, 3), dtype=torch.float32, device="cuda") for _ in range(n_ret)]
    rd = [torch.empty((1, h, w), dtype=torch.int32, device="cuda") for _ in range(n_ret)]
    ts = torch.empty((1, w), dtype=torch.int64, device="cuda")
    mid = torch.empty((1, w), dtype=torch.int16, device="cuda")
    status = torch.empty((1, w), dtype=torch.int32, device="cuda")
    dec.decode_batch(1, t_pk, n, psz, n * psz, outs, lut=lut, pixel_shift_by_row=shifts if n_ret else None,
                     xyz=xyz or None, range_destaggered=rd or None, timestamp=ts, measurement_id=mid,
                     status=status, stream=st)
    torch.cuda.synchronize()
    for name, t in outs.items():
        assert np.array_equal(t[0].cpu().numpy().view(src.field(name).dtype), src.field(name)), name
    assert np.array_equal(ts[0].cpu().numpy().view(np.uint64), src.timestamp)
    assert np.array_equal(mid[0].cpu().numpy().view(np.uint16), src.measurement_id)
    assert np.array_equal(status[0].cpu().numpy().view(np.uint32), src.status)
    for r, nm in enumerate(("RANGE", "RANGE2")[:n_ret]):
        assert np.array_equal(xyz[r][0].cpu().numpy(), orc.cartesian(src.field(nm), d, o)), nm
        assert np.array_equal(rd[r][0].cpu().numpy().view(np.uint32), orc.destagger(src.field(nm), shifts)), nm


def _error_case(pf, src, what):
    layout, fields = decoder_desc_from_oracle(pf, src)
    _, _, headers = oracle_packets(pf, src)
    psz = pf.lidar_packet_size
    io = frame_io(src, fields, headers, None, psz)
    with_crc = True
    if what == "columns":
        layout["columns_per_frame"] = pf.columns_per_frame + 8
        msg = "Mismatch between expected number of packets and PacketFormat.columns_per_packet"
    elif what == "stride":
        io["stride"] = psz - 4
        msg = "packet_stride smaller than the lidar packet size"
    elif what == "header_bytes":
        io["headers"] = np.ascontiguousarray(headers[:, :pf.packet_header_size - 1])
        io["header_bytes"] = pf.packet_header_size - 1
        msg = "packet_header_bytes smaller than the packet header"
    else:   # "crc": a packet size that is not a multiple of 4
        layout["packet_size"] = psz + 2
        io["stride"] = psz + 2
        msg = "packet size must be a multiple of 4 for the CRC64 footer"
    return layout, fields, io, with_crc, msg


@pytest.mark.parametrize("what", ["columns", "stride", "header_bytes", "crc"])
@pytest.mark.parametrize("where", ["host", "device"])
def test_errors_leave_the_output_untouched(ob, what, where):
    pf = oracle_pf("RNG19_RFL8_SIG16_NIR16", 16, 256)
    src = random_frame(pf, seed=99)
    layout, fields, io, with_crc, msg = _error_case(pf, src, what)
    dec = ob.Decoder(layout, fields)
    nbytes = 16 * (pf.lidar_packet_size + 2)
    if where == "device":
        torch = pytest.importorskip("torch")
        io["packets"] = torch.full((nbytes,), SENTINEL, dtype=torch.uint8, device="cuda")
    else:
        io["packets"] = np.full(nbytes, SENTINEL, np.uint8)
    with pytest.raises(ValueError, match=msg):
        encode(ob, dec, [io], with_crc)
    out = io["packets"].cpu().numpy() if where == "device" else io["packets"]
    assert np.all(out == SENTINEL)
    if what == "crc":   # without the CRC footer the same odd-sized layout encodes through the byte stores
        encode(ob, dec, [io], False)
        psz = layout["packet_size"]
        got = out if where == "host" else io["packets"].cpu().numpy()
        refs, emitted, _ = oracle_packets(pf, src)
        for k in range(len(refs)):
            assert np.array_equal(got[k * psz:k * psz + pf.lidar_packet_size - 8], refs[k, :-8]), k
