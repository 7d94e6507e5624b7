"""Shared helpers for the test-suite (fixture loading, synthetic inputs)."""
import json
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

PCAP_FIXTURES = [
    "OS-0-128-U1_v2.3.0_1024x10",
    "OS-0-32-U1_v2.2.0_1024x10",
    "OS-1-128_767798045_1024x10_20230712_120049",
    "OS-2-128-U1_v2.3.0_1024x10",
    "OS-2-32-U0_v2.0.0_1024x10",
    "OS-1-32-G_v2.1.1_1024x10",
]


def load_fixture(name):
    meta = json.load(open(os.path.join(GOLDEN, name + ".json")))
    packets = np.load(os.path.join(GOLDEN, name + ".npz"))["packets"]
    return meta, packets


def fw_has_window(meta):
    """WINDOW is in the default field set only for fw >= 3.2 (lidar_frame.cpp:1097-1110);
    every committed fixture is older."""
    return False


def random_range(h, w, seed, p_zero=0.5, max_range=(1 << 19) - 1):
    """Synthetic range image as tests/benchmarks/benchmark_utils.h:93-110 draws it:
    ~p_zero zeros, valid returns uniform in [1, max_range]."""
    rng = np.random.default_rng(seed)
    r = rng.integers(1, max_range + 1, size=(h, w), dtype=np.uint32)
    r[rng.random((h, w)) < p_zero] = 0
    return r


def random_lut(n, seed, dtype=np.float32):
    """Random LUT as tests/benchmarks/benchmark_utils.h:112-126: dir in U(0.5,1.5), off in U(0,0.01)."""
    rng = np.random.default_rng(seed)
    d = (rng.random((n, 3)) + 0.5).astype(dtype)
    o = (rng.random((n, 3)) * 0.01).astype(dtype)
    return d, o


# ------------------------------------------------------------------------------------------------
# decode helpers (test infrastructure: descriptors and column maps derived from the ORACLE tables,
# so the kernel is checked independently of the product's own host-side PacketFormat)
# ------------------------------------------------------------------------------------------------
def oracle_pf(meta_or_profile, h=None, w=None, cpp=16, header="STANDARD"):
    from oracle import oracle as orc
    if isinstance(meta_or_profile, dict):
        m = meta_or_profile
        return orc.PacketFormat(m["profile"], m["h"], m["w"], m["columns_per_packet"],
                                orc.HEADER_FUSA if m["header_type"] == "FUSA" else orc.HEADER_STANDARD)
    return orc.PacketFormat(meta_or_profile, h, w, cpp,
                            orc.HEADER_FUSA if header == "FUSA" else orc.HEADER_STANDARD)


def decoder_desc_from_oracle(pf, frame):
    """(layout, fields) for ob.Decoder from an oracle PacketFormat and an oracle Frame."""
    fi = lambda i: (i.offset, i.mask, i.shift)
    layout = {
        "packet_header_size": pf.packet_header_size, "col_header_size": pf.col_header_size,
        "channel_data_size": pf.channel_data_size, "col_size": pf.col_size,
        "packet_size": pf.lidar_packet_size, "columns_per_packet": pf.columns_per_packet,
        "pixels_per_column": pf.pixels_per_column, "columns_per_frame": pf.columns_per_frame,
        "col_timestamp": fi(pf.c.col_timestamp_info),
        "col_measurement_id": fi(pf.c.col_measurement_id_info),
        "col_status": fi(pf.c.col_status_info),
    }
    fields = []
    for name in pf.field_names:          # std::map order
        if not frame.has_field(name):
            continue
        info = pf.field_info(name)
        a = frame.field(name)
        es = a.dtype.itemsize * (3 if name == "RGB" else 1)
        fields.append({"name": name, "offset": info.offset, "mask": info.mask, "shift": info.shift,
                       "elem_size": es,
                       "range_return": {"RANGE": 0, "RANGE2": 1}.get(name, -1),
                       "zero_pattern": 0x7e00 if name == "RGB" else 0})
    return layout, fields


def col_map_from_packets(pf, packets):
    """Final-state rule of FrameBatcher (SURVEY 8a'-3): frame column m_id takes the LAST arriving
    valid (status & 1) packet column with that measurement id; everything else is zero-filled."""
    w, cpp = pf.columns_per_frame, pf.columns_per_packet
    col_src = np.full(w, -1, np.int32)
    for slot, buf in enumerate(packets):
        for c in range(cpp):
            base = pf.packet_header_size + c * pf.col_size
            col = np.concatenate([buf[base: base + pf.col_size], np.zeros(8, np.uint8)])
            from oracle import oracle as orc
            import ctypes as C
            m_id = orc.lib().orc_field_get(C.byref(pf.c.col_measurement_id_info), col.ctypes.data) & 0xffff
            status = orc.lib().orc_field_get(C.byref(pf.c.col_status_info), col.ctypes.data) & 0xffffffff
            if (status & 1) and m_id < w:
                col_src[m_id] = slot * cpp + c
    return col_src


def random_frame(pf, seed, with_window=True, frame_id=700, extra_fields=()):
    """Random LidarFrame as tests/packet_format_test.cpp:246-266 builds it: every profile field
    drawn within its value mask, headers iota, status 1.  extra_fields: [(name, orc type tag)] added to
    the frame's default fields (and drawn too when the profile carries them)."""
    from oracle import oracle as orc
    f = orc.Frame(pf, with_window=with_window, extra_fields=extra_fields)
    rs = np.random.default_rng(seed)
    w = pf.columns_per_frame
    f.measurement_id[:] = np.arange(w)
    f.timestamp[:] = 1000 + np.arange(w)
    f.status[:] = 1
    f.packet_timestamp[:] = 10 + np.arange(f.c.n_packets)
    f.alert_flags[:] = rs.integers(0, 256, f.c.n_packets)
    f.frame_id = frame_id
    for name in pf.field_names:
        if not f.has_field(name):
            continue
        a = f.field(name)
        mask = pf.value_mask(name)
        if name == "RGB":
            a[...] = rs.integers(0, 1 << 16, size=a.shape, dtype=np.uint64).astype(np.uint16)
        else:
            vals = rs.integers(0, mask + 1 if mask < (1 << 63) else (1 << 63), size=a.shape, dtype=np.uint64) & np.uint64(mask)
            a[...] = vals.astype(a.dtype)
    return f


# ---- BASELINE configs[0]: default OS1-64 1024x64 sensor (sensor_info.cpp:163-222, data_format.cpp:79-126)
def default_os1_64(w=1024):
    top = [16.611, 16.084, 15.557, 15.029, 14.502, 13.975, 13.447, 12.920, 12.393, 11.865, 11.338, 10.811,
           10.283, 9.756, 9.229, 8.701, 8.174, 7.646, 7.119, 6.592, 6.064, 5.537, 5.010, 4.482, 3.955, 3.428,
           2.900, 2.373, 1.846, 1.318, 0.791, 0.264]
    alt = np.array(top + [-a for a in reversed(top)])
    az = np.tile(np.array([3.164, 1.055, -1.055, -3.164]), 16)
    unit = {512: 3, 1024: 6, 2048: 12, 4096: 24}[w]
    shifts = np.tile(np.array([3, 2, 1, 0], np.int32) * unit, 16)
    b2l = np.eye(4)
    b2l[0, 3] = 15.806
    l2s = np.diag([-1.0, -1.0, 1.0, 1.0])
    l2s[2, 3] = 36.18
    return {"h": 64, "w": w, "beam_altitude_angles": alt, "beam_azimuth_angles": az,
            "pixel_shift_by_row": shifts, "beam_to_lidar_transform": b2l, "lidar_to_sensor_transform": l2s}
