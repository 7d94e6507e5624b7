"""Python mirror of the reference's LidarScan / ScanBatcher / PacketFormat objects over the host
C ABI (include/ouster_b200_host.h).  Names follow python/src/ouster/sdk/core/__init__.py:140-142
(LidarFrame/LidarScan, FrameBatcher/ScanBatcher)."""
import ctypes as C

import numpy as np

from ._capi import FieldDesc, PacketLayout, check, lib
from .core import _Handle

vp, sz, i32, u32, u64, i64 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32, C.c_uint64, C.c_int64
PP = C.POINTER


def _sig(name, restype, *argtypes):
    f = getattr(lib, name)
    f.restype, f.argtypes = restype, list(argtypes)


_sig("obh_set_device", i32, i32)
_sig("obh_get_device", i32)
_sig("obh_sensor_create", i32, C.c_char_p, i32, u32, u32, u32, vp, u32, u64, C.c_char_p, u32, u32, PP(vp))
_sig("obh_sensor_set_intrinsics", i32, vp, vp, sz, vp, sz, vp, vp, vp)
_sig("obh_sensor_set_custom_fields", i32, vp, sz, PP(C.c_char_p), vp, vp, vp, vp, sz)
_sig("obh_sensor_layout", i32, vp, PP(PacketLayout))
_sig("obh_sensor_n_fields", sz, vp)
_sig("obh_sensor_field", i32, vp, sz, C.c_char_p, sz, PP(C.c_int32), PP(u64), PP(u64), PP(C.c_int32),
     PP(C.c_int32), PP(u64))
_sig("obh_sensor_block_parsable", i32, vp)
_sig("obh_sensor_frame_id_difference", i32, vp, u32, u32)
_sig("obh_sensor_packet_frame_id", u32, vp, vp)
_sig("obh_sensor_packet_init_id", u32, vp, vp)
_sig("obh_sensor_packet_prod_sn", u64, vp, vp)
_sig("obh_sensor_calculate_crc", u64, vp, vp, sz)
_sig("obh_sensor_destroy", i32, vp)
_sig("obh_frame_create", i32, vp, PP(vp))
_sig("obh_frame_add_field", i32, vp, C.c_char_p, C.c_int32, sz)
_sig("obh_frame_add_field_class", i32, vp, C.c_char_p, C.c_int32, sz, C.c_int32)
_sig("obh_frame_del_field", i32, vp, C.c_char_p)
_sig("obh_frame_field_shape", i32, vp, C.c_char_p, PP(C.c_int32), PP(sz), PP(sz))
_sig("obh_frame_n_fields", sz, vp)
_sig("obh_frame_field_at", i32, vp, sz, C.c_char_p, sz, PP(C.c_int32), PP(sz), PP(vp))
_sig("obh_frame_field", i32, vp, C.c_char_p, PP(C.c_int32), PP(sz), PP(vp))
_sig("obh_frame_headers", i32, vp, PP(vp), PP(vp), PP(vp), PP(vp), PP(vp), PP(sz), PP(sz), PP(sz))
_sig("obh_frame_body_to_world", i32, vp, PP(vp))
_sig("obh_frame_valid_columns", i32, vp, PP(i32), PP(i32))
_sig("obh_frame_get_frame_id", i64, vp)
_sig("obh_frame_set_frame_id", None, vp, i64)
_sig("obh_frame_get_status", u64, vp, PP(C.c_uint8), PP(C.c_uint8))
_sig("obh_frame_set_status", None, vp, u64, C.c_uint8, C.c_uint8)
_sig("obh_frame_destroy", i32, vp)
_sig("obh_frame_to_packets", i32, vp, vp, u32, u64, vp, vp, PP(sz))
_sig("obh_frame_to_packets_device", i32, vp, vp, u32, u64, vp, vp, PP(sz))
_sig("obh_batcher_create", i32, vp, PP(vp))
_sig("obh_batcher_batch", i32, vp, vp, sz, u64, vp, PP(i32))
_sig("obh_batcher_flush", i32, vp, vp)
_sig("obh_batcher_batch_burst", i32, vp, vp, sz, sz, sz, vp, vp, PP(sz), PP(i32))
_sig("obh_batcher_reset", i32, vp)
_sig("obh_batcher_batched_packets", sz, vp)
_sig("obh_batcher_dropped_packets", sz, vp)
_sig("obh_batcher_gpu_launches", sz, vp)
_sig("obh_batcher_set_max_cache_size", i32, vp, sz)
_sig("obh_batcher_set_fused", i32, vp, vp, vp, sz)
_sig("obh_batcher_set_headers_only", i32, vp, i32)
_sig("obh_batcher_fused_outputs", i32, vp, i32, PP(vp), PP(sz), PP(vp))
_sig("obh_batcher_set_device_outputs", i32, vp, sz, PP(C.c_char_p), PP(vp), PP(vp), PP(vp))
_sig("obh_batcher_set_pipeline_depth", i32, vp, sz)
_sig("obh_batcher_wait", i32, vp, vp)
_sig("obh_batcher_destroy", i32, vp)
_sig("obh_pcap_open", i32, C.c_char_p, sz, C.c_uint16, sz, PP(vp))
_sig("obh_pcap_next_burst", i32, vp, sz, PP(vp), PP(sz), PP(vp), PP(sz))
_sig("obh_pcap_packets_read", sz, vp)
_sig("obh_pcap_skipped", sz, vp)
_sig("obh_pcap_close", i32, vp)


class Slot(C.Structure):
    """obh_slot (include/ouster_b200_host.h)."""
    _fields_ = [("frame", vp), ("xyz", vp * 2), ("range_destaggered", vp * 2), ("xyz_bytes", sz)]


_sig("obh_pipeline_create", i32, vp, sz, vp, vp, sz, PP(vp))
_sig("obh_pipeline_push_burst", i32, vp, vp, sz, sz, sz, vp, PP(sz), PP(Slot))
_sig("obh_pipeline_drain", i32, vp, PP(Slot))
_sig("obh_pipeline_stats", i32, vp, vp)
_sig("obh_pipeline_in_flight", sz, vp)
_sig("obh_pipeline_gpu_launches", sz, vp)
_sig("obh_pipeline_dropped_packets", sz, vp)
_sig("obh_pipeline_destroy", i32, vp)

# ChanFieldType tags (chanfield.h:111-128)
TAG_NP = {1: np.uint8, 2: np.uint16, 3: np.uint32, 4: np.uint64, 5: np.int8, 6: np.int16,
          7: np.int32, 8: np.int64, 9: np.float32, 10: np.float64, 12: np.uint16}
NP_TAG = {np.dtype(np.uint8): 1, np.dtype(np.uint16): 2, np.dtype(np.uint32): 3,
          np.dtype(np.uint64): 4, np.dtype(np.int8): 5, np.dtype(np.int16): 6,
          np.dtype(np.int32): 7, np.dtype(np.int64): 8, np.dtype(np.float32): 9,
          np.dtype(np.float64): 10}


def set_device(device):
    """CUDA device for this thread's FrameBatcher / host-mirror objects (b200::set_device)."""
    check(lib.obh_set_device(int(device)))


def get_device():
    return lib.obh_get_device()


def _as_array(ptr, dtype, shape):
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    if n == 0:
        return np.empty(shape, dtype)
    raw = np.ctypeslib.as_array((C.c_uint8 * n).from_address(ptr))
    return raw.view(dtype).reshape(shape)


class SensorInfo(_Handle):
    """SensorInfo + PacketFormat of one sensor stream."""
    _release = "obh_sensor_destroy"

    def __init__(self, profile, h, w, columns_per_packet=16, header_type="STANDARD",
                 pixel_shift_by_row=None, init_id=0, sn=0, fw_rev="UNKNOWN", column_window=None, prod_line=""):
        cw = column_window or (0, w - 1)
        sh = None
        if pixel_shift_by_row is not None:
            sh = np.ascontiguousarray(pixel_shift_by_row, np.int32)
            if sh.size != h:
                raise ValueError("pixel_shift_by_row must have one entry per row")
        hd = vp()
        check(lib.obh_sensor_create(profile.encode(), int(header_type == "FUSA"), h, w,
                                    columns_per_packet, sh.ctypes.data if sh is not None else None,
                                    init_id, sn, fw_rev.encode(), cw[0], cw[1], C.byref(hd)))
        self._h = hd
        self.profile, self.h, self.w, self.columns_per_packet = profile, h, w, columns_per_packet
        self.pixel_shift_by_row = sh if sh is not None else np.zeros(h, np.int32)
        self.init_id, self.sn = init_id, sn
        self.header_type, self.fw_rev, self.column_window = header_type, fw_rev, tuple(cw)
        self.prod_line = prod_line

    @classmethod
    def from_meta(cls, meta, fw_rev="UNKNOWN"):
        """From a tests/golden/*.json fixture dict."""
        s = cls(meta["profile"], meta["h"], meta["w"], meta["columns_per_packet"], meta["header_type"],
                meta["pixel_shift_by_row"], meta["init_id"], meta["prod_sn"], fw_rev,
                tuple(meta["column_window"]), meta.get("prod_line", ""))
        s.set_intrinsics(meta["beam_azimuth_angles"], meta["beam_altitude_angles"],
                         meta["beam_to_lidar_transform"], meta["lidar_to_sensor_transform"])
        return s

    def set_intrinsics(self, az, alt, beam_to_lidar, lidar_to_sensor, sensor_to_body=None):
        az = np.ascontiguousarray(az, np.float64)
        alt = np.ascontiguousarray(alt, np.float64)
        b2l = np.ascontiguousarray(beam_to_lidar, np.float64).reshape(16)
        l2s = np.ascontiguousarray(lidar_to_sensor, np.float64).reshape(16)
        s2b = None if sensor_to_body is None else np.ascontiguousarray(sensor_to_body, np.float64).reshape(16)
        check(lib.obh_sensor_set_intrinsics(self._h, az.ctypes.data, az.size, alt.ctypes.data, alt.size,
                                            b2l.ctypes.data, l2s.ctypes.data,
                                            s2b.ctypes.data if s2b is not None else None))
        self.beam_azimuth_angles, self.beam_altitude_angles = az, alt
        self.beam_to_lidar_transform, self.lidar_to_sensor_transform = b2l.reshape(4, 4), l2s.reshape(4, 4)
        self.sensor_to_body = None if s2b is None else s2b.reshape(4, 4)

    def set_custom_fields(self, fields, channel_data_size):
        """fields: list of (name, ty_tag, offset, mask, shift) -- add_custom_profile analogue."""
        n = len(fields)
        names = (C.c_char_p * n)(*[f[0].encode() for f in fields])
        tags = np.array([f[1] for f in fields], np.int32)
        offs = np.array([f[2] for f in fields], np.uint64)
        masks = np.array([f[3] for f in fields], np.uint64)
        shifts = np.array([f[4] for f in fields], np.int32)
        check(lib.obh_sensor_set_custom_fields(self._h, n, names, tags.ctypes.data, offs.ctypes.data,
                                               masks.ctypes.data, shifts.ctypes.data, channel_data_size))

    @property
    def layout(self):
        L = PacketLayout()
        check(lib.obh_sensor_layout(self._h, C.byref(L)))
        return L

    @property
    def lidar_packet_size(self):
        return self.layout.packet_size

    def fields(self):
        """[(name, ty_tag, offset, mask, shift, num_elements, value_mask)] in PacketFormat order."""
        out = []
        for i in range(lib.obh_sensor_n_fields(self._h)):
            name = C.create_string_buffer(32)
            tag, sh, nel = C.c_int32(), C.c_int32(), C.c_int32()
            off, mask, vm = u64(), u64(), u64()
            check(lib.obh_sensor_field(self._h, i, name, 32, C.byref(tag), C.byref(off), C.byref(mask),
                                       C.byref(sh), C.byref(nel), C.byref(vm)))
            out.append((name.value.decode(), tag.value, off.value, mask.value, sh.value, nel.value, vm.value))
        return out

    def block_parsable(self):
        return lib.obh_sensor_block_parsable(self._h)

    def frame_id_difference(self, cur, other):
        return lib.obh_sensor_frame_id_difference(self._h, cur, other)

    def _pad(self, buf):
        b = np.frombuffer(bytes(buf), np.uint8) if not isinstance(buf, np.ndarray) else buf
        return np.concatenate([b, np.zeros(8, np.uint8)])

    def frame_id(self, packet):
        p = self._pad(packet)
        return lib.obh_sensor_packet_frame_id(self._h, p.ctypes.data)

    def packet_init_id(self, packet):
        p = self._pad(packet)
        return lib.obh_sensor_packet_init_id(self._h, p.ctypes.data)

    def packet_prod_sn(self, packet):
        p = self._pad(packet)
        return lib.obh_sensor_packet_prod_sn(self._h, p.ctypes.data)

    def calculate_crc(self, packet):
        p = np.ascontiguousarray(packet)
        return lib.obh_sensor_calculate_crc(self._h, p.ctypes.data, p.size)


class LidarFrame(_Handle):
    """LidarFrame / LidarScan: named row-major fields + per-column / per-packet headers (host)."""
    _release = "obh_frame_destroy"

    def __init__(self, info, _borrowed=None):
        if _borrowed is None:
            hd = vp()
            check(lib.obh_frame_create(info._h, C.byref(hd)))
            self._owned = True
        else:  # view of a frame owned by a FramePipeline slot
            hd = vp(_borrowed)
            self._owned = False
        self._h, self.info = hd, info
        self.sensor_info = info   # None for a frame selected without update_metadata (frame_ops)
        ts, mid, st, pts, af = vp(), vp(), vp(), vp(), vp()
        w, h, npk = sz(), sz(), sz()
        check(lib.obh_frame_headers(hd, C.byref(ts), C.byref(mid), C.byref(st), C.byref(pts), C.byref(af),
                                    C.byref(w), C.byref(h), C.byref(npk)))
        self.w, self.h, self.n_packets = w.value, h.value, npk.value
        self.timestamp = _as_array(ts.value, np.uint64, (self.w,))
        self.measurement_id = _as_array(mid.value, np.uint16, (self.w,))
        self.status = _as_array(st.value, np.uint32, (self.w,))
        self.packet_timestamp = _as_array(pts.value, np.uint64, (self.n_packets,))
        self.alert_flags = _as_array(af.value, np.uint8, (self.n_packets,))
        b2w = vp()
        check(lib.obh_frame_body_to_world(hd, C.byref(b2w)))
        self.body_to_world = _as_array(b2w.value, np.float64, (self.w, 4, 4))   # identity on construction
        self.pose = self.body_to_world                                           # deprecated spelling

    def get_first_valid_column(self):
        a, b = i32(0), i32(0)
        if not lib.obh_frame_valid_columns(self._h, C.byref(a), C.byref(b)):
            raise RuntimeError("No valid columns in LidarFrame")
        return a.value

    def get_last_valid_column(self):
        a, b = i32(0), i32(0)
        if not lib.obh_frame_valid_columns(self._h, C.byref(a), C.byref(b)):
            raise RuntimeError("No valid columns in LidarFrame")
        return b.value

    def add_field(self, name, dtype, extra_dim=1, tag=None, field_class=1):
        """`tag`: a ChanFieldType tag for types numpy does not name (12: FLOAT16, stored as uint16 bits);
        `field_class`: a FieldClass (1 PIXEL_FIELD, 2 COLUMN_FIELD, 3 PACKET_FIELD, 4 FRAME_FIELD)."""
        check(lib.obh_frame_add_field_class(self._h, name.encode(),
                                            NP_TAG[np.dtype(dtype)] if tag is None else int(tag), extra_dim,
                                            int(field_class)))

    def del_field(self, name):
        """LidarFrame::del_field: drops the field (ValueError when the frame has none of that name)."""
        check(lib.obh_frame_del_field(self._h, name.encode()))

    def field_class(self, name):
        """FieldClass of a field (1 PIXEL_FIELD, 2 COLUMN_FIELD, 3 PACKET_FIELD, 4 FRAME_FIELD)."""
        return self._shape(name)[0]

    def _shape(self, name):
        cls, nd, shp = C.c_int32(), sz(), (sz * 8)()
        check(lib.obh_frame_field_shape(self._h, name.encode(), C.byref(cls), C.byref(nd), shp))
        return cls.value, tuple(shp[i] for i in range(min(nd.value, 8)))

    def field_tag(self, name):
        """ChanFieldType tag of a field."""
        tag = C.c_int32()
        check(lib.obh_frame_field(self._h, name.encode(), C.byref(tag), None, None))
        return tag.value

    @property
    def fields(self):
        out = []
        for i in range(lib.obh_frame_n_fields(self._h)):
            name = C.create_string_buffer(32)
            check(lib.obh_frame_field_at(self._h, i, name, 32, None, None, None))
            out.append(name.value.decode())
        return out

    def has_field(self, name):
        return name in self.fields

    def field(self, name):
        tag, eb, data = C.c_int32(), sz(), vp()
        check(lib.obh_frame_field(self._h, name.encode(), C.byref(tag), C.byref(eb), C.byref(data)))
        dt = np.dtype(TAG_NP.get(tag.value, np.uint8))
        return _as_array(data.value, dt, self._shape(name)[1])

    @property
    def frame_id(self):
        return lib.obh_frame_get_frame_id(self._h)

    @frame_id.setter
    def frame_id(self, v):
        lib.obh_frame_set_frame_id(self._h, v)

    @property
    def frame_status(self):
        return lib.obh_frame_get_status(self._h, None, None)

    def status_tuple(self):
        a, b = C.c_uint8(), C.c_uint8()
        s = lib.obh_frame_get_status(self._h, C.byref(a), C.byref(b))
        return s, a.value, b.value

    def set_status(self, frame_status, shutdown_countdown=0, shot_limiting_countdown=0):
        lib.obh_frame_set_status(self._h, frame_status, shutdown_countdown, shot_limiting_countdown)


def frame_to_packets(frame, info, init_id=0, prod_sn=0, device=False):
    """impl::frame_to_packets -> (packets uint8 [n, size], host_ts uint64 [n]).  device=True: the
    GPU encoder (K4: set_block of every field + CRC64 in one launch), byte-identical output."""
    psz = info.lidar_packet_size
    out = np.zeros((frame.n_packets, psz), np.uint8)
    ts = np.zeros(frame.n_packets, np.uint64)
    n = sz()
    fn = lib.obh_frame_to_packets_device if device else lib.obh_frame_to_packets
    check(fn(frame._h, info._h, init_id, prod_sn, out.ctypes.data, ts.ctypes.data, C.byref(n)))
    return out[:n.value].copy(), ts[:n.value].copy()


class PcapLidarSource(_Handle):
    """Capture file -> page-locked ring of lidar packets (include/ouster/core/pcap_source.h; replaces the
    read loop of ouster_pcap/src/pcap_packet_source.cpp for this path).  `next_burst` returns numpy VIEWS of
    the ring ([n, packet_size] uint8 with the ring's stride, [n] uint64 capture timestamps in ns), valid
    until the next call -- feed them to FrameBatcher.batch_burst / FramePipeline.push_burst as they are."""
    _release = "obh_pcap_close"

    def __init__(self, path, lidar_packet_size, dst_port=0, ring_packets=256):
        hd = vp()
        check(lib.obh_pcap_open(str(path).encode(), int(lidar_packet_size), int(dst_port), int(ring_packets),
                                C.byref(hd)))
        self._h, self.packet_size = hd, int(lidar_packet_size)

    def next_burst(self, max_packets):
        pk, ts, stride, n = vp(), vp(), sz(), sz()
        check(lib.obh_pcap_next_burst(self._h, int(max_packets), C.byref(pk), C.byref(stride), C.byref(ts),
                                      C.byref(n)))
        if n.value == 0:
            return np.zeros((0, self.packet_size), np.uint8), np.zeros(0, np.uint64)
        raw = np.ctypeslib.as_array(C.cast(pk, C.POINTER(C.c_uint8)), shape=(n.value * stride.value,))
        packets = np.lib.stride_tricks.as_strided(raw, shape=(n.value, self.packet_size),
                                                  strides=(stride.value, 1), writeable=False)
        tsv = np.ctypeslib.as_array(C.cast(ts, C.POINTER(C.c_uint64)), shape=(n.value,))
        return packets, tsv

    def __iter__(self):
        while True:
            p, t = self.next_burst(64)
            if len(t) == 0:
                return
            yield p, t

    @property
    def packets_read(self):
        return lib.obh_pcap_packets_read(self._h)

    @property
    def skipped(self):
        return lib.obh_pcap_skipped(self._h)

    def close(self):
        if self._h:
            lib.obh_pcap_close(self._h)
            self._h = None


class FrameBatcher(_Handle):
    """FrameBatcher / ScanBatcher: host state machine + one fused GPU decode per frame."""
    _release = "obh_batcher_destroy"

    def __init__(self, info):
        hd = vp()
        check(lib.obh_batcher_create(info._h, C.byref(hd)))
        self._h, self.info = hd, info
        self._lut = None

    def batch(self, packet, host_timestamp, frame):
        b = packet if isinstance(packet, np.ndarray) else np.frombuffer(bytes(packet), np.uint8)
        done = i32(0)
        check(lib.obh_batcher_batch(self._h, b.ctypes.data, b.size, int(host_timestamp), frame._h,
                                    C.byref(done)))
        return bool(done.value)

    __call__ = batch

    def batch_burst(self, packets, host_timestamps, frame):
        """Feed a [n, packet_size] uint8 burst; returns (packets consumed, frame complete)."""
        ts = np.ascontiguousarray(host_timestamps, np.uint64)
        n, stride = packets.shape[0], packets.strides[0]
        used, done = sz(0), i32(0)
        check(lib.obh_batcher_batch_burst(self._h, packets.ctypes.data, n, stride, packets.shape[1],
                                          ts.ctypes.data, frame._h, C.byref(used), C.byref(done)))
        return used.value, bool(done.value)

    def flush(self, frame):
        check(lib.obh_batcher_flush(self._h, frame._h))

    def reset(self):
        check(lib.obh_batcher_reset(self._h))

    @property
    def batched_packets(self):
        return lib.obh_batcher_batched_packets(self._h)

    @property
    def dropped_packets(self):
        return lib.obh_batcher_dropped_packets(self._h)

    @property
    def gpu_launches(self):
        return lib.obh_batcher_gpu_launches(self._h)

    def set_max_cache_size(self, n):
        check(lib.obh_batcher_set_max_cache_size(self._h, n))

    def set_headers_only(self, on=True):
        check(lib.obh_batcher_set_headers_only(self._h, int(on)))

    def set_fused_cloud(self, lut, pixel_shift_by_row=None):
        self._lut = lut
        sh, n = None, 0
        if pixel_shift_by_row is not None:
            sh = np.ascontiguousarray(pixel_shift_by_row, np.int32)
            n = sh.size
        check(lib.obh_batcher_set_fused(self._h, lut._h if lut is not None else None,
                                        sh.ctypes.data if sh is not None else None, n))

    def set_device_outputs(self, fields=None, xyz=None, range_destaggered=None):
        """FrameBatcher::set_device_outputs: `fields` maps a field name to a CUDA tensor / device
        pointer holder (h x w of the field's dtype); xyz / range_destaggered are per-return lists of
        CUDA tensors (need set_fused_cloud).  The decode then writes there instead of the host frame,
        so the results stay in HBM.  Call with no arguments to detach.  Tensors are kept alive here."""
        from .core import _ptr
        self._dev_keep = (fields, xyz, range_destaggered)
        if not fields and not xyz and not range_destaggered:
            check(lib.obh_batcher_set_device_outputs(self._h, 0, None, None, None, None))
            return
        names = list((fields or {}).keys())
        c_names = (C.c_char_p * max(len(names), 1))(*[n.encode() for n in names])
        c_ptrs = (vp * max(len(names), 1))(*[_ptr(fields[n]) for n in names])

        def two(lst):
            if not lst:
                return None
            a = (vp * 2)()
            for r, t in enumerate(lst[:2]):
                a[r] = _ptr(t) if t is not None else None
            return a
        check(lib.obh_batcher_set_device_outputs(self._h, len(names), c_names, c_ptrs, two(xyz),
                                                 two(range_destaggered)))

    def set_pipeline_depth(self, n):
        """n >= 2: batch() returns True once the frame's GPU pass is submitted; wait(frame) before
        reading pixel fields (FrameBatcher::set_pipeline_depth, lidar_frame.h)."""
        check(lib.obh_batcher_set_pipeline_depth(self._h, int(n)))

    def wait(self, frame=None):
        check(lib.obh_batcher_wait(self._h, frame._h if frame is not None else None))

    def fused_outputs(self, ret):
        xyz, nb, rd = vp(), sz(), vp()
        check(lib.obh_batcher_fused_outputs(self._h, ret, C.byref(xyz), C.byref(nb), C.byref(rd)))
        dt = self._lut.dtype
        n = nb.value // dt.itemsize
        pts = _as_array(xyz.value, dt, (n // 3, 3)) if n else None
        h, w = self.info.h, self.info.w
        rdd = _as_array(rd.value, np.uint32, (h, w)) if rd.value else None
        return pts, rdd


class FinishedSlot:
    """A finished FramePipeline slot: .frame (LidarFrame view), .xyz[r], .range_destaggered[r].
    Valid until the pipeline returns its next slot; the views are built on first access."""

    def __init__(self, info, slot, dtype):
        self._info, self._dtype = info, np.dtype(dtype)
        self._frame_h, self._xyz_p = slot.frame, (slot.xyz[0], slot.xyz[1])
        self._rd_p, self._nb = (slot.range_destaggered[0], slot.range_destaggered[1]), slot.xyz_bytes
        self._frame = self._xyz = self._rd = None

    @property
    def frame(self):
        if self._frame is None:
            self._frame = LidarFrame(self._info, _borrowed=self._frame_h)
        return self._frame

    @property
    def xyz(self):
        if self._xyz is None:
            n = self._nb // self._dtype.itemsize
            self._xyz = [(_as_array(p, self._dtype, (n // 3, 3)) if p else None) for p in self._xyz_p]
        return self._xyz

    @property
    def range_destaggered(self):
        if self._rd is None:
            hw = (self._info.h, self._info.w)
            self._rd = [(_as_array(p, np.uint32, hw) if p else None) for p in self._rd_p]
        return self._rd


class FramePipeline(_Handle):
    """Ring of LidarFrames with `depth` frames in flight on the GPU (frame_pipeline.h): the host
    state machine of frame k+1 overlaps the H2D / fused kernel / D2H of frame k."""
    _release = "obh_pipeline_destroy"

    def __init__(self, info, depth=3, lut=None, pixel_shift_by_row=None):
        sh, n = None, 0
        if pixel_shift_by_row is not None:
            sh = np.ascontiguousarray(pixel_shift_by_row, np.int32)
            n = sh.size
        hd = vp()
        check(lib.obh_pipeline_create(info._h, int(depth), lut._h if lut is not None else None,
                                      sh.ctypes.data if sh is not None else None, n, C.byref(hd)))
        self._h, self.info, self._lut = hd, info, lut
        self._dtype = lut.dtype if lut is not None else np.float32

    def _wrap(self, slot):
        return FinishedSlot(self.info, slot, self._dtype) if slot.frame else None

    def push_burst(self, packets, host_timestamps):
        """Feed a [n, packet_size] uint8 burst; returns (packets consumed, FinishedSlot or None)."""
        ts = np.ascontiguousarray(host_timestamps, np.uint64)
        used, slot = sz(0), Slot()
        check(lib.obh_pipeline_push_burst(self._h, packets.ctypes.data, packets.shape[0], packets.strides[0],
                                          packets.shape[1], ts.ctypes.data, C.byref(used), C.byref(slot)))
        return used.value, self._wrap(slot)

    def drain(self):
        """Oldest frame still in flight (waited for), or None."""
        slot = Slot()
        check(lib.obh_pipeline_drain(self._h, C.byref(slot)))
        return self._wrap(slot)

    @property
    def in_flight(self):
        return lib.obh_pipeline_in_flight(self._h)

    def stats(self):
        """Cumulative host-thread time by phase (FrameBatcher::Stats), seconds."""
        a = np.zeros(5, np.uint64)
        check(lib.obh_pipeline_stats(self._h, a.ctypes.data))
        return {"burst_s": a[0] * 1e-9, "upload_wait_s": a[1] * 1e-9, "submit_s": a[2] * 1e-9,
                "wait_s": a[3] * 1e-9, "frames": int(a[4])}

    @property
    def gpu_launches(self):
        return lib.obh_pipeline_gpu_launches(self._h)

    @property
    def dropped_packets(self):
        return lib.obh_pipeline_dropped_packets(self._h)


LidarScan = LidarFrame
ScanBatcher = FrameBatcher
