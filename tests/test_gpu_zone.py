"""GPU tests of zone monitoring (ouster-sdk_b200/csrc/ob_zone.cu): Zone::render bit for bit against the CPU oracle
(oracle/orc_zone.c) on the same LUT, the per-frame occupancy equal to a numpy restatement of EmulatedZoneMon, the
reference's known answers through pyapi, a device chain from packets, and replay from a CUDA graph."""
import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import zone as oz
from tests.test_oracle_zone import ZDIR, s2b_z1, sensor_meta, stl_tris

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


def device_luts(ob, meta, s2b):
    """BeamConfig's LUTs as the package builds them (float64, on the GPU), and their host copies for the oracle"""
    cfg = ob.pyapi.BeamConfig.from_sensor_info(meta, s2b)
    host = lambda lut: None if lut is None else (lut.direction.copy(), lut.offset.copy())
    return cfg, host(cfg.lut), host(cfg.lut_no_sensor_to_body_transform)


def render_both(ob, meta, zones, s2b):
    """GPU render of `zones` (list of (triangles, frame)) in one launch and the oracle's, zone by zone"""
    cfg, body, sensor = device_luts(ob, meta, s2b)
    h, w = meta["h"], meta["w"]
    specs = [{"triangles": t, "coordinate_frame": f} for t, f in zones]
    near, far, px = ob.zone_render(specs, h, w, cfg.lut_no_sensor_to_body_transform, cfg.lut, device_out=False)
    for k, (t, f) in enumerate(zones):
        d, o = body if f == 1 else sensor
        rn, rf, rpx = oz.render(t, d, o, h, w)
        assert np.array_equal(near[k], rn), k
        assert np.array_equal(far[k], rf), k
        assert px[k] == rpx, k
    return near, far, px


def test_render_fixtures_both_frames(ob):
    for name, s2b in (("785.json", s2b_z1()), ("OS-0-128_v3.0.1_1024x10.2.json", np.eye(4))):
        meta = sensor_meta(name)
        zones = [(stl_tris(f"{i}.stl"), f) for i in (0, 1) for f in (1, 2)]
        render_both(ob, meta, zones, s2b)


def subsample(meta, h, w):
    m = dict(meta)
    idx = np.linspace(0, meta["h"] - 1, h).astype(int)
    m["beam_altitude_angles"] = list(np.asarray(meta["beam_altitude_angles"])[idx])
    m["beam_azimuth_angles"] = list(np.asarray(meta["beam_azimuth_angles"])[idx])
    m["h"], m["w"] = h, w
    return m


@pytest.mark.parametrize("h", [32, 64, 128])
@pytest.mark.parametrize("w", [512, 1024, 2048])
def test_render_shapes(ob, h, w):
    meta = subsample(sensor_meta("785.json"), h, w)
    render_both(ob, meta, [(stl_tris("0.stl"), 1), (stl_tris("1.stl"), 2)], s2b_z1())


def grid_mesh(n_side, z0, seed):
    """a closed-ish height field of 2 * n_side^2 triangles sharing edges, 1-3 m in front of the sensor"""
    rs = np.random.default_rng(seed)
    xs = np.linspace(-2, 2, n_side + 1, dtype=np.float32)
    ys = np.linspace(-2, 2, n_side + 1, dtype=np.float32)
    zz = (z0 + 0.3 * rs.random((n_side + 1, n_side + 1))).astype(np.float32)
    tris = []
    for i in range(n_side):
        for j in range(n_side):
            a = (xs[i], ys[j], zz[i, j])
            b = (xs[i + 1], ys[j], zz[i + 1, j])
            c = (xs[i], ys[j + 1], zz[i, j + 1])
            d = (xs[i + 1], ys[j + 1], zz[i + 1, j + 1])
            tris += [a + b + c, b + d + c]
    return np.array(tris, np.float32)


def synthetic_zones():
    """16 zones: full 2048-triangle shared-edge meshes in several orientations, degenerate and NaN triangles,
    meshes behind the sensor, triangles parallel to rays, and walls seen from inside the bounding sphere"""
    zones = []
    base = grid_mesh(32, 1.5, 0)  # 2048 triangles
    assert len(base) == 2048
    for k in range(6):  # rotate the height field to face each axis direction
        t = base.reshape(-1, 3, 3).copy()
        t = np.roll(t, k % 3, axis=2)
        if k >= 3:
            t = -t
        zones.append((t.reshape(-1, 9), 1 + (k % 2)))
    degen = base[:300].copy()
    degen[::3, 3:6] = degen[::3, 0:3]          # zero-area triangles
    zones.append((degen, 2))
    behind = base.copy()
    behind.reshape(-1, 3, 3)[..., 2] *= -1     # the same mesh below the sensor's xy plane
    zones.append((behind, 2))
    par = np.array([[0, 0, 0, 5, 0, 0, 0, 5, 0], [0, 0, 0, 0, 5, 0, 0, 0, 5], [0, 0, 0, 5, 0, 0, 0, 0, 5]],
                   np.float32)                 # planes through the sensor origin: rays lie in them
    zones.append((np.concatenate([par, par + np.float32(1e-7)]), 2))
    box = []
    for ax in range(3):
        for s in (-1, 1):
            q = grid_mesh(4, 0, ax).reshape(-1, 3, 3)
            q[..., 2] = 3 * s
            box.append(np.roll(q, ax, axis=2).reshape(-1, 9))
    zones.append((np.concatenate(box), 2))     # a box around the sensor: every ray exits through one wall
    zones.append((grid_mesh(20, 0.5, 3), 1))
    zones.append((grid_mesh(8, 10.0, 4), 2))
    zones.append((base[:1], 1))                # a single triangle: (0, t) hits
    zones.append((np.concatenate([base[:512], base[:512]]), 2))  # every triangle twice: t == t ties
    zones.append((grid_mesh(32, 2.5, 5), 1))
    nan_mesh = degen.copy()
    nan_mesh[1::7, 4] = np.nan                 # NaN vertices: the bounding sphere is NaN, so every ray misses
    zones.append((nan_mesh, 2))
    assert len(zones) == 16
    return zones


def test_render_16_zones_one_launch(ob):
    meta = subsample(sensor_meta("785.json"), 64, 512)
    before = ob.kernel_launch_count("zone")
    near, far, px = render_both(ob, meta, synthetic_zones(), s2b_z1())
    assert ob.kernel_launch_count("zone") - before == 1
    assert (px > 0).sum() >= 6 and px[15] == 0
    assert np.any((near > 0) & (near == far))  # ties give (t, t)
    assert np.any((near == 0) & (far > 0))     # single hits give (0, t)


def test_render_device_outputs(ob):
    import torch
    meta = sensor_meta("785.json")
    cfg, body, _ = device_luts(ob, meta, s2b_z1())
    near, far, px = ob.zone_render([{"triangles": stl_tris("0.stl"), "coordinate_frame": 1}], meta["h"], meta["w"],
                                   cfg.lut_no_sensor_to_body_transform, cfg.lut)
    assert near.is_cuda and far.is_cuda
    rn, rf, rpx = oz.render(stl_tris("0.stl"), *body, meta["h"], meta["w"])
    assert np.array_equal(near[0].cpu().numpy().view(np.uint32), rn)
    assert np.array_equal(far[0].cpu().numpy().view(np.uint32), rf) and px[0] == rpx
    # LUT arrays as CUDA tensors work too
    t = lambda a: torch.from_numpy(a).cuda()
    n2, f2, _ = ob.zone_render([{"triangles": stl_tris("0.stl"), "coordinate_frame": 1}], meta["h"], meta["w"],
                               (t(body[0]), t(body[1])), (t(body[0]), t(body[1])))
    assert torch.equal(n2, near) and torch.equal(f2, far)


def test_render_errors(ob):
    meta = subsample(sensor_meta("785.json"), 32, 512)
    cfg, _, sensor = device_luts(ob, meta, None)
    h, w = meta["h"], meta["w"]
    run = lambda z, body=None: ob.zone_render(z, h, w, cfg.lut_no_sensor_to_body_transform, body, device_out=False)
    t0 = stl_tris("0.stl")
    with pytest.raises(ValueError, match=r"^Zone: Error rendering zone, STL has too many triangles\.$"):
        run([{"triangles": np.zeros((2049, 9), np.float32), "coordinate_frame": 2}])
    with pytest.raises(ValueError, match=r"^Zone: Error rendering zone, STL has no triangles\.$"):
        run([{"triangles": np.zeros((0, 9), np.float32), "coordinate_frame": 2}])
    with pytest.raises(ValueError, match=r"sensor_to_body_transform not set for BODY coordinate frame\.$"):
        run([{"triangles": t0, "coordinate_frame": 1}])
    with pytest.raises(ValueError, match=r"^Zone: point_count must be in \[1, 262143\]$"):
        run([{"triangles": t0, "coordinate_frame": 2, "point_count": 0}])
    _, _, px = run([{"triangles": t0, "coordinate_frame": 2}])
    assert px[0] > 0
    with pytest.raises(RuntimeError, match=rf"Zone: area of rendered zone \({px[0]}\) is smaller than point_count "
                                           rf"\({px[0] + 1}\) specified in zone\.$"):
        run([{"triangles": t0, "coordinate_frame": 2, "point_count": int(px[0]) + 1}])
    # a wall 5000 km away: t * 1000 exceeds UINT32_MAX
    wall = np.array([[-1e9, -1e9, 5e6, 1e9, -1e9, 5e6, 0, 1e9, 5e6], [-1e9, -1e9, -5e6, 1e9, -1e9, -5e6, 0, 1e9, -5e6],
                     [5e6, -1e9, -1e9, 5e6, 1e9, -1e9, 5e6, 0, 1e9]], np.float32)
    with pytest.raises(RuntimeError, match=r"Zone::render: range overflow$"):
        oz.render(wall, *sensor, h, w)
    with pytest.raises(RuntimeError, match=r"Zone::render: range overflow$"):
        run([{"triangles": wall, "coordinate_frame": 2}])


class RefZoneMon:
    """numpy restatement of EmulatedZoneMon (zone_common.py:14-136) over (id, mode, point_count, frame_count,
    near, far) zones, live in list order"""

    def __init__(self, zones):
        self.zones = zones
        self.triggers = [0] * len(zones)
        self.alerts = [0] * len(zones)
        self.max_counts = [int(np.count_nonzero(z[4] < z[5])) for z in zones]

    def calc(self, r, bitmask):
        pkt = np.zeros(16, ZSD)
        pkt["id"] = 255
        for i, (zid, mode, pc, fc, near, far) in enumerate(self.zones):
            m = np.logical_and(r > 0, np.logical_and(near <= r, r <= far))
            cnt = int(np.count_nonzero(m))
            inv = int(np.count_nonzero(np.logical_and(r == 0, near > 0)))
            occ = int(np.count_nonzero(np.logical_and(r > 0, r <= near)))
            pts = r[m]
            avg, mn, mx = (np.mean(pts), np.min(pts), np.max(pts)) if len(pts) else (0, 0, 0)
            bitmask[m] |= np.uint32(1 << i)
            if (cnt >= pc and mode == 1) or (cnt < pc and mode == 2):
                self.triggers[i] += 1
            else:
                self.triggers[i] = 0
            self.alerts[i] = self.alerts[i] + 1 if self.triggers[i] >= fc else 0
            rec = pkt[i]
            rec["live"], rec["id"], rec["count"], rec["occlusion_count"] = 1, zid, cnt, occ
            rec["invalid_count"], rec["max_count"] = inv, self.max_counts[i]
            rec["trigger_status"], rec["trigger_type"] = self.alerts[i] > 0, mode
            rec["triggered_frames"], rec["min_range"], rec["max_range"] = self.alerts[i], mn, mx
            rec["mean_range"] = avg  # float64 mean, truncated into the uint32 record
        return pkt


ZSD = None


def random_zones(h, w, n, seed):
    rs = np.random.default_rng(seed)
    zones = []
    for i in range(n):
        near = rs.integers(0, 4000, (h, w)).astype(np.uint32)
        far = (near + rs.integers(0, 3000, (h, w))).astype(np.uint32)
        hole = rs.random((h, w)) < 0.5
        near[hole] = 0
        far[hole & (rs.random((h, w)) < 0.7)] = 0
        zones.append((rs.integers(0, 128), 1 + (i % 2), int(rs.integers(1, 2 * h * w // 10)), int(rs.integers(1, 4)),
                      near, far))
    return zones


def random_range(zones, h, w, seed):
    rs = np.random.default_rng(seed)
    r = rs.integers(1, 8000, (h, w)).astype(np.uint32)
    r[rs.random((h, w)) < 0.2] = 0
    z = zones[int(rs.integers(len(zones)))]
    pick = rs.random((h, w))
    r[pick < 0.1] = z[4][pick < 0.1]           # exactly at near
    r[(pick >= 0.1) & (pick < 0.2)] = z[5][(pick >= 0.1) & (pick < 0.2)]  # exactly at far
    if seed % 3 == 0:
        r[:] = 0                                # an empty frame: VACANCY triggers, OCCUPANCY resets
    return r


@pytest.mark.parametrize("dev", [False, True])
def test_occupancy_equals_numpy_restatement(ob, dev):
    import torch
    global ZSD
    ZSD = ob.core.ZONE_STATE_DTYPE
    h, w = 64, 1024
    zones = random_zones(h, w, 16, 1)
    live = [{"id": z[0], "mode": z[1], "point_count": z[2], "frame_count": z[3], "near_mm": z[4], "far_mm": z[5]}
            for z in zones]
    mon = ob.ZoneMonitor(live, h, w)
    ref = RefZoneMon(zones)
    for f in range(12):
        r = random_range(zones, h, w, f)
        bm_ref = np.zeros((h, w), np.uint32)
        bm_ref[0, :7] = 1 << 31             # bits already set are kept
        want = ref.calc(r, bm_ref)
        if dev:
            bm = torch.zeros((h, w), dtype=torch.int32, device="cuda")
            bm[0, :7] = -(1 << 31)
            mon.update(torch.from_numpy(r.view(np.int32)).cuda(), bm)
            st = mon.states(device=True).cpu().numpy().view(ZSD).reshape(16)
            bm = bm.cpu().numpy().view(np.uint32)
        else:
            bm = np.zeros((h, w), np.uint32)
            bm[0, :7] = 1 << 31
            mon.update(r, bm)
            st = mon.states()
        assert np.array_equal(st, want), f
        assert np.array_equal(bm, bm_ref), f
    trig, alerts, sums = mon.counters()
    assert trig == ref.triggers and alerts == ref.alerts
    assert sums == [int(r[(r > 0) & (z[4] <= r) & (r <= z[5])].astype(np.uint64).sum()) for z in zones]


def test_occupancy_sequences(ob):
    """OCCUPANCY and VACANCY over frame_count sequences: triggers count consecutive frames, alerts start at
    frame_count and reset with the triggers"""
    global ZSD
    ZSD = ob.core.ZONE_STATE_DTYPE
    h, w = 32, 512
    near = np.full((h, w), 1000, np.uint32)
    far = np.full((h, w), 2000, np.uint32)
    zones = [(3, 1, 100, 3, near, far), (4, 2, 100, 2, near, far)]
    mon = ob.ZoneMonitor([{"id": z[0], "mode": z[1], "point_count": z[2], "frame_count": z[3], "near_mm": z[4],
                           "far_mm": z[5]} for z in zones], h, w)
    ref = RefZoneMon(zones)
    for k, n_in in enumerate([200, 200, 200, 200, 0, 200, 200, 200, 50, 50, 50]):
        r = np.full((h, w), 5000, np.uint32)
        r.reshape(-1)[:n_in] = 1500
        want = ref.calc(r, np.zeros((h, w), np.uint32))
        mon.update(r)
        assert np.array_equal(mon.states(), want), k
    assert ref.alerts == [0, 2]


def make_zone_set(ob, meta_name, s2b, stls, live, frame_counts=None, frame=1):
    api = ob.pyapi
    zs = api.ZoneSet()
    zs.sensor_to_body_transform = s2b
    zs.power_on_live_ids = live
    for i, name in enumerate(stls):
        z = api.Zone()
        z.point_count, z.frame_count = 1, (frame_counts or {}).get(i, 1)
        z.mode = api.ZoneMode.OCCUPANCY
        z.stl = api.Stl(f"{ZDIR}/{name}")
        z.stl.coordinate_frame = api.CoordinateFrame(frame)
        zs.zones[i] = z
    zs.render(sensor_meta(meta_name))
    return zs


def test_known_answers_through_pyapi(ob):
    api = ob.pyapi
    zs = make_zone_set(ob, "785.json", s2b_z1(), ["0.stl", "1.stl"], [0, 1], {1: 4})
    ezm = api.EmulatedZoneMon(zs)
    assert ezm.max_counts == {0: 12096, 1: 3098}
    assert ezm.zone_counts == {} and ezm.zone_triggers == [0] * 128 and ezm.triggered_zone_ids == []
    assert ezm.live_zones == [0, 1] and ezm.update_count == 0 and not ezm.debug
    assert zs.zones[0].zrb.near_range_mm.shape == (128, 1024)

    zs = make_zone_set(ob, "OS-0-128_v3.0.1_1024x10.2.json", np.eye(4), ["0.stl"], [0])
    ezm = api.EmulatedZoneMon(zs)
    rng = np.full((128, 1024), 1000, np.uint32)
    bm = np.zeros((128, 1024), np.uint32)
    ezm.calc_triggers(rng, bm)
    p = ezm.get_packet()
    assert p[0]["id"] == 0 and p[0]["live"] == 1 and p[0]["count"] == 1218
    assert p[0]["min_range"] == p[0]["max_range"] == p[0]["mean_range"] == 1000
    assert p[0]["trigger_status"] == 1 and p[0]["triggered_frames"] == 1
    assert all(p[k]["id"] == 255 for k in range(1, 16))
    assert np.count_nonzero(bm) == 1218 and ezm.triggered_zone_ids == [0]
    assert ezm.zone_counts == {0: 1218} and ezm.zone_avgs == {0: 1000.0}
    assert ezm.zone_mins == {0: 1000} and ezm.zone_maxes == {0: 1000}


def test_zone_avgs_is_the_float_mean(ob):
    """zone_avgs is np.mean of the triggering ranges (float64), the record's mean_range its truncation"""
    api = ob.pyapi
    zs = api.ZoneSet()
    z = api.Zone()
    z.point_count, z.frame_count, z.mode = 1, 1, api.ZoneMode.OCCUPANCY
    z.zrb = api.Zrb(np.full((8, 16), 100, np.uint32), np.full((8, 16), 5000, np.uint32))
    zs.zones, zs.power_on_live_ids = {0: z}, [0]
    rs = np.random.default_rng(3)
    r = rs.integers(0, 6000, (8, 16)).astype(np.uint32)
    ezm = api.EmulatedZoneMon(zs)
    ezm.calc_triggers(r, np.zeros((8, 16), np.uint32))
    pts = r[(r > 0) & (100 <= r) & (r <= 5000)]
    assert ezm.zone_avgs == {0: np.mean(pts)} and ezm.get_packet()[0]["mean_range"] == int(np.mean(pts))
    assert ezm.zone_avgs[0] != int(ezm.zone_avgs[0])


def test_bitmask_must_be_contiguous_int32(ob):
    import torch
    near, far = np.zeros((4, 8), np.uint32), np.full((4, 8), 10, np.uint32)
    mon = ob.ZoneMonitor([{"id": 0, "mode": 1, "point_count": 1, "frame_count": 1, "near_mm": near, "far_mm": far}],
                         4, 8)
    r = torch.full((4, 8), 5, dtype=torch.int32, device="cuda")
    for bad in (torch.zeros((4, 8), dtype=torch.float32, device="cuda"),
                torch.zeros((8, 4), dtype=torch.int32, device="cuda").t(),
                torch.zeros((4, 16), dtype=torch.int32, device="cuda")[:, ::2],
                np.zeros((4, 8), np.float32), np.zeros((8, 4), np.uint32).T):
        with pytest.raises(ValueError, match="bitmask must be a contiguous"):
            mon.update(r, bad)
    ok = torch.zeros((4, 8), dtype=torch.int32, device="cuda")
    mon.update(r, ok)
    assert int(ok.sum()) == 32


def test_zone_set_errors(ob):
    api = ob.pyapi
    with pytest.raises(RuntimeError, match=r"^ZoneSet::render: zone 0 was out of sensor FOV\.$"):
        make_zone_set(ob, "785.json", None, ["0.stl"], [0])   # BODY without sensor_to_body
    far = np.array([[0, 0, -500, 1, 0, -500, 0, 1, -500]], np.float32)  # straight down, 500 m: no beam reaches it
    zs = api.ZoneSet()
    z = api.Zone()
    z.point_count = z.frame_count = 1
    z.mode = api.ZoneMode.VACANCY
    z.stl = api.Stl(b"\0" * 80 + np.uint32(1).tobytes() + np.zeros(3, np.float32).tobytes() + far.tobytes() + b"\0\0")
    z.stl.coordinate_frame = api.CoordinateFrame.SENSOR
    zs.zones = {7: z}
    with pytest.raises(RuntimeError, match=r"^ZoneSet::render: zone 7 was out of sensor FOV\.$"):
        zs.render(sensor_meta("785.json"))


def test_device_chain_from_packets(ob):
    """DeviceScanBatcher's RANGE (K2, on the GPU) straight into the monitor; the second frame's update is replayed
    from a CUDA graph, which capture would refuse if it synchronised with the host; equal to the host path"""
    import torch
    from tests.helpers import load_fixture
    api = ob.pyapi
    meta, packets = load_fixture("OS-1-128_767798045_1024x10_20230712_120049")
    info = api.SensorInfo.from_meta(meta)
    zmeta = {"w": info.w, "h": info.h, "beam_to_lidar_transform": meta["beam_to_lidar_transform"],
             "lidar_to_sensor_transform": meta["lidar_to_sensor_transform"],
             "beam_azimuth_angles": meta["beam_azimuth_angles"], "beam_altitude_angles": meta["beam_altitude_angles"]}
    zs = api.ZoneSet()
    zs.sensor_to_body_transform = np.eye(4)
    zs.power_on_live_ids = [0, 1]
    box = synthetic_zones()[9][0]  # the box around the sensor: every beam is inside it
    for i, t in enumerate([box, box * np.float32(2)]):
        z = api.Zone()
        z.point_count, z.frame_count, z.mode = 100, 1, api.ZoneMode(1 + i)
        z.stl = api.Stl(b"\0" * 80 + np.uint32(len(t)).tobytes() + b"".join(
            np.zeros(3, np.float32).tobytes() + row.tobytes() + b"\0\0" for row in t))
        z.stl.coordinate_frame = api.CoordinateFrame.SENSOR
        zs.zones[i] = z
    zs.render(zmeta)
    batcher = api.DeviceScanBatcher(info)
    scan = batcher.new_scan()
    done = [batcher(p, 77, scan) for p in packets]
    if not done[-1]:
        batcher.flush(scan)
    dev_mon, host_mon = api.EmulatedZoneMon(zs), api.EmulatedZoneMon(zs)
    bm_dev = torch.zeros((info.h, info.w), dtype=torch.int32, device="cuda")
    rng = scan.field("RANGE")
    assert rng.is_cuda
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        dev_mon.calc_triggers(rng, bm_dev)  # builds the monitor (allocates, uploads the zone images)
        # the next frame's update, captured: a host synchronisation inside it would fail the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            dev_mon.calc_triggers(rng, bm_dev)
    torch.cuda.current_stream().wait_stream(side)
    g.replay()
    torch.cuda.synchronize()
    bm_host = np.zeros((info.h, info.w), np.uint32)
    for _ in range(2):
        host_mon.calc_triggers(rng.cpu().numpy().view(np.uint32), bm_host)
    assert np.array_equal(dev_mon.get_packet(), host_mon.get_packet())
    assert dev_mon.zone_triggers == host_mon.zone_triggers and max(host_mon.zone_triggers) == 2
    assert np.array_equal(bm_dev.cpu().numpy().view(np.uint32), bm_host)
    assert host_mon.zone_counts[0] > 0 and np.count_nonzero(bm_host) > 0


def test_update_from_cuda_graph(ob):
    import torch
    global ZSD
    ZSD = ob.core.ZONE_STATE_DTYPE
    h, w = 128, 2048
    zones = random_zones(h, w, 16, 7)
    live = [{"id": z[0], "mode": z[1], "point_count": z[2], "frame_count": z[3], "near_mm": z[4], "far_mm": z[5]}
            for z in zones]
    frames = [random_range(zones, h, w, s) for s in range(1, 5)]
    # eager reference run
    eager = ob.ZoneMonitor(live, h, w)
    want = []
    for r in frames:
        bm = torch.zeros((h, w), dtype=torch.int32, device="cuda")
        eager.update(torch.from_numpy(r.view(np.int32)).cuda(), bm)
        want.append((eager.states(device=True).clone(), bm.clone()))
    # the same frames replayed from one captured update
    mon = ob.ZoneMonitor(live, h, w)
    r_in = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    bm = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    st_out = torch.zeros((16, 37), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        stream = ob.Stream(0, cuda_stream=s.cuda_stream)
        with torch.cuda.graph(g, stream=s):
            bm.zero_()
            mon.update(r_in, bm, stream=stream)
            ob._capi.check(ob._capi.lib.ob_zone_monitor_states(mon._h, st_out.data_ptr(), stream.h))
    torch.cuda.current_stream().wait_stream(s)
    for r, (st_want, bm_want) in zip(frames, want):
        r_in.copy_(torch.from_numpy(r.view(np.int32)))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(st_out, st_want)
        assert torch.equal(bm, bm_want)
