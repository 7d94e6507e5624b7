"""Synthetic point-cloud pairs with a known relative pose, for the align_clouds tests.

Each scene of tests/ground_scenes.py is ray-cast twice: once from the target sensor (at the origin) and once from
the source sensor, moved by a known pose (yaw, translation and a Z offset).  Both clouds are returned in their own
sensor's frame, so `truth` maps source points onto the target ones.  The two scans sample the surfaces at different
places, as two real scans would.  Normals are the exact normals of the surface each ray hit.
"""
import numpy as np

from tests import ground_scenes as gs


def _room():
    # an 18 m x 14 m room with a ceiling; a pillar and a cabinet break its 180 degree symmetry
    walls = [(9.0, 9.3, -7.3, 7.3, 0.0, 3.0), (-9.3, -9.0, -7.3, 7.3, 0.0, 3.0),
             (-9.3, 9.3, 7.0, 7.3, 0.0, 3.0), (-9.3, 9.3, -7.3, -7.0, 0.0, 3.0)]
    inner = [(3.0, 3.6, 2.0, 2.6, 0.0, 3.0), (-8.9, -7.9, -6.9, -3.0, 0.0, 1.8), (-2.0, -1.8, 1.0, 7.0, 0.0, 3.0),
             (5.0, 8.9, -3.2, -3.0, 0.0, 3.0)]
    return gs.Scene(gs.flat, boxes=walls + inner,
                    ceiling=3.0, max_range=24.0, fov=(45.0, -45.0))


def _box_island():
    return gs.Scene(gs.flat, boxes=[(10.0, 12.0, 2.0, 4.0, 0.0, 1.0), (-12.0, -6.0, 6.0, 11.0, 0.0, 3.0),
                                    (4.0, 5.0, -9.0, -6.0, 0.0, 2.0)], max_range=20.0, fov=(15.0, -25.0))


def _wall():
    return gs.Scene(gs.flat, boxes=[(14.0, 14.4, -15.0, 15.0, 0.0, 3.0), (5.0, 6.0, 6.0, 7.0, 0.0, 2.5),
                                    (-4.0, -3.0, -7.0, -6.0, 0.0, 1.5), (8.0, 14.0, -9.0, -8.5, 0.0, 2.0),
                                    (-9.0, -8.0, 4.0, 10.0, 0.0, 2.0)], max_range=24.0, fov=(15.0, -25.0))


def _open():
    boxes = [(30.0, 34.0, -5.0, 6.0, 0.0, 4.0), (-36.0, -31.0, 8.0, 20.0, 0.0, 6.0), (12.0, 14.0, 25.0, 40.0, 0.0, 3.0),
             (-8.0, 4.0, -35.0, -32.0, 0.0, 5.0), (6.0, 7.0, 4.0, 5.0, 0.0, 2.0), (-15.0, -13.0, -12.0, -9.0, 0.0, 2.5)]
    return gs.Scene(gs.flat, boxes=boxes, max_range=55.0, fov=(10.0, -15.0))


SCENES = {"room": _room, "box_island": _box_island, "wall": _wall, "open": _open}


def pose(yaw_deg, t=(0.0, 0.0, 0.0)):
    p = np.eye(4)
    c, s = np.cos(np.radians(yaw_deg)), np.sin(np.radians(yaw_deg))
    p[:2, :2] = [[c, -s], [s, c]]
    p[:3, 3] = t
    return p


def _normals(scene, p, label, origin):
    """Exact surface normal (unit, facing the sensor) at each hit point."""
    n = np.zeros_like(p)
    n[..., 2] = 1.0
    obj = label == 2
    if scene.ceiling is not None:
        n[obj & (np.abs(p[..., 2] - scene.ceiling) < 1e-2)] = (0.0, 0.0, -1.0)
    best = np.full(p.shape[:-1], np.inf)
    for x0, x1, y0, y1, z0, z1 in scene.boxes:
        lo, hi = np.array([x0, y0, z0]), np.array([x1, y1, z1])
        d_lo, d_hi = np.abs(p - lo), np.abs(p - hi)
        inside = np.all((p >= lo - 1e-2) & (p <= hi + 1e-2), axis=-1) & obj
        face = np.minimum(d_lo, d_hi)
        axis = np.argmin(face, axis=-1)
        dist = np.take_along_axis(face, axis[..., None], -1)[..., 0]
        take = inside & (dist < best)
        e = np.zeros_like(p)
        np.put_along_axis(e, axis[..., None], 1.0, -1)
        n = np.where(take[..., None], e, n)
        best = np.where(take, dist, best)
    flip = np.sum(n * (origin - p), -1) < 0
    return np.where(flip[..., None], -n, n)


def scan(name, sensor_pose=None, h=32, w=512, seed=0, noise=0.0):
    """One scan from `sensor_pose` (4x4; the sensor's pose relative to the target sensor): (points, normals) in the
    scanning sensor's frame, no-return rows dropped."""
    scene = SCENES[name]()
    sp = np.eye(4) if sensor_pose is None else np.asarray(sensor_pose, np.float64)
    world = sp.copy()
    world[2, 3] += scene.sensor_z                      # the sensor's pose in the scene
    d = gs.beams(h, w, scene.fov, seed=seed) @ world[:3, :3].T
    t, label = scene.cast(d, world[:3, 3])
    ok = np.isfinite(t) & (label > 0)
    p = world[:3, 3] + np.round(np.where(ok, t, 0.0) * 1000.0)[..., None] * 0.001 * d
    n = _normals(scene, p, label, world[:3, 3])
    p, n = p[ok], n[ok]
    if noise:
        p = p + np.random.default_rng(seed + 7).normal(0.0, noise, p.shape)
    inv = np.linalg.inv(world)
    return p @ inv[:3, :3].T + inv[:3, 3], n @ inv[:3, :3].T


def pair(name, truth, h=32, w=512, seed=0, noise=0.0):
    """(source, source normals, target, target normals): the target scanned at the origin, the source from `truth`
    (so truth @ source ~ target)."""
    tp, tn = scan(name, None, h, w, seed, noise)
    sp, sn = scan(name, truth, h, w, seed + 1, noise)
    return sp, sn, tp, tn


def pose_error(p, truth):
    """(translation error m, rotation error deg) of 4x4 p against truth."""
    d = np.linalg.inv(truth) @ p
    ang = np.degrees(np.arccos(np.clip((np.trace(d[:3, :3]) - 1.0) / 2.0, -1.0, 1.0)))
    return float(np.linalg.norm(d[:3, 3])), float(ang)
