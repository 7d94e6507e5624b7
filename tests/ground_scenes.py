"""Synthetic lidar frames with known ground, for the ground-segmentation tests.

A sensor 1.8 m (or 4.5 m) above the origin looks at a scene made of a ground surface and a few solids.  Every pixel's range is
ray-cast exactly (rounded to the millimetre), so the surface it hit, and hence its true label, is known by
construction.  Frames come as a range image (one or two returns), a LUT (direction in metres per millimetre and a
zero offset), column status and column poses.
"""
import numpy as np

SENSOR_Z = 1.8


def beams(h, w, alt_deg=(11.0, -11.0), seed=0):
    """Unit beam directions (H, W, 3): altitudes evenly spread with a little seeded jitter, azimuths around 360°."""
    rs = np.random.default_rng(seed)
    alt = np.radians(np.linspace(alt_deg[0], alt_deg[1], h) + rs.normal(0, 0.02, h))
    az = 2 * np.pi * (np.arange(w) + 0.5) / w
    d = np.stack([np.cos(alt)[:, None] * np.cos(az)[None, :], np.cos(alt)[:, None] * np.sin(az)[None, :],
                  np.sin(alt)[:, None] * np.ones((1, w))], axis=-1)
    return d


class Scene:
    """Surfaces: ground z = g(x, y) and axis-aligned boxes [(x0, x1, y0, y1, z0, z1), ...] standing on it, plus
    optional holes in the ground [(x0, x1, y0, y1)] that return nothing, and a ceiling height.  The room is seen by
    a ±45° sensor, the outdoor scenes by a ±11° one."""

    def __init__(self, ground, boxes=(), holes=(), ceiling=None, max_range=60.0, fov=(11.0, -11.0),
                 sensor_z=SENSOR_Z):
        self.ground, self.boxes, self.holes, self.ceiling, self.max_range = ground, list(boxes), list(holes), \
            ceiling, max_range
        self.fov = fov  # altitude of the top and bottom beams, degrees
        self.sensor_z = sensor_z

    def cast(self, d, o):
        """Rays from o along unit d -> (t (..,) metres or inf, label (..,) 0 none / 1 ground / 2 object)."""
        o = np.asarray(o, np.float64)
        t_best = np.full(d.shape[:-1], np.inf)
        label = np.zeros(d.shape[:-1], np.int8)
        # ground: march to the first sign change of f(t) = o_z + t d_z - g(o_x + t d_x, o_y + t d_y), then bisect
        ts = np.linspace(0.0, self.max_range, 1201)
        f = np.stack([(o[2] + t * d[..., 2]) - self.ground(o[0] + t * d[..., 0], o[1] + t * d[..., 1]) for t in ts])
        below = f <= 0
        first = np.argmax(below, axis=0)
        crossed = below.any(axis=0) & (first > 0)
        lo = ts[np.maximum(first - 1, 0)]
        hi = ts[first]
        for _ in range(60):
            mid = 0.5 * (lo + hi)
            fm = (o[2] + mid * d[..., 2]) - self.ground(o[0] + mid * d[..., 0], o[1] + mid * d[..., 1])
            up = fm > 0
            lo = np.where(up, mid, lo)
            hi = np.where(up, hi, mid)
        hit = np.where(crossed, hi, np.inf)
        p = o + np.where(np.isfinite(hit), hit, 0.0)[..., None] * d
        in_hole = np.zeros(d.shape[:-1], bool)
        for x0, x1, y0, y1 in self.holes:
            in_hole |= (p[..., 0] >= x0) & (p[..., 0] <= x1) & (p[..., 1] >= y0) & (p[..., 1] <= y1)
        hit = np.where(in_hole, np.inf, hit)
        t_best = np.minimum(t_best, hit)
        label = np.where(np.isfinite(hit), 1, label)
        for b in self.boxes:
            t = _slab(o, d, b)
            closer = t < t_best
            t_best = np.where(closer, t, t_best)
            label = np.where(closer, 2, label)
        if self.ceiling is not None:
            with np.errstate(divide="ignore", invalid="ignore"):
                t = np.where(d[..., 2] > 0, (self.ceiling - o[2]) / d[..., 2], np.inf)
            closer = t < t_best
            t_best = np.where(closer, t, t_best)
            label = np.where(closer, 2, label)
        far = t_best > self.max_range
        return np.where(far, np.inf, t_best), np.where(far, 0, label)


def _slab(o, d, box):
    x0, x1, y0, y1, z0, z1 = box
    lo = np.array([x0, y0, z0])
    hi = np.array([x1, y1, z1])
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        t0 = (lo - o) * inv
        t1 = (hi - o) * inv
    tmin = np.nanmax(np.minimum(t0, t1), axis=-1)
    tmax = np.nanmin(np.maximum(t0, t1), axis=-1)
    ok = (tmax >= np.maximum(tmin, 0.0))
    return np.where(ok, np.maximum(tmin, 0.0), np.inf)


def flat(x, y):
    return np.zeros_like(x)


def tilted(deg):
    s = np.tan(np.radians(deg))
    return lambda x, y: s * x


def ramp(x, y):
    """Flat to x = 5 m, then rising at 8 % to x = 25 m, flat again beyond."""
    return np.clip(x - 5.0, 0.0, 20.0) * 0.08


SCENES = {
    "flat": lambda: Scene(flat),
    "tilted5": lambda: Scene(tilted(5.0)),
    "ramp": lambda: Scene(ramp),
    # a sensor 4.5 m up (on a truck) sees the top of the 3 m island
    "box_rooftop": lambda: Scene(flat, boxes=[(10.0, 12.0, 2.0, 4.0, 0.0, 1.0), (-20.0, -12.0, 6.0, 14.0, 0.0, 3.0)],
                                 sensor_z=4.5),
    "wall": lambda: Scene(flat, boxes=[(14.0, 14.4, -15.0, 15.0, 0.0, 3.0)]),
    "room": lambda: Scene(flat, boxes=[(9.0, 9.3, -10.0, 10.0, 0.0, 3.0), (-9.3, -9.0, -10.0, 10.0, 0.0, 3.0),
                                       (-9.0, 9.0, 7.0, 7.3, 0.0, 3.0), (-9.0, 9.0, -7.3, -7.0, 0.0, 3.0)],
                          ceiling=3.0, max_range=24.0, fov=(45.0, -45.0)),
    "hole": lambda: Scene(flat, holes=[(12.0, 20.0, -6.0, 6.0)]),
}


def make_frame(name, h=64, w=1024, seed=0, dual=False, pose=None):
    """-> dict with ranges (list of (H, W) uint32), label (H, W), points (H, W, 3) true hit points in the world,
    direction, offset (H*W x 3), status, poses (W x 16), sensor_to_body (16,).  pose: optional 4x4 world pose of
    the sensor applied to every column (the LUT stays in the sensor frame)."""
    scene = SCENES[name]()
    d = beams(h, w, scene.fov, seed=seed)
    pose = np.eye(4) if pose is None else np.asarray(pose, np.float64)
    # the scene lives in the world; rays leave the sensor along R d from the sensor's world position
    dw = d @ pose[:3, :3].T
    t, label = scene.cast(dw, pose[:3, 3] + np.array([0.0, 0.0, scene.sensor_z]))
    rng = np.where(np.isfinite(t), np.round(t * 1000.0), 0).astype(np.uint32)
    # the measured range keeps the true surface label; a hit rounded to 0 mm is no return
    label = np.where(rng > 0, label, 0)
    direction = (d * 0.001).reshape(-1, 3)
    offset = np.zeros_like(direction)
    # the column pose carries the sensor's height above the world origin
    col_pose = pose.copy()
    col_pose[:3, 3] = pose[:3, 3] + np.array([0.0, 0.0, scene.sensor_z])
    poses = np.repeat(col_pose.reshape(1, 16), w, axis=0)
    ranges = [rng]
    if dual:
        # second return: the same surface 5 % of the time, scattered a little further, else nothing
        rs = np.random.default_rng(seed + 1)
        r2 = np.where(rs.random(rng.shape) < 0.05, rng + rs.integers(1, 30, rng.shape).astype(np.uint32), 0)
        ranges.append(np.where(rng > 0, r2, 0).astype(np.uint32))
    world = (np.where(np.isfinite(t), t, 0.0)[..., None] * dw) + col_pose[:3, 3]
    return {"ranges": ranges, "label": label, "points": world, "direction": direction, "offset": offset,
            "status": np.ones(w, np.uint32), "poses": poses, "sensor_to_body": np.eye(4).reshape(16),
            "scene": scene, "h": h, "w": w}


def truth_sets(frame, clearance=1.0, min_height=0.5):
    """Boolean (H, W) sets the thresholds apply to: ground pixels farther than `clearance` (horizontally) from every
    object, and object pixels more than `min_height` above the ground under them."""
    scene, p, label = frame["scene"], frame["points"], frame["label"]
    ground = label == 1
    for x0, x1, y0, y1, _, _ in scene.boxes:
        dx = np.maximum(np.maximum(x0 - p[..., 0], p[..., 0] - x1), 0.0)
        dy = np.maximum(np.maximum(y0 - p[..., 1], p[..., 1] - y1), 0.0)
        ground &= np.hypot(dx, dy) > clearance
    obj = (label == 2) & (p[..., 2] - scene.ground(p[..., 0], p[..., 1]) > min_height)
    return ground, obj
