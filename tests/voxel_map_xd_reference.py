"""Plain-Python statement of VoxelHashMapXd (ouster_core/include/ouster/core/voxel_hash_map.h:287-305, 352-517,
ouster_core/src/voxel_hash_map.cpp:14-247) with first_n_point insertion, and of the map exporter's per-return step
(python/src/ouster/cli/plugins/map_export.py:589-617), for the tests of the device map with attributes.

Points are 3 + num_attributes doubles; voxels, the gate, the cull and the closest-neighbour search read x, y, z only
(impl::spatial_view).  Voxels are listed in creation order (DESIGN 9): a dict keeps insertion order, an erased voxel
leaves it, a voxel created again goes to the end.  Arithmetic is IEEE double without contraction, summed in the
reference's order, so results compare bit for bit with the oracle (oracle/orc_icp.c) and the GPU.
"""
import math

import numpy as np

from oracle import icp as oi
from oracle import oracle as orc

DBL_MAX = oi.DBL_MAX

# VOXEL_SHIFTS (voxel_hash_map.cpp), the order get_closest_neighbor visits the 27 voxels in
SHIFTS = [(0, 0, 0), (1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1), (1, 1, 0), (1, -1, 0),
          (-1, 1, 0), (-1, -1, 0), (1, 0, 1), (1, 0, -1), (-1, 0, 1), (-1, 0, -1), (0, 1, 1), (0, 1, -1), (0, -1, 1),
          (0, -1, -1), (1, 1, 1), (1, 1, -1), (1, -1, 1), (1, -1, -1), (-1, 1, 1), (-1, 1, -1), (-1, -1, 1),
          (-1, -1, -1)]


def _i32(v):
    """wrap to int32"""
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= (1 << 31) else v


def voxel_coord(v):
    """static_cast<int>(std::floor(v)) as x86 evaluates it: NaN and out-of-range give INT32_MIN."""
    if math.isnan(v):
        return -(1 << 31)
    f = math.floor(v) if math.isfinite(v) else v
    if not (-2147483648.0 <= f < 2147483648.0):
        return -(1 << 31)
    return int(f)


class VoxelHashMapXd:
    def __init__(self, voxel_size, max_distance=100.0, max_points_per_voxel=20, min_pts_threshold=1,
                 num_attributes=0):
        if max_points_per_voxel == 0:
            raise ValueError("max_points_per_voxel must be greater than 0")
        if voxel_size <= 0:
            raise ValueError("voxel_size must be greater than 0")
        if max_distance <= 0:
            raise ValueError("max_distance must be greater than 0")
        self.voxel_size, self.max_distance = float(voxel_size), float(max_distance)
        self.max_pts, self.cols = int(max_points_per_voxel), 3 + int(num_attributes)
        self.res_sq = self.voxel_size * self.voxel_size / float(self.max_pts)
        self.inv = 1.0 / self.voxel_size
        self.vox = {}

    def _key(self, p):
        return tuple(voxel_coord(float(p[d]) * self.inv) for d in range(3))

    @property
    def empty(self):
        return not self.vox

    def clear(self):
        self.vox = {}

    def size(self):
        return len(self.vox), sum(len(b) for b in self.vox.values())

    def add_points(self, rows):
        rows = np.ascontiguousarray(rows, np.float64)
        if rows.ndim != 2 or rows.shape[1] != self.cols:
            raise ValueError("VoxelHashMap::add_points received unexpected point dimension")
        for row in rows:
            b = self.vox.setdefault(self._key(row), [])
            if len(b) == self.max_pts:
                continue
            x, y, z = float(row[0]), float(row[1]), float(row[2])
            near = False
            for q in b:
                dx, dy, dz = q[0] - x, q[1] - y, q[2] - z
                if (dx * dx + dy * dy) + dz * dz < self.res_sq:
                    near = True
                    break
            if not near:
                b.append(row.copy())

    def _rows(self, buckets):
        rows = [r for b in buckets for r in b]
        return np.array(rows).reshape(-1, self.cols) if rows else np.empty((0, self.cols))

    def point_cloud(self):
        return self._rows(self.vox.values())

    def extract_voxels_far_from_location(self, origin):
        o = self._key(np.asarray(origin, np.float64).reshape(-1)[:3])
        thr = oi.cull_threshold(self.max_distance, self.voxel_size)
        out = []
        for k in list(self.vox):
            d = [(k[i] - o[i]) & 0xFFFFFFFF for i in range(3)]
            if _i32(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) >= thr:
                out.append(self.vox.pop(k))
        return self._rows(out)

    def remove_voxels_far_from_location(self, origin):
        self.extract_voxels_far_from_location(origin)

    def get_closest_neighbor(self, query, max_distance_sq=DBL_MAX):
        q = [float(v) for v in np.asarray(query, np.float64).reshape(-1)[:3]]
        v = self._key(q)
        best, nb = float(max_distance_sq), np.zeros(self.cols)
        for s in SHIFTS:
            w = tuple(_i32(v[d] + s[d]) for d in range(3))
            lb = 0.0
            for d in range(3):
                lo = float(w[d]) * self.voxel_size
                hi = lo + self.voxel_size
                if q[d] < lo:
                    lb += (lo - q[d]) * (lo - q[d])
                elif q[d] > hi:
                    lb += (q[d] - hi) * (q[d] - hi)
            if lb >= best:
                continue
            for p in self.vox.get(w, ()):
                dx, dy, dz = p[0] - q[0], p[1] - q[1], p[2] - q[2]
                d2 = (dx * dx + dy * dy) + dz * dz
                if d2 < best:
                    best, nb = d2, p
        return np.array(nb, np.float64), best

    def get_closest_neighbors(self, queries, max_distance_sq=DBL_MAX):
        queries = np.asarray(queries, np.float64)
        res = [self.get_closest_neighbor(q, max_distance_sq) for q in queries]
        nb = np.array([r[0] for r in res]).reshape(-1, self.cols)
        return nb, np.array([r[1] for r in res])


def map_rows(items):
    """map_export.py:589-617 for every item {direction, offset, range [h, w], poses [w, 4, 4], fields}:
    orc_cartesian_f64 -> orc_dewarp_f64 -> [range > 0] -> the fields [range > 0] as columns ->
    np.concatenate(..., axis=1).astype(float64); the items' rows one after the other."""
    out = []
    for it in items:
        rng = np.ascontiguousarray(it["range"], np.uint32)
        h, w = rng.shape
        pts = orc.cartesian(rng, it["direction"], it["offset"]).reshape(h, w, 3)
        dewarped = orc.dewarp(pts, it["poses"])
        valid = rng > 0
        points = dewarped[valid]
        chunks = []
        for f in it.get("fields", []):
            f = np.asarray(f)
            chunks.append(f[valid].reshape(-1, 1) if f.ndim == 2 else f[valid].reshape(-1, f.shape[-1]))
        if chunks:   # map_export.py:609-613, then add_points :475-476
            out.append(np.concatenate([points, np.concatenate(chunks, axis=1)], axis=1).astype(np.float64))
        else:
            out.append(points.astype(np.float64))
    return np.concatenate(out, axis=0)
