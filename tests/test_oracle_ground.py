"""CPU checks of the ground-segmentation oracle (oracle/orc_ground.c) against scenes whose ground is known by
construction (tests/ground_scenes.py), plus its error texts, early returns and return handling."""
import numpy as np
import pytest

from oracle import ground as og
from tests import ground_scenes as gs

# Fixed thresholds: share of far-from-object ground pixels labelled ground, and of object pixels more than 0.5 m
# above the ground labelled non-ground.
MIN_GROUND_RECALL = 0.99
MIN_OBJECT_REJECTION = 0.99

_cache = {}


def _frame(name, **kw):
    key = (name, tuple(sorted(kw.items())))
    if key not in _cache:
        _cache[key] = gs.make_frame(name, **kw)
    return _cache[key]


def _run(f, ranges=None, normals="computed", stop=og.FINAL):
    ranges = f["ranges"] if ranges is None else ranges
    if normals == "computed":
        normals = og.computed_normals(ranges[:2], f["direction"], f["offset"], f["poses"], f["sensor_to_body"])
    return og.run(ranges, f["status"], f["direction"], f["offset"], f["poses"], normals, stop=stop)


def _check_truth(f, mask):
    ground, obj = gs.truth_sets(f)
    m = mask.astype(bool)
    assert ground.sum() > 1000
    assert m[ground].mean() >= MIN_GROUND_RECALL, m[ground].mean()
    if obj.any():
        assert (~m[obj]).mean() >= MIN_OBJECT_REJECTION, (~m[obj]).mean()


@pytest.mark.parametrize("name", list(gs.SCENES))
def test_scene_known_ground(name):
    f = _frame(name)
    masks, model, _ = _run(f)
    assert model["valid"] == 1
    _check_truth(f, masks[0])


def test_scenes_with_objects_have_objects():
    for name in ("box_rooftop", "wall", "room"):
        _, obj = gs.truth_sets(_frame(name))
        assert obj.sum() > 500, name


def test_indoor_and_outdoor_scenes():
    """The room's 95th-percentile footprint is under 25 m (indoor tolerances), the outdoor scenes' above it."""
    assert _run(_frame("room"))[1]["footprint_bound"] <= 25.0
    assert _run(_frame("flat"))[1]["footprint_bound"] > 25.0


def test_world_frame_pose():
    """A sensor yawed and moved in the world: the same scene, segmented in the world frame."""
    c, s = np.cos(0.7), np.sin(0.7)
    pose = np.array([[c, -s, 0, 3.0], [s, c, 0, -2.0], [0, 0, 1, 0.0], [0, 0, 0, 1]])
    f = gs.make_frame("wall", pose=pose)
    masks, _, _ = _run(f)
    _check_truth(f, masks[0])


def test_world_frame_pose_island_side_face():
    """The 3 m island seen by a yawed and moved sensor.  Its top is rejected whole, but part of the low band of the
    side faces (0.5-1.35 m above the ground) is labelled ground: the prune removes the top's cells, the fills then
    give the cells along the island's edge heights of up to 1.14 m taken from the faces' own points, and the lower
    face points fall within the local tolerance of those cells.  This is the reference's algorithm (DESIGN §9); the
    counts are pinned so that a change in it shows here."""
    c, s = np.cos(0.7), np.sin(0.7)
    pose = np.array([[c, -s, 0, 3.0], [s, c, 0, -2.0], [0, 0, 1, 0.0], [0, 0, 0, 1]])
    f = gs.make_frame("box_rooftop", pose=pose)
    masks, model, grids = _run(f)
    ground, obj = gs.truth_sets(f)
    m = masks[0].astype(bool)
    assert m[ground].mean() >= MIN_GROUND_RECALL
    z = f["points"][..., 2]
    top = obj & (z > 2.999)
    side = obj & ~top
    band = side & (z <= 1.35)
    assert top.sum() == 233 and not m[top].any()
    assert not m[side & ~band].any()
    assert band.sum() == 380 and m[band].sum() == 148
    # the island's cells after the passes: none at the top's height, the highest from the faces
    gx = (np.arange(model["cols"]) + 0.5) * 0.5 + model["origin_x"]
    gy = (np.arange(model["rows"]) + 0.5) * 0.5 + model["origin_y"]
    island = ((gx[None, :] > -19.0) & (gx[None, :] < -13.0)) & ((gy[:, None] > 7.0) & (gy[:, None] < 13.0))
    assert grids["valid"][island].all()
    assert 0.5 < grids["height"][island].max() < 1.2


def test_dual_return_and_precomputed_normals():
    f = _frame("box_rooftop", dual=True)
    masks, model, grids = _run(f)
    assert len(masks) == 2
    _check_truth(f, masks[0])
    second = f["ranges"][1] > 0
    assert second.sum() > 100
    ground, _ = gs.truth_sets(f)
    assert masks[1][second & ground].mean() >= MIN_GROUND_RECALL
    # NORMALS present but not NORMALS2: the second return is classified without normals
    n = og.computed_normals(f["ranges"], f["direction"], f["offset"], f["poses"], f["sensor_to_body"])
    frame = {"sensor_info": {"num_returns": 2, "sensor_to_body": f["sensor_to_body"]},
             "fields": {"RANGE": f["ranges"][0], "RANGE2": f["ranges"][1], "NORMALS": n[0].astype(np.float32)},
             "status": f["status"], "poses": f["poses"], "direction": f["direction"], "offset": f["offset"]}
    got = og.get_ground_mask(frame)
    want, _, _ = _run(f, normals=[n[0].astype(np.float32).astype(np.float64), None])
    assert all(np.array_equal(a, b) for a, b in zip(got, want))


def test_third_return_is_classified_without_normals_and_leaves_the_model_alone():
    f = _frame("box_rooftop", dual=True)
    third = f["ranges"][0].copy()
    masks3, model3, grids3 = _run(f, ranges=f["ranges"] + [third])
    masks2, model2, grids2 = _run(f)
    assert len(masks3) == 3
    assert model3 == model2
    for k in grids2:
        assert np.array_equal(grids2[k], grids3[k], equal_nan=True), k
    assert np.array_equal(masks3[0], masks2[0]) and np.array_equal(masks3[1], masks2[1])
    # the same points as the first return, without normals: the model is the same, so the ground agrees
    _check_truth(f, masks3[2])


def test_stages_are_the_passes_in_order():
    f = _frame("box_rooftop")
    prev = None
    for stop in range(og.FINAL + 1):
        _, model, grids = _run(f, stop=stop)
        assert (model["rows"], model["cols"]) == (grids["valid"].shape)
        if prev is not None:
            # floor and obstacle columns are fixed by the cell pass; the passes only move valid / height / roughness
            assert np.array_equal(prev["floor_z"], grids["floor_z"], equal_nan=True)
            assert np.array_equal(prev["obstacle"], grids["obstacle"])
        if og.STAGES[stop].startswith("fill") and prev is not None:
            assert grids["valid"].sum() >= prev["valid"].sum()
            changed = prev["valid"] == 1
            assert np.array_equal(prev["height"][changed], grids["height"][changed])
        if og.STAGES[stop] in ("prune", "components") and prev is not None:
            assert grids["valid"].sum() <= prev["valid"].sum()
        invalid = grids["valid"] == 0
        if stop > 0:
            assert np.all(np.isnan(grids["height"][invalid & ~(prev["valid"] == 1)]))
        prev = grids
    # no cell over the 3 m rooftop keeps its height: the passes remove it and the last fill puts ground there
    gx = (np.arange(model["cols"]) + 0.5) * 0.5 + model["origin_x"]
    gy = (np.arange(model["rows"]) + 0.5) * 0.5 + model["origin_y"]
    roof = ((gx[None, :] > -19.0) & (gx[None, :] < -13.0)) & ((gy[:, None] > 7.0) & (gy[:, None] < 13.0))
    _, _, cells = _run(f, stop=0)
    assert np.nanmax(cells["height"][roof]) > 2.5
    assert not np.any(grids["height"][roof] > 0.5)


def test_hole_wider_than_the_fill_radius():
    """A hole 8 x 12 m: its centre is 8 cells from any return, beyond one fill's radius of 6, so the first fill leaves
    it open; the later fills start from the first one's output and close it (ground_seg.cpp:921-942)."""
    f = _frame("hole")
    centre = None
    for stop, want in ((og.STAGES.index("cells"), 0), (og.STAGES.index("fill1"), 0), (og.FINAL, 1)):
        _, model, grids = _run(f, stop=stop)
        if centre is None:
            gx = (np.arange(model["cols"]) + 0.5) * 0.5 + model["origin_x"]
            gy = (np.arange(model["rows"]) + 0.5) * 0.5 + model["origin_y"]
            centre = ((gx[None, :] > 15.5) & (gx[None, :] < 16.5)) & ((gy[:, None] > -0.5) & (gy[:, None] < 0.5))
            assert centre.sum() == 4
        assert np.all(grids["valid"][centre] == want), og.STAGES[stop]


def test_error_texts():
    f = _frame("flat")
    base = {"sensor_info": {"num_returns": 1, "sensor_to_body": f["sensor_to_body"]},
            "fields": {"RANGE": f["ranges"][0]}, "status": f["status"], "poses": f["poses"],
            "direction": f["direction"], "offset": f["offset"]}
    with pytest.raises(ValueError) as ei:
        og.get_ground_mask(dict(base, sensor_info=None))
    assert str(ei.value) == "frame.sensor_info is required for get_ground_mask"
    with pytest.raises(ValueError) as ei:
        og.get_ground_mask(dict(base, fields={}))
    assert str(ei.value) == "frame must contain RANGE field for get_ground_mask"
    for g in (0.0, -0.5, float("nan"), float("inf")):
        with pytest.raises(ValueError) as ei:
            og.check_grid_size(g)
        assert str(ei.value) == "GroundSegConfig.grid_size must be > 0"


def test_no_valid_column_returns_zero_masks():
    f = _frame("flat")
    masks, model, grids = og.run(f["ranges"], np.zeros(f["w"], np.uint32), f["direction"], f["offset"], f["poses"])
    assert model["has_columns"] == 0 and model["valid"] == 0 and grids is None
    assert not masks[0].any()
    # bit 0 decides the first / last valid column; inside that span any non-zero status counts
    st = np.zeros(f["w"], np.uint32)
    st[100], st[300] = 1, 1
    st[101:300] = 2
    st[500:] = 2
    masks, model, _ = og.run(f["ranges"], st, f["direction"], f["offset"], f["poses"])
    assert model["valid"] == 1
    assert masks[0][:, 101:300].any()
    assert not masks[0][:, :100].any() and not masks[0][:, 301:].any()


def test_empty_frame():
    h, w = 8, 0
    masks, model, grids = og.run([np.zeros((h, w), np.uint32)], np.zeros(w, np.uint32), np.zeros((0, 3)),
                                 np.zeros((0, 3)), np.zeros((0, 16)))
    assert masks[0].shape == (h, w) and grids is None and model["has_columns"] == 0


def test_frame_without_model_points_uses_the_indoor_fallback():
    """Every return closer than 0.15 m: no model point, the footprint is 0 (indoor) and the fallback z is 0, so
    points up to 0.3 m high are ground."""
    h, w = 4, 16
    rs = np.random.default_rng(3)
    d = rs.normal(size=(h * w, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d *= 0.001
    rng = rs.integers(1, 140, size=(h, w)).astype(np.uint32)
    rng[0, 0] = 0
    poses = np.repeat(np.eye(4).reshape(1, 16), w, axis=0)
    masks, model, grids = og.run([rng], np.ones(w, np.uint32), d, np.zeros_like(d), poses)
    assert model["valid"] == 0 and model["has_columns"] == 1 and grids is None
    z = (rng.reshape(-1).astype(np.float64)[:, None] * d)[:, 2].reshape(h, w)
    assert np.array_equal(masks[0], ((rng > 0) & (z <= 0.3)).astype(np.uint8))
