"""Layered clustering without a device (include/lmot.h, lmot_set_layers): the NumPy restatement of steps 1-6 (tests/layer_scenes.py) is
componentClustering at one slice, behaves as the definition says on hand-built voxel cases, and -- through the per-cluster reference
oracle of step 7 -- gives boxes to cars under canopies that the plain reference loses."""
import numpy as np
import pytest

import layer_scenes as ls

f32 = np.float32


def _ref():
    from oracle import ref
    if not ref.have_ref("intended"):
        pytest.skip("oracle/_ref not built")
    return ref.RefOracle("intended")


def _grid_ids(elev, grid):
    xi, yi, ok = ls.columns(elev)
    return np.where(ok, grid[xi, yi], 0).astype(np.int32)


@pytest.mark.parametrize("seed", [3, 11])
def test_one_slice_is_component_clustering(synth, seed):
    ref = _ref()
    cfg = synth.SceneConfig(rings=32, azimuths=900, n_objects=30, seed=seed)
    for _, pts in synth.frames(cfg, 2):
        e, _ = ref.ground_remove(pts)
        grid, k = ref.component_clustering(e)
        ids, k1 = ls.point_clusters(e, n_slices=1, gap_slices=0)
        assert k1 == k
        assert np.array_equal(ids, _grid_ids(e, grid))


@pytest.mark.parametrize("seed", [1, 2])
def test_one_slice_on_uniform_clouds(synth, seed):
    ref = _ref()
    cloud = synth.uniform_cloud(20000, seed, half=30.0)[:, :3]
    grid, k = ref.component_clustering(cloud)
    ids, k1 = ls.point_clusters(cloud, n_slices=1, gap_slices=0)
    assert k1 == k and np.array_equal(ids, _grid_ids(cloud, grid))


def _pts(cells):
    """two points per (x, y, slice) voxel of the default setting (sensor_height 2, slice 0.2 m from z = -0.5 above the ground)"""
    out = []
    for x, y, s in cells:
        cx = (x + 0.5) * 0.2 - 25.0
        cy = (y + 0.5) * 0.2 - 25.0
        z = -2.0 - 0.5 + (s + 0.5) * 0.2
        out += [(cx, cy, z), (cx + 0.01, cy, z)]
    return np.array(out, f32)


@pytest.mark.parametrize("g", [0, 1, 2, 3])
def test_gap_join_and_split(g):
    """seeds with exactly 2g empty slices between them join; 2g + 1 separate"""
    join = ls.point_clusters(_pts([(100, 100, 5), (100, 100, 5 + 2 * g + 1)]), gap_slices=g)
    split = ls.point_clusters(_pts([(100, 100, 5), (100, 100, 5 + 2 * g + 2)]), gap_slices=g)
    assert join[1] == 1 and split[1] == 2
    assert list(split[0][::2]) == [1, 2]


def test_diagonal_adjacency():
    # dilated by one column and g = 0 slices, seeds two columns and one slice apart touch only diagonally (26-adjacency)
    ids, k = ls.point_clusters(_pts([(100, 100, 5), (102, 102, 6)]), gap_slices=0)
    assert k == 1
    ids, k = ls.point_clusters(_pts([(100, 100, 5), (102, 102, 7)]), gap_slices=0)
    assert k == 2
    ids, k = ls.point_clusters(_pts([(100, 100, 5), (104, 100, 5)]), gap_slices=0)
    assert k == 2


def test_clamping_at_both_ends():
    low = np.array([[0.0, 0.0, -30.0], [0.01, 0.0, -29.0], [0.0, 0.0, -2.0 - 0.5 + 0.05]], f32)
    ids, k = ls.point_clusters(low, gap_slices=0)
    assert k == 1 and (ids == 1).all()                    # far below slice 0: clamped into it
    high = np.array([[0.0, 0.0, 50.0], [0.01, 0.0, 80.0], [0.0, 0.0, -2.0 - 0.5 + 31 * 0.2 + 0.1]], f32)
    ids, k = ls.point_clusters(high, gap_slices=0)
    assert k == 1 and (ids == 1).all()
    assert list(ls.slices(high, 2.0)) == [31, 31, 31]


def test_single_point_column():
    """a one-point column is no seed: its point is labelled where a neighbour's reach covers its voxel, 0 elsewhere"""
    seed = _pts([(100, 100, 10)])
    c100, c101 = (100 + 0.5) * 0.2 - 25.0, (101 + 0.5) * 0.2 - 25.0
    near = np.array([[c101, c100, -2.0 - 0.5 + 12.5 * 0.2]], f32)   # column (101, 100), slice 12: within g = 2
    far = np.array([[c100, c101, -2.0 - 0.5 + 13.5 * 0.2]], f32)    # column (100, 101), slice 13: outside
    ids, k = ls.point_clusters(np.concatenate([seed, near, far]))
    assert k == 1 and list(ids) == [1, 1, 1, 0]


def test_id_order():
    """ids follow each component's smallest (x, y, s): x outermost, then y, then the slice"""
    cells = [(120, 50, 20), (120, 50, 2), (110, 200, 9), (120, 10, 15)]
    ids, k = ls.point_clusters(_pts(cells), gap_slices=1)
    assert k == 4 and list(ids[::2]) == [4, 3, 1, 2]


def test_points_outside_the_roi():
    p = np.array([[30.0, 0.0, -1.0], [30.0, 0.01, -1.0], [0.0, 0.0, -1.0], [0.01, 0.0, -1.0]], f32)
    ids, k = ls.point_clusters(p)
    assert k == 1 and list(ids) == [0, 0, 1, 1]


# objects the per-cluster reference oracle finds on layer_scenes.render(sensor), with layers (defaults) and without: car_canopy /
# ped_shelter / car_gantry / truck / car_open / ped_open
FOUND = {
    "64": {"plain": [0, 0, 0, 0, 2, 3], "layers": [2, 0, 0, 0, 2, 3]},
    "32": {"plain": [0, 1, 0, 0, 3, 3], "layers": [2, 1, 0, 0, 3, 3]},
}
KINDS = ["car_canopy", "ped_shelter", "car_gantry", "truck", "car_open", "ped_open"]


@pytest.mark.parametrize("sensor", ["64", "32"])
def test_canopy_scene(sensor):
    ref = _ref()
    pts, objects = ls.render(sensor)
    e, _ = ref.ground_remove(pts)
    grid, k = ref.component_clustering(e)
    plain, _ = ref.box_fitting(e, grid, k)
    lay = ls.ref_layers_detect(ref, pts)
    assert [ls.found(plain, objects, t) for t in KINDS] == FOUND[sensor]["plain"]
    assert [ls.found(lay["boxes"], objects, t) for t in KINDS] == FOUND[sensor]["layers"]
    # the truck's points stay in one cluster
    tx, ty, _ = [o for o in objects if o[2] == "truck"][0]
    near = np.hypot(lay["elev"][:, 0] - tx, lay["elev"][:, 1] - ty) < 2.0
    assert len(set(lay["ids"][near]) - {0}) == 1
