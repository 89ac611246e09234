"""Merging rigs without a device: the overlapping scene shows the problem separate detection has, what the merged oracle does about it,
and where the merged oracle's own remaining second boxes come from.

Four sensors at quarter-turn yaws with 180 degree fields of view see every direction twice.  Detected separately (the reference per
sensor, boxes moved into the vehicle frame), objects get two boxes -- one per sensor.  Detected from the merged cloud, the two sensors'
points of an object fall into one set of cells.  The merged cloud of this rig is, point for point, the vehicle's whole view with every
elevated point twice; the reference's seed rule ("more than one point in a 0.2 m cell", component_clustering.cpp:136) then also seeds
cells that hold a single return of the view, and around sparse, far objects those can form a separate small component that passes the
rule filter.  So on some scenes (seed 91 below) the merged oracle still boxes an object twice -- exactly where the reference boxes the
doubled view twice, never from the overlap.  A one-sensor identity rig's merged oracle is the reference on that cloud.
"""
import numpy as np
import pytest

from rig_merge_scenes import (boxes_per_object, doubled_view_detection, merged_detection, overlap_rig, overlap_ticks,
                              separate_detection)
from test_sensor_rig_gpu import H_DEFAULT, ref_detect

RIG4 = overlap_rig(4, heights=[2.0, 1.2, 0.8, 1.8])


def test_separate_detection_duplicates_and_merge_does_not(ref_intended, synth):
    """seed 5: separate detection boxes objects twice, the merged oracle never does (a property of this scene, see the next test)"""
    ref = ref_intended
    dup_sep, max_merged, seen = 0, 0, 0
    for ts, frames, pos, size in overlap_ticks(synth, RIG4, 6):
        sep = boxes_per_object(separate_detection(ref, RIG4, frames), pos, size)
        _, b, _, cut = merged_detection(ref, RIG4, frames)
        mer = boxes_per_object(b, pos, size)
        assert not cut
        dup_sep += int((sep > 1).sum())
        max_merged = max(max_merged, int(mer.max()))
        seen += int((mer == 1).sum())
    assert dup_sep > 0              # the scene exhibits the problem
    assert max_merged <= 1          # the merged oracle removes it
    assert seen > 20                # and still boxes the objects


@pytest.mark.parametrize("seed", [5, 91])
def test_remaining_second_boxes_are_the_doubled_density(ref_intended, synth, seed):
    """every sensor at the same height: per object and tick, the merged oracle's box count equals the reference's on the whole view
    with every elevated point twice; on seed 91 that count is 2 for some objects (on seed 5 never), while separate detection gives far
    more second boxes"""
    ref = ref_intended
    rig = overlap_rig(4)
    cfg = dict(seed=seed, n_objects=30, rings=32, azimuths=900)
    views = [p for _, p in synth.frames(synth.SceneConfig(**cfg), 12)]
    dup_mer = dup_sep = 0
    for (ts, frames, pos, size), view in zip(overlap_ticks(synth, rig, 12, **cfg), views):
        mer = boxes_per_object(merged_detection(ref, rig, frames)[1], pos, size)
        dbl = boxes_per_object(doubled_view_detection(ref, view), pos, size)
        assert np.array_equal(mer, dbl), (ts, mer, dbl)
        dup_mer += int((mer > 1).sum())
        dup_sep += int((boxes_per_object(separate_detection(ref, rig, frames), pos, size) > 1).sum())
    assert (dup_mer > 0) == (seed == 91), dup_mer
    assert dup_sep > 5 * max(dup_mer, 1), (dup_sep, dup_mer)


def test_one_identity_sensor_is_the_reference(ref_intended, synth):
    ref = ref_intended
    rig = overlap_rig(1)
    assert np.array_equal(rig[0][0], np.eye(3, 4, dtype=np.float32))
    for ts, frames, _, _ in overlap_ticks(synth, rig, 3, seed=9):
        rows, b, E, _ = merged_detection(ref, rig, frames)
        counts, want = ref_detect(ref, frames[0], H_DEFAULT)
        assert rows == [counts]
        assert b.shape == want.shape and np.array_equal(b.view(np.uint32), want.view(np.uint32))
        e, _ = ref.ground_remove(frames[0])
        assert np.array_equal(E.view(np.uint32), e.view(np.uint32))
