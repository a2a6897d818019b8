"""CPU: the scenes of the point-average grid's input-order sums (tests/_grid_order_scenes.py) reach the cases the GPU
tests rely on.  Runs of thousands of points and sub-normal addends occur, and summing each voxel in the opposite order
changes the float32 bits of many voxels, so a GPU grid that equals `oracle.numpy_grid` on these scenes has summed in
input order.  With the compiled reference built, `numpy_grid` equals it on the stress scene."""

import numpy as np
import pytest

import oracle
from tests import _grid_order_scenes as O
from tests._util import sort_dump


def _changed_share(a, b):
    """Share of the voxels with two or more points whose position or colour sum bits differ between two grids."""
    assert np.array_equal(a.keys, b.keys) and np.array_equal(a.count, b.count)
    multi = a.count >= 2
    diff = np.any(a.pos.view(np.uint32) != b.pos.view(np.uint32), axis=1)
    diff |= np.any(a.col.view(np.uint32) != b.col.view(np.uint32), axis=1)
    return float(diff[multi].mean())


def test_stress_scene_has_long_runs_and_reverse_order_changes_its_sums():
    pts, _, cols = O.stress_scene()
    assert len(pts) >= 100_000
    longest, p99 = O.longest_runs([(pts, cols)])
    assert longest >= 1000 and p99 >= 100
    assert np.unique(O.numpy_grid_of([(pts, None)]).keys, axis=0).shape[0] <= 400
    share = _changed_share(O.numpy_grid_of([(pts, cols)]), O.reversed_dump([(pts, cols)]))
    assert share > 0.5, share


def test_float64_and_subnormal_scenes_reach_their_cases():
    p64, c = O.float64_scene()
    assert p64.dtype == np.float64
    assert O.longest_runs([(p64, c)])[0] >= 1000
    assert _changed_share(O.numpy_grid_of([(p64, c)]), O.reversed_dump([(p64, c)])) > 0.5
    pts, cols = O.subnormal_scene()
    assert O.is_subnormal(pts).sum() > 10_000 and O.is_subnormal(cols).sum() > 10_000
    G = O.numpy_grid_of([(pts, cols)])
    row = G.keys[:, 1] > 8
    assert row.sum() >= 10 and O.is_subnormal(G.pos[row, 0]).all()     # the far row's x sums stay sub-normal
    assert not O.is_subnormal(G.pos[~row]).any()
    assert _changed_share(G, O.reversed_dump([(pts, cols)])) > 0.5


def test_real_frames_reverse_order_changes_many_voxels():
    batches = O.frame_points()
    assert len(batches) == O.N_FRAMES and all(len(p) > 100_000 for p, _ in batches)
    share = _changed_share(O.numpy_grid_of(batches), O.reversed_dump(batches))
    assert share > 0.2, share


@pytest.mark.skipif(not oracle.have_ref(), reason="compiled reference (oracle/_ref) not built")
def test_numpy_grid_equals_compiled_reference_on_the_stress_scene():
    pts, u8, _ = O.stress_scene()
    ref = oracle.RefGrid(O.VS, 8)
    G = oracle.numpy_grid(O.VS)
    for part in np.array_split(np.arange(len(pts)), 3):
        ref.integrate(pts[part], u8[part])
        G.integrate(pts[part], u8[part])
    a, b = G.dump(), sort_dump(ref.dump_blocks())
    for k in ("keys", "count", "pos_sum", "col_sum"):
        assert np.array_equal(a[k], b[k]), k
