"""CPU: the edge scenes of tests/test_gpu_tsdf_edges.py reach what they are built for, and the twin
(oracle/tsdf_oracle.c) stays the right truth on them.

- Tile census: every §1 scene drives the allocate kernel's capacity fallbacks (the capacities are read from
  b2v_tsdf.cu, so a later change of a capacity fails here instead of silently making a scene vacuous).
- The twin equals the Open3D-order restatement (oracle/open3d_order.c) on the unit-16 scenes and on the boundary
  inputs (special depths, voxels behind / on the camera plane, a principal point off the image).
- oracle.numpy_point_cloud agrees with the zero-crossing count definition of ExtractPointCloud."""

import numpy as np
import pytest

import oracle
from pyslam_b200 import synthetic as S
from tests import _edge_scenes as E
from tests._util import sort_dump, sorted_keys


# ---------------------------------------------------------------------------------------------------------------------
# tile census
# ---------------------------------------------------------------------------------------------------------------------

def _census(name):
    sc = E.SCENES[name]
    return [E.tile_census(sc, sc.frame(s)[0]) for s in E.SEEDS]


def test_capacities_are_read_from_the_kernel_source():
    k = E.kernel_constants()
    assert k["kAllocTile"] == 8 and k["kKeySet"] >= k["kListCap"] > 0 and k["kBoxSet"] >= k["kBoxList"] > 0


def test_noisy_d1_saturates_the_key_set_and_overflows_the_lists():
    """Per tile: more distinct keys than the key set holds (its 96-probe exit and the s_keys overflow are taken), and
    more keys that belong to that tile alone than s_new / s_act hold (whichever CTA inserts a shared key first, a
    tile's own keys are new in it and first touched by it)."""
    k = E.kernel_constants()
    for census in _census("noisy-D1"):
        assert len(census) == 4
        for t in census.values():
            assert t["units"] > 2 * k["kKeySet"]
            assert t["own_blocks"] > 4 * k["kListCap"]
            assert t["max_n"] <= 15 and t["box_span"] < 32768 and t["key_span"] < 1024   # the regular box / key path


def test_noisy_u16_overflows_the_lists_with_unit_sub_blocks():
    k = E.kernel_constants()
    for census in _census("noisy-U16"):
        for t in census.values():
            assert t["units"] < k["kListCap"]          # the units fit the key set and s_keys: only the blocks overflow
            assert t["own_blocks"] > 2 * k["kListCap"]


def test_far_u16_puts_units_out_of_rel_key_reach_whatever_the_reference():
    """A unit-key span of at least 1024 means some unit is more than 511 units from any reference key of the tile;
    the boxes themselves still fit the box set (span < 32768, at most 15 units a side)."""
    for census in _census("far-U16"):
        assert len(census) == 4
        for t in census.values():
            assert t["key_span"] >= 1024
            assert t["box_span"] < 32768 and t["max_n"] <= 15


def test_veryfar_d1_puts_boxes_beyond_the_box_offset_range():
    for census in _census("veryfar-D1"):
        assert len(census) == 1
        for t in census.values():
            assert t["box_span"] >= 65536


def test_widebox_d1_boxes_exceed_15_blocks_a_side():
    for census in _census("widebox-D1"):
        for t in census.values():
            assert t["min_max_n"] > 15                     # every sample's box takes the over-sized path


# ---------------------------------------------------------------------------------------------------------------------
# the twin against the Open3D-order restatement
# ---------------------------------------------------------------------------------------------------------------------

def _twin_vs_open3d(vs, tau, trunc, frames, unit=16):
    o3 = oracle.Open3DOrderVolume(vs, tau, unit, 4)
    tw = oracle.TsdfOracle(vs, tau, trunc, unit_resolution=unit)
    sub = np.stack(np.meshgrid(*[np.arange(unit // 8)] * 3, indexing="ij"), -1).reshape(-1, 3)
    for d, c, K, T in frames:
        o3.integrate(d, c, K, T, trunc, nthreads=4)
        tw.integrate(d, c, K, T, nthreads=4)
        u = o3.last_touched_units()
        assert np.array_equal(sorted_keys((u[:, None, :] * (unit // 8) + sub[None]).reshape(-1, 3)),
                              sorted_keys(tw.last_touched()))
    a, b = sort_dump(o3.dump_blocks()), sort_dump(tw.dump_blocks())
    assert np.array_equal(a["keys"], b["keys"])
    assert np.array_equal(a["vox"][:, 1], b["vox"][:, 1].astype(np.float64)), "weights differ"
    assert np.array_equal(a["vox"][:, 0], b["vox"][:, 0].astype(np.float64)), "tsdf differs"
    assert np.abs(a["vox"][:, 2:] - b["vox"][:, 2:]).max() < 1e-3
    return int((b["vox"][:, 1] > 0).sum())


@pytest.mark.parametrize("name", ["noisy-U16", "far-U16"])
def test_twin_equals_open3d_order_on_unit16_scenes(name):
    sc = E.SCENES[name]
    frames = [sc.frame(s)[:2] + (np.array(sc.K), np.eye(4)) for s in E.SEEDS[:2]]
    assert _twin_vs_open3d(sc.voxel_size, sc.sdf_trunc, sc.depth_trunc, frames) > 100000


def test_twin_equals_open3d_order_on_special_depths():
    cfg = S.CONFIGS["T0"]
    d, c, T = E.specials_frame()
    d1, c1, T1 = S.render_frame(cfg, 1)
    assert _twin_vs_open3d(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, [(d, c, cfg.K, T), (d1, c1, cfg.K, T1),
                                                                           (d, c, cfg.K, T1)]) > 10000


def test_twin_equals_open3d_order_with_the_camera_inside_the_band():
    """Flat depth 0.03 m with tau 0.08: voxels behind the camera and, with the second pose, a layer of voxel centres
    at camera z = +0.0 exactly (both skip the voxel)."""
    cfg = S.CONFIGS["T0"]
    frames = E.band_frames(cfg)
    assert frames[1][3][2, 3] == -float(np.float32(cfg.voxel_size) * np.float32(0.5))
    assert _twin_vs_open3d(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, frames) > 500


def test_twin_equals_open3d_order_with_the_principal_point_off_the_image():
    cfg = S.CONFIGS["T0"]
    frames = []
    for i, K in ((0, (80.0, 95.0, -20.25, cfg.height + 10.5)), (1, (80.0, 80.0, 0.0, 0.0))):
        d, c, T = S.render_frame(cfg, i)
        frames.append((d, c, np.array(K), T))
    assert _twin_vs_open3d(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, frames) > 500


# ---------------------------------------------------------------------------------------------------------------------
# the point-cloud restatement
# ---------------------------------------------------------------------------------------------------------------------

def _count_definition(dump):
    """ExtractPointCloud's zero crossings counted straight from a dump, voxel by voxel (A.4)."""
    idx = {tuple(k): i for i, k in enumerate(dump["keys"])}
    expect = 0
    for bi, key in enumerate(dump["keys"]):
        f = dump["vox"][bi, 0].reshape(8, 8, 8)   # [z, y, x]
        w = dump["vox"][bi, 1].reshape(8, 8, 8)
        for axis, dk in ((2, (1, 0, 0)), (1, (0, 1, 0)), (0, (0, 0, 1))):
            nk = (key[0] + dk[0], key[1] + dk[1], key[2] + dk[2])
            if nk in idx:
                fn = dump["vox"][idx[nk], 0].reshape(8, 8, 8)
                wn = dump["vox"][idx[nk], 1].reshape(8, 8, 8)
            else:
                fn, wn = np.zeros((8, 8, 8), np.float32), np.zeros((8, 8, 8), np.float32)
            f1 = np.concatenate([np.take(f, range(1, 8), axis), np.take(fn, [0], axis)], axis)
            w1 = np.concatenate([np.take(w, range(1, 8), axis), np.take(wn, [0], axis)], axis)
            ok0 = (w != 0) & (f < 0.98) & (f >= -0.98)
            ok1 = (w1 != 0) & (f1 < 0.98) & (f1 >= -0.98)
            expect += int((ok0 & ok1 & (f * f1 < 0)).sum())
    return expect


def test_numpy_point_cloud_matches_the_count_definition():
    cfg = S.CONFIGS["T0"]
    tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    for i in range(3):
        d, c, T = S.render_frame(cfg, i)
        tw.integrate(d, c, cfg.K, T)
    for dump in (tw.dump_blocks(), dict(zip(("keys", "vox"), E.random_blocks()))):
        pc = oracle.numpy_point_cloud(dump, cfg.voxel_size, 16)
        assert len(pc["points"]) == _count_definition(dump) > 100
        assert len(np.unique(pc["edges"], axis=0)) == len(pc["edges"])
        # every point lies on its edge, between the two voxel centres (inclusive: a tiny |f| rounds to an end)
        e = pc["edges"]
        for a in range(3):
            on = e[:, 3] == a
            lo = (e[on, a] + 0.5) * cfg.voxel_size
            assert np.all(pc["points"][on, a] >= lo - 1e-9) and np.all(pc["points"][on, a] <= lo + cfg.voxel_size + 1e-9)
        assert pc["colors"].min() >= 0.0 and pc["colors"].max() <= 1.0 + 1e-6   # float32 blend: may round up


def test_random_blocks_reach_every_cube_case():
    keys, vox = E.random_blocks()
    assert keys.min() < 0 and len(keys) == 300
    cases = E.cube_cases(keys, vox)
    assert set(np.unique(cases).tolist()) >= set(range(1, 255))
    mk, mv = E.max_output_blocks()
    c = E.cube_cases(mk, mv)
    assert len(c) >= 512 and set(np.unique(c).tolist()) == {0x5A, 0xA5}   # every edge of every cube crosses
