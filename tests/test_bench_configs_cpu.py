"""CPU: the kernels' twin (oracle/tsdf_oracle.c) against the Open3D-order restatement (oracle/open3d_order.c) on the
bench's KITTI-shaped street far from the origin and on consecutive ScanNet-shaped frames: the blocks each frame
touches, keys, tsdf and weights bit for bit, colour within 1e-3 (float32 against float64 running means), and the
meshes' edges, triangles and float64 vertices.  The GPU tests of tests/test_gpu_bench_configs.py compare the kernels
with the twin at bench scale and with the Open3D-order restatement on the same runs; this file keeps the chain
GPU = twin = Open3D order valid where they rely on it."""

import numpy as np
import pytest

import oracle
from pyslam_b200 import synthetic as S
from tests import _bench_configs as B
from tests import _color64 as C64
from tests._util import sort_dump, sorted_keys


def _both(name, frames):
    """Twin and Open3D-order restatement frame by frame; each frame's touched blocks are the sub-blocks of the units
    Open3D touches."""
    cfg = S.CONFIGS[name]
    o3 = oracle.Open3DOrderVolume(cfg.voxel_size, cfg.sdf_trunc, 16, 4)
    tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    for i in frames:
        d, c, T = S.render_frame(cfg, i)
        n3 = o3.integrate(d, c, cfg.K, T, cfg.depth_trunc, nthreads=B.NT)
        nt = tw.integrate(d, c, cfg.K, T, nthreads=B.NT)
        assert nt == 8 * n3
        assert np.array_equal(B.unit_blocks(o3.last_touched_units()), sorted_keys(tw.last_touched())), i
    return cfg, o3, tw


RUNS = {
    "C5-far": list(range(B.FAR_C5[1], B.FAR_C5[1] + 8)),   # the GPU test's far run (z 1975 .. 1978 m)
    "C5-end": [4538, 4539, 4540],                          # the last frames of the street, z 1997 m
    "C5-mid": list(range(2262, 2270)),                     # z ~ 1000 m
    "C4-run": list(range(B.RUN_C4[1], B.RUN_C4[1] + 6)),   # 4 mm voxels, consecutive frames
}


@pytest.mark.parametrize("run", list(RUNS))
def test_twin_equals_open3d_order_far_and_consecutive(run):
    cfg, o3, tw = _both(run[:2], RUNS[run])
    a, b = sort_dump(o3.dump_blocks()), sort_dump(tw.dump_blocks())
    n_obs, wmax = B.equal_to_open3d_order(b, a)
    assert n_obs > (30_000 if cfg.name == "C5" else 1_000_000)
    assert wmax >= 2                                   # consecutive frames overlap: voxels take several updates
    print(f"\n[{run}] frames {RUNS[run][0]}..{RUNS[run][-1]}: blocks {len(a['keys'])}, observed voxels {n_obs}, "
          f"max weight {wmax:.0f}")


@pytest.mark.parametrize("run", ["C5-far", "C5-end", "C4-run"])
def test_twin_mesh_equals_open3d_order_mesh(run):
    cfg, o3, tw = _both(run[:2], RUNS[run])
    ca, cb = B.canon(o3.extract_triangle_mesh()), B.canon(tw.extract_mesh())
    B.same_topology_and_vertices(ca, cb)
    assert np.abs(ca["colors"] - cb["colors"]).max() < 1e-5
    assert len(ca["triangles"]) > (10_000 if cfg.name == "C5" else 100_000)
    if cfg.name == "C5":                               # the vertices really are ~2 km out
        assert np.abs(ca["vertices"][:, 2]).min() > 1900.0


def test_far_c5_float64_colour_restatement_equals_open3d_order():
    """tests/_color64.py's float64 colour restatement, which the GPU float64-colour volume equals, against Open3D's
    float64 colours at the far end of the street."""
    cfg = S.CONFIGS["C5"]
    o3 = oracle.Open3DOrderVolume(cfg.voxel_size, cfg.sdf_trunc, 16, 4)
    tw = C64.Color64Twin(cfg)
    for i in RUNS["C5-far"]:
        d, c, T = S.render_frame(cfg, i)
        o3.integrate(d, c, cfg.K, T, cfg.depth_trunc, nthreads=B.NT)
        tw.integrate(d, c, cfg.K, T, nthreads=B.NT)
    a, b = sort_dump(o3.dump_blocks()), sort_dump(tw.dump_blocks())
    assert np.array_equal(a["keys"], b["keys"])
    assert np.array_equal(a["vox"][:, :2], b["vox"][:, :2].astype(np.float64))
    assert np.array_equal(a["vox"][:, 2:].view(np.uint64), b["rgb64"].view(np.uint64))
    ma = B.canon(o3.extract_triangle_mesh())
    mb = B.canon(C64.mesh(tw.tw.extract_mesh(), tw.dump_blocks()))
    B.same_topology_and_vertices(ma, mb)
    assert np.array_equal(ma["colors"].view(np.uint64), mb["colors"].view(np.uint64))


def test_the_far_street_is_far():
    """Census of the far runs: the camera is over 1.9 km from the origin, voxel centres have a float32 ulp of at least
    1e-4 m (a tenth of a millimetre, 1/1000 of a 10 cm voxel), and the bench's C5 frames reach the same distance."""
    cfg = S.CONFIGS["C5"]
    for i in RUNS["C5-far"] + RUNS["C5-end"]:
        Twc = S.inv_T(S.pose_Tcw(cfg, i))
        assert np.linalg.norm(Twc[:3, 3]) > 1900.0
    _, _, tw = _both("C5", RUNS["C5-far"][:2])
    keys = tw.dump_blocks()["keys"]
    assert B.centre_ulp(keys, cfg.voxel_size) >= 1e-4
    # the bench's 300 C5 frames: every 15th frame of the street, the last at z = 0.44 * 4485 m
    step = cfg.n_frames // B.BENCH_FRAMES
    assert step == 15 and 0.44 * step * (B.BENCH_FRAMES - 1) > 1970.0
