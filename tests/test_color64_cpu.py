"""CPU: the float64-colour restatement of tests/_color64.py against the literal Open3D-order restatement
(oracle/open3d_order.c), whose TSDFVoxel keeps an Eigen::Vector3d colour updated as (c * w + rgb) / (w + 1) in float64
(open3d_order.c:253-254), and against the float64 colours of tsdf_T0.npz.  Voxel colours and mesh colours are equal bit
for bit; keys, tsdf and weights are the block twin's.  Also the C ABI's config layout."""

import os

import numpy as np
import pytest

import oracle
from pyslam_b200 import synthetic as S
from tests import _color64 as C64
from tests._util import GOLDEN, sort_dump


def _run(cfg, frames):
    o3 = oracle.Open3DOrderVolume(cfg.voxel_size, cfg.sdf_trunc, 16, 4)
    tw = C64.Color64Twin(cfg)
    for i in frames:
        d, c, T = S.render_frame(cfg, i)
        o3.integrate(d, c, cfg.K, T, cfg.depth_trunc, nthreads=4)
        tw.integrate(d, c, cfg.K, T, nthreads=4)
    return o3, tw


@pytest.mark.parametrize("cfg_name,frames", [("T0", [0, 1, 2, 3]), ("C1", [0, 7]), ("C2", list(range(30))),
                                             ("C3", [0]), ("C4", [3]), ("C5", [0, 1])])
def test_f64_colour_equals_open3d_order(cfg_name, frames):
    o3, tw = _run(S.CONFIGS[cfg_name], frames)
    a, b = sort_dump(o3.dump_blocks()), sort_dump(tw.dump_blocks())
    assert np.array_equal(a["keys"], b["keys"])
    assert np.array_equal(a["vox"][:, :2], b["vox"][:, :2].astype(np.float64))
    assert np.array_equal(a["vox"][:, 2:].view(np.uint64), b["rgb64"].view(np.uint64)), "float64 colours differ"
    assert np.array_equal(b["vox"][:, 2:], b["rgb64"].astype(np.float32))   # vox holds them rounded
    assert (a["vox"][:, 1] > 0).sum() > 1000


def test_f64_mesh_colours_equal_open3d_order_and_the_golden():
    z = np.load(os.path.join(GOLDEN, "tsdf_T0.npz"))
    cfg = S.CONFIGS["T0"]
    o3, tw = _run(cfg, range(int(z["n_frames"])))
    ma = o3.extract_triangle_mesh()
    mb = C64.mesh(tw.tw.extract_mesh(), tw.dump_blocks())
    ca = oracle.canonical_mesh(ma["vertices"], ma["colors"], ma["edges"], ma["triangles"])
    cb = oracle.canonical_mesh(mb["vertices"], mb["colors"], mb["edges"], mb["triangles"])
    assert np.array_equal(ca["edges"], cb["edges"]) and np.array_equal(ca["triangles"], cb["triangles"])
    assert np.array_equal(ca["vertices"], cb["vertices"])
    assert np.array_equal(ca["colors"], cb["colors"])
    assert np.array_equal(cb["colors"], z["o3d_mesh_colors"])
    d = sort_dump(tw.dump_blocks())
    assert np.array_equal(d["keys"], z["keys"])
    assert np.array_equal(d["rgb64"], z["o3d_rgb64"])


def test_uploaded_weights_saturate_at_2_24():
    """Seeded blocks at weights 2^24 - 1 and 2^24: the restatement's weights stay the twin's (2^24 + 1 rounds to 2^24)
    and its colours follow (c * 2^24 + x) / 2^24 where the weight saturated."""
    cfg = S.CONFIGS["T0"]
    frames = [S.render_frame(cfg, i) for i in range(3)]
    seed = C64.Color64Twin(cfg)
    seed.integrate(*frames[0][:2], cfg.K, frames[0][2])
    s = sort_dump(seed.dump_blocks())
    for w in (16777215.0, 16777216.0):
        vox = s["vox"].copy()
        vox[:, 1] = np.where(vox[:, 1] > 0, np.float32(w), 0.0)
        tw = C64.Color64Twin(cfg)
        tw.upload(s["keys"], vox, s["rgb64"] + 1.0 / 3.0)
        for d, c, T in frames[1:]:
            tw.integrate(d, c, cfg.K, T)
        out = sort_dump(tw.dump_blocks())   # checks the weights against the twin's
        assert out["vox"][:, 1].max() == 16777216.0


def test_point_colours_take_float64_voxel_colours():
    """The point colour formula by hand on one point; the points and edges are oracle.numpy_point_cloud's."""
    cfg = S.CONFIGS["T0"]
    _, tw = _run(cfg, [0, 1, 2, 3])
    d = tw.dump_blocks()
    p64 = C64.point_cloud(d, cfg.voxel_size)
    p32 = oracle.numpy_point_cloud(dict(keys=d["keys"], vox=d["vox"]), cfg.voxel_size)
    assert len(p64["points"]) > 1000
    assert np.array_equal(p64["points"], p32["points"]) and np.array_equal(p64["edges"], p32["edges"])
    assert np.abs(p64["colors"] - p32["colors"]).max() < 1e-6
    assert not np.array_equal(p64["colors"], p32["colors"])
    e = p64["edges"][0]
    keys = {tuple(k): i for i, k in enumerate(d["keys"].tolist())}

    def voxel(g):
        b = keys[tuple(int(x) // 8 for x in g)]
        v = int(g[0] % 8) + 8 * int(g[1] % 8) + 64 * int(g[2] % 8)
        return d["vox"][b, 0, v], d["rgb64"][b, :, v]
    g1 = e[:3].copy()
    g1[e[3]] += 1
    (f0, c0), (f1, c1) = voxel(e[:3]), voxel(g1)
    r0, r1 = np.abs(f0), np.abs(f1)
    want = (c0 * np.float64(r1) + c1 * np.float64(r0)) / np.float64(r0 + r1) / 255.0
    assert np.array_equal(p64["colors"][0], want)


def test_config_with_color_f64_matches_the_header(tmp_path):
    """b2v_config's color_f64 is its last field, at the ctypes mirror's offset, and the struct keeps its size."""
    import ctypes
    import shutil
    import subprocess
    from pyslam_b200._lib import B2VConfig, B2VConfigEx
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    if not gcc:
        pytest.skip("gcc not available")
    names = [f[0] for f in B2VConfigEx._fields_]
    assert names[-1] == "color_f64"
    src = tmp_path / "layout.c"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b2v.h"\nint main(void) {\n'
                   + "".join(f'    printf("%zu\\n", offsetof(b2v_config, {n}));\n' for n in names)
                   + '    printf("%zu\\n", sizeof(b2v_config));\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    r = subprocess.run([gcc, "-std=c11", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    assert got == [getattr(B2VConfigEx, n).offset for n in names] + [ctypes.sizeof(B2VConfigEx)]
    assert ctypes.sizeof(B2VConfig) == ctypes.sizeof(B2VConfigEx)
