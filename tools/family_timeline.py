"""Run every kernel family once or twice on C2-shape frames, a short timeline of the grid_*, sem_*, remap_*,
shadow_*, depth_u16_*, mesh_* and lambda kernels for a profiler.
    python tools/family_timeline.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pyslam_b200 import (B200TsdfVolume, VoxelBlockGrid, VoxelBlockSemanticProbabilisticGrid, VoxelBlockSemanticGrid,  # noqa: E402
                         filter_shadow_points)
from pyslam_b200 import synthetic as S  # noqa: E402

cfg, depth, color, Tcw = bench.load_frames("C2", 16, 0, 1)
H, W = depth.shape[1:]
# point-average grid: fused RGBD front-end (+ shadow filter), get_voxels
g = VoxelBlockGrid(cfg.voxel_size, 8, capacity_blocks=1 << 17)
for i in range(4):
    g.integrate_rgbd(depth[i], color[i], cfg.K, S.inv_T(Tcw[i]), max_depth=cfg.depth_trunc, filter_shadow_points=(i % 2 == 0))
v = g.get_voxels(2)
print("grid voxels", len(v.points))
filter_shadow_points(depth[0])
# semantic grids: Bayesian and voting fusion through the RGBD front-end, read-outs
lab = (np.arange(H * W, dtype=np.int32).reshape(H, W) // 9973) % 40
for Cls in (VoxelBlockSemanticProbabilisticGrid, VoxelBlockSemanticGrid):
    sg = Cls(0.015, 8, capacity_blocks=1 << 16)
    for i in range(3):
        sg.integrate_rgbd(depth[i], color[i], cfg.K, S.inv_T(Tcw[i]), class_image=lab, object_image=lab % 7,
                          max_depth=cfg.depth_trunc)
    print("semantic voxels", len(sg.get_voxels(1, 0.0).points), "objects", len(sg.get_object_segments(1, 0.0).object_vector))
    sg.close()
# TSDF volume with GPU rectification + raw 16-bit depth + mesh / point extraction
vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 17)
jj, ii = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32))
vol.set_rectification(jj + 0.25, ii - 0.25, swap_rb=True)
raw = np.round(depth * 5000.0).astype(np.uint16)
vol.integrate_batch(raw[:8], color[:8], cfg.K, Tcw[:8], depth_scale=np.float32(1 / 5000.0))
vol.integrate(raw[8], color[8], cfg.K, Tcw[8], depth_scale=np.float32(1 / 5000.0))
m = vol.extract_mesh()
pc = vol.extract_point_cloud()
print("mesh", len(m.vertices), len(m.triangles), "points", len(pc.points))
