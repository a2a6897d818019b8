"""pyslam_b200 — H100-native volumetric TSDF integrator behind pySLAM's dense-mapping plugin API.

Scope: the hot path of SURVEY.md §8 only (voxel-block hash allocation, projective TSDF + colour
update, per-block marching cubes, and the point-average compat grid).  `csrc/` holds the sm_90a
CUDA kernels and the C ABI (include/b2v.h); the Python modules mirror the reference's interface.
"""

from .volume import (B200TsdfVolume, BoundingBox3D, CameraFrustrum, PointCloud, TBBUtils, TriangleMesh,
                     VoxelBlockGrid, VoxelBlockSemanticGrid, VoxelBlockSemanticProbabilisticGrid, VoxelGridData,
                     VoxelSemanticGrid, VoxelSemanticGridProbabilistic, filter_shadow_points, remap,
                     remap_instance_ids)

__all__ = ["B200TsdfVolume", "BoundingBox3D", "CameraFrustrum", "PointCloud", "TBBUtils", "TriangleMesh",
           "VoxelBlockGrid", "VoxelBlockSemanticGrid", "VoxelBlockSemanticProbabilisticGrid", "VoxelGridData",
           "VoxelSemanticGrid", "VoxelSemanticGridProbabilistic", "filter_shadow_points", "remap",
           "remap_instance_ids"]
