"""TEST INFRASTRUCTURE ONLY.  CPU oracle for the volumetric-integration hot path.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s `cpu_baseline` / `--impl reference`
legs may import this package; the product (`pyslam_b200/`) never does.

* `RefGrid`     - the UNMODIFIED reference `volumetric::VoxelBlockGrid` compiled from
                  /root/reference/cpp/volumetric (oracle/_ref/libref_grid.so): truth for block keys,
                  `BlockKeyHash`, local voxel index, counts and point/colour running sums.
* `RefSemanticGrid` - the UNMODIFIED reference `VoxelBlockSemanticGrid` / `VoxelBlockSemanticProbabilisticGrid`
                  (oracle/_ref/libref_semantic.so): truth for label voting / Bayesian label fusion.
* `TsdfOracle`  - C restatement of Open3D's legacy ScalableTSDFVolume under decision D1
                  (oracle/tsdf_oracle.c): truth for tsdf / weight / rgb and the mesh.
                  PARITY UNPINNED against Open3D itself (not installed, not vendored).
* `Open3DOrderVolume` - ScalableTSDFVolume restated in OPEN3D'S OWN operation order and types (16^3 units,
                  incremental `p += vl*E[:,2]`, true divisions, float64 colour; oracle/open3d_order.c): the independent
                  truth the twin above and the kernels are measured against, with the tolerances of SURVEY.md 8c.
* `numpy_tsdf`  - a second, independent numpy restatement of A.3 used to pin the C oracle.
* `numpy_point_cloud` - numpy restatement of the documented ExtractPointCloud formulas (DESIGN §3) on a block dump.
* `numpy_grid`  - numpy restatement of the point-average `VoxelBlockGrid` (keys, sums, queries, carve).
* `numpy_semantic_grid` - plain Python / numpy restatement of both semantic block grids (label voting, Bayesian label
                  fusion with the kernel's 8-slot eviction, read-outs, edits, carve, instance association).
* `numpy_shadow_filter` - numpy restatement of the reference's `filter_shadow_points` (median threshold).
"""

from .oracle import (EigenOps, Open3DOrderVolume, have_eigen_ops, open3d_order_inverse4, RefGrid, RefSemanticGrid, TsdfOracle, build, canonical_mesh, have_ref, have_ref_semantic, numpy_grid, numpy_integrate_block,
                     numpy_point_cloud, numpy_semantic_grid, numpy_shadow_filter, numpy_touched_blocks, ref_block_key_hash, ref_floor_div, ref_keys)

__all__ = ["EigenOps", "have_eigen_ops", "open3d_order_inverse4", "Open3DOrderVolume", "RefGrid", "RefSemanticGrid", "TsdfOracle", "build", "canonical_mesh", "have_ref", "have_ref_semantic", "numpy_grid", "numpy_integrate_block",
           "numpy_point_cloud", "numpy_semantic_grid", "numpy_shadow_filter", "numpy_touched_blocks", "ref_block_key_hash", "ref_floor_div", "ref_keys"]
