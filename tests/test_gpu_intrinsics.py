"""GPU: a change of intrinsics within one volume.  The update kernels read the depth-to-camera-distance multiplier
from the volume's lambda image, which is rewritten when K (or the image size) changes; update kernels of the previous
batch may still be running at that moment, on the library's streams or on the caller's."""

import numpy as np
import pytest

import oracle
from pyslam_b200 import B200TsdfVolume
from pyslam_b200 import synthetic as S
from tests._util import sort_dump

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("group,fused,device_inputs", [
    (32, True, True),      # fused groups, device frames on a caller stream
    (3, True, False),      # fused groups, host frames through the library's streams
    (16, False, True),     # frame by frame, device frames on a caller stream
])
def test_batches_with_different_intrinsics_back_to_back_match_oracle(group, fused, device_inputs):
    import torch
    cfg = S.CONFIGS["C1"]
    frames = [S.render_frame(cfg, i) for i in range(40)]
    D, Cc, T = (np.stack([f[k] for f in frames]) for k in range(3))
    K1 = cfg.K
    K2 = cfg.K * np.array([1.07, 0.96, 1.0, 1.0]) + np.array([0.0, 0.0, 5.5, -3.25])
    vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 16)
    vol.set_group_size(group)
    vol.set_fusion(fused)
    orc = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    halves = [(slice(0, 20), K1), (slice(20, 40), K2), (slice(0, 20), K1)]
    if device_inputs:
        stream = torch.cuda.Stream()
        Dd, Cd = torch.from_numpy(D).cuda(), torch.from_numpy(Cc).cuda()
        torch.cuda.synchronize()
        for sl, K in halves:   # enqueued back to back on the caller's stream, no synchronisation in between
            vol.integrate_batch(Dd[sl], Cd[sl], K, T[sl], stream=stream.cuda_stream)
        stream.synchronize()
    else:
        for sl, K in halves:
            vol.integrate_batch(D[sl], Cc[sl], K, T[sl])
    for sl, K in halves:
        for i in range(sl.start, sl.stop):
            orc.integrate(D[i], Cc[i], K, T[i])
    a, b = sort_dump(vol.dump_blocks()), sort_dump(orc.dump_blocks())
    for name in ("keys", "hashes", "vox"):
        assert np.array_equal(a[name], b[name]), name
