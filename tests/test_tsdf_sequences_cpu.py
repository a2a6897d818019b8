"""CPU: the committed call sequences of tests/_tsdf_sequences.py reach every transition they are for (stream switches,
with and without a stall before them; frame shape, intrinsics and input-kind changes; mode switches; lifecycle calls),
and each sequence stays valid: device-only options go with device frames, maps fit the frames they rectify."""

import numpy as np

from tests import _tsdf_sequences as Q


def test_committed_seeds_reach_every_transition():
    seen = set()
    for seed in Q.SEEDS:
        seen |= Q.transitions(Q.generate(seed))
    assert Q.REQUIRED - seen == set()


def test_sequences_are_deterministic_and_valid():
    for seed in Q.SEEDS:
        steps = Q.generate(seed)
        assert steps == Q.generate(seed) and 55 <= len(steps) <= 65
        rect = None
        n_checks = 0
        for s in steps:
            if s["op"] == "rectify":
                rect = s["value"]
            elif s["op"] == "extract":
                n_checks += s["what"] in ("mesh", "points")
            elif s["op"] == "frames":
                dev = s["kind"] in Q.DEVICE_KINDS
                assert dev or (s["stream"] is None and not s["event"] and not s["stall"] and s["offset"] == 0)
                assert s["kind"] != "cuda_u16" or s["entry"] == "batch"
                assert len(s["frames"]) == (1 if s["entry"] == "integrate" else len(s["frames"])) >= 1
                assert rect is None or rect == s["shape"]
                assert all(0 <= i < Q.N_FRAME_INDICES for i in s["frames"])
        assert n_checks >= 3


def test_intrinsics_variants_keep_the_size_and_change_k():
    for shape in Q.SHAPES:
        ks = [Q.intrinsics(shape, v) for v in Q.KVARS]
        assert all(np.all(k[:2] > 0) for k in ks)
        assert not np.array_equal(ks[0], ks[1]) and not np.array_equal(ks[0], ks[2])
