"""GPU: the TSDF volume's asynchronous host code across call sequences, against the CPU twin (oracle/tsdf_oracle.c)
fed the same frames in call order.

The deterministic tests hold one stream back with a bounded `torch.cuda._sleep` (a "stall", ~50 ms, never more than
200 ms) so that work enqueued after it would run out of order every time, not sometimes.  Each asserts that the stall
is still pending when it makes the call under test; if it is not, the test fails with a message saying that its
premise did not hold (it neither skips nor retries).  Three kinds of ordering are pinned down:

* calls on different streams (a caller's, another caller's, the library's own) update the map in call order, and
  every synchronising call (dump, extraction, reset, save, capacity) waits for all of them;
* the wrapper keeps device and pinned host inputs referenced until the work that reads them is done, so torch's
  caching allocators cannot hand their memory to a new tensor while queued kernels or copies still read it;
* device frames passed without a stream are read after the work torch queued before the call (their producers).

Every test ends with its work synchronised."""

import numpy as np
import pytest

import oracle
from pyslam_b200 import B200TsdfVolume
from pyslam_b200 import synthetic as S
from tests import _tsdf_sequences as Q
from tests._util import sort_dump, sorted_keys

pytestmark = pytest.mark.gpu

STALL_MS, STALL_MS_MAX = 50.0, 200.0
T0 = S.CONFIGS["T0"]


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def stall_cycles(torch):
    """`torch.cuda._sleep` cycles of one ~50 ms stall, calibrated once with CUDA events; a stall measured above 200 ms
    fails the calibration."""
    s = torch.cuda.Stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(cycles):
        with torch.cuda.stream(s):
            e0.record(s)
            torch.cuda._sleep(cycles)
            e1.record(s)
        e1.synchronize()
        return e0.elapsed_time(e1)

    timed(1 << 20)
    probe = 1 << 22
    cycles = int(probe * STALL_MS / max(timed(probe), 1e-3))
    ms = timed(cycles)
    assert 0.5 * STALL_MS < ms <= STALL_MS_MAX, f"stall calibration: {cycles} cycles took {ms:.1f} ms"
    torch.cuda.synchronize()
    return cycles


@pytest.fixture
def stall(torch, stall_cycles):
    """stall(stream) holds `stream` back: it waits for an event that fires when a ~50 ms sleep on a stream of its own
    ends; returns the event.  The sleep does not run on `stream` itself: a kernel running on a stream can also hold up
    work on other streams (here: pageable uploads), which would hide the misordering under test."""
    sleeper = torch.cuda.Stream()

    def _stall(stream):
        with torch.cuda.stream(sleeper):
            torch.cuda._sleep(stall_cycles)
        ev = torch.cuda.Event()
        ev.record(sleeper)
        stream.wait_event(ev)
        return ev
    yield _stall
    torch.cuda.synchronize()


def _assert_pending(ev, what):
    assert ev.query() is False, (f"premise not met: the stall had already ended when {what} was called, so this run "
                                 "says nothing about the ordering under test")


def _frames(cfg, idx):
    return [S.render_frame(cfg, i) for i in idx]


def _pair(cfg, capacity=1 << 14, max_capacity=None):
    """A volume primed for `cfg`'s frames, and its twin.  Priming (one frame, then a reset) sizes the staging and
    writes the lambda image, the two steps that drain the whole device: a first call would otherwise wait for the
    stall it is meant to queue behind."""
    vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=capacity,
                         max_capacity_blocks=max_capacity)
    d, c, T = S.render_frame(cfg, 0)
    vol.integrate(d, c, cfg.K, T)
    vol.reset()
    orc = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    return vol, orc


def _feed(orc, cfg, frames):
    for d, c, T in frames:
        orc.integrate(d, c, cfg.K, T, nthreads=8)


def _dev(torch, frames):
    """device [n,H,W] depth and [n,H,W,3] colour of `frames`, and the [n,4,4] poses"""
    D = torch.from_numpy(np.stack([f[0] for f in frames])).cuda()
    Cc = torch.from_numpy(np.stack([f[1] for f in frames])).cuda()
    return D, Cc, np.stack([f[2] for f in frames])


def _assert_same_blocks(got, orc, what=""):
    a, b = sort_dump(got), sort_dump(orc.dump_blocks())
    assert len(b["keys"]) > 0
    assert np.array_equal(a["keys"], b["keys"]), f"{what}: block keys differ from the twin"
    if "hashes" in a:
        assert np.array_equal(a["hashes"], b["hashes"]), f"{what}: block hashes differ from the twin"
    for p, name in enumerate(("tsdf", "weight", "r", "g", "b")):
        assert np.array_equal(a["vox"][:, p], b["vox"][:, p]), f"{what}: the {name} plane differs from the twin"


def _assert_same_mesh(m, orc):
    got = oracle.canonical_mesh(m.vertices, m.vertex_colors, m.edge_ids, m.triangles)
    ref = orc.extract_mesh()
    want = oracle.canonical_mesh(ref["vertices"], ref["colors"], ref["edges"], ref["triangles"])
    assert len(want["triangles"]) > 0
    for k in want:
        assert np.array_equal(got[k], want[k]), f"mesh {k} differ from the twin's"


# ---------------------------------------------------------------------------------------------------------------
# calls on different streams
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("drain", ["dump_blocks", "extract_mesh", "reset", "save_state", "capacity"])
def test_drains_wait_for_every_stream(torch, stall, drain, tmp_path):
    """Frames on a stalled caller stream, then a host frame on the library's streams, then a synchronising call:
    it waits for the caller stream's frames too (a reset must not clear the pool under their updates; a growable
    volume's skipped groups are replayed after them)."""
    fr = _frames(T0, range(6))
    growable = drain == "capacity"
    vol, orc = _pair(T0, capacity=64 if growable else 1 << 14, max_capacity=1 << 14 if growable else None)
    vol.set_overlap(False)
    D, Cc, T = _dev(torch, fr[:3])
    s = torch.cuda.Stream()
    ev = stall(s)
    vol.integrate_batch(D, Cc, T0.K, T, stream=s.cuda_stream)
    _assert_pending(ev, "the library-stream integrate")
    vol.integrate(*fr[3][:2], T0.K, fr[3][2])
    _assert_pending(ev, drain)
    if drain == "dump_blocks":
        got = vol.dump_blocks()
    elif drain == "extract_mesh":
        m = vol.extract_mesh()
    elif drain == "reset":
        vol.reset()
        for d, c, t in fr[4:]:
            vol.integrate(d, c, T0.K, t)
    elif drain == "save_state":
        path = str(tmp_path / "map.npz")
        vol.save_state(path)
    else:
        cap, growths = vol.capacity()
    _feed(orc, T0, fr[:4])
    if drain == "reset":
        orc.reset()
        _feed(orc, T0, fr[4:])
    elif drain == "extract_mesh":
        _assert_same_mesh(m, orc)
    elif drain == "save_state":
        vol, _ = _pair(T0)
        vol.load_state(path)
    elif drain == "capacity":
        assert growths >= 1 and cap >= orc.num_blocks()
    _assert_same_blocks(got if drain == "dump_blocks" else vol.dump_blocks(), orc, drain)
    torch.cuda.synchronize()


def test_library_streams_then_caller_stream(torch, stall):
    """Device frames on the library's streams held back by a stalled input event (overlap off), then frames on a
    caller stream: the caller stream's updates wait for the library's."""
    fr = _frames(T0, range(6))
    vol, orc = _pair(T0)
    vol.set_overlap(False)
    A, B = _dev(torch, fr[:3]), _dev(torch, fr[3:])
    ev = stall(torch.cuda.Stream())
    vol.set_input_event(ev.cuda_event)
    vol.integrate_batch(*A[:2], T0.K, A[2])
    s2 = torch.cuda.Stream()
    _assert_pending(ev, "the caller-stream integrate")
    vol.integrate_batch(*B[:2], T0.K, B[2], stream=s2.cuda_stream)
    _feed(orc, T0, fr)
    _assert_same_blocks(vol.dump_blocks(), orc, "library -> S")
    torch.cuda.synchronize()


def test_caller_stream_then_another_caller_stream(torch, stall):
    """Frames on a stalled caller stream S1, then frames on S2 (overlap off)."""
    fr = _frames(T0, range(6))
    vol, orc = _pair(T0)
    vol.set_overlap(False)
    A, B = _dev(torch, fr[:3]), _dev(torch, fr[3:])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    ev = stall(s1)
    vol.integrate_batch(*A[:2], T0.K, A[2], stream=s1.cuda_stream)
    _assert_pending(ev, "the S2 integrate")
    vol.integrate_batch(*B[:2], T0.K, B[2], stream=s2.cuda_stream)
    _feed(orc, T0, fr)
    _assert_same_blocks(vol.dump_blocks(), orc, "S1 -> S2")
    torch.cuda.synchronize()


def test_caller_stream_then_library_streams_with_overlap_on_a_large_batch(torch, stall):
    """A 64-frame C2 batch on a stalled caller stream, then single device frames on the library's streams with overlap
    on (their allocation may overlap the batch's updates, their updates may not).  Device frames: a pageable upload
    could wait for the stalled batch and so hold the calls under test back until the stall is over."""
    cfg = S.CONFIGS["C2"]
    fr = _frames(cfg, range(0, 136, 2))
    vol, orc = _pair(cfg, capacity=1 << 17)
    D, Cc, T = _dev(torch, fr[:64])
    B = _dev(torch, fr[64:])
    s = torch.cuda.Stream()
    ev = stall(s)
    vol.integrate_batch(D, Cc, cfg.K, T, stream=s.cuda_stream)
    _assert_pending(ev, "the library-stream integrate")
    for k in range(len(fr) - 64):
        vol.integrate(B[0][k], B[1][k], cfg.K, B[2][k])
    _assert_pending(ev, "the last library-stream integrate returned")
    _feed(orc, cfg, fr)
    _assert_same_blocks(vol.dump_blocks(), orc, "S -> library, overlap on")
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------
# input lifetime
# ---------------------------------------------------------------------------------------------------------------
def _hold_back_allocation(torch, vol, stall, fr, group_size=16):
    """A device batch of `fr` whose allocation waits for a stalled input event: every later allocation of the volume
    (and every host upload into a group buffer that batch uses) queues behind it.  Returns the event."""
    D, Cc, T = _dev(torch, fr)
    vol.set_group_size(group_size)
    ev = stall(torch.cuda.Stream())
    vol.set_input_event(ev.cuda_event)
    vol.integrate_batch(D, Cc, T0.K, T)
    return ev


def _overwrite_freed(torch, shapes, pinned=False):
    """New tensors of the freed frames' sizes, filled with other data on torch's stream; their addresses"""
    junk = []
    for shape, dtype, value in shapes:
        t = torch.empty(shape, dtype=dtype, pin_memory=True) if pinned else torch.empty(shape, dtype=dtype,
                                                                                           device="cuda")
        t.fill_(value)
        junk.append(t)
    return junk, {t.data_ptr() for t in junk}


def test_device_frames_outlive_the_wrapper_references(torch, stall):
    """Ten single device frames only the wrapper references (it used to keep the last eight), while their allocation
    is held back; torch then allocates and fills tensors of the same sizes."""
    fr = _frames(T0, range(14))
    vol, orc = _pair(T0)
    H, W = T0.height, T0.width
    shapes = [((H, W), torch.float32, 1.5), ((H, W, 3), torch.uint8, 200)] * 10
    warm, _ = _overwrite_freed(torch, shapes * 3)   # cached free memory: the overwrite below allocates no new memory
    del warm
    inputs = [(torch.from_numpy(d).cuda(), torch.from_numpy(c).cuda()) for d, c, _ in fr[4:]]
    ptrs = {x.data_ptr() for pair in inputs for x in pair}
    ev = _hold_back_allocation(torch, vol, stall, fr[:4])
    for _, _, t in fr[4:]:
        _assert_pending(ev, "integrate")
        vol.integrate(*inputs.pop(0), T0.K, t)
    junk, reused = _overwrite_freed(torch, shapes)
    _assert_pending(ev, "the overwrite")
    _feed(orc, T0, fr)
    _assert_same_blocks(vol.dump_blocks(), orc, f"{len(reused & ptrs)} freed input buffers reused")
    torch.cuda.synchronize()


def test_device_frame_outlives_a_following_host_batch(torch, stall):
    """One single device frame only the wrapper references, then a host batch (which used to replace the held
    list), then torch reuses memory of the frame's size."""
    fr = _frames(T0, range(8))
    vol, orc = _pair(T0)
    dd, cc = torch.from_numpy(fr[4][0]).cuda(), torch.from_numpy(fr[4][1]).cuda()
    ptrs = {dd.data_ptr(), cc.data_ptr()}
    ev = _hold_back_allocation(torch, vol, stall, fr[:4])
    _assert_pending(ev, "integrate")
    vol.integrate(dd, cc, T0.K, fr[4][2])
    del dd, cc
    vol.integrate_batch(np.stack([f[0] for f in fr[5:]]), np.stack([f[1] for f in fr[5:]]), T0.K,
                        np.stack([f[2] for f in fr[5:]]))
    H, W = T0.height, T0.width
    junk, reused = _overwrite_freed(torch, [((H, W), torch.float32, 1.5), ((H, W, 3), torch.uint8, 200)] * 2)
    _assert_pending(ev, "the overwrite")
    _feed(orc, T0, fr)
    _assert_same_blocks(vol.dump_blocks(), orc, f"{len(reused & ptrs)} freed input buffers reused")
    torch.cuda.synchronize()


def test_pinned_host_frames_outlive_the_wrapper_references(torch, stall):
    """Ten single pinned host frames whose uploads wait for group buffers held back by a stalled allocation (four
    one-frame groups); torch's pinned allocator then hands out and fills blocks of the same size."""
    fr = _frames(T0, range(14))
    vol, orc = _pair(T0)
    inputs = [(torch.from_numpy(d).pin_memory(), torch.from_numpy(c).pin_memory()) for d, c, _ in fr[4:]]
    ptrs = {x.data_ptr() for pair in inputs for x in pair}
    ev = _hold_back_allocation(torch, vol, stall, fr[:4], group_size=1)
    for _, _, t in fr[4:]:
        _assert_pending(ev, "integrate")
        vol.integrate(*inputs.pop(0), T0.K, t)
    H, W = T0.height, T0.width
    junk, reused = _overwrite_freed(torch, [((H, W), torch.float32, 1.5), ((H, W, 3), torch.uint8, 200)] * 10,
                                    pinned=True)
    _assert_pending(ev, "the overwrite")
    _feed(orc, T0, fr)
    _assert_same_blocks(vol.dump_blocks(), orc, f"{len(reused & ptrs)} freed pinned buffers reused")
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------
# producers of device frames
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch", [False, True])
def test_device_frames_without_a_stream_follow_their_producer(torch, stall, batch):
    """The frames are copied into zeroed tensors on torch's current stream behind a stall, then integrated with no
    stream: the map is the real frames' map, not the zeros'."""
    fr = _frames(T0, range(3) if batch else range(1))
    vol, orc = _pair(T0)
    src_d, src_c, T = _dev(torch, fr)
    dst_d, dst_c = torch.zeros_like(src_d), torch.zeros_like(src_c)
    torch.cuda.synchronize()
    ev = stall(torch.cuda.current_stream())
    dst_d.copy_(src_d)
    dst_c.copy_(src_c)
    _assert_pending(ev, "integrate")
    if batch:
        vol.integrate_batch(dst_d, dst_c, T0.K, T)
    else:
        vol.integrate(dst_d[0], dst_c[0], T0.K, T[0])
    _feed(orc, T0, fr)
    _assert_same_blocks(vol.dump_blocks(), orc, "producer on torch's stream")
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------
# randomised call sequences (tests/_tsdf_sequences.py) on a fixed volume, a growable one and three hash shards
# ---------------------------------------------------------------------------------------------------------------
_SETUPS = ([dict(name="fixed", capacity_blocks=1 << 16),
            dict(name="growable", capacity_blocks=64, max_capacity_blocks=1 << 16)]
           + [dict(name=f"shard{r}", capacity_blocks=1 << 16, shard_rank=r, shard_count=3) for r in range(3)])
_RECT_D = np.array([0.05, -0.02, 0.001, -0.001, 0.0])


class _SequenceRunner:
    """Feeds one step at a time to every setup and to the twin (the frames in call order, rectified with cv2.remap,
    uint16 depth widened as float32(d) * float32(scale)), and checks the setups against the twin."""

    def __init__(self, torch, stall, tmp_path):
        self.torch, self.stall, self.tmp = torch, stall, tmp_path
        self.vols = [self._new(spec) for spec in _SETUPS]
        self.orc = oracle.TsdfOracle(T0.voxel_size, T0.sdf_trunc, T0.depth_trunc)
        self.settings = {}            # mode calls made so far, replayed into volumes loaded from a state file
        self.rect = None              # (shape, map_x, map_y, swap)
        self.streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        self.cache = {}
        self.n_mesh_checks = 0

    @staticmethod
    def _new(spec):
        kw = {k: v for k, v in spec.items() if k != "name"}
        return B200TsdfVolume(T0.voxel_size, T0.sdf_trunc, T0.depth_trunc, **kw)

    def _frame(self, shape, kvar, i):
        key = (shape, kvar, i)
        if key not in self.cache:
            import dataclasses
            w, h = Q.SHAPES[shape]
            fx, fy, cx, cy = Q.intrinsics(shape, kvar)
            self.cache[key] = S.render_frame(dataclasses.replace(T0, width=w, height=h, fx=fx, fy=fy, cx=cx, cy=cy), i)
        return self.cache[key]

    def _apply_settings(self, vol):
        for op, arg in self.settings.items():
            if op == "rectify":
                vol.set_rectification(arg[1], arg[2], swap_rb=arg[3])
            else:
                getattr(vol, "set_" + op)(arg)

    # ---- steps ----
    def step(self, s):
        op = s["op"]
        if op == "frames":
            self._frames(s)
            return
        if op in ("group_size", "fusion", "overlap"):
            self.settings[op] = s["value"]
            for v in self.vols:
                getattr(v, "set_" + op)(s["value"])
        elif op == "rectify":
            self._rectify(s)
        elif op == "upload":
            self._upload(s)
        elif op == "reset":
            for v in self.vols:
                v.reset()
            self.orc.reset()
        elif op == "save_load":
            loaded = []
            for spec, v in zip(_SETUPS, self.vols):
                path = str(self.tmp / f"{spec['name']}.npz")
                v.save_state(path)
                v.close()
                w = self._new(spec)
                w.load_state(path)
                self._apply_settings(w)
                loaded.append(w)
            self.vols = loaded
        elif s["what"] == "capacity":
            for v in self.vols:
                v.capacity()
        elif s["what"] == "dump":
            for v in self.vols:
                v.dump_blocks()
        else:
            self._check_extraction(s["what"])
        self.check_blocks(op)

    def _rectify(self, s):
        import cv2
        if s["value"] is None:
            self.rect = None
            self.settings.pop("rectify", None)
            for v in self.vols:
                v.set_rectification(None, None)
            return
        w, h = Q.SHAPES[s["value"]]
        fx, fy, cx, cy = Q.intrinsics(s["value"], "base")
        Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])
        mx, my = cv2.initUndistortRectifyMap(Km, _RECT_D, None, Km, (w, h), cv2.CV_32FC1)
        self.rect = (s["value"], mx, my, s["swap"])
        self.settings["rectify"] = self.rect
        for v in self.vols:
            v.set_rectification(mx, my, swap_rb=s["swap"])

    def _upload(self, s):
        from pyslam_b200.sharding import owner_of
        rng = np.random.default_rng(s["seed"])
        have = self.orc.dump_blocks()["keys"]
        taken = {tuple(k) for k in have}
        keys = [tuple(have[i]) for i in rng.choice(len(have), min(s["n_replace"], len(have)), replace=False)]
        while len(keys) < s["n_replace"] + s["n_new"]:
            k = tuple(int(x) for x in rng.integers(-24, 24, 3))
            if k not in taken:
                taken.add(k)
                keys.append(k)
        keys = np.array(keys, np.int32).reshape(-1, 3)
        vox = np.empty((len(keys), 5, 512), np.float32)
        vox[:, 0] = rng.uniform(-1, 1, (len(keys), 512))
        vox[:, 1] = rng.integers(0, 6, (len(keys), 512))
        vox[:, 2:] = rng.uniform(0, 255, (len(keys), 3, 512))
        for k, x in zip(keys, vox):
            self.orc.set_block(k, x)
        own = owner_of(keys, 3)
        for spec, v in zip(_SETUPS, self.vols):
            sel = own == spec["shard_rank"] if "shard_rank" in spec else np.ones(len(keys), bool)
            if sel.any():
                v.upload_blocks(keys[sel], vox[sel])

    def _frames(self, s):
        import cv2
        torch = self.torch
        fr = [self._frame(s["shape"], s["kvar"], i) for i in s["frames"]]
        K = Q.intrinsics(s["shape"], s["kvar"])
        D, Cc, T = (np.stack([f[k] for f in fr]) for k in range(3))
        u16 = s["kind"] in ("host_u16", "cuda_u16")
        D16 = np.clip(np.round(D / Q.DEPTH_SCALE), 0, 65535).astype(np.uint16) if u16 else None
        Dt = D16.astype(np.float32) * np.float32(Q.DEPTH_SCALE) if u16 else D
        Ct = Cc
        Cl = np.ascontiguousarray(Cc[..., ::-1]) if self.rect and self.rect[3] else Cc   # BGR in with swap_rb
        if self.rect:
            _, mx, my, _ = self.rect
            Dt = np.stack([cv2.remap(d, mx, my, cv2.INTER_NEAREST) for d in Dt])
            Ct = np.stack([cv2.remap(c, mx, my, cv2.INTER_LINEAR) for c in Cc])
        n, off = len(fr), s["offset"]
        dsrc = D16 if u16 else D
        if s["kind"] in Q.DEVICE_KINDS:
            dd = torch.zeros((off + n,) + dsrc.shape[1:], dtype=torch.from_numpy(dsrc[:1]).dtype, device="cuda")
            cc = torch.zeros((off + n,) + Cl.shape[1:], dtype=torch.uint8, device="cuda")
            dd[off:].copy_(torch.from_numpy(dsrc))
            cc[off:].copy_(torch.from_numpy(Cl))
            depth, color = dd[off:], cc[off:]
        elif s["kind"] == "pinned":
            depth, color = torch.from_numpy(dsrc).pin_memory(), torch.from_numpy(Cl).pin_memory()
        else:
            depth, color = dsrc, Cl
        stream = self.streams[s["stream"]] if s["stream"] is not None else None
        if s["stall"]:
            self.stall(stream if stream is not None else torch.cuda.current_stream())
        sh = stream.cuda_stream if stream is not None else None
        scale = Q.DEPTH_SCALE if u16 else None
        for v in self.vols:
            if s["event"]:
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream())
                v.set_input_event(ev.cuda_event)
            if s["entry"] == "batch":
                v.integrate_batch(depth, color, K, T, stream=sh, depth_scale=scale)
            else:
                v.integrate(depth[0], color[0], K, T[0], stream=sh, depth_scale=scale)
        del depth, color
        for d, c, t in zip(Dt, Ct, T):
            self.orc.integrate(d, c, K, t, nthreads=8)
        if s["entry"] == "integrate":
            want = sorted_keys(self.orc.last_touched())
            for v in self.vols[:2]:
                assert np.array_equal(sorted_keys(v.last_touched_keys()), want), "last touched keys"
                assert v.last_frame_stats()[0] == len(want), "last frame stats"

    # ---- checks ----
    def check_blocks(self, what):
        from pyslam_b200.sharding import merge_dumps
        want = sort_dump(self.orc.dump_blocks())
        parts = [v.dump_blocks() for v in self.vols[2:]]
        for r, p in enumerate(parts):
            assert np.all(p["hashes"] % np.uint64(3) == r), f"after {what}: shard {r} holds a block it does not own"
        for name, got in (("fixed", self.vols[0].dump_blocks()), ("growable", self.vols[1].dump_blocks()),
                          ("shards", merge_dumps(parts))):
            got = sort_dump(got)
            assert np.array_equal(got["keys"], want["keys"]), f"after {what}: {name} block keys differ from the twin"
            assert np.array_equal(got["hashes"], want["hashes"]), f"after {what}: {name} hashes differ"
            assert np.array_equal(got["vox"], want["vox"]), f"after {what}: {name} voxels differ from the twin"

    def _check_extraction(self, what):
        if self.orc.num_blocks() == 0:
            return
        self.n_mesh_checks += 1
        if what == "mesh":
            for v in self.vols[:2]:
                _assert_same_mesh(v.extract_mesh(), self.orc)
            return
        pw = oracle.numpy_point_cloud(self.orc.dump_blocks(), T0.voxel_size, 16)
        ow = np.lexsort(pw["points"].T[::-1])
        for v in self.vols[:2]:
            pc = v.extract_point_cloud()
            o = np.lexsort(pc.points.T[::-1])
            assert np.array_equal(pc.points[o], pw["points"][ow]), "point cloud positions"
            assert np.array_equal(pc.colors[o], pw["colors"][ow]), "point cloud colours"


@pytest.mark.parametrize("seed", Q.SEEDS)
def test_random_call_sequence_equals_the_twin(torch, stall, tmp_path, seed):
    """A seeded sequence of about 60 steps (frames of every input kind, stream, shape and intrinsics, mode switches,
    rectification, uploads, resets, save -> load -> continue, extractions) on a fixed volume, a growable one that
    starts at 64 blocks and three hash shards: bit for bit equal to the twin after every synchronising step and at the
    end; last touched keys and frame stats after every single frame; mesh and point cloud at 3 or more points."""
    run = _SequenceRunner(torch, stall, tmp_path)
    for s in Q.generate(seed):
        run.step(s)
    run.check_blocks("the sequence")
    assert run.n_mesh_checks >= 3
    for v in run.vols:
        v.synchronize()
    torch.cuda.synchronize()
