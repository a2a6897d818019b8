"""Multi-GPU partitioning of the voxel-block hash space (SURVEY.md §8e).

One process per GPU.  A block belongs to rank `BlockKeyHash(key) % world` — the reference's own hash
(`cpp/volumetric/voxel_hashing.h:106-113`), so ownership is reproducible from the keys alone.  Every rank
integrates every frame into the blocks it owns (`b2v_config.shard_rank / shard_count`).

* Ingest (`FrameIngest`): a frame crosses PCIe ONCE in the whole job - rank r uploads 1/world of every chunk of
  frames over its own link and the chunk is completed GPU <-> GPU by an NCCL all-gather over NVLink / NVSwitch on a
  side stream, overlapped with the kernels of the previous chunk.
* Mesh extraction needs the +1-voxel halos of blocks that may live on another rank.  `extract_mesh_sharded` /
  `extract_point_cloud_sharded` exchange only those faces (one all_to_all of halo records) and mesh every shard on its
  own GPU; the pieces are welded on one rank (DESIGN.md §7).  The per-rank steps are public (`halo_records`,
  `mesh_piece`, `point_piece`, `weld`) so that N shards held in one process can run them too.
  `extract_mesh_distributed` is the older route: `gather_blocks_device` collects all shards on one rank GPU-to-GPU over
  NCCL (`gather_blocks` is the host-array variant used with gloo in the CPU tests), which then meshes the union.

The point-average and semantic grids shard the same way (`shard_rank` / `shard_count`; DESIGN.md §7, "Sharded grids"):
every rank is fed every frame and keeps its own blocks, voxel edits apply per rank, and the read-outs are gathered
(`get_voxels_sharded`, `get_object_segments_sharded`, ...).  The one step that is not per voxel, the instance -> object
association, exchanges vote triples: `association_votes` on every rank, then `resolve_association` of all ranks'
triples on every rank (`assign_object_ids_to_instance_ids_sharded` runs both over a process group).
"""

from __future__ import annotations

import numpy as np


def block_key_hash(keys) -> np.ndarray:
    """`BlockKeyHash` of int32 keys [n,3] as uint64 (sign-extending, like libstdc++'s identity hash)."""
    k = np.asarray(keys, dtype=np.int32).reshape(-1, 3).astype(np.int64).astype(np.uint64)
    return k[:, 0] ^ (k[:, 1] << np.uint64(1)) ^ (k[:, 2] << np.uint64(2))


def owner_of(keys, world: int) -> np.ndarray:
    """Rank owning each block key."""
    return (block_key_hash(keys) % np.uint64(world)).astype(np.int64)


def merge_dumps(dumps):
    """Union of per-rank block dumps, sorted by key: any dicts of per-block arrays with a "keys" entry, such as
    `B200TsdfVolume.dump_blocks` (keys / hashes / vox) or a grid's `dump_blocks`."""
    keys = np.concatenate([d["keys"] for d in dumps])
    order = np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))
    return {name: np.concatenate([d[name] for d in dumps])[order] for name in dumps[0]}


def chunk_plan(n_frames: int, world: int, chunk_frames: int):
    """Split a batch into chunks of <= chunk_frames frames.  -> [(first frame, frame count, q)]: rank r uploads the
    frames [first + r*q, first + min((r+1)*q, count)) of the chunk (q = ceil(count / world)) into segment r of the
    chunk buffer, so after the all-gather of the world q-frame segments the chunk's frames are contiguous and in
    frame order (the last segments of a ragged chunk may be partly or wholly padding)."""
    plan = []
    c0 = 0
    while c0 < n_frames:
        cnt = min(chunk_frames, n_frames - c0)
        plan.append((c0, cnt, -(-cnt // world)))
        c0 += cnt
    return plan


class FrameIngest:
    """Frame-split ingest of a hash-sharded volume: `integrate_batch(depths, colors, K, poses)` with HOST frames
    (pinned numpy arrays or torch tensors; every rank passes the same batch) is, per chunk of `chunk_frames`:

        upload stream   H2D of this rank's 1/world share of the chunk (its own PCIe link)
        gather stream   all-gather of the shares (NCCL over NVLink; in place in the chunk buffer)
        compute stream  volume.integrate_batch(chunk buffer, device pointers)   [allocate + fused update kernels]

    with `buffers` chunk buffers in rotation: the upload of chunk c+2, the all-gather of chunk c+1 and the kernels of
    chunk c run concurrently (three streams, events between them).
    Frame order is unchanged, so the result is bit-identical to a single-GPU `integrate_batch` of the batch.
    world = 1 (or no process group) degenerates to a chunked, double-buffered upload.  `depth_scale`: the depths are
    raw uint16 (2 bytes per pixel over PCIe AND NVLink), widened on the GPU."""

    def __init__(self, volume, group=None, chunk_frames: int = 64, buffers: int = 4, device=None):
        import torch
        import torch.distributed as dist
        self.volume = volume
        self.group = group
        self.dist = dist if (dist.is_available() and dist.is_initialized()) else None
        self.world = self.dist.get_world_size(group) if self.dist else 1
        self.rank = self.dist.get_rank(group) if self.dist else 0
        self.chunk_frames = int(chunk_frames)
        self.device = torch.device(device) if device is not None else torch.device("cuda", volume.device)
        self.cuda = self.device.type == "cuda"
        self.n_buffers = int(buffers)
        self._bufs = None
        self._shape = None
        if self.cuda:
            self.s_up = torch.cuda.Stream(self.device)
            self.s_gather = torch.cuda.Stream(self.device)
            self.s_int = torch.cuda.Stream(self.device)
        self.h2d_bytes = 0       # bytes this rank uploaded (accounting for bench.py)
        self.gather_bytes = 0    # bytes this rank received from its peers

    def _ensure(self, H, W, ddtype):
        import torch
        shape = (H, W, ddtype)
        if self._shape == shape:
            return
        if self.cuda and self._bufs is not None:
            torch.cuda.synchronize(self.device)
        cap = -(-self.chunk_frames // self.world) * self.world   # room for world equal segments
        self._bufs = []
        for _ in range(self.n_buffers):
            b = dict(depth=torch.empty((cap, H, W), dtype=ddtype, device=self.device),
                     color=torch.empty((cap, H, W, 3), dtype=torch.uint8, device=self.device))
            if self.cuda:
                b["free"] = torch.cuda.Event()
                b["uploaded"] = torch.cuda.Event()
                b["ready"] = torch.cuda.Event()
            self._bufs.append(b)
        self._shape = shape

    def integrate_batch(self, depths, colors, K, poses, depth_scale=None):
        import contextlib
        import torch
        D = depths if torch.is_tensor(depths) else torch.from_numpy(np.ascontiguousarray(depths))
        Cc = colors if torch.is_tensor(colors) else torch.from_numpy(np.ascontiguousarray(colors))
        T = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(-1, 4, 4))
        n, H, W = int(D.shape[0]), int(D.shape[1]), int(D.shape[2])
        if tuple(Cc.shape) != (n, H, W, 3) or T.shape[0] != n:
            raise RuntimeError("depths must be [n,H,W], colors [n,H,W,3], poses [n,4,4]")
        if depth_scale is None and D.dtype != torch.float32:
            raise RuntimeError("depths must be float32 (or uint16 with depth_scale)")
        self._ensure(H, W, D.dtype)
        world, r = self.world, self.rank
        up = torch.cuda.stream(self.s_up) if self.cuda else contextlib.nullcontext()
        ga = torch.cuda.stream(self.s_gather) if self.cuda else contextlib.nullcontext()
        for i, (c0, cnt, q) in enumerate(chunk_plan(n, world, self.chunk_frames)):
            b = self._bufs[i % self.n_buffers]
            lo, hi = min(r * q, cnt), min((r + 1) * q, cnt)
            with up:
                if self.cuda:
                    self.s_up.wait_event(b["free"])      # the kernels that read this buffer last are done
                if hi > lo:
                    b["depth"][lo:hi].copy_(D[c0 + lo:c0 + hi], non_blocking=True)
                    b["color"][lo:hi].copy_(Cc[c0 + lo:c0 + hi], non_blocking=True)
                    self.h2d_bytes += (hi - lo) * H * W * (D.element_size() + 3)
                if self.cuda:
                    b["uploaded"].record(self.s_up)
            with ga:
                if self.cuda:
                    self.s_gather.wait_event(b["uploaded"])
                if world > 1:
                    # in place: segment r of the buffer is this rank's contribution
                    for t in (b["depth"], b["color"]):
                        if t.dtype == torch.uint16:      # no uint16 in NCCL / gloo: gather the same bytes as uint8
                            t = t.view(torch.uint8)
                        self.dist.all_gather_into_tensor(t[:world * q], t[r * q:(r + 1) * q], group=self.group)
                    self.gather_bytes += (cnt - (hi - lo)) * H * W * (D.element_size() + 3)
                if self.cuda:
                    b["ready"].record(self.s_gather)
            if self.cuda:
                if hasattr(self.volume, "set_input_event"):
                    # the allocate kernels of this chunk wait for the upload / all-gather only, not for the update
                    # kernels of the previous chunk that are queued on the compute stream
                    self.volume.set_input_event(b["ready"].cuda_event)
                else:
                    self.s_int.wait_event(b["ready"])
                self.volume.integrate_batch(b["depth"][:cnt], b["color"][:cnt], K, T[c0:c0 + cnt],
                                            stream=self.s_int.cuda_stream, depth_scale=depth_scale)
                b["free"].record(self.s_int)
            else:   # CPU / gloo (host-logic tests with a stand-in volume)
                self.volume.integrate_batch(b["depth"][:cnt], b["color"][:cnt], K, T[c0:c0 + cnt],
                                            depth_scale=depth_scale)

    def synchronize(self):
        import torch
        if self.cuda:
            self.s_up.synchronize()
            self.s_gather.synchronize()
            self.s_int.synchronize()
        self.volume.synchronize()


def gather_blocks(keys, vox, dst: int = 0, group=None, device=None):
    """Gather every rank's blocks on `dst` with torch.distributed (padded all_gather of sizes, then
    gather of the payloads).  keys int32 [n,3], vox float32 [n,5,512] numpy arrays.
    Returns (keys, vox) on dst, (None, None) elsewhere."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    dev = torch.device(device) if device is not None else torch.device("cpu")
    n = torch.tensor([len(keys)], dtype=torch.int64, device=dev)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n, group=group)
    sizes = [int(s.item()) for s in sizes]
    nmax = max(max(sizes), 1)
    k = torch.zeros((nmax, 3), dtype=torch.int32, device=dev)
    v = torch.zeros((nmax,) + tuple(np.asarray(vox).shape[1:]), dtype=torch.float32, device=dev)
    if len(keys):
        k[:len(keys)] = torch.from_numpy(np.ascontiguousarray(keys, np.int32)).to(dev)
        v[:len(keys)] = torch.from_numpy(np.ascontiguousarray(vox, np.float32)).to(dev)
    if rank == dst:
        ks = [torch.zeros_like(k) for _ in range(world)]
        vs = [torch.zeros_like(v) for _ in range(world)]
    else:
        ks = vs = None
    dist.gather(k, ks, dst=dst, group=group)
    dist.gather(v, vs, dst=dst, group=group)
    if rank != dst:
        return None, None
    out_k = np.concatenate([ks[r][:sizes[r]].cpu().numpy() for r in range(world)])
    out_v = np.concatenate([vs[r][:sizes[r]].cpu().numpy() for r in range(world)])
    return out_k, out_v


def gather_blocks_device(volume, dst: int = 0, group=None):
    """Device-resident gather over NCCL: every rank exports its blocks device-to-device
    (`b2v_export_blocks`), the payloads travel GPU to GPU (NVLink), nothing touches host memory.
    Returns (keys int32 [n,4], vox float32 [n,5,512], or a float64-colour volume's raw layout [n,4096]) CUDA tensors
    on dst, (None, None) elsewhere."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    keys, vox = volume.export_blocks_torch()
    n = torch.tensor([keys.shape[0]], dtype=torch.int64, device=keys.device)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n, group=group)
    sizes = [int(s.item()) for s in sizes]
    nmax = max(max(sizes), 1)
    k = torch.zeros((nmax, 4), dtype=torch.int32, device=keys.device)
    v = torch.zeros((nmax,) + tuple(vox.shape[1:]), dtype=torch.float32, device=keys.device)
    k[:keys.shape[0]] = keys
    v[:vox.shape[0]] = vox
    ks = [torch.zeros_like(k) for _ in range(world)] if rank == dst else None
    vs = [torch.zeros_like(v) for _ in range(world)] if rank == dst else None
    dist.gather(k, ks, dst=dst, group=group)
    dist.gather(v, vs, dst=dst, group=group)
    if rank != dst:
        return None, None
    return (torch.cat([ks[r][:sizes[r]] for r in range(world)]).contiguous(),
            torch.cat([vs[r][:sizes[r]] for r in range(world)]).contiguous())


def extract_mesh_distributed(volume, dst: int = 0, group=None, device=None, capacity_blocks=None):
    """Mesh of a sharded volume: gather all shards on `dst`, load them into a scratch single-GPU
    volume there and run the marching-cubes kernels on the union.  Returns a TriangleMesh on dst,
    None elsewhere.  With the NCCL backend the blocks stay on the GPUs (`gather_blocks_device`); any other
    backend (gloo in the CPU tests) goes through host arrays (`gather_blocks`)."""
    import torch.distributed as dist
    from .volume import B200TsdfVolume

    on_device = dist.get_backend(group) == "nccl"
    if on_device:
        keys, vox = gather_blocks_device(volume, dst=dst, group=group)
    else:   # the blocks in the volume's raw layout, which gather_blocks moves word for word
        keys4, raw = volume._export_blocks(np.empty)
        keys, vox = gather_blocks(keys4[:, :3], raw, dst=dst, group=group, device=device)
    if dist.get_rank(group) != dst:
        return None
    cap = capacity_blocks or max(2 * len(keys), 1024)
    scratch = getattr(volume, "_mesh_scratch", None)   # kept between extractions (one per output tick)
    if scratch is None or scratch.capacity_blocks < len(keys) + 1:
        if scratch is not None:
            scratch.close()
        scratch = B200TsdfVolume(volume.voxel_length, volume.sdf_trunc, volume.depth_trunc,
                                 capacity_blocks=cap, device=volume.device,
                                 volume_unit_resolution=volume.volume_unit_resolution,
                                 color_float64=volume.color_float64)
        volume._mesh_scratch = scratch
    else:
        scratch.reset()
    if on_device:
        scratch.import_blocks_torch(keys, vox)
    else:
        scratch._upload_raw(keys, vox)
    return scratch.extract_mesh()


# ---- sharded extraction: face-halo exchange ----------------------------------------------------------------------

def halo_records(volume, world: int):
    """The halo records `volume` (one shard of a `world`-rank sharding) sends each rank: a list of `world` pairs
    (headers int32 [n,4] = {x,y,z,mask}, payload float32 [m,5], or [m,8] with float64 colour) of CUDA tensors; the
    volume's own rank gets empty ones."""
    headers, payload, nrec, nvox = volume.export_halo_torch(world)
    return list(zip(headers.split(nrec), payload.split(nvox)))


def _concat_records(records):
    """`records`: one (headers, payload) pair or a list of them (the records a rank received, any order)."""
    import torch
    if isinstance(records, tuple) and len(records) == 2 and not isinstance(records[0], tuple):
        return records
    records = list(records)
    if not records:
        return torch.zeros((0, 4), dtype=torch.int32), torch.zeros((0, 5), dtype=torch.float32)
    return torch.cat([torch.as_tensor(h).reshape(-1, 4) for h, _ in records]), \
        torch.cat([torch.as_tensor(x).reshape(-1, torch.as_tensor(x).shape[-1]) for _, x in records])


def mesh_piece(volume, records):
    """The mesh of the cubes rooted in `volume`'s blocks, given the halo records the other shards sent it: a
    TriangleMesh with edge_ids; seam vertices may repeat across pieces (`weld` merges them)."""
    h, x = _concat_records(records)
    return volume.extract_mesh_with_halo(h, x)


def point_piece(volume, records):
    """The zero crossings rooted in `volume`'s blocks: a PointCloud with edge_ids; pieces of different shards are
    disjoint."""
    h, x = _concat_records(records)
    return volume.extract_point_cloud_with_halo(h, x)


def weld(pieces, device: int = 0):
    """One mesh from the mesh pieces of every shard, in rank order: the first vertex of each edge id is kept, in order
    of first occurrence, and the triangles (rank-major) are re-indexed (b2v_weld_mesh_device, on `device`)."""
    import ctypes as C
    import torch
    from . import _lib
    from .volume import TriangleMesh
    L = _lib.load()
    pieces = list(pieces)
    dev = torch.device("cuda", device)
    nv = (C.c_int64 * len(pieces))(*[len(p.vertices) for p in pieces])
    nt = (C.c_int64 * len(pieces))(*[len(p.triangles) for p in pieces])

    def cat(name, dtype, width):
        arrs = [np.asarray(getattr(p, name), dtype).reshape(-1, width) for p in pieces]
        return torch.from_numpy(np.ascontiguousarray(np.concatenate(arrs) if arrs else np.zeros((0, width), dtype))).to(dev)

    V, Cc = cat("vertices", np.float64, 3), cat("vertex_colors", np.float64, 3)
    E, T = cat("edge_ids", np.int32, 4), cat("triangles", np.int32, 3)
    oV, oC, oE, oT = torch.empty_like(V), torch.empty_like(Cc), torch.empty_like(E), torch.empty_like(T)
    torch.cuda.current_stream(dev).synchronize()
    n = C.c_int64(0)
    rc = L.b2v_weld_mesh_device(device, len(pieces), nv, nt, V.data_ptr(), Cc.data_ptr(), E.data_ptr(), T.data_ptr(),
                                oV.data_ptr(), oC.data_ptr(), oE.data_ptr(), oT.data_ptr(), C.byref(n))
    if rc != _lib.B2V_OK:
        raise RuntimeError(f"b2v_weld_mesh_device failed (status {rc}): {L.b2v_weld_last_error().decode()}")
    k = n.value
    return TriangleMesh(oV[:k].cpu().numpy(), oT.cpu().numpy(), oC[:k].cpu().numpy(), oE[:k].cpu().numpy())


def _exchange_halo(volume, group):
    """All-to-all of the halo records: -> (headers, payload) this rank received (on the volume's GPU), and the halo
    bytes each rank sent."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    on_device = dist.get_backend(group) == "nccl"
    headers, payload, nrec, nvox = volume.export_halo_torch(world)
    dev = headers.device if on_device else torch.device("cpu")
    headers, payload = headers.to(dev), payload.to(dev)
    # row 2: the payload's words per voxel, which tell the ranks' colour precisions apart
    mine = torch.tensor([nrec, nvox, [payload.shape[1]] * world], dtype=torch.int64, device=dev)
    sizes = [torch.zeros_like(mine) for _ in range(world)]
    dist.all_gather(sizes, mine, group=group)
    sizes = [s.cpu() for s in sizes]
    if any(int(sizes[s][2, 0]) != payload.shape[1] for s in range(world)):
        raise ValueError("the ranks of a sharded volume must all keep float32 colour or all float64 colour")
    in_rec = [int(sizes[s][0, rank]) for s in range(world)]
    in_vox = [int(sizes[s][1, rank]) for s in range(world)]
    rh = torch.empty((sum(in_rec), 4), dtype=torch.int32, device=dev)
    rx = torch.empty((sum(in_vox), payload.shape[1]), dtype=torch.float32, device=dev)
    dist.all_to_all_single(rh, headers, output_split_sizes=in_rec, input_split_sizes=nrec, group=group)
    dist.all_to_all_single(rx, payload, output_split_sizes=in_vox, input_split_sizes=nvox, group=group)
    sent = [int(sizes[s][0].sum()) * 16 + int(sizes[s][1].sum()) * 4 * payload.shape[1] for s in range(world)]
    return rh, rx, sent


def _gather_rows(arr, dst, group, on_device, device):
    """Variable-length row arrays (numpy, or torch tensors on any device) of every rank, as numpy arrays in rank order:
    on dst, or on every rank with dst=None; None elsewhere.  The rows travel as CUDA tensors on `device` with NCCL
    (on_device), as host tensors otherwise."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    dev = torch.device("cuda", device) if on_device else torch.device("cpu")
    t = (arr if torch.is_tensor(arr) else torch.from_numpy(np.ascontiguousarray(arr))).to(dev)
    n = torch.tensor([t.shape[0]], dtype=torch.int64, device=dev)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n, group=group)
    sizes = [int(s.item()) for s in sizes]
    pad = torch.zeros((max(max(sizes), 1),) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
    pad[:t.shape[0]] = t
    if dst is None:
        bufs = [torch.zeros_like(pad) for _ in range(world)]
        dist.all_gather(bufs, pad, group=group)
    else:
        bufs = [torch.zeros_like(pad) for _ in range(world)] if dist.get_rank(group) == dst else None
        dist.gather(pad, bufs, dst=dst, group=group)
    if bufs is None:
        return None
    return [bufs[r][:sizes[r]].cpu().numpy() for r in range(world)]


def _sharded(volume, dst, group, gather, points):
    import torch.distributed as dist
    from .volume import PointCloud, TriangleMesh
    rh, rx, sent = _exchange_halo(volume, group)
    volume.last_halo_bytes = sent
    piece = point_piece(volume, (rh, rx)) if points else mesh_piece(volume, (rh, rx))
    if not gather:
        return piece
    on_device = dist.get_backend(group) == "nccl"
    names = (("points", "colors", "edge_ids") if points else ("vertices", "vertex_colors", "edge_ids", "triangles"))
    parts = {k: _gather_rows(getattr(piece, k), dst, group, on_device, volume.device) for k in names}
    if dist.get_rank(group) != dst:
        return None
    if points:
        return PointCloud(*(np.concatenate(parts[k]) for k in names))
    ranks = range(len(parts["edge_ids"]))
    return weld([TriangleMesh(parts["vertices"][r], parts["triangles"][r], parts["vertex_colors"][r],
                              parts["edge_ids"][r]) for r in ranks], device=volume.device)


def extract_mesh_sharded(volume, dst: int = 0, group=None, gather: bool = True):
    """Mesh of a hash-sharded volume with each rank meshing its own blocks: one all-gather of the per-destination
    sizes, one all_to_all of halo headers and one of halo voxels (GPU to GPU with NCCL, host tensors with any other
    backend), the mesh piece of the rank's blocks on its GPU, then the pieces gathered to `dst` and welded there.
    Returns the welded TriangleMesh (with edge_ids) on dst and None elsewhere; `gather=False` returns every rank's own
    piece instead.  `volume.last_halo_bytes` lists the halo bytes each rank sent."""
    return _sharded(volume, dst, group, gather, points=False)


def extract_point_cloud_sharded(volume, dst: int = 0, group=None, gather: bool = True):
    """Point cloud of a hash-sharded volume, like `extract_mesh_sharded`: each rank extracts the zero crossings rooted
    in its own blocks; the disjoint pieces are concatenated in rank order on `dst` (a PointCloud with edge_ids)."""
    return _sharded(volume, dst, group, gather, points=True)


# ---- sharded point-average and semantic grids ------------------------------------------------------------------------

def association_votes(grid, camera_frustrum, class_ids_image, semantic_instances_image, depth_image=None,
                      depth_threshold: float = 0.1, do_carving: bool = False, device: bool = False):
    """The votes step of `assign_object_ids_to_instance_ids` on one shard of a semantic grid (b2v_sgrid_assoc_votes):
    the shard's frustum voxels vote, pending voxels are marked and `do_carving` carves, as in the unsharded call.
    Returns the shard's sorted unique vote triples int32 [n,3] = (instance id, object id or `_lib.B2V_ASSOC_PENDING`,
    count): numpy, or a CUDA tensor on the grid's device with `device=True` (for NCCL).  None when the label images are
    empty or wrongly sized (the reference's soft failure, which `resolve_association` repeats)."""
    import ctypes as C
    from . import _lib
    hold = []
    imgs = grid._assoc_images((camera_frustrum.height, camera_frustrum.width), class_ids_image,
                              semantic_instances_image, depth_image, hold)
    if imgs is None:
        return None
    K, T = camera_frustrum._args()
    n = grid._L.b2v_sgrid_assoc_votes(grid._h, K.ctypes.data, camera_frustrum.width, camera_frustrum.height,
                                      T.ctypes.data, camera_frustrum.depth_max, camera_frustrum.depth_min, *imgs,
                                      float(depth_threshold), 1 if do_carving else 0)
    if n < 0:
        raise RuntimeError(grid._L.b2v_sgrid_last_error(grid._h).decode())
    if device:
        import torch
        out = torch.empty((n, 3), dtype=torch.int32, device=torch.device("cuda", grid.device))
        torch.cuda.synchronize(out.device)
        ptr = out.data_ptr()
    else:
        out = np.zeros((n, 3), np.int32)
        ptr = out.ctypes.data
    grid._check(grid._L.b2v_sgrid_copy_assoc_votes(grid._h, C.c_void_p(ptr) if n else None),
                "b2v_sgrid_copy_assoc_votes")
    return out


def resolve_association(grid, votes_list, class_ids_image, semantic_instances_image, min_vote_ratio: float = 0.5,
                        min_votes: int = 3) -> dict:
    """The resolve step on one shard (b2v_sgrid_assoc_resolve): the triples of every rank (`association_votes`, any
    order, numpy or tensors) are summed, new object ids go to the instances with a pending triple in ascending
    instance order, the reference's winner rule picks each instance's object, and the shard's pending voxels take
    their instance's id.  Every rank that resolves the same triples returns the unsharded map and advances
    `next_object_id` alike.  No integrate, edit or clear may come between the votes and the resolve."""
    import torch
    parts = [v for v in votes_list if v is not None]
    if len(parts) < len(votes_list):
        return {}
    hw = tuple(getattr(class_ids_image, "shape", None) or np.shape(class_ids_image))
    hold = []
    imgs = grid._assoc_images(hw, class_ids_image, semantic_instances_image, None, hold) if len(hw) == 2 else None
    if imgs is None:
        return {}
    t = np.ascontiguousarray(np.concatenate([np.asarray(v.cpu() if torch.is_tensor(v) else v, np.int32).reshape(-1, 3)
                                             for v in parts] or [np.zeros((0, 3), np.int32)]))
    H, W = hw
    n = grid._L.b2v_sgrid_assoc_resolve(grid._h, t.ctypes.data, len(t), W, H, imgs[0], imgs[1],
                                        float(min_vote_ratio), int(min_votes))
    return grid._instance_map(n)


def _on_device(group):
    import torch.distributed as dist
    return dist.get_backend(group) == "nccl"


def assign_object_ids_to_instance_ids_sharded(grid, camera_frustrum, class_ids_image, semantic_instances_image,
                                              depth_image=None, depth_threshold: float = 0.1,
                                              do_carving: bool = False, min_vote_ratio: float = 0.5,
                                              min_votes: int = 3, group=None) -> dict:
    """`assign_object_ids_to_instance_ids` of a hash-sharded semantic grid over a process group, called on every rank
    with the same frame: the votes of every rank, one all-gather of the vote triples (GPU to GPU with NCCL, host
    tensors with any other backend), then the resolve on every rank.  Every rank returns the map of the unsharded grid
    and its voxels are those of the unsharded grid it owns."""
    on_device = _on_device(group)
    votes = association_votes(grid, camera_frustrum, class_ids_image, semantic_instances_image, depth_image,
                              depth_threshold, do_carving, device=on_device)
    if votes is None:   # the same images on every rank: all ranks return here
        return {}
    parts = _gather_rows(votes, None, group, on_device, grid.device)
    return resolve_association(grid, parts, class_ids_image, semantic_instances_image, min_vote_ratio, min_votes)


def _gather_voxels(grid, v, dst, group):
    """A read-out (VoxelGridData) of every rank, concatenated in rank order on dst; None elsewhere."""
    import torch.distributed as dist
    from .volume import VoxelGridData
    names = [k for k in ("points", "colors", "class_ids", "object_ids", "confidences") if getattr(v, k) is not None]
    parts = {k: _gather_rows(getattr(v, k), dst, group, _on_device(group), grid.device) for k in names}
    if dist.get_rank(group) != dst:
        return None
    out = VoxelGridData(np.concatenate(parts["points"]), np.concatenate(parts["colors"]))
    for k in names[2:]:
        setattr(out, k, np.concatenate(parts[k]))
    return out


def get_voxels_sharded(grid, min_count: int = 1, min_confidence: float = 0.0, dst: int = 0, group=None):
    """`get_voxels` of a hash-sharded grid: every rank's voxels, rank-major on `dst` (the reference leaves the order
    unspecified); None elsewhere."""
    return _gather_voxels(grid, grid.get_voxels(min_count, min_confidence), dst, group)


def get_voxels_in_bb_sharded(grid, bbox, min_count: int = 1, min_confidence: float = 0.0, dst: int = 0, group=None):
    """`get_voxels_in_bb` of a hash-sharded grid, gathered like `get_voxels_sharded`."""
    return _gather_voxels(grid, grid.get_voxels_in_bb(bbox, min_count, min_confidence), dst, group)


def get_voxels_in_camera_frustrum_sharded(grid, camera_frustrum, min_count: int = 1, min_confidence: float = 0.0,
                                          dst: int = 0, group=None):
    """`get_voxels_in_camera_frustrum` of a hash-sharded grid, gathered like `get_voxels_sharded`."""
    return _gather_voxels(grid, grid.get_voxels_in_camera_frustrum(camera_frustrum, min_count, min_confidence), dst,
                          group)


def _segments_sharded(grid, by_class, min_count, min_confidence, dst, group):
    from .volume import segment_min_count, segments
    v = get_voxels_sharded(grid, segment_min_count(min_count), min_confidence, dst, group)
    return None if v is None else segments(v, by_class)


def get_object_segments_sharded(grid, min_count: int = 1, min_confidence: float = 0.0, dst: int = 0, group=None):
    """`get_object_segments` of a hash-sharded semantic grid: the voxels gathered on `dst`, then grouped there (same
    ids, voxels and confidence ranges as the unsharded grid; the voxels of a segment come rank-major).  None
    elsewhere."""
    return _segments_sharded(grid, False, min_count, min_confidence, dst, group)


def get_class_segments_sharded(grid, min_count: int = 1, min_confidence: float = 0.0, dst: int = 0, group=None):
    """`get_class_segments` of a hash-sharded semantic grid, like `get_object_segments_sharded`."""
    return _segments_sharded(grid, True, min_count, min_confidence, dst, group)


def _all_sum(grid, x: int, group) -> int:
    import torch
    import torch.distributed as dist
    dev = torch.device("cuda", grid.device) if _on_device(group) else torch.device("cpu")
    t = torch.tensor([int(x)], dtype=torch.int64, device=dev)
    dist.all_reduce(t, group=group)
    return int(t.item())


def num_blocks_sharded(grid, group=None) -> int:
    """Blocks of a hash-sharded grid over all ranks (an all-reduce; the ranks' blocks are disjoint)."""
    return _all_sum(grid, grid.num_blocks(), group)


def size_sharded(grid, group=None) -> int:
    """`size()` (non-empty voxels) of a hash-sharded grid over all ranks (an all-reduce)."""
    return _all_sum(grid, grid.size(), group)
