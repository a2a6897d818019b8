"""Cost of a loop-closure rebuild through the TSDF plugin, with and without the keyframe store
(kVolumetricIntegrationB200KeyframeStoreFrames).  N C2 keyframes (the 300 frames of bench.py's sequence, repeated, with
their own ids and timestamps) go through the stand-in plugin (tests/plugin_standins.py) with GPU rectification on
identity maps, as pySLAM's calibrated cameras do.  Then, timed: RESET, every keyframe again with a corrected pose, the
queue drained and the device synchronised - pySLAM's rebuild(map) (base.py:1242-1318).  The input queue pickles every
task, as a multiprocessing queue does, so the bytes that cross it and the time spent pickling are counted.

Per N and mode, over `--reps` alternating repetitions: wall time from RESET to a drained queue (seconds, each rep),
bytes pickled through q_in, light tasks sent, the store's frames and device bytes, and whether the rebuilt map's mesh
equals the store-off plugin's.  Prints one JSON line with the card's name and power limit read in the same run.

--plugin voxel_grid / semantic: the same rebuild through the point-average grid plugin (C2 frames, input-order sums)
or the semantic plugin (C3 frames with class and instance images, voting and Bayesian fusion), keyframes taken
round-robin from --distinct rendered frames.  Their output check compares the rebuilt grids' block dumps bit for bit,
and each run also times one keyframe's staging with CUDA events: `set_frame` from the host images against
`stage_stored` of its slot (mean over 20 of each, after a warm-up).
python tools/rebuild_cost.py [--plugin tsdf|voxel_grid|semantic] [--keyframes 300 1000] [--reps 2] [--distinct N]
                             [--out FILE]"""
import argparse
import json
import os
import pickle
import queue
import subprocess
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import bench  # noqa: E402
import oracle  # noqa: E402
from pyslam_b200 import keyframe_store  # noqa: E402
from pyslam_b200 import synthetic as S  # noqa: E402
from tests import plugin_standins as P  # noqa: E402
from tests._util import sort_dump  # noqa: E402


class PicklingQueue(queue.Queue):
    """queue.Queue that carries each task pickled, like multiprocessing.Queue, and counts the bytes."""

    def __init__(self):
        super().__init__()
        self.bytes = self.light = 0

    def put(self, item, block=True, timeout=None):
        b = pickle.dumps(item, protocol=pickle.HIGHEST_PROTOCOL)
        self.bytes += len(b)
        self.light += keyframe_store.is_stored(item)
        super().put(b, block, timeout)

    def get(self, block=True, timeout=None):
        return pickle.loads(super().get(block, timeout))

    def get_nowait(self):
        return self.get(False)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, limit = (r.stdout.strip().split(", ") + ["?", "?"])[:2]
    return name, limit


def corrected(T):
    """A loop closure's pose correction: a small rotation about y and a few millimetres of translation."""
    a = 0.003
    D = np.eye(4)
    D[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    D[:3, 3] = [0.004, -0.002, 0.003]
    return T @ D


def run(cfg, frames, n, store):
    depth, bgr, Tcw = frames
    Cls = P.standalone_integrator_class()
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)
    y, x = np.mgrid[:cfg.height, :cfg.width].astype(np.float32)
    integ = Cls(cam, P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF", calib_maps=(x, y),
                kVolumetricIntegrationVoxelLength=cfg.voxel_size, kVolumetricIntegrationTSdfTrunc=cfg.sdf_trunc,
                kVolumetricIntegrationB200KeyframeStoreFrames=n if store else 0,
                kVolumetricIntegrationOutputTimeInterval=1e9)
    integ.q_in = PicklingQueue()
    m = len(depth)
    kds = [P.VolumetricIntegrationKeyframeData(id=i, pose=Tcw[i % m], img=bgr[i % m], depth=depth[i % m],
                                               timestamp=0.1 * i) for i in range(n)]
    for kd in kds:
        integ.add_keyframe_data(kd)
    integ.run_pending()
    integ.volume.synchronize()
    integ.q_in.bytes = integ.q_in.light = 0
    for kd in kds:
        kd.pose = corrected(kd.pose)
    t0 = time.perf_counter()
    integ.reset()
    for kd in kds:
        integ.add_keyframe_data(kd)
    integ.run_pending()
    integ.volume.synchronize()
    wall = time.perf_counter() - t0
    m = integ.volume.extract_mesh()
    mesh = oracle.canonical_mesh(m.vertices, m.vertex_colors, m.edge_ids, m.triangles)
    stats = integ.volume.frame_store_stats()
    out = dict(wall_s=wall, pickled_bytes=integ.q_in.bytes, light_tasks=integ.q_in.light, store_frames=stats[0],
               store_bytes=stats[1], blocks=integ.volume.num_blocks(), triangles=int(len(m.triangles)))
    integ.quit()
    return out, mesh


# ---- grid plugins ----------------------------------------------------------------------------------------------------

def grid_frames(kind, distinct):
    """(cfg, [keyframe image dicts]) of `distinct` rendered frames: C2 for the point-average grid, C3 with class and
    instance images for the semantic grids."""
    cfg, depth, color, Tcw = bench.load_frames("C2" if kind == "voxel_grid" else "C3", distinct, 0, 1)
    out = []
    for i in range(len(depth)):
        f = dict(depth=depth[i], img=np.ascontiguousarray(color[i][..., ::-1]), pose=Tcw[i])
        if kind != "voxel_grid":
            cls = S.render_class_ids(cfg, i)
            inst = np.where(cls % 3 == 0, -1, cls * 7 + (np.arange(cls.shape[1])[None, :] // 400)).astype(np.int32)
            inst[depth[i] == 0] = 0
            f.update(semantic_img=cls, semantic_instances_img=inst)
        out.append(f)
    return cfg, out


def stage_times(grid, f, slot, reps=20):
    """Mean ms of set_frame from the host images and of stage_stored(slot), CUDA events around each call."""
    import torch
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        fn()
        total = 0.0
        for _ in range(reps):
            ev[0].record()
            fn()
            ev[1].record()
            ev[1].synchronize()
            total += ev[0].elapsed_time(ev[1])
        return total / reps

    kw = dict(class_image=f.get("semantic_img"), instance_image=f.get("semantic_instances_img"))
    if "semantic_img" not in f:
        kw = {}
    return dict(set_frame_ms=timed(lambda: grid.set_frame(f["depth"], f["img"], filter_shadow_points=True, **kw)),
                stage_stored_ms=timed(lambda: grid.stage_stored(slot)))


def run_grid(kind, prob, cfg, frames, n, store):
    from pyslam_b200 import integrator_semantic as IS
    make = IS.make_voxel_grid_integrator_class if kind == "voxel_grid" else IS.make_semantic_integrator_class
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)
    y, x = np.mgrid[:cfg.height, :cfg.width].astype(np.float32)
    kw = dict(use_semantic_probabilistic=True) if prob else {}
    integ = make(P.StandaloneIntegratorBase, P.API)(
        cam, P.DatasetEnvironmentType.INDOOR, None, "B200", calib_maps=(x, y),
        kVolumetricIntegrationB200KeyframeStoreFrames=n if store else 0, kVolumetricIntegrationOutputTimeInterval=1e9,
        kVolumetricIntegrationB200InputOrderSums=True, kVolumetricIntegrationB200CapacityBlocks=1 << 14,
        kVolumetricIntegrationB200MaxCapacityBlocks=1 << 20, **kw)
    integ.q_in = PicklingQueue()
    m = len(frames)
    kds = [P.VolumetricIntegrationKeyframeData(id=i, timestamp=0.1 * i, **frames[i % m]) for i in range(n)]
    for kd in kds:
        integ.add_keyframe_data(kd)
    integ.run_pending()
    integ.q_in.bytes = integ.q_in.light = 0
    for kd in kds:
        kd.pose = corrected(kd.pose)
    t0 = time.perf_counter()
    integ.reset()
    for kd in kds:
        integ.add_keyframe_data(kd)
    integ.run_pending()
    integ.volume.num_blocks()   # synchronises
    wall = time.perf_counter() - t0
    dump = sort_dump(integ.volume.dump_blocks(8) if kind == "semantic" else integ.volume.dump_blocks())
    stats = integ.volume.frame_store_stats()
    out = dict(wall_s=wall, pickled_bytes=integ.q_in.bytes, light_tasks=integ.q_in.light, store_frames=stats[0],
               store_bytes=stats[1], blocks=integ.volume.num_blocks())
    if store:
        out.update(stage_times(integ.volume, frames[0], 0))
    integ.quit()
    return out, dump


def main_grid(a, name, limit):
    cfg, frames = grid_frames(a.plugin, a.distinct)
    res = {"gpu": name, "power_limit": limit, "plugin": a.plugin, "config": cfg.name,
           "distinct_frames": len(frames), "runs": {}}
    variants = [("point", False)] if a.plugin == "voxel_grid" else [("voting", False), ("bayesian", True)]
    for label, prob in variants:
        run_grid(a.plugin, prob, cfg, frames[:8], 8, True)   # module loads, first allocations
        for n in a.keyframes:
            per, dumps = {"off": [], "on": []}, {}
            for _ in range(a.reps):
                for mode in ("off", "on"):
                    r, dumps[mode] = run_grid(a.plugin, prob, cfg, frames, n, mode == "on")
                    per[mode].append(r)
            same = dumps["off"].keys() == dumps["on"].keys() and all(
                np.array_equal(dumps["off"][k], dumps["on"][k]) for k in dumps["off"])
            entry = {mode: dict(wall_s=[r["wall_s"] for r in rs], **{k: v for k, v in rs[-1].items() if k != "wall_s"})
                     for mode, rs in per.items()}
            entry["map_equal"] = bool(same)
            res["runs"][f"{label}_{n}"] = entry
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--plugin", choices=("tsdf", "voxel_grid", "semantic"), default="tsdf")
    ap.add_argument("--keyframes", type=int, nargs="+", default=[300, 1000])
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--distinct", type=int, default=60, help="grid plugins: rendered frames the keyframes cycle over")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.plugin != "tsdf":
        name, limit = card()
        emit(main_grid(a, name, limit), a.out)
        return
    cfg, depth, color, Tcw = bench.load_frames("C2", 300, 0, 1)
    bgr = np.ascontiguousarray(color[..., ::-1])
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "config": "C2", "runs": {}}
    run(cfg, (depth[:32], bgr[:32], Tcw[:32]), 32, True)   # module loads, first allocations
    for n in a.keyframes:
        per = {"off": [], "on": []}
        meshes = {}
        for _ in range(a.reps):
            for mode in ("off", "on"):
                r, mesh = run(cfg, (depth, bgr, Tcw), n, mode == "on")
                per[mode].append(r)
                meshes[mode] = mesh
        same = all(np.array_equal(meshes["off"][k], meshes["on"][k]) for k in ("edges", "triangles", "vertices",
                                                                              "colors"))
        res["runs"][str(n)] = {mode: dict(wall_s=[r["wall_s"] for r in rs],
                                          **{k: v for k, v in rs[-1].items() if k != "wall_s"})
                               for mode, rs in per.items()}
        res["runs"][str(n)]["mesh_equal"] = bool(same)
    emit(res, a.out)


def emit(res, out):
    line = json.dumps(res)
    print(line)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
