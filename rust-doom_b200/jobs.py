"""The BASELINE.json configurations as runnable jobs (bench.py --config ..., cli).

* c2  (bench.py default)  one map, 1000-pose fly-through, 1920x1080, device resident
* c3  all E1 maps batched, 1920x1080, one GPU: nine renderers, batches interleaved round-robin
* c4  MAP01-MAP10, 3840x2160, four GPUs one-map-per-GPU (3/3/2/2), no collective
* c5  100 k random poses, 1920x1080, 8 GPUs, chunked NCCL all-gather of finished frames overlapped with rendering
      (b2d_render_sharded), gathered frames validated by per-frame checksums on every rank and against the oracle

Every runner returns a dict of device-timed numbers (max over ranks where there are ranks); bench.py turns them into
its JSON line and checks the frames against the oracle (the checker lives there, not in the product package).
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import Comm, Renderer, Scene, _lib, frame_checksums_device, make_view

C3_MAPS = tuple("E1M%d" % i for i in range(1, 10))
C4_MAPS = tuple("MAP%02d" % i for i in range(1, 11))


# ------------------------------------------------------------------------------------------------ host binding
def gpu_numa_node(device_index: int) -> Optional[int]:
    """NUMA node the GPU hangs off (sysfs), or None."""
    try:
        import torch
        props = torch.cuda.get_device_properties(device_index)
        bus = "%04x:%02x:%02x.0" % (props.pci_domain_id, props.pci_bus_id, props.pci_device_id)
        with open("/sys/bus/pci/devices/%s/numa_node" % bus) as f:
            node = int(f.read().strip())
        return node if node >= 0 else None
    except Exception:  # noqa: BLE001
        return None


def _parse_cpulist(text: str) -> List[int]:
    cpus: List[int] = []
    for part in text.strip().split(","):
        if not part:
            continue
        if "-" in part:
            a, b = part.split("-")
            cpus.extend(range(int(a), int(b) + 1))
        else:
            cpus.append(int(part))
    return cpus


def bind_to_gpu_numa(device_index: int) -> Dict[str, object]:
    """Pin this process to the CPUs of the GPU's NUMA node so that the pinned host buffers it allocates afterwards are
    first-touched on the memory next to the GPU's PCIe root.
    Returns what was done (for the bench line)."""
    node = gpu_numa_node(device_index)
    info: Dict[str, object] = {"numa_node": node, "bound": False}
    if node is None:
        return info
    try:
        with open("/sys/devices/system/node/node%d/cpulist" % node) as f:
            cpus = set(_parse_cpulist(f.read()))
        allowed = os.sched_getaffinity(0) & cpus
        if allowed:
            os.sched_setaffinity(0, allowed)
            info["bound"] = True
            info["cpus"] = len(allowed)
    except Exception as e:  # noqa: BLE001
        info["error"] = str(e)
    return info


def usable_cores() -> int:
    """Cores this process may run on: affinity mask, capped by the cgroup cpu.max quota."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        with open("/sys/fs/cgroup/cpu.max") as f:
            quota, period = f.read().split()
        if quota != "max":
            n = max(1, min(n, int(int(quota) / int(period))))
    except Exception:  # noqa: BLE001
        pass
    return n


# ------------------------------------------------------------------------------------------------ communicator
def make_comm(local_rank: int) -> Comm:
    """b2d communicator for the torch.distributed job this process belongs to (the unique id travels by broadcast)."""
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    box = [Comm.unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    return Comm(box[0], rank, world, local_rank)


def single_comm(device: int = 0) -> Comm:
    return Comm(Comm.unique_id(), 0, 1, device)


# ------------------------------------------------------------------------------------------------ c5
def global_pose_index(q: int, per: int, first: int, j: int) -> int:
    """Pose shown by frame j of rank q's slice of the chunk that starts at local pose `first` (include/b2d.h)."""
    return q * per + first + j


class ChecksumTable:
    """Per-frame checksums of every gathered frame, laid out [world, per] on the device; filled by the chunk callback."""

    def __init__(self, world: int, per: int, npix: int, dev):
        import torch
        self.world, self.per, self.npix = world, per, npix
        self.table = torch.zeros((world, per), dtype=torch.int32, device=dev)

    def on_chunk(self, k, first, cnt, ptr, ranks, stream):
        for q in range(ranks):
            frame_checksums_device(ptr + q * cnt * self.npix, cnt, self.npix,
                                   self.table.data_ptr() + 4 * (q * self.per + first), stream)

    def host(self) -> np.ndarray:
        return self.table.cpu().numpy().view(np.uint32)


def run_c5(scene: Scene, poses: np.ndarray, width: int, height: int, local_rank: int, comm: Comm, chunk: int = 256,
           reps: int = 1) -> Dict[str, object]:
    """Render-only, gather-only and joint (overlapped) passes over the whole pose list; then a joint pass with the
    checksum consumer whose table is returned for verification."""
    import torch
    import torch.distributed as dist
    dev = torch.device("cuda", local_rank)
    world = comm.world
    n_total = len(poses)
    per = (n_total + world - 1) // world
    chunk = min(chunk, per)
    view = make_view(width, height)
    r = Renderer(scene, view, device=local_rank, max_batch=chunk)
    npix = width * height

    def timed(mode, on_chunk=None):
        best = None
        for _ in range(max(reps, 1)):
            if world > 1:
                dist.barrier()
            torch.cuda.synchronize()
            st = r.render_sharded(comm, poses, chunk, mode, on_chunk)
            t = torch.tensor([st["total_ms"], st["render_ms"], st["gather_ms"]], dtype=torch.float64, device=dev)
            if world > 1:
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
            st["total_ms"], st["render_ms"], st["gather_ms"] = (float(x) for x in t.tolist())
            if best is None or st["total_ms"] < best["total_ms"]:
                best = st
        return best

    timed(_lib.SHARD_RENDER_GATHER)                       # warm-up: buffers, registration, NCCL channels
    render = timed(_lib.SHARD_RENDER_ONLY)
    gather = timed(_lib.SHARD_GATHER_ONLY)
    joint = timed(_lib.SHARD_RENDER_GATHER)
    table = ChecksumTable(world, per, npix, dev)
    checked = timed(_lib.SHARD_RENDER_GATHER, table.on_chunk)
    status = r.status()
    frames = per * world                                 # padded job size actually rendered and gathered
    out = {
        "n_total": n_total, "frames": frames, "per_rank": per, "chunk_frames": chunk, "chunks": joint["chunks"],
        "render_only_ms": render["total_ms"], "gather_only_ms": gather["total_ms"], "joint_ms": joint["total_ms"],
        "joint_checked_ms": checked["total_ms"],
        "render_only_fps": frames / (render["total_ms"] / 1e3),
        "gather_only_fps": frames / (gather["total_ms"] / 1e3),
        "joint_fps": frames / (joint["total_ms"] / 1e3),
        "joint_checked_fps": frames / (checked["total_ms"] / 1e3),
        "gather_gbs_received_per_rank": (world - 1) * per * npix / (gather["total_ms"] / 1e3) / 1e9 if world > 1 else 0.0,
        "joint_gbs_received_per_rank": (world - 1) * per * npix / (joint["total_ms"] / 1e3) / 1e9 if world > 1 else 0.0,
        "registration": joint["registration"], "nccl_version": comm.nccl_version, "status_bits": status,
        "table": table, "renderer": r,
    }
    return out


# ------------------------------------------------------------------------------------------------ c3 / c4
def map_assignment(n_maps: int, world: int) -> List[List[int]]:
    """Maps per rank, contiguous, sizes differing by at most one with the larger shares first: 10 maps on 4 ranks ->
    3/3/2/2 (BASELINE.json configs[3])."""
    base, extra = divmod(n_maps, world)
    out, k = [], 0
    for r in range(world):
        cnt = base + (1 if r < extra else 0)
        out.append(list(range(k, k + cnt)))
        k += cnt
    return out


def run_maps(scenes: Sequence[Scene], poses: Sequence[np.ndarray], width: int, height: int, local_rank: int,
             batch: int, steps: int, warmup: int, interleave: bool, raster_streams: int = 2) -> Dict[str, object]:
    """Device-resident render of several maps on one GPU.  interleave=True: one pass = every map's pose list in batches
    of `batch`, round-robin over the maps (c3: 'one scene handle per map, batches interleaved'); False: map after map
    (c4).  raster_streams=2: consecutive launches raster on two alternating streams (they write disjoint frames), so the
    first CTAs of launch i+1 use the SMs the last CTAs of launch i leave idle.  Returns total / raster / walk milliseconds
    per pass (CUDA events; with two raster streams the per-launch event pairs also span a launch's wait for SMs, so
    raster_ms_per_pass is then the pass itself) and the renderers (for parity probes)."""
    import torch
    dev = torch.device("cuda", local_rank)
    view = make_view(width, height)
    rs = [Renderer(s, view, device=local_rank, max_batch=batch) for s in scenes]
    d_poses = [torch.from_numpy(p.view(np.int32).reshape(-1, 4).copy()).to(dev) for p in poses]
    npix = width * height
    nmax = max((len(p) for p in poses), default=0)
    # one output buffer per map (c3 keeps all nine resident: 9 x 2.07 GB at 1080p x 1000)
    outs = [torch.empty((len(p), height, width), dtype=torch.uint8, device=dev) for p in poses]
    main_stream = torch.cuda.current_stream()
    # rasters that defer masked entries (two-sided middle textures, sprites) share one arena per renderer and are ordered by
    # an event whatever streams they are on: a second stream buys nothing there
    masked = any(s.info.n_masked_mids + s.info.n_sprites > 0 for s in scenes)
    side = [torch.cuda.Stream(device=dev) for _ in range(2)] if raster_streams > 1 and not masked else None

    # the launches of one pass, in order: (map, first pose, count); c3 interleaves the maps batch by batch
    items = []
    if interleave:
        for b0 in range(0, nmax, batch):
            for m in range(len(rs)):
                if b0 < len(poses[m]):
                    items.append((m, b0, min(batch, len(poses[m]) - b0)))
    else:
        for m in range(len(rs)):
            for b0 in range(0, len(poses[m]), batch):
                items.append((m, b0, min(batch, len(poses[m]) - b0)))
    walk_stream = torch.cuda.Stream(device=dev, priority=-1)

    def walk(i):
        m, b0, cnt = items[i]
        return rs[m].walk_device(d_poses[m].data_ptr() + 16 * b0, cnt, walk_stream.cuda_stream)

    def one_pass():
        # pipelined like bench.py's c2 step: the BSP walk of item i+1 (a background grid) runs under the raster of item i
        if side:
            for t in side:
                t.wait_stream(main_stream)
        ticket = walk(0)
        for i, (m, b0, cnt) in enumerate(items):
            st = side[i & 1] if side else main_stream
            rs[m].raster_device(ticket, outs[m].data_ptr() + npix * b0, 0, st.cuda_stream)
            if i + 1 < len(items):
                ticket = walk(i + 1)
        if side:
            for t in side:
                main_stream.wait_stream(t)

    for _ in range(max(warmup, 1)):
        one_pass()
    torch.cuda.synchronize()
    for r in rs:
        r.profile(True)
        r.profile_read()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    launches0 = sum(r.launch_count for r in rs)
    e0.record()
    for _ in range(steps):
        one_pass()
    e1.record()
    torch.cuda.synchronize()
    walk = raster = 0.0
    for r in rs:
        w, ra, _ = r.profile_read()
        r.profile(False)
        walk += w
        raster += ra
    status = 0
    for r in rs:
        status |= r.status()
    ms_pass = e0.elapsed_time(e1) / steps
    return {"ms_per_pass": ms_pass, "raster_ms_per_pass": ms_pass if side else raster / steps, "walk_ms_per_pass": walk / steps,
            "raster_streams": 2 if side else 1,
            "frames_per_pass": int(sum(len(p) for p in poses)), "launches": sum(r.launch_count for r in rs) - launches0,
            "renderers": rs, "outs": outs, "status_bits": status}
