"""Level sets on the sharded path (b2d_render_sharded_levels_states) against one renderer per map (b2d_render_sharded), and
the per-frame-level palette kernel against K3.

    python tools/sharded_levels_bench.py [--poses 222] [--steps 5] [--warmup 1]              # one GPU, world 1
    torchrun --nproc-per-node N tools/sharded_levels_bench.py --c4                          # N GPUs (c4 shape)

One GPU, world 1, RENDER_ONLY: the c3 shape of tools/levels_states_bench.py (synthetic E1M1-E1M9, seeds 11-19, a
fly-through of --poses per map, 1920x1080).  (a) nine single-level renderers, one b2d_render_sharded call per map, each at
its map's own clock (1000 m: the call renders at the renderer's time); (b) one level set, one
b2d_render_sharded_levels_states call over all maps' poses, pose i of map m at tic 1000 m + i.  The arms alternate
(a, b, b, a) after a warm-up; each prints ms (the calls' device time) and launches per pass.  (b)'s frames are checked,
by device checksum, against each map's own renderer rendering the same poses at the same tics (b2d_render_device_states).

--c4 under torchrun: ten generated maps (seeds 11-20, --poses each, 1920x1080).  (a) jobs.map_assignment's whole maps per
rank, one world-1 b2d_render_sharded call per map; (b) one level set of the ten maps sharded by pose across all ranks.
Prints the max over ranks of each arm's device time.

The palette kernel: 1000 random 1920x1080 index frames through b2d_palette_lut_levels_device (levels alternating over the
nine maps) and through K3 (b2d_palette_lut_device) over the same bytes, alternated; ms and GB/s at 5 bytes per pixel.
The card's name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.levels_bench import gpu_info  # noqa: E402

W, H = 1920, 1080


def maps(seeds, poses_per_map):
    import rust_doom_b200 as b2d
    from rust_doom_b200 import poses as P, synthwad
    scenes = [b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(s, ("E1M%d" % (1 + (s - 11) % 9),))), 0) for s in seeds]
    return scenes, [P.flythrough_poses(s, poses_per_map, 2) for s in scenes]


def one_gpu(args):
    import torch
    import rust_doom_b200 as b2d
    from rust_doom_b200 import _lib, jobs
    scenes, poses = maps(range(11, 20), args.poses)
    nmap, npix = len(scenes), W * H
    view = b2d.make_view(W, H)
    chunk = 128
    comm = jobs.single_comm(0)
    rs = [b2d.Renderer(s, view, max_batch=chunk) for s in scenes]
    for m, r in enumerate(rs):
        r.set_time(1000 * m)
    allp = np.concatenate(poses)
    lv = np.repeat(np.arange(nmap, dtype=np.uint32), args.poses)
    tics = np.concatenate([np.arange(args.poses, dtype=np.uint32) + 1000 * m for m in range(nmap)])
    ls = b2d.Renderer.from_levels(scenes, view, max_batch=chunk)

    def arm_a():
        l0 = sum(r.launch_count for r in rs)
        ms = sum(r.render_sharded(comm, p, chunk, _lib.SHARD_RENDER_ONLY)["total_ms"] for r, p in zip(rs, poses))
        return ms, sum(r.launch_count for r in rs) - l0

    def arm_b():
        l0 = ls.launch_count
        ms = ls.render_sharded_levels_states(comm, allp, lv, tics, None, chunk, _lib.SHARD_RENDER_ONLY)["total_ms"]
        return ms, ls.launch_count - l0

    for _ in range(max(args.warmup, 1)):
        arm_a(), arm_b()
    res = {"a": [], "b": []}
    for _ in range(args.steps):
        for name, arm in (("a", arm_a), ("b", arm_b), ("b", arm_b), ("a", arm_a)):
            res[name].append(arm())
    # (b)'s frames against each map's own renderer at the same poses and tics
    n = len(allp)
    table = jobs.ChecksumTable(1, n, npix, torch.device("cuda", 0))
    ls.render_sharded_levels_states(comm, allp, lv, tics, None, chunk, _lib.SHARD_RENDER_ONLY, table.on_chunk)
    got = table.host()[0]
    want = torch.zeros(n, dtype=torch.int32, device="cuda")
    out = torch.empty((chunk, H, W), dtype=torch.uint8, device="cuda")
    for m, r in enumerate(rs):
        dp = torch.from_numpy(poses[m].view(np.int32).reshape(-1, 4).copy()).cuda()
        for b0 in range(0, args.poses, chunk):
            cnt = min(chunk, args.poses - b0)
            r.render_device_states(dp.data_ptr() + 16 * b0, tics[m * args.poses + b0:m * args.poses + b0 + cnt], cnt, out.data_ptr())
            b2d.frame_checksums_device(out.data_ptr(), cnt, npix, want.data_ptr() + 4 * (m * args.poses + b0))
    torch.cuda.synchronize()
    same = bool(np.array_equal(got, want.cpu().numpy().view(np.uint32)))
    status = ls.status()
    for r in rs:
        status |= r.status()
    line = dict(gpu_info(), bench="sharded_levels_world1", width=W, height=H, maps=nmap, poses_per_map=args.poses, chunk=chunk,
                frames_per_pass=n, nine_renderers_ms_per_pass=[round(t[0], 3) for t in res["a"]],
                nine_renderers_launches_per_pass=res["a"][0][1], level_set_ms_per_pass=[round(t[0], 3) for t in res["b"]],
                level_set_launches_per_pass=res["b"][0][1], level_set_frames_equal_per_map_renderers=same, status_bits=int(status))
    print(json.dumps(line), flush=True)
    comm.close()
    palette(ls, nmap)


def palette(r, nmap, frames=1000, reps=5):
    import torch
    npix = W * H
    idx = torch.randint(0, 256, (frames * npix,), dtype=torch.uint8, device="cuda")
    out = torch.empty(frames * npix, dtype=torch.int32, device="cuda")
    lv = [f % nmap for f in range(frames)]
    runs = {"k3": lambda: r.palette_lut_device(idx.data_ptr(), out.data_ptr(), frames * npix),
            "levels": lambda: r.palette_lut_levels_device(idx.data_ptr(), lv, frames, out.data_ptr())}
    for f in runs.values():
        f()
    ms = {k: [] for k in runs}
    for _ in range(reps):
        for k in ("k3", "levels", "levels", "k3"):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            runs[k]()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    gbs = {k: round(5 * frames * npix / (min(v) / 1e3) / 1e9, 1) for k, v in ms.items()}
    print(json.dumps(dict(gpu_info(), bench="palette_levels", frames=frames, width=W, height=H, bytes_per_pixel=5,
                          k3_ms=[round(x, 3) for x in ms["k3"]], levels_ms=[round(x, 3) for x in ms["levels"]],
                          k3_gbs_best=gbs["k3"], levels_gbs_best=gbs["levels"])), flush=True)


def c4(args):
    import torch
    import torch.distributed as dist
    import rust_doom_b200 as b2d
    from rust_doom_b200 import _lib, jobs
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, world = dist.get_rank(), dist.get_world_size()
    scenes, poses = maps(range(11, 21), args.poses)
    view = b2d.make_view(W, H)
    chunk = 128
    mine = jobs.map_assignment(len(scenes), world)[rank]
    solo = jobs.single_comm(local)
    comm = jobs.make_comm(local)
    rs = {m: b2d.Renderer(scenes[m], view, device=local, max_batch=chunk) for m in mine}
    ls = b2d.Renderer.from_levels(scenes, view, device=local, max_batch=chunk)
    allp = np.concatenate(poses)
    lv = np.repeat(np.arange(len(scenes), dtype=np.uint32), args.poses)
    tics = np.zeros(len(allp), np.uint32)

    def arm_a():
        return sum(rs[m].render_sharded(solo, poses[m], chunk, _lib.SHARD_RENDER_ONLY)["total_ms"] for m in mine)

    def arm_b():
        return ls.render_sharded_levels_states(comm, allp, lv, tics, None, chunk, _lib.SHARD_RENDER_ONLY)["total_ms"]

    def worst(ms):
        t = torch.tensor([ms], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    for _ in range(max(args.warmup, 1)):
        dist.barrier(); arm_a(); dist.barrier(); arm_b()
    res = {"a": [], "b": []}
    for _ in range(args.steps):
        for name, arm in (("a", arm_a), ("b", arm_b), ("b", arm_b), ("a", arm_a)):
            dist.barrier()
            res[name].append(round(worst(arm()), 3))
    if rank == 0:
        print(json.dumps(dict(gpu_info(), bench="sharded_levels_c4", world=world, maps=len(scenes), poses_per_map=args.poses,
                              width=W, height=H, maps_per_rank=[len(x) for x in jobs.map_assignment(len(scenes), world)],
                              whole_maps_max_rank_ms=res["a"], level_set_max_rank_ms=res["b"])), flush=True)
    solo.close()
    comm.close()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=222, help="poses per map")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--c4", action="store_true", help="the ten-map job under torchrun")
    args = ap.parse_args()
    from rust_doom_b200 import build
    build.build()
    c4(args) if args.c4 else one_gpu(args)


if __name__ == "__main__":
    main()
