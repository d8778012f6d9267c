"""The resolved sharded call (b2d_render_sharded_resolved) against the unresolved one (b2d_render_sharded): what the
resolve adds to each rank's chunk loop, and the bytes per frame the exchange carries.

    python tools/sharded_resolve_bench.py [--poses 1024] [--chunk 128] [--rounds 5] [--out FILE.json]     # one GPU
    torchrun --nproc-per-node N tools/sharded_resolve_bench.py                                          # N GPUs

Job: the c5 poses (poses.random_poses, seed 5) on the c5 level (synthetic SYN_E1M1, seed 1), chunks of --chunk frames.
Variants at 1920x1080: index frames (unresolved), grey k=2, planar RGB k=2 and RGB k=1; at 3840x2160: index frames and
RGB k=2, the 2x anti-aliased 1080p frame.  Each round runs every variant once per mode, alternating; reported are the
medians over rounds of render_ms (raster plus resolve, summed over chunks) and total_ms (first launch to last consumer)
from the call's stats, with the gathered bytes per frame.  World 1 runs RENDER_ONLY: there is no exchange.  With N > 1
ranks it also runs RENDER_GATHER and GATHER_ONLY, and each number is the max over ranks.  The card's name, power limit
and SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.levels_bench import gpu_info  # noqa: E402

VARIANTS = [((1920, 1080), None), ((1920, 1080), (2, "gray")), ((1920, 1080), (2, "rgb_planar")), ((1920, 1080), (1, "rgb")),
            ((3840, 2160), None), ((3840, 2160), (2, "rgb"))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=1024)
    ap.add_argument("--chunk", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "sharded_resolve_bench measures on a GPU; there is no CPU number"
    import rust_doom_b200 as b2d
    from rust_doom_b200 import _lib, build, jobs
    from rust_doom_b200 import poses as P, synthwad
    build.build()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        comm = jobs.make_comm(local)
    else:
        comm = jobs.single_comm(local)
    scene = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",))), 0)
    poses = P.random_poses(scene, args.poses, 5)
    renderers = {wh: b2d.Renderer(scene, b2d.make_view(*wh), device=local, max_batch=args.chunk) for wh in {v[0] for v in VARIANTS}}
    modes = [("render_only", _lib.SHARD_RENDER_ONLY)]
    if world > 1:
        modes += [("render_gather", _lib.SHARD_RENDER_GATHER), ("gather_only", _lib.SHARD_GATHER_ONLY)]

    def worst(x):
        if world == 1:
            return x
        t = torch.tensor([x], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def run(v, mode):
        wh, res = v
        if world > 1:
            dist.barrier()
        st = renderers[wh].render_sharded(comm, poses, args.chunk, mode, resolve=res)
        return worst(st["render_ms"]), worst(st["total_ms"]), st

    for v in VARIANTS:                                   # warm-up: buffers, staging, kernels at every size
        for _, mode in modes:
            run(v, mode)
    times = {(i, m): [] for i in range(len(VARIANTS)) for m, _ in modes}
    stats = {}
    for _ in range(args.rounds):
        for m, mode in modes:
            for i, v in enumerate(VARIANTS):
                rm, tm, st = run(v, mode)
                times[(i, m)].append((rm, tm))
                stats[(i, m)] = st
    status = 0
    for r in renderers.values():
        status |= r.status()
    rows = []
    for i, (wh, res) in enumerate(VARIANTS):
        r = renderers[wh]
        fb = wh[0] * wh[1] if res is None else r.resolve_frame_bytes(res[0], b2d.RESOLVE_FORMATS[res[1]])
        row = {"view": "%dx%d" % wh, "resolve": "index" if res is None else "%s k=%d" % (res[1], res[0]),
               "gathered_bytes_per_frame": fb, "bytes_vs_index": round(fb / (wh[0] * wh[1]), 4)}
        for m, _ in modes:
            t = times[(i, m)]
            row[m + "_render_ms"] = round(statistics.median(x[0] for x in t), 3)
            row[m + "_total_ms"] = round(statistics.median(x[1] for x in t), 3)
            row[m + "_total_ms_range"] = [round(min(x[1] for x in t), 3), round(max(x[1] for x in t), 3)]
            if m != "render_only":
                row[m + "_bytes_received"] = stats[(i, m)]["bytes_received"]
        rows.append(row)
    res = dict(gpu_info(), bench="sharded_resolve", world=world, poses=args.poses, chunk=args.chunk, rounds=args.rounds,
               per_rank=stats[(0, "render_only")]["frames_local"], chunks=stats[(0, "render_only")]["chunks"], rows=rows,
               status_bits=int(status))
    if int(os.environ.get("RANK", "0")) == 0:
        for row in rows:
            print("%-9s %-14s %9d B/frame  " % (row["view"], row["resolve"], row["gathered_bytes_per_frame"]) +
                  "  ".join("%s render %.3f total %.3f ms" % (m, row[m + "_render_ms"], row[m + "_total_ms"]) for m, _ in modes))
        print(json.dumps(res), flush=True)
        if args.out:
            with open(args.out, "w") as f:
                json.dump(res, f, indent=1)
    comm.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
