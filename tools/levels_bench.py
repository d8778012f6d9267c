"""Nine maps on one GPU, two ways: nine renderers with their batches interleaved (jobs.run_maps, bench.py --config c3) and
one level-set renderer (b2d_renderer_create_levels) whose batches mix the nine maps.

    python tools/levels_bench.py [--poses 222] [--batches 8,32,111] [--steps 20] [--warmup 2]

The c3 shape: synthetic E1M1-E1M9 (seeds 11-19), a fly-through per map, 1920x1080, index frames only.  For each per-map
batch size B, one pass renders every map's poses: (a) in batches of B per map, round-robin over the maps; (b) in batches
of 9 B frames that take B poses of every map (frame j of a batch is on map j mod 9).  Both run the same loop -- the
background walk of the next batch under the raster of the current one, rasters alternating between two streams, CUDA
events around the timed passes only, no per-launch profiling in either arm -- and alternate (a, b, b, a) per batch size.
Prints one JSON line per batch size with ms and launches per pass of both, and checks that (b)'s frames equal (a)'s byte
for byte.  Then one line on the walk alone: the c2 level's 1000-pose fly-through at 1080p through a level set of one, the
plain walk (render_device / walk_device) against the per-frame-level walk (render_device_levels / walk_device_levels),
walk kernel times from the library's per-launch events, taken the same way for both.  The card name, power limit and SM
clock are read in the same run (nvidia-smi, right after each measurement).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # noqa: BLE001
        return {"gpu_info_error": str(e)}


def pipelined(renderer_of, items, walk, out_of, steps, warmup):
    """time `steps` passes over `items` (CUDA events, after `warmup` passes): the background walk of item i+1 under the
    raster of item i, rasters alternating between two streams.  walk(i, stream) -> ticket; renderer_of(i) rasters it into
    out_of(i).  -> ms per pass"""
    import torch
    main = torch.cuda.current_stream()
    side = [torch.cuda.Stream() for _ in range(2)]
    walk_stream = torch.cuda.Stream(priority=-1)

    def one_pass():
        for t in side:
            t.wait_stream(main)
        ticket = walk(0, walk_stream.cuda_stream)
        for i in range(len(items)):
            renderer_of(i).raster_device(ticket, out_of(i), 0, side[i & 1].cuda_stream)
            if i + 1 < len(items):
                ticket = walk(i + 1, walk_stream.cuda_stream)
        for t in side:
            main.wait_stream(t)

    for _ in range(max(warmup, 1)):
        one_pass()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        one_pass()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


class NineRenderers:
    """(a): one renderer per map, batches of `batch` poses round-robin over the maps (the loop of jobs.run_maps with c3's
    interleave, without its per-launch profiling)"""

    def __init__(self, scenes, poses, width, height, batch):
        import torch
        import rust_doom_b200 as b2d
        self.rs = [b2d.Renderer(s, b2d.make_view(width, height), max_batch=batch) for s in scenes]
        self.dp = [torch.from_numpy(p.view(np.int32).reshape(-1, 4).copy()).cuda() for p in poses]
        self.outs = [torch.empty((len(p), height, width), dtype=torch.uint8, device="cuda") for p in poses]
        self.npix = width * height
        self.items = [(m, b0, min(batch, len(poses[m]) - b0)) for b0 in range(0, max(len(p) for p in poses), batch)
                      for m in range(len(scenes)) if b0 < len(poses[m])]

    def run(self, steps, warmup):
        def walk(i, st):
            m, b0, cnt = self.items[i]
            return self.rs[m].walk_device(self.dp[m].data_ptr() + 16 * b0, cnt, st)

        l0 = sum(r.launch_count for r in self.rs)
        ms = pipelined(lambda i: self.rs[self.items[i][0]], self.items, walk,
                       lambda i: self.outs[self.items[i][0]].data_ptr() + self.npix * self.items[i][1], steps, warmup)
        return ms, (sum(r.launch_count for r in self.rs) - l0) // (steps + max(warmup, 1))

    def status(self):
        bits = 0
        for r in self.rs:
            bits |= r.status()
        return bits


class LevelSet:
    """(b): one renderer over the maps; a batch takes `batch` poses of every map, frame j of a batch on map j % maps"""

    def __init__(self, scenes, poses, width, height, batch):
        import torch
        import rust_doom_b200 as b2d
        nmap = len(scenes)
        self.r = b2d.Renderer.from_levels(scenes, b2d.make_view(width, height), max_batch=batch * nmap)
        npose = len(poses[0])
        assert all(len(p) == npose for p in poses)
        self.order, levels = [], []
        for b0 in range(0, npose, batch):
            cnt = min(batch, npose - b0)
            for j in range(cnt * nmap):
                self.order.append((j % nmap, b0 + j // nmap))
                levels.append(j % nmap)
        flat = np.concatenate([poses[m][i:i + 1] for m, i in self.order])
        self.levels = np.array(levels, np.uint32)
        self.dp = torch.from_numpy(flat.view(np.int32).reshape(-1, 4).copy()).cuda()
        self.out = torch.empty((len(flat), height, width), dtype=torch.uint8, device="cuda")
        self.npix = width * height
        self.items = [(f0, min(batch * nmap, len(flat) - f0)) for f0 in range(0, len(flat), batch * nmap)]

    def run(self, steps, warmup):
        def walk(i, st):
            f0, cnt = self.items[i]
            return self.r.walk_device_levels(self.dp.data_ptr() + 16 * f0, self.levels[f0:f0 + cnt], cnt, st)

        l0 = self.r.launch_count
        ms = pipelined(lambda i: self.r, self.items, walk, lambda i: self.out.data_ptr() + self.npix * self.items[i][0],
                       steps, warmup)
        return ms, (self.r.launch_count - l0) // (steps + max(warmup, 1))


def walk_cost(scene, poses, width, height, rounds=3, steps=10):
    """walk kernel ms per batch of len(poses) frames on a level set of one: plain walk against the per-frame-level walk,
    foreground (render_device / render_device_levels: one CTA per frame, nothing to hide behind) and background
    (walk_device / walk_device_levels: the persistent grid, rastered on the same stream afterwards).  Medians of
    `rounds` alternated rounds; every walk timed by the library's per-launch events."""
    import torch
    import rust_doom_b200 as b2d
    n = len(poses)
    r = b2d.Renderer.from_levels([scene], b2d.make_view(width, height), max_batch=n)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    out = torch.empty((n, height, width), dtype=torch.uint8, device="cuda")
    zeros = np.zeros(n, np.uint32)
    st = torch.cuda.current_stream().cuda_stream
    arms = {
        "foreground_plain": lambda: r.render_device(dp.data_ptr(), n, out.data_ptr(), 0, st),
        "foreground_levels": lambda: r.render_device_levels(dp.data_ptr(), zeros, n, out.data_ptr(), 0, st),
        "background_plain": lambda: r.raster_device(r.walk_device(dp.data_ptr(), n, st), out.data_ptr(), 0, st),
        "background_levels": lambda: r.raster_device(r.walk_device_levels(dp.data_ptr(), zeros, n, st), out.data_ptr(), 0, st),
    }
    got = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            for _ in range(2):
                fn()
            torch.cuda.synchronize()
            r.profile(True)
            r.profile_read()
            for _ in range(steps):
                fn()
            w, _, b = r.profile_read()
            r.profile(False)
            got[k].append(w / b)
    return {k + "_walk_ms": round(float(np.median(v)), 4) for k, v in got.items()}, r.status()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=222, help="poses per map")
    ap.add_argument("--batches", default="8,32,111", help="per-map batch sizes")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    import rust_doom_b200 as b2d
    from rust_doom_b200 import build, poses as P, synthwad
    build.build()
    width, height = 1920, 1080
    scenes = [b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(10 + i, ("E1M%d" % i,))), 0) for i in range(1, 10)]
    poses = [P.flythrough_poses(s, args.poses, 2) for s in scenes]
    for batch in [int(b) for b in args.batches.split(",")]:
        a, b = NineRenderers(scenes, poses, width, height, batch), LevelSet(scenes, poses, width, height, batch)
        ta, tb = [], []
        for arm in (a, b, b, a):                                 # alternated, so drift falls on both arms alike
            ms, launches = arm.run(args.steps, args.warmup)
            (ta if arm is a else tb).append((ms, launches))
        info = gpu_info()
        same = all(torch.equal(b.out[k], a.outs[m][i]) for k, (m, i) in enumerate(b.order))
        line = dict(info, width=width, height=height, maps=len(scenes), poses_per_map=args.poses, per_map_batch=batch,
                    frames_per_pass=int(sum(len(p) for p in poses)),
                    nine_renderers_ms_per_pass=[round(t[0], 3) for t in ta], nine_renderers_launches_per_pass=ta[0][1],
                    level_set_ms_per_pass=[round(t[0], 3) for t in tb], level_set_launches_per_pass=tb[0][1],
                    level_set_batch=batch * len(scenes), frames_identical=bool(same),
                    status_bits=int(a.status()) | int(b.r.status()))
        print(json.dumps(line), flush=True)
        del a, b
        torch.cuda.empty_cache()
    c2 = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",))), 0)
    walk, bits = walk_cost(c2, P.flythrough_poses(c2, 1000, 2), width, height)
    print(json.dumps(dict(gpu_info(), what="walk kernel ms per 1000-frame batch, c2 level, 1080p, level set of one",
                          status_bits=int(bits), **walk)), flush=True)


if __name__ == "__main__":
    main()
