"""Nine maps on one GPU with a running clock per map, two ways: nine renderers through per-frame states
(b2d_walk_device_states + b2d_raster_device) and one level set through per-frame states and levels
(b2d_walk_device_levels_states).

    python tools/levels_states_bench.py [--poses 222] [--batches 8,32,111] [--steps 20] [--warmup 2]

The c3 shape of tools/levels_bench.py (synthetic E1M1-E1M9, seeds 11-19, with the generator's default light effects; a
fly-through per map; 1920x1080 index frames), with a clock: pose i of map m is at level time 1000 m + i, as
tools/timeline_bench.py runs one map.  For each per-map batch size B, one pass renders every map's poses: (a) in batches of
B per map, round-robin over the maps, each map's renderer walking its batch at the batch's tics; (b) in batches of 9 B
frames that take B poses of every map (frame j of a batch on map j mod 9), each frame at its own tic.  Both run
tools/levels_bench.py's `pipelined` loop and alternate (a, b, b, a) per batch size.  Prints one JSON line per batch size
with ms and launches per pass of both arms, the host-to-device bytes per batch (summed from the memcpy records of one
profiled pass, so they follow the distinct table sets each batch uploads), the distinct table sets per pass, and whether
(b)'s frames equal (a)'s byte for byte.  The card name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.levels_bench import gpu_info, pipelined  # noqa: E402


def h2d_bytes(fn):
    """host-to-device bytes copied by the work `fn` enqueues (torch.profiler's memcpy records), and the number of copies"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    copies = [e for e in trace.get("traceEvents", []) if e.get("cat") == "gpu_memcpy" and "HtoD" in e.get("name", "")]
    return sum(int(e.get("args", {}).get("bytes", 0)) for e in copies), len(copies)


class NineRenderers:
    """(a): one renderer per map, batches of `batch` poses round-robin over the maps, per-frame states"""

    def __init__(self, scenes, poses, tics, width, height, batch):
        import torch
        import rust_doom_b200 as b2d
        self.rs = [b2d.Renderer(s, b2d.make_view(width, height), max_batch=batch) for s in scenes]
        self.dp = [torch.from_numpy(p.view(np.int32).reshape(-1, 4).copy()).cuda() for p in poses]
        self.tics = tics
        self.outs = [torch.empty((len(p), height, width), dtype=torch.uint8, device="cuda") for p in poses]
        self.npix = width * height
        self.items = [(m, b0, min(batch, len(poses[m]) - b0)) for b0 in range(0, max(len(p) for p in poses), batch)
                      for m in range(len(scenes)) if b0 < len(poses[m])]

    def walk(self, i, st):
        m, b0, cnt = self.items[i]
        return self.rs[m].walk_device_states(self.dp[m].data_ptr() + 16 * b0, self.tics[m][b0:b0 + cnt], cnt, None, st)

    def run(self, steps, warmup):
        l0 = sum(r.launch_count for r in self.rs)
        ms = pipelined(lambda i: self.rs[self.items[i][0]], self.items, self.walk,
                       lambda i: self.outs[self.items[i][0]].data_ptr() + self.npix * self.items[i][1], steps, warmup)
        return ms, (sum(r.launch_count for r in self.rs) - l0) // (steps + max(warmup, 1))

    def sets_per_pass(self):
        n = 0
        for i in range(len(self.items)):
            r = self.rs[self.items[i][0]]
            r.raster_device(self.walk(i, 0), self.outs[self.items[i][0]].data_ptr() + self.npix * self.items[i][1])
            n += int(r.state_slots(self.items[i][2]).max()) + 1
        return n

    def status(self):
        bits = 0
        for r in self.rs:
            bits |= r.status()
        return bits


class LevelSet:
    """(b): one renderer over the maps; a batch takes `batch` poses of every map, frame j of a batch on map j % maps, each
    frame at its own tic"""

    def __init__(self, scenes, poses, tics, width, height, batch):
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
        self.tics = np.array([tics[m][i] for m, i in self.order], np.uint32)
        self.dp = torch.from_numpy(flat.view(np.int32).reshape(-1, 4).copy()).cuda()
        self.out = torch.empty((len(flat), height, width), dtype=torch.uint8, device="cuda")
        self.npix = width * height
        self.items = [(f0, min(batch * nmap, len(flat) - f0)) for f0 in range(0, len(flat), batch * nmap)]

    def walk(self, i, st):
        f0, cnt = self.items[i]
        return self.r.walk_device_levels_states(self.dp.data_ptr() + 16 * f0, self.levels[f0:f0 + cnt], self.tics[f0:f0 + cnt],
                                                cnt, None, st)

    def run(self, steps, warmup):
        l0 = self.r.launch_count
        ms = pipelined(lambda i: self.r, self.items, self.walk, lambda i: self.out.data_ptr() + self.npix * self.items[i][0],
                       steps, warmup)
        return ms, (self.r.launch_count - l0) // (steps + max(warmup, 1))

    def sets_per_pass(self):
        n = 0
        for i in range(len(self.items)):
            self.r.raster_device(self.walk(i, 0), self.out.data_ptr() + self.npix * self.items[i][0])
            slots = self.r.state_slots(self.items[i][1])
            n += len(set(slots.tolist()) - {0xFFFFFFFF})
        return n


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
    tics = [np.arange(args.poses, dtype=np.uint32) + 1000 * m for m in range(len(scenes))]
    for batch in [int(b) for b in args.batches.split(",")]:
        a = NineRenderers(scenes, poses, tics, width, height, batch)
        b = LevelSet(scenes, poses, tics, width, height, batch)
        ta, tb = [], []
        for arm in (a, b, b, a):                                 # alternated, so drift falls on both arms alike
            ms, launches = arm.run(args.steps, args.warmup)
            (ta if arm is a else tb).append((ms, launches))
        info = gpu_info()
        same = all(torch.equal(b.out[k], a.outs[m][i]) for k, (m, i) in enumerate(b.order))
        ha, ca = h2d_bytes(lambda: a.run(1, 0))                 # run(1, 0): two passes (one untimed warm-up pass)
        hb, cb = h2d_bytes(lambda: b.run(1, 0))
        line = dict(info, width=width, height=height, maps=len(scenes), poses_per_map=args.poses, per_map_batch=batch,
                    frames_per_pass=int(sum(len(p) for p in poses)),
                    nine_renderers_ms_per_pass=[round(t[0], 3) for t in ta], nine_renderers_launches_per_pass=ta[0][1],
                    level_set_ms_per_pass=[round(t[0], 3) for t in tb], level_set_launches_per_pass=tb[0][1],
                    level_set_batch=batch * len(scenes),
                    nine_renderers_h2d_bytes_per_batch=round(ha / (2 * len(a.items))), nine_renderers_h2d_copies_per_pass=ca // 2,
                    level_set_h2d_bytes_per_batch=round(hb / (2 * len(b.items))), level_set_h2d_copies_per_pass=cb // 2,
                    nine_renderers_sets_per_pass=a.sets_per_pass(), level_set_sets_per_pass=b.sets_per_pass(),
                    frames_identical=bool(same), status_bits=int(a.status()) | int(b.r.status()))
        print(json.dumps(line), flush=True)
        del a, b
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
