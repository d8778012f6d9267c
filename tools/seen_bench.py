"""The seen raster variant (b2d_raster_device_seen, DESIGN.md C20) against the plain raster, in bench.py's pipelined loop.

    python tools/seen_bench.py [--frames 1000] [--steps 20] [--rounds 5] [--out FILE.json]

Workload: the c2 level (synthetic SYN_E1M1, seed 1, as bench.py) with a 1000-pose fly-through, at 1920x1080 and
3840x2160, index frames only.  A step is bench.py's pipelined step: the raster of the walked batch of all frames on one of
two raster streams, then the walk of the next batch on a high-priority walk stream.  Each round times `steps` steps with
b2d_raster_device, then `steps` steps with b2d_raster_device_seen into one row per frame (zeroed once: the rows
accumulate, as an agent's would), CUDA events around each group; the two alternate round by round.  Reported: the median
over rounds of ms per step and the range, and the seen variant's cost against the plain raster.  The card's name, power
limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.levels_bench import gpu_info  # noqa: E402

SIZES = ((1920, 1080), (3840, 2160))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    import torch

    import rust_doom_b200 as b2d
    from rust_doom_b200 import poses as P
    from rust_doom_b200 import synthwad
    if not torch.cuda.is_available():
        raise SystemExit("seen_bench needs a GPU")
    n = args.frames
    scene = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",))), 0)
    poses = P.flythrough_poses(scene, n, 2)
    dp = torch.from_numpy(np.ascontiguousarray(poses).view(np.uint8).reshape(-1).copy()).cuda()
    info = gpu_info()
    rows = []
    for w, h in SIZES:
        r = b2d.Renderer(scene, b2d.make_view(w, h), max_batch=n)
        outs = [torch.empty((n, h, w), dtype=torch.uint8, device="cuda") for _ in range(2)]
        seen = torch.zeros((n, r.seen_words), dtype=torch.int32, device="cuda")
        main_stream = torch.cuda.current_stream()
        walk_stream = torch.cuda.Stream(priority=-1)
        raster_streams = [torch.cuda.Stream() for _ in range(2)]
        pending = [r.walk_device(dp.data_ptr(), n, walk_stream.cuda_stream)]
        turn = [0]

        def step(with_seen):
            b = turn[0] % 2
            turn[0] += 1
            rs = raster_streams[b].cuda_stream
            if with_seen:
                r.raster_device_seen(pending[0], outs[b].data_ptr(), seen.data_ptr(), rs)
            else:
                r.raster_device(pending[0], outs[b].data_ptr(), 0, rs)
            pending[0] = r.walk_device(dp.data_ptr(), n, walk_stream.cuda_stream)

        def timed(with_seen):
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for t in raster_streams:
                t.wait_stream(main_stream)
            a.record()
            for _ in range(args.steps):
                step(with_seen)
            for t in raster_streams:
                main_stream.wait_stream(t)
            e.record()
            e.synchronize()
            return a.elapsed_time(e) / args.steps

        timed(False)                 # warm-up: both variants' modules and the seen tables
        timed(True)
        times = {"raster_device": [], "raster_device_seen": []}
        for _ in range(args.rounds):
            times["raster_device"].append(timed(False))
            times["raster_device_seen"].append(timed(True))
        torch.cuda.synchronize()
        assert r.status() == 0
        lines = len(b2d.seen_lines(np.bitwise_or.reduce(seen.cpu().numpy().view(np.uint32), axis=0)))
        base = statistics.median(times["raster_device"])
        for k, t in times.items():
            rows.append({"size": "%dx%d" % (w, h), "case": k, "frames": n, "ms_median": statistics.median(t), "ms_min": min(t),
                         "ms_max": max(t), "vs_plain_pct": 100.0 * (statistics.median(t) / base - 1.0), "lines_seen": lines})
        r.raster_device(pending[0], outs[0].data_ptr(), 0)
        torch.cuda.synchronize()
        r.close()
    for row in rows:
        print("%-9s %-19s %8.3f ms/step (%.3f-%.3f)  %+6.2f %%  (%d lines seen)" % (
            row["size"], row["case"], row["ms_median"], row["ms_min"], row["ms_max"], row["vs_plain_pct"], row["lines_seen"]))
    print(json.dumps(info))
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"bench": "seen", "gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
