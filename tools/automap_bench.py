"""The automap kernel K5 (b2d_automap_device) against K3 per level (b2d_palette_lut_levels_device) and the render itself.

    python tools/automap_bench.py [--frames 1000] [--rounds 5] [--reps 3] [--out FILE.json]

Workloads: the c2 level (synthetic SYN_E1M1, seed 1) and the content-rich level (the same map with masked middles,
sprites and animated content, as bench.py's `rich`), 1000-pose fly-throughs, at 1920x1080 and 320x200.  Each round
times, per level and size, `reps` automap calls over all frames for every flag combination at Doom's default scale (0.2
pixels per map unit), then `reps` K3-per-level calls over the same number of frames (a host level array on both, so both
stage it), then the frames rendered with b2d_render_device batches of 250; CUDA events around each group.  Reported:
median over rounds of ms per call and the range, and the automap's cost per frame against the render's.  The card's name,
power limit and SM clock are read in the same run.
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

SIZES = ((1920, 1080), (320, 200))
FLAGS = {0: "north-up", 1: "rotate", 2: "all", 4: "things", 7: "rotate,all,things"}


def timed(fn, reps):
    """ms per call of fn(), CUDA events around `reps` calls"""
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    import torch

    import rust_doom_b200 as b2d
    from rust_doom_b200 import poses as P
    from rust_doom_b200 import synthwad
    if not torch.cuda.is_available():
        raise SystemExit("automap_bench needs a GPU")
    n = args.frames
    levels = {"c2": synthwad.build_iwad(1, ("E1M1",)),
              "rich": synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=30, thing_pct=40, anim=True))}
    info = gpu_info()
    rows = []
    for name, data in levels.items():
        scene = b2d.Scene(b2d.Archive.from_bytes(data), 0)
        poses = P.flythrough_poses(scene, n, 2)
        dp = torch.from_numpy(np.ascontiguousarray(poses).view(np.uint8).reshape(-1).copy()).cuda()
        lv = [0] * n
        for w, h in SIZES:
            r = b2d.Renderer(scene, b2d.make_view(w, h), max_batch=250)
            out = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
            rgba = torch.empty((n, h, w), dtype=torch.int32, device="cuda")
            cases = {"automap " + FLAGS[f]: (lambda f=f: r.automap_device(dp.data_ptr(), n, out.data_ptr(), 13107, f, lv))
                     for f in FLAGS}
            cases["K3 per level"] = lambda: r.palette_lut_levels_device(out.data_ptr(), lv, n, rgba.data_ptr())

            def render():
                for i in range(0, n, 250):
                    m = min(250, n - i)
                    r.render_device(dp.data_ptr() + 16 * i, m, out.data_ptr() + w * h * i)
            cases["render"] = render
            for fn in cases.values():            # warm-up: every shape once
                fn()
            torch.cuda.synchronize()
            times = {k: [] for k in cases}
            for _ in range(args.rounds):
                for k, fn in cases.items():
                    times[k].append(timed(fn, args.reps))
            assert r.status() == 0
            for k, t in times.items():
                rows.append({"level": name, "size": "%dx%d" % (w, h), "case": k, "frames": n, "ms_median": statistics.median(t),
                             "ms_min": min(t), "ms_max": max(t), "us_per_frame": statistics.median(t) * 1000.0 / n})
            r.close()
    result = {"bench": "automap", "gpu": info, "rows": rows}
    for row in rows:
        print("%-5s %-9s %-26s %8.3f ms (%.3f-%.3f)  %7.2f us/frame" % (row["level"], row["size"], row["case"], row["ms_median"],
                                                                         row["ms_min"], row["ms_max"], row["us_per_frame"]))
    print(json.dumps(info))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
