#!/usr/bin/env python3
"""Device-resident frames/s of the walk+raster step at several resolutions (CUDA events, 3 warm-ups, inputs and
outputs in HBM).  Informational table; the headline number is bench.py's.
usage: python tools/sweep_res.py [n_poses]"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rust_doom_b200 as b2d  # noqa: E402
from rust_doom_b200 import poses as P, synthwad  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 400
    rows = []
    cases = [("SYN_E1M1 seed 1", 1, ("E1M1",), synthwad.SynthConfig()),
             ("SYN_E1M1 seed 1 + masked middles, sprites, animation", 1, ("E1M1",),
              synthwad.SynthConfig(mid_pct=30, thing_pct=50, anim=True))]
    if os.environ.get("B2D_SWEEP_PARTS"):      # which kind of content costs what (1080p only)
        cases = [("plain", 1, ("E1M1",), synthwad.SynthConfig()),
                 ("masked middles only", 1, ("E1M1",), synthwad.SynthConfig(mid_pct=30)),
                 ("sprites only", 1, ("E1M1",), synthwad.SynthConfig(thing_pct=50)),
                 ("animation / light effects only", 1, ("E1M1",), synthwad.SynthConfig(anim=True))]
    if os.environ.get("B2D_SWEEP_FULL"):       # the content-rich level alone (for ncu captures)
        cases = cases[1:]
    for name, seed, maps, cfg in cases:
        sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(seed, maps, cfg=cfg)), 0)
        poses = P.flythrough_poses(sc, n, 2)
        dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
        for (w, h) in (((1920, 1080),) if (os.environ.get("B2D_SWEEP_PARTS") or os.environ.get("B2D_SWEEP_FULL")) else ((320, 200), (1280, 720), (1920, 1080), (3840, 2160))):
            m = n if w < 3000 else n // 4
            r = b2d.Renderer(sc, b2d.make_view(w, h), max_batch=m)
            out = torch.empty((m, h, w), dtype=torch.uint8, device="cuda")
            for _ in range(3):
                r.render_device(dp.data_ptr(), m, out.data_ptr())
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 10
            e0.record()
            for _ in range(reps):
                r.render_device(dp.data_ptr(), m, out.data_ptr())
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            rows.append({"level": name, "w": w, "h": h, "frames": m, "ms_per_batch": ms, "frames_per_s": m / ms * 1e3,
                         "GBps": m * w * h / ms / 1e6})
            del r, out
    print(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
