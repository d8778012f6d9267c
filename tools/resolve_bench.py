"""The resolve kernel K4 (b2d_resolve_device) against K3 per level (b2d_palette_lut_levels_device), and what 2x
anti-aliasing costs per frame.

    python tools/resolve_bench.py [--frames 1000] [--rounds 5] [--reps 5] [--out FILE.json] [--palettes]

Frames: the c2 fly-through (synthetic SYN_E1M1, seed 1, 1920x1080), rendered once on the device.  Each round times, for
every factor in 1, 2, 4 and every format, `reps` resolve calls over all frames and, right after, `reps` K3-per-level calls
over the same frames (both with a host level array, so both stage it); CUDA events around each group.  Reported: the
median over rounds of ms per call, and GB/s of bytes read plus written (K4: W*H + (W/k)*(H/k)*bytes per pixel per frame;
K3: 5 bytes per pixel).  Then the render alone at 1920x1080 and at 3840x2160 (plain b2d_render_device batches, events
around the batches) and the 2x resolve of the 4K frames: the per-frame cost of 2x anti-aliasing.  The card's name, power
limit and SM clock are read in the same run.

--palettes times per-frame palettes instead: b2d_resolve_device against b2d_resolve_palettes_device with every frame on
palette 0 and with seeded random palettes 0..13, the three calls alternated within each round, at 1080p grey k=2, 1080p
planar RGB k=2, 1080p RGB k=1 and 4K RGB k=2 (the 4K frames rendered from the same poses).  Both calls stage one u32 per
frame and run the same kernel, so the expectation is equal times within noise.
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

W, H = 1920, 1080
FORMATS = ("rgba", "rgb", "rgb_planar", "gray")
BPP = {"rgba": 4, "rgb": 3, "rgb_planar": 3, "gray": 1}


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


def render_frames(b2d, scene, poses, w, h, batch):
    """(renderer, device index frames [n, h, w], fn that renders them all again)"""
    import torch
    n = len(poses)
    r = b2d.Renderer.from_levels([scene], b2d.make_view(w, h), max_batch=batch)
    dp = torch.from_numpy(np.ascontiguousarray(poses).view(np.int32).reshape(-1, 4).copy()).cuda()
    idx = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")

    def run():
        for i in range(0, n, batch):
            m = min(batch, n - i)
            r.render_device(dp[i:i + m].data_ptr(), m, idx[i:i + m].data_ptr())
    run()
    torch.cuda.synchronize()
    assert r.status() == 0
    return r, idx, run


def palette_rows(b2d, scene, poses, args):
    """--palettes: ms per call of the three calls at each shape, median and spread over rounds"""
    import torch
    n = len(poses)
    levels = np.zeros(n, np.uint32)
    zero = np.zeros(n, np.uint32)
    rand = np.random.default_rng(14).integers(0, 14, n).astype(np.uint32)
    rows = []
    for (w, h), k, fmt in (((W, H), 2, "gray"), ((W, H), 2, "rgb_planar"), ((W, H), 1, "rgb"), ((2 * W, 2 * H), 2, "rgb")):
        r, idx, _ = render_frames(b2d, scene, poses, w, h, 250 if w == W else 125)
        code = b2d.RESOLVE_FORMATS[fmt]
        out = torch.empty(n * r.resolve_frame_bytes(k, code), dtype=torch.uint8, device="cuda")
        calls = {"resolve_device": lambda: r.resolve_device(idx.data_ptr(), n, k, code, out.data_ptr(), levels),
                 "palettes_0": lambda: r.resolve_device(idx.data_ptr(), n, k, code, out.data_ptr(), levels, palettes=zero),
                 "palettes_random": lambda: r.resolve_device(idx.data_ptr(), n, k, code, out.data_ptr(), levels, palettes=rand)}
        for fn in calls.values():
            fn()
        torch.cuda.synchronize()
        t = {c: [] for c in calls}
        for _ in range(args.rounds):
            for c, fn in calls.items():
                t[c].append(timed(fn, args.reps))
        row = {"view": "%dx%d" % (w, h), "factor": k, "format": fmt}
        for c in calls:
            row[c] = {"ms": round(statistics.median(t[c]), 3), "ms_min": round(min(t[c]), 3), "ms_max": round(max(t[c]), 3)}
        rows.append(row)
        print("%s k=%d %-10s " % (row["view"], k, fmt) + "  ".join("%s %.3f ms (%.3f .. %.3f)" % (c, v["ms"], v["ms_min"], v["ms_max"])
                                                                 for c, v in ((c, row[c]) for c in calls)))
        del r, idx, out
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--palettes", action="store_true", help="time per-frame palettes against b2d_resolve_device")
    args = ap.parse_args()
    import torch
    import rust_doom_b200 as b2d
    from rust_doom_b200 import poses as P, synthwad
    assert torch.cuda.is_available(), "resolve_bench measures on a GPU; there is no CPU number"
    n = args.frames
    scene = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",))), 0)
    poses = P.flythrough_poses(scene, n, 2)
    if args.palettes:
        res = {"frames": n, "rounds": args.rounds, "reps": args.reps, "palettes": palette_rows(b2d, scene, poses, args)}
        res.update(gpu_info())
        print(json.dumps(res))
        if args.out:
            with open(args.out, "w") as f:
                json.dump(res, f, indent=1)
        return
    r, idx, render_1x = render_frames(b2d, scene, poses, W, H, 250)
    levels = np.zeros(n, np.uint32)
    out = torch.empty(n * W * H * 4, dtype=torch.uint8, device="cuda")
    cases = [(k, f) for k in (1, 2, 4) for f in FORMATS]

    def k4(k, fmt):
        return lambda: r.resolve_device(idx.data_ptr(), n, k, b2d.RESOLVE_FORMATS[fmt], out.data_ptr(), levels)

    def k3():
        r.palette_lut_levels_device(idx.data_ptr(), levels, n, out.data_ptr())

    for k, fmt in cases:                                  # warm-up: every kernel and the staging at full size
        k4(k, fmt)()
    k3()
    torch.cuda.synchronize()
    t4 = {c: [] for c in cases}
    t3 = []
    for _ in range(args.rounds):
        for c in cases:
            t4[c].append(timed(k4(*c), args.reps))
            t3.append(timed(k3, args.reps))
    rows = []
    k3_ms = statistics.median(t3)
    k3_gbs = n * W * H * 5 / (k3_ms * 1e-3) / 1e9
    for k, fmt in cases:
        ms = statistics.median(t4[(k, fmt)])
        moved = n * (W * H + (W // k) * (H // k) * BPP[fmt])
        rows.append({"factor": k, "format": fmt, "ms": round(ms, 3), "gbs": round(moved / (ms * 1e-3) / 1e9, 1),
                     "ms_min": round(min(t4[(k, fmt)]), 3), "ms_max": round(max(t4[(k, fmt)]), 3)})
    # 2x anti-aliasing: the render at 1x, at 2x, and the 2x resolve to 1x RGB
    del out
    rr, idx4, render_2x = render_frames(b2d, scene, poses, 2 * W, 2 * H, 125)
    rgb = torch.empty((n, H, W, 3), dtype=torch.uint8, device="cuda")

    def aa_resolve():
        rr.resolve_device(idx4.data_ptr(), n, 2, b2d.RESOLVE_RGB8, rgb.data_ptr(), levels)
    aa_resolve()
    t1, t2, tr = [], [], []
    for _ in range(args.rounds):
        t1.append(timed(render_1x, 1))
        t2.append(timed(render_2x, 1))
        tr.append(timed(aa_resolve, 1))
    r1, r2, rs = (statistics.median(t) for t in (t1, t2, tr))
    aa = {"render_1080p_ms_per_frame": round(r1 / n, 4), "render_4k_ms_per_frame": round(r2 / n, 4),
          "resolve_4k_to_1080p_rgb_ms_per_frame": round(rs / n, 4),
          "aa2x_cost_ms_per_frame": round((r2 + rs - r1) / n, 4), "aa2x_over_1x": round((r2 + rs) / r1, 2)}
    res = {"frames": n, "view": "%dx%d" % (W, H), "rounds": args.rounds, "reps": args.reps,
           "k3_levels": {"ms": round(k3_ms, 3), "gbs": round(k3_gbs, 1), "ms_min": round(min(t3), 3), "ms_max": round(max(t3), 3)},
           "k4": rows, "aa2x": aa}
    res.update(gpu_info())
    print("K3 per level: %.3f ms  %.0f GB/s" % (k3_ms, k3_gbs))
    for row in rows:
        print("K4 k=%d %-10s %8.3f ms  %6.0f GB/s  (%.3f .. %.3f)" % (row["factor"], row["format"], row["ms"], row["gbs"],
                                                                    row["ms_min"], row["ms_max"]))
    print("2x AA: " + json.dumps(aa))
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
