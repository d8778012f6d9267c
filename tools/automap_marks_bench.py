"""The marks automap (b2d_automap_marks_device, DESIGN.md C22) against the state automap (b2d_automap_states_device) on
the same frames.

    python tools/automap_marks_bench.py [--frames 1000] [--rounds 5] [--reps 3] [--out FILE.json]

Workload: the c2 level (synthetic SYN_E1M1, seed 1) and the content-rich level (tests/test_lights.py rich_wad), each
with ten digit patches from a PWAD overlay, a 1000-pose fly-through, Doom's default scale 0.2, at 1920x1080 and 320x200.
Cases, alternated within each round: the state automap at rest without arrows; the marks automap with the grid off and
no marks; with the grid on; with the grid on and 10 marks per frame (digits 0..9 around the pose, most on screen).
CUDA events around `reps` calls per case; the host builds the argument arrays once, outside the timing, so the times
include the call's host checks, its staging copy and the kernel.  Reported: median over rounds of ms per call, the
range, the difference from the state automap per frame, and for the grid the difference from grid off per 128 x 32
tile.  The card's name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.automap_bench import timed  # noqa: E402
from tools.levels_bench import gpu_info  # noqa: E402

SIZES = ((1920, 1080), (320, 200))


def _marks(poses, n):
    """10 marks per frame, digits 0..9, spread within 200 map units of the frame's pose"""
    rng = np.random.default_rng(7)
    out = []
    for i in range(n):
        px, py = int(poses["x"][i]), int(poses["y"][i])
        out.append([(int(np.clip(px + int(rng.integers(-200, 201)) * 65536, -2 ** 31, 2 ** 31 - 1)),
                     int(np.clip(py + int(rng.integers(-200, 201)) * 65536, -2 ** 31, 2 ** 31 - 1)), d) for d in range(10)])
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    import torch

    import rust_doom_b200 as b2d
    from rust_doom_b200 import _check, _frame_marks, _lib
    from rust_doom_b200 import poses as P
    from rust_doom_b200 import synthwad
    from tests.test_automap_marks import digit_images, digit_pwad
    from tests.test_lights import rich_wad
    if not torch.cuda.is_available():
        raise SystemExit("automap_marks_bench needs a GPU")
    n = args.frames
    overlay = digit_pwad(digit_images(1))
    info = gpu_info()
    L = _lib.load()
    rows = []
    for name, data in (("c2", synthwad.build_iwad(1, ("E1M1",))), ("rich", rich_wad())):
        scene = b2d.Scene(b2d.Archive.from_bytes(data, overlays=(overlay,)), 0)
        poses = P.flythrough_poses(scene, n, 2)
        dp = torch.from_numpy(np.ascontiguousarray(poses).view(np.uint8).reshape(-1).copy()).cuda()
        ten = _frame_marks(_marks(poses, n), n)
        for w, h in SIZES:
            r = b2d.Renderer(scene, b2d.make_view(w, h), max_batch=250)
            out = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
            tiles = ((w + 127) // 128) * ((h + 31) // 32)

            def marks_call(flags, marks=(None, None, 0)):
                return lambda: _check(L.b2d_automap_marks_device(r._h, dp.data_ptr(), None, None, None, 0, None, None, 0, None, n,
                                                                 13107, flags, out.data_ptr(), None, *marks))
            cases = {"states, at rest": lambda: _check(L.b2d_automap_states_device(r._h, dp.data_ptr(), None, None, None, 0, None,
                                                                                   None, 0, None, n, 13107, 0, out.data_ptr(),
                                                                                   None)),
                     "marks, grid off": marks_call(0),
                     "marks, grid on": marks_call(16),
                     "marks, grid on, 10 marks": marks_call(16, ten)}
            for fn in cases.values():                # warm-up: every case once
                fn()
            torch.cuda.synchronize()
            times = {k: [] for k in cases}
            for _ in range(args.rounds):
                for k, fn in cases.items():
                    times[k].append(timed(fn, args.reps))
            base = statistics.median(times["states, at rest"])
            off = statistics.median(times["marks, grid off"])
            for k, t in times.items():
                med = statistics.median(t)
                row = {"level": name, "size": "%dx%d" % (w, h), "case": k, "frames": n, "ms_median": med, "ms_min": min(t),
                       "ms_max": max(t), "us_per_frame": med * 1000.0 / n, "us_per_frame_over_states": (med - base) * 1000.0 / n}
                if k != "states, at rest":
                    row["ns_per_tile_over_grid_off"] = (med - off) * 1e6 / (n * tiles)
                rows.append(row)
            r.close()
    result = {"bench": "automap_marks", "gpu": info, "rows": rows}
    for row in rows:
        print("%-5s %-9s %-26s %8.3f ms (%.3f-%.3f)  %7.3f us/frame  %+7.3f us/frame over states  %s" % (
            row["level"], row["size"], row["case"], row["ms_median"], row["ms_min"], row["ms_max"], row["us_per_frame"],
            row["us_per_frame_over_states"],
            "" if "ns_per_tile_over_grid_off" not in row else "%+7.2f ns/tile over grid off" % row["ns_per_tile_over_grid_off"]))
    print(json.dumps(info))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
