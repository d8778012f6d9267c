"""The state automap (b2d_automap_states_device, DESIGN.md C21) against the seen automap (b2d_automap_seen_device) on the
same frames.

    python tools/automap_states_bench.py [--frames 1000] [--rounds 5] [--reps 3] [--out FILE.json]

Workload: the c2 level (synthetic SYN_E1M1, seed 1) with 16 sectors declared dynamic (tests/refcheck/moves.py's
declaration), a 1000-pose fly-through, Doom's default scale 0.2, flags 0, a NULL seen row, at 1920x1080 and 320x200.
Cases, alternated within each round: the seen automap; the state automap at rest without arrows; a different random
state per frame; 4 arrows per frame (a co-op team: the frame's own pose and the next three); 63 arrows per frame (the
other agents of a 64-agent batch).  CUDA events around `reps` calls per case; the host builds the argument arrays once,
outside the timing, so the times include the call's host checks, its staging copy and the kernel.  Reported: median over
rounds of ms per call, the range, and the difference from the seen automap per frame.  The card's name, power limit and
SM clock are read in the same run.
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


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    import torch

    import rust_doom_b200 as b2d
    from oracle import wad as W
    from rust_doom_b200 import _check, _frame_arrows, _frame_states, _lib
    from rust_doom_b200 import poses as P
    from rust_doom_b200 import synthwad
    from tests.refcheck import moves as MV
    if not torch.cuda.is_available():
        raise SystemExit("automap_states_bench needs a GPU")
    n = args.frames
    data = synthwad.build_iwad(1, ("E1M1",))
    level = W.Level(W.Archive(data), 0)
    dynamic = MV.declare(level, 5, 16)
    scene = b2d.Scene(b2d.Archive.from_bytes(data), 0, dynamic=dynamic)
    poses = P.flythrough_poses(scene, n, 2)
    dp = torch.from_numpy(np.ascontiguousarray(poses).view(np.uint8).reshape(-1).copy()).cuda()
    per_state = [MV.state(level, dynamic, 1000 + i, hole_free=False) for i in range(n)]
    team = [[(int(p["x"]), int(p["y"]), int(p["angle"]), c) for p, c in zip(poses[i:i + 4], (112, 96, 64, 176))]
            for i in range(n)]
    batch = [[(int(p["x"]), int(p["y"]), int(p["angle"]), 96) for p in poses[(i // 64) * 64:(i // 64) * 64 + 64]][:63]
             for i in range(n)]
    info = gpu_info()
    L = _lib.load()
    rows = []
    for w, h in SIZES:
        r = b2d.Renderer(scene, b2d.make_view(w, h), max_batch=250)
        out = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")

        def states_call(states=None, arrows=None):
            st, mv, nm = _frame_states(0, states, n) if states is not None else (None, None, 0)
            rg, ar, na = _frame_arrows(arrows, n) if arrows is not None else (None, None, 0)
            return lambda: _check(L.b2d_automap_states_device(r._h, dp.data_ptr(), None, st, mv, nm, rg, ar, na, None, n, 13107, 0,
                                                              out.data_ptr(), None))
        cases = {"seen automap": lambda: _check(L.b2d_automap_seen_device(r._h, dp.data_ptr(), None, None, n, 13107, 0,
                                                                          out.data_ptr(), None)),
                 "states, at rest": states_call([[]] * n, [[]] * n),
                 "states, a state per frame": states_call(per_state),
                 "states, 4 arrows per frame": states_call(None, team),
                 "states, 63 arrows per frame": states_call(None, batch)}
        for fn in cases.values():                # warm-up: every case once
            fn()
        torch.cuda.synchronize()
        times = {k: [] for k in cases}
        for _ in range(args.rounds):
            for k, fn in cases.items():
                times[k].append(timed(fn, args.reps))
        base = statistics.median(times["seen automap"])
        for k, t in times.items():
            rows.append({"size": "%dx%d" % (w, h), "case": k, "frames": n, "ms_median": statistics.median(t), "ms_min": min(t),
                         "ms_max": max(t), "us_per_frame": statistics.median(t) * 1000.0 / n,
                         "us_per_frame_over_seen": (statistics.median(t) - base) * 1000.0 / n})
        r.close()
    result = {"bench": "automap_states", "gpu": info, "rows": rows}
    for row in rows:
        print("%-9s %-28s %8.3f ms (%.3f-%.3f)  %7.3f us/frame  %+7.3f us/frame over seen" % (
            row["size"], row["case"], row["ms_median"], row["ms_min"], row["ms_max"], row["us_per_frame"],
            row["us_per_frame_over_seen"]))
    print(json.dumps(info))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
