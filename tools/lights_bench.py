"""The cost of the player's light effects (DESIGN.md C18) on the c3 level set: one renderer over nine maps through
b2d_walk_device_levels_states_lights + b2d_raster_device, frames without lights against a mix with fixed colormaps and
extra light.

    python tools/lights_bench.py [--poses 222] [--batch 32] [--fixed 0.1] [--extra 0.1] [--steps 20] [--warmup 2]

The shape of tools/levels_states_bench.py's level-set arm (synthetic E1M1-E1M9, seeds 11-19, a fly-through per map,
1920x1080 index frames, pose i of map m at level time 1000 m + i, batches of `batch` poses of every map).  Arm `plain`
passes no lights; arm `lit` gives a seeded `fixed` share of the frames fixed colormap 32 (invulnerability) and another
`extra` share extra light 1 or 2 (weapon flashes).  The arms alternate (plain, lit, lit, plain) in one process, through
tools/levels_bench.py's `pipelined` loop.  Prints one JSON line: ms and launches per pass of both arms, the table sets per
pass of both, and the card name, power limit and SM clock, read in the same run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.levels_bench import gpu_info, pipelined  # noqa: E402
from tools.levels_states_bench import LevelSet  # noqa: E402


class LitLevelSet(LevelSet):
    """LevelSet with a (fixed_colormap, extralight) per frame (None: the call without lights)"""

    def __init__(self, scenes, poses, tics, width, height, batch, lights):
        super().__init__(scenes, poses, tics, width, height, batch)
        self.lights = lights

    def walk(self, i, st):
        f0, cnt = self.items[i]
        return self.r.walk_device_levels_states(self.dp.data_ptr() + 16 * f0, self.levels[f0:f0 + cnt], self.tics[f0:f0 + cnt],
                                                cnt, None, st, lights=None if self.lights is None else self.lights[f0:f0 + cnt])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=222, help="poses per map")
    ap.add_argument("--batch", type=int, default=32, help="per-map batch size")
    ap.add_argument("--fixed", type=float, default=0.1, help="share of frames with fixed colormap 32")
    ap.add_argument("--extra", type=float, default=0.1, help="share of frames with extra light 1 or 2")
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
    plain = LitLevelSet(scenes, poses, tics, width, height, args.batch, None)
    n = len(plain.levels)
    rng = np.random.default_rng(7)
    u = rng.random(n)
    lights = [(32, 0) if u[i] < args.fixed else (-1, int(rng.integers(1, 3))) if u[i] < args.fixed + args.extra else (-1, 0)
              for i in range(n)]
    lit = LitLevelSet(scenes, poses, tics, width, height, args.batch, lights)
    tp, tl = [], []
    for arm in (plain, lit, lit, plain):                         # alternated, so drift falls on both arms alike
        l0 = arm.r.launch_count
        ms = pipelined(lambda i: arm.r, arm.items, arm.walk, lambda i: arm.out.data_ptr() + arm.npix * arm.items[i][0],
                       args.steps, args.warmup)
        (tp if arm is plain else tl).append((ms, (arm.r.launch_count - l0) // (args.steps + max(args.warmup, 1))))
    line = dict(gpu_info(), width=width, height=height, maps=len(scenes), poses_per_map=args.poses,
                level_set_batch=args.batch * len(scenes), frames_per_pass=n,
                fixed_share=args.fixed, extra_share=args.extra,
                frames_fixed=sum(1 for f, _ in lights if f >= 0), frames_extra=sum(1 for _, e in lights if e),
                plain_ms_per_pass=[round(t[0], 3) for t in tp], plain_launches_per_pass=tp[0][1],
                lit_ms_per_pass=[round(t[0], 3) for t in tl], lit_launches_per_pass=tl[0][1],
                plain_sets_per_pass=plain.sets_per_pass(), lit_sets_per_pass=lit.sets_per_pass(),
                status_bits=int(plain.r.status()) | int(lit.r.status()))
    print(json.dumps(line), flush=True)
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
