"""Timelines whose level time changes every frame: what per-frame states cost against a time fixed per batch.

    python tools/timeline_bench.py [--rounds 3] [--batches 4] [--out DIR]

Workload: the bench.py c2 level (SYN_E1M1, seed 1) and its content-rich variant, the benchmark's 1000-pose fly-through at
1920x1080 (index frames), with a timeline of one tic per pose that continues across batches (batch k: tics 1000k ..).
Arms, alternated in one process, `--rounds` times each:
  A   time fixed per batch: set_time_async to the batch's first tic + the pipelined walk_device / raster_device pair (the
      ceiling: every frame of a batch shares one table set)
  B   walk_device_states / raster_device, pipelined the same way: every frame at its own tic
  B1  B with every frame of a batch at the batch's first tic, so that all frames share one table set (separates the cost of
      the per-frame addressing from the cost of 1000 table sets' L2 footprint)
  C   set_time_async + render_device per pose: what a per-pose timeline cost before per-frame states (one batch per round)
Per arm: ms per 1000 frames and frames/s (CUDA events around the arm's batches), host ms per batch in the calls that
build and enqueue states or tables, H2D bytes per batch (B: the batch's distinct compact states, counted from the
table-set index of every frame, plus one set index per frame).  Before timing, sampled frames of batch 0 are checked: B equal to
C and to the oracle at each frame's tic, A equal to the oracle at the batch's tic.  The card, its power limit and SM clock
are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import rust_doom_b200 as b2d  # noqa: E402
from oracle import render, scene as S  # noqa: E402
from rust_doom_b200 import poses as P, synthwad  # noqa: E402

LEVELS = {"c2": {}, "rich": dict(mid_pct=30, thing_pct=40, anim=True)}      # bench.py's c2 / rich levels
N, W, H = 1000, 1920, 1080
SAMPLE = (0, 333, 999)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def state_bytes(blob):
    """bytes of one compact state: 2 words + 2 per dynamic sector + the light bytes of the effect sectors, four to a word"""
    h = S.header(blob)
    n = h[S.H_NSECTORS]
    kinds = np.frombuffer(blob, "<u4", 8 * n, h[S.H_OFF_LIGHTS]).reshape(n, 8)[:, 0]
    return 4 * (2 + 2 * h[S.H_NDYN] + (int((kinds != 0).sum()) + 3) // 4)


def run_level(name, cfg, rounds, batches):
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(**cfg))
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    poses = P.flythrough_poses(sc, N, 2)
    view = b2d.make_view(W, H)
    r = b2d.Renderer(sc, view, max_batch=N)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    outs = [torch.empty((N, H, W), dtype=torch.uint8, device="cuda") for _ in range(2)]
    s_walk = torch.cuda.Stream(priority=-1)
    s_r = [torch.cuda.Stream(), torch.cuda.Stream()]
    main = torch.cuda.current_stream()
    table_bytes = len(sc.tables_at(0))
    tl = lambda k: (np.arange(N, dtype=np.uint64) + N * k).astype(np.uint32)     # noqa: E731

    host = {"A": 0.0, "B": 0.0, "B1": 0.0, "C": 0.0}

    def pipelined(arm, ks):
        """walk of batch k+1 under the raster of batch k (two raster streams), as bench.py's c2 step"""
        def walk(k):
            t0 = time.perf_counter()
            if arm == "A":
                r.set_time_async(int(tl(k)[0]), s_walk.cuda_stream)
                t = r.walk_device(dp.data_ptr(), N, s_walk.cuda_stream)
            elif arm == "B":
                t = r.walk_device_states(dp.data_ptr(), tl(k), N, None, s_walk.cuda_stream)
            else:
                t = r.walk_device_states(dp.data_ptr(), int(tl(k)[0]), N, None, s_walk.cuda_stream)
            host[arm] += time.perf_counter() - t0
            return t

        for s in [s_walk] + s_r:
            s.wait_stream(main)
        ticket = walk(ks[0])
        for j, k in enumerate(ks):
            r.raster_device(ticket, outs[j % 2].data_ptr(), 0, s_r[j % 2].cuda_stream)
            if j + 1 < len(ks):
                ticket = walk(ks[j + 1])
        for s in [s_walk] + s_r:
            main.wait_stream(s)

    def per_pose(k):
        t = tl(k)
        for i in range(N):
            t0 = time.perf_counter()
            r.set_time_async(int(t[i]), main.cuda_stream)
            host["C"] += time.perf_counter() - t0
            r.render_device(dp.data_ptr() + 16 * i, 1, outs[0].data_ptr() + i * W * H, 0, main.cuda_stream)

    # ---- parity: sampled frames of batch 0
    oblob = sc.blob
    oview = render.make_view(W, H)
    t0 = tl(0)
    pipelined("B", [0])
    torch.cuda.synchronize()
    fb_b = outs[0][list(SAMPLE)].cpu().numpy()
    per_pose(0)
    torch.cuda.synchronize()
    fb_c = outs[0][list(SAMPLE)].cpu().numpy()
    pipelined("A", [0])
    torch.cuda.synchronize()
    fb_a = outs[0][list(SAMPLE)].cpu().numpy()
    for j, i in enumerate(SAMPLE):
        want = render.render(oblob, oview, poses[i:i + 1], threads=os.cpu_count(), tics=int(t0[i]))[0]
        assert np.array_equal(fb_b[j], fb_c[j]), "B and C differ at frame %d" % i
        assert np.array_equal(fb_b[j], want), "B differs from the oracle at frame %d" % i
        want_a = render.render(oblob, oview, poses[i:i + 1], threads=os.cpu_count(), tics=int(t0[0]))[0]
        assert np.array_equal(fb_a[j], want_a), "A differs from the oracle at frame %d" % i
    assert r.status() == 0

    # ---- timing, arms alternated
    times = {a: [] for a in host}
    for a in host:
        host[a] = 0.0
    for rnd in range(rounds):
        for arm in ("A", "B", "B1", "C"):
            ks = list(range(rnd * batches, (rnd + 1) * batches)) if arm != "C" else [rnd]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            if arm == "C":
                per_pose(ks[0])
            else:
                pipelined(arm, ks)
            e1.record()
            torch.cuda.synchronize()
            times[arm].append(e0.elapsed_time(e1) / (len(ks) * N) * 1000.0)
    assert r.status() == 0
    # distinct states per batch of arm B, counted from the table-set index of every frame (outside the timed region)
    distinct = []
    for k in range(rounds * batches):
        ticket = r.walk_device_states(dp.data_ptr(), tl(k), N, None, s_walk.cuda_stream)
        distinct.append(int(r.state_slots(N).max()) + 1)
        r.raster_device(ticket, outs[0].data_ptr(), 0, s_walk.cuda_stream)
    torch.cuda.synchronize()
    nb = {"A": rounds * batches, "B": rounds * batches, "B1": rounds * batches, "C": rounds}
    sb = state_bytes(sc.blob)
    h2d = {"A": table_bytes, "B": round(float(np.mean(distinct)) * sb) + 4 * N, "B1": sb + 4 * N, "C": N * table_bytes}
    res = {}
    for arm in host:
        med = float(np.median(times[arm]))
        res[arm] = {"ms_per_1000_frames": round(med, 3), "range": [round(min(times[arm]), 3), round(max(times[arm]), 3)],
                    "frames_per_s": round(1e6 / med), "host_ms_per_batch": round(1e3 * host[arm] / nb[arm], 3),
                    "h2d_bytes_per_batch": h2d[arm]}
    return {"level": name, "table_bytes": table_bytes, "state_bytes": sb, "distinct_states_per_batch_B": distinct, "arms": res}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=int, default=4, help="pipelined batches per round (arms A, B, B1)")
    ap.add_argument("--out", default="", help="also write the results as JSON into this directory")
    args = ap.parse_args()
    from rust_doom_b200 import build as B
    B.build()
    info = card()
    print("card: %s (name, power limit, SM clock, max SM clock)" % info)
    out = {"card": info, "levels": []}
    for name, cfg in LEVELS.items():
        res = run_level(name, cfg, args.rounds, args.batches)
        out["levels"].append(res)
        print("%s: tables %d B, compact state %d B, distinct states per batch in B: %s" % (
            name, res["table_bytes"], res["state_bytes"], res["distinct_states_per_batch_B"]))
        for arm, v in res["arms"].items():
            print("  %-2s %9.3f ms / 1000 frames (%.3f-%.3f)  %8d frames/s  host %7.3f ms/batch  H2D %9d B/batch" % (
                arm, v["ms_per_1000_frames"], v["range"][0], v["range"][1], v["frames_per_s"], v["host_ms_per_batch"],
                v["h2d_bytes_per_batch"]))
    out["card_after"] = card()
    print("card after: %s" % out["card_after"])
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "timeline.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
