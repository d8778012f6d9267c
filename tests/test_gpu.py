"""-m gpu: parity of the CUDA path (through the C ABI) against the oracle, plus size-independent
properties at BASELINE.json's full sizes."""
import json
import os

import numpy as np
import pytest

from oracle import render
from tests.conftest import oracle_blob, sample_poses

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frames.json")


def _assert_same(ofb, gfb, what=""):
    bad = [(i, int((ofb[i] != gfb[i]).sum())) for i in range(len(ofb)) if not np.array_equal(ofb[i], gfb[i])]
    assert not bad, "%s: frames differ (index, pixels): %s" % (what, bad[:6])


def _loaded_native():
    from rust_doom_b200 import _lib
    maps = open("/proc/self/maps").read()
    assert _lib.LIB_PATH in maps, "libb2d.so is not mapped into this process"


def test_gpu_matches_oracle_320x200(b2d, product_scene):
    poses = sample_poses(b2d, product_scene, 96, 31)
    r = b2d.Renderer(product_scene, b2d.make_view(320, 200), max_batch=40)     # forces 3 batches
    gfb = r.render(poses)
    _loaded_native()
    ofb = render.render(product_scene.blob, render.make_view(320, 200), poses, threads=8)
    _assert_same(ofb, gfb, "320x200")
    assert r.launch_count == 6          # 3 batches of <= 40 frames: walk + raster each


def test_gpu_matches_oracle_odd_width(b2d, product_scene):
    poses = sample_poses(b2d, product_scene, 12, 32)
    for (w, h) in ((333, 187), (64, 48), (1000, 10)):
        gfb = b2d.Renderer(product_scene, b2d.make_view(w, h), max_batch=16).render(poses)
        ofb = render.render(product_scene.blob, render.make_view(w, h), poses, threads=8)
        _assert_same(ofb, gfb, "%dx%d" % (w, h))


def test_gpu_matches_oracle_1080p_and_4k(b2d, product_scene, oracle_scene):
    """The oracle renders from the scene ITS OWN compiler built (oracle/scene.py), the GPU from libb2d's."""
    poses = sample_poses(b2d, product_scene, 10, 33)
    gfb = b2d.Renderer(product_scene, b2d.make_view(1920, 1080), max_batch=16).render(poses)
    ofb = render.render(oracle_scene, render.make_view(1920, 1080), poses, threads=8)
    _assert_same(ofb, gfb, "1080p")
    gfb = b2d.Renderer(product_scene, b2d.make_view(3840, 2160), max_batch=4).render(poses[:3])
    ofb = render.render(oracle_scene, render.make_view(3840, 2160), poses[:3], threads=8)
    _assert_same(ofb, gfb, "4K")


@pytest.mark.parametrize("seed,maps,level", [(7, ("E2M3",), 0), (21, ("MAP01", "MAP12"), 1), (3, ("E1M1", "E1M2", "E1M3"), 2)])
def test_gpu_matches_oracle_other_maps(b2d, seed, maps, level):
    from rust_doom_b200 import synthwad
    sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(seed, maps)), level)
    poses = sample_poses(b2d, sc, 48, seed)
    gfb = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=64).render(poses)
    ofb = render.render(sc.blob, render.make_view(320, 200), poses, threads=8)
    _assert_same(ofb, gfb, str(maps))


def test_gpu_micro_level_extremes(b2d):
    from tests.test_scene import _micro_level
    sc = b2d.Scene(b2d.Archive.from_bytes(_micro_level()), 0)
    poses = np.concatenate([
        b2d.make_pose(-0.01, 128, 60, 0), b2d.make_pose(0, 128, 60, 180), b2d.make_pose(-255.99, 0.01, 1, 45),
        b2d.make_pose(-128, 128, 127.99, 270), b2d.make_pose(-5000, 9000, 60, 300), b2d.make_pose(128, 128, 30, 123.4),
    ])
    gfb = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=8).render(poses)
    ofb = render.render(sc.blob, render.make_view(320, 200), poses)
    _assert_same(ofb, gfb, "micro")


def test_gpu_golden_crcs(b2d):
    from rust_doom_b200 import synthwad
    for c in json.load(open(GOLDEN)):
        data = synthwad.build_iwad(c["seed"], c["maps"], cfg=synthwad.SynthConfig(**c.get("cfg", {})))
        sc = b2d.Scene(b2d.Archive.from_bytes(data), c["level"])
        poses = np.array([tuple(p) for p in c["poses"]], dtype=b2d.POSE_DTYPE)
        r = b2d.Renderer(sc, b2d.make_view(c["w"], c["h"]), max_batch=max(1, len(poses)))
        r.set_time(c.get("tics", 0))
        gfb = r.render(poses)
        assert [render.crc32(gfb[i]) for i in range(len(poses))] == c["frame_crc"], c["name"]


def test_gpu_worklist_matches_hostcheck(b2d, hostcheck, product_scene):
    import torch
    poses = sample_poses(b2d, product_scene, 24, 35)
    view = b2d.make_view(640, 400)
    r = b2d.Renderer(product_scene, view, max_batch=32)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    out = torch.empty((len(poses), 400, 640), dtype=torch.uint8, device="cuda")
    r.render_device(dp.data_ptr(), len(poses), out.data_ptr(), 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    counts, ids = r.worklist(len(poses))
    hfb, hcounts, hids = hostcheck(product_scene.blob, view, poses)
    assert counts.tolist() == hcounts.tolist()
    for i in range(len(poses)):
        assert ids[i, :counts[i]].tolist() == hids[i, :hcounts[i]].tolist()
    assert np.array_equal(out.cpu().numpy(), hfb)


def test_gpu_rgba_and_palette_kernel(b2d, product_scene):
    import torch
    poses = sample_poses(b2d, product_scene, 6, 36)
    r = b2d.Renderer(product_scene, b2d.make_view(640, 400), max_batch=8)
    idx, rgba = r.render(poses, rgba=True)
    ofb, orgba = render.render(product_scene.blob, render.make_view(640, 400), poses, rgba=True)
    assert np.array_equal(idx, ofb) and np.array_equal(rgba, orgba)
    # 1080p RGBA on a level without masked content: the unmasked variant of the kernel compiled for W = 1920 with RGBA
    idx2, rgba2 = b2d.Renderer(product_scene, b2d.make_view(1920, 1080), max_batch=4).render(poses[:3], rgba=True)
    oi2, orgba2 = render.render(product_scene.blob, render.make_view(1920, 1080), poses[:3], rgba=True, threads=8)
    _assert_same(oi2, idx2, "1080p RGBA (index)")
    assert np.array_equal(rgba2, orgba2)
    # stand-alone palette kernel, incl. a pixel count that is not a multiple of 16
    for npx in (640 * 400 * 6, 1003):
        di = torch.from_numpy(ofb.reshape(-1)[:npx].copy()).cuda()
        do = torch.zeros(npx, dtype=torch.int32, device="cuda")
        r.palette_lut_device(di.data_ptr(), do.data_ptr(), npx, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert np.array_equal(do.cpu().numpy().view(np.uint32), orgba.reshape(-1)[:npx])


def test_gpu_every_pixel_written_once_full_size(b2d, product_scene):
    """Full-size property: the raster never leaves a byte of the frame untouched -- two runs over
    differently poisoned buffers must agree everywhere (1920x1080, 64 poses)."""
    import torch
    poses = sample_poses(b2d, product_scene, 64, 37)
    r = b2d.Renderer(product_scene, b2d.make_view(1920, 1080), max_batch=64)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    outs = []
    for poison in (0x5A, 0xC3):
        out = torch.full((64, 1080, 1920), poison, dtype=torch.uint8, device="cuda")
        r.render_device(dp.data_ptr(), 64, out.data_ptr(), 0, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    # determinism + checksum-of-checksums against the oracle on a subsample
    ofb = render.render(product_scene.blob, render.make_view(1920, 1080), poses[::16], threads=8)
    assert np.array_equal(outs[0][::16].cpu().numpy(), ofb)


def test_gpu_device_and_host_paths_agree(b2d, product_scene):
    import torch
    poses = sample_poses(b2d, product_scene, 20, 38)
    r = b2d.Renderer(product_scene, b2d.make_view(320, 200), max_batch=7)
    host = r.render(poses)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    out = torch.empty((7, 200, 320), dtype=torch.uint8, device="cuda")
    r.render_device(dp.data_ptr(), 7, out.data_ptr(), 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), host[:7])
    with pytest.raises(b2d.B2dError):
        r.render_device(dp.data_ptr(), 8, out.data_ptr())          # n > max_batch


# ---- BASELINE.json configs as parity cases (sizes the oracle finishes in seconds) ---------------------
def test_config3_all_e1_maps_batched_1080p(b2d):
    """configs[2]: every E1 map, 1920x1080, one renderer per map, frames vs oracle."""
    from rust_doom_b200 import poses as P
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, synthwad.E1_MAPS, map_seeds=list(range(11, 20)))
    arch = b2d.Archive.from_bytes(data)
    assert arch.num_levels() == 9
    view = b2d.make_view(1920, 1080)
    for lvl in range(9):
        sc = b2d.Scene(arch, lvl)
        poses = P.flythrough_poses(sc, 3, 2)
        gfb = b2d.Renderer(sc, view, max_batch=4).render(poses)
        ofb = render.render(oracle_blob(data, lvl), render.make_view(1920, 1080), poses, threads=8)   # the oracle's own scene
        _assert_same(ofb, gfb, "E1M%d" % (lvl + 1))


def test_config4_doom2_maps_4k(b2d):
    """configs[3]: MAP01-MAP10 stand-ins at 3840x2160 (one map per GPU in the real config)."""
    from rust_doom_b200 import poses as P
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(2, synthwad.MAP_NAMES_DOOM2, map_seeds=list(range(21, 31)))
    arch = b2d.Archive.from_bytes(data)
    view = b2d.make_view(3840, 2160)
    for lvl in (0, 4, 9):
        sc = b2d.Scene(arch, lvl)
        poses = P.flythrough_poses(sc, 2, 2)
        gfb = b2d.Renderer(sc, view, max_batch=2).render(poses)
        ofb = render.render(oracle_blob(data, lvl), render.make_view(3840, 2160), poses, threads=8)
        _assert_same(ofb, gfb, "MAP%02d" % (lvl + 1))


def test_config5_random_poses_1080p(b2d, product_scene, oracle_scene):
    """configs[4]: random poses (splitmix64, sector_at acceptance); 512 rendered, every 32nd checked vs oracle,
    all checked for determinism across two launches."""
    import torch
    from rust_doom_b200 import poses as P
    poses = P.random_poses(product_scene, 512, 5)
    r = b2d.Renderer(product_scene, b2d.make_view(1920, 1080), max_batch=512)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    a = torch.empty((512, 1080, 1920), dtype=torch.uint8, device="cuda")
    bb = torch.full((512, 1080, 1920), 7, dtype=torch.uint8, device="cuda")
    r.render_device(dp.data_ptr(), 512, a.data_ptr())
    r.render_device(dp.data_ptr(), 512, bb.data_ptr())
    torch.cuda.synchronize()
    assert torch.equal(a, bb)
    ofb = render.render(oracle_scene, render.make_view(1920, 1080), poses[::32], threads=8)
    assert np.array_equal(a[::32].cpu().numpy(), ofb)


def test_gpu_edge_sizes(b2d, product_scene):
    """Empty pose list, 1x2 and the maximum 4096x2160 view."""
    poses = sample_poses(b2d, product_scene, 3, 41)
    r = b2d.Renderer(product_scene, b2d.make_view(320, 200), max_batch=4)
    assert r.render(poses[:0]).shape == (0, 200, 320)
    for (w, h) in ((1, 2), (31, 3), (4096, 2160)):
        gfb = b2d.Renderer(product_scene, b2d.make_view(w, h), max_batch=2).render(poses[:2])
        ofb = render.render(product_scene.blob, render.make_view(w, h), poses[:2], threads=2)
        _assert_same(ofb, gfb, "%dx%d" % (w, h))


def test_gpu_large_batch(b2d, product_scene):
    poses = sample_poses(b2d, product_scene, 130, 42)
    r = b2d.Renderer(product_scene, b2d.make_view(320, 200), max_batch=130)
    gfb = r.render(poses)
    assert r.launch_count == 2
    ofb = render.render(product_scene.blob, render.make_view(320, 200), poses, threads=8)
    _assert_same(ofb, gfb, "batch of 130")
    counts, ids = r.worklist(130)
    assert (counts > 0).all()


def test_gpu_fuzzed_levels_match_oracle(b2d):
    """Corrupt level lumps (random bytes in SEGS/NODES/SECTORS/...) that still load must render identically
    on the GPU and in the oracle, or be reported incomplete by the walk -- and never fault the device."""
    import struct
    import torch
    from oracle import scene as S
    from oracle import wad as W
    from rust_doom_b200 import synthwad
    base = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(gx=4, gy=3, origin=(-512, -384)))
    oa0 = W.Archive(base)
    rng = synthwad.SplitMix64(77)
    view, oview = b2d.make_view(160, 100), render.make_view(160, 100)
    poses = np.concatenate([b2d.make_pose(-300 + 150 * i, -100 + 60 * i, 30 + 7 * i, 47 * i) for i in range(4)])
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    compared = 0
    for it in range(60):
        data = bytearray(base)
        idx = oa0.levels[0] + 2 + rng.below(7)            # LINEDEFS .. SECTORS
        _, pos, size = oa0.lumps[idx]
        for _ in range(1 + rng.below(5)):
            data[pos + rng.below(size)] = rng.below(256)
        data = bytes(data)
        try:
            oa = W.Archive(data)
            ob = S.compile_scene(oa, W.TextureDirectory(oa), 0)
            sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
        except (W.WadError, b2d.B2dError):
            continue
        assert sc.blob == ob
        r = b2d.Renderer(sc, view, max_batch=4)
        out = torch.full((4, 100, 160), 0xEE, dtype=torch.uint8, device="cuda")
        r.render_device(dp.data_ptr(), 4, out.data_ptr())
        torch.cuda.synchronize()
        counts, _ = r.worklist(4)
        if (counts < 0).any():
            continue                                      # walk reported an incomplete traversal (cyclic BSP)
        ofb = render.render(ob, oview, poses)
        _assert_same(ofb, out.cpu().numpy(), "fuzz iteration %d" % it)
        compared += 1
    assert compared > 20


def test_gpu_masked_middle_textures(b2d):
    """Masked two-sided middle textures: deferred per-strip lists + back-to-front pass, index and RGBA."""
    from rust_doom_b200 import synthwad
    sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=45))), 0)
    poses = sample_poses(b2d, sc, 48, 61)
    for (w, h) in ((320, 200), (1920, 1080)):
        p = poses if w == 320 else poses[:6]
        r = b2d.Renderer(sc, b2d.make_view(w, h), max_batch=48)
        idx, rgba = r.render(p, rgba=True)
        ofb, orgba = render.render(sc.blob, render.make_view(w, h), p, rgba=True, threads=8)
        _assert_same(ofb, idx, "masked %dx%d" % (w, h))
        assert np.array_equal(rgba, orgba)
    # 4K index frames only: the masked variant of the kernel compiled for W = 3840 (RGBA at 4K takes the generic one)
    gfb = b2d.Renderer(sc, b2d.make_view(3840, 2160), max_batch=2).render(poses[:2])
    _assert_same(render.render(sc.blob, render.make_view(3840, 2160), poses[:2], threads=8), gfb, "masked 4K")


def test_gpu_full_benchmark_workload_matches_oracle(b2d, product_scene):
    """BASELINE.json configs[1] at full size: every one of the 1000 fly-through frames at 1920x1080 is compared
    with the oracle (the GPU box has enough host cores for the oracle to finish this in seconds)."""
    import os
    from rust_doom_b200 import poses as P
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1",))
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    oblob = oracle_blob(data, 0)
    poses = P.flythrough_poses(sc, 1000, 2)
    r = b2d.Renderer(sc, b2d.make_view(1920, 1080), max_batch=250)
    gfb = r.render(poses)
    threads = len(os.sched_getaffinity(0))
    bad = []
    for c0 in range(0, 1000, 250):
        ofb = render.render(oblob, render.make_view(1920, 1080), poses[c0:c0 + 250], threads=threads)
        bad += [c0 + i for i in range(250) if not np.array_equal(ofb[i], gfb[c0 + i])]
    assert not bad, "frames differ: %s" % bad[:10]


def test_gpu_decoration_sprites(b2d, hostcheck):
    """Thing sprites + masked middles on the GPU: frames vs oracle, worklist (with sprite entries) vs hostcheck."""
    import torch
    from rust_doom_b200 import synthwad
    sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=30, thing_pct=70))), 0)
    poses = sample_poses(b2d, sc, 48, 81)
    for (w, h) in ((320, 200), (1920, 1080)):
        p = poses if w == 320 else poses[:6]
        r = b2d.Renderer(sc, b2d.make_view(w, h), max_batch=48)
        idx, rgba = r.render(p, rgba=True)
        ofb, orgba = render.render(sc.blob, render.make_view(w, h), p, rgba=True, threads=8)
        _assert_same(ofb, idx, "sprites %dx%d" % (w, h))
        assert np.array_equal(rgba, orgba)
    gfb = b2d.Renderer(sc, b2d.make_view(3840, 2160), max_batch=2).render(poses[:2])     # masked W = 3840 kernel, index only
    _assert_same(render.render(sc.blob, render.make_view(3840, 2160), poses[:2], threads=8), gfb, "sprites 4K")
    view = b2d.make_view(320, 200)
    r = b2d.Renderer(sc, view, max_batch=48)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    out = torch.empty((48, 200, 320), dtype=torch.uint8, device="cuda")
    r.render_device(dp.data_ptr(), 48, out.data_ptr())
    torch.cuda.synchronize()
    counts, ids = r.worklist(48)
    hfb, hcounts, hids = hostcheck(sc.blob, view, poses)
    assert counts.tolist() == hcounts.tolist()
    assert any((ids[i, :counts[i]] < 0).any() for i in range(48)), "no sprite entry (negative id) in any worklist"
    for i in range(48):
        assert ids[i, :counts[i]].tolist() == hids[i, :hcounts[i]].tolist()


def test_gpu_animated_and_scrolling(b2d):
    """Level time (C14) through b2d_renderer_set_time: animated flats / walls, scrolling walls; going back to an
    earlier time restores the earlier frames; the device path sees the same tables as the host path."""
    import torch
    from oracle import scene as S
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=20, thing_pct=30, anim=True))
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    assert S.header(sc.blob)[S.H_NANIM] >= 6
    poses = sample_poses(b2d, sc, 24, 91)
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=16)
    oview = render.make_view(320, 200)
    for tics in (0, 1, 8, 23, 12345, 8, (1 << 24) + 5, 0xFFFFFFFF, 0):
        r.set_time(tics)
        _assert_same(render.render(sc.blob, oview, poses, threads=8, tics=tics), r.render(poses), "tics %d" % tics)
    r.set_time(77)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    out = torch.empty((16, 200, 320), dtype=torch.uint8, device="cuda")
    r.render_device(dp.data_ptr(), 16, out.data_ptr())
    torch.cuda.synchronize()
    _assert_same(render.render(sc.blob, oview, poses[:16], threads=8, tics=77), out.cpu().numpy(), "device path")
    r2 = b2d.Renderer(sc, b2d.make_view(1920, 1080), max_batch=4)
    r2.set_time(1001)
    _assert_same(render.render(sc.blob, render.make_view(1920, 1080), poses[:4], threads=8, tics=1001), r2.render(poses[:4]), "1080p")


def test_gpu_moving_sectors(b2d):
    """Doors / lifts as a per-batch state (DESIGN.md C16): b2d_renderer_set_sector_moves re-derives the height-dependent
    tables on the host and uploads them in stream order; the frames equal the oracle's render of its own scene with the
    same moves applied (oracle/scene.py apply_moves); moves compose with the level time; going back to rest restores the
    rest frames; the async variant orders the upload between two batches without a host wait."""
    import torch
    from oracle import scene as S, wad as W
    from rust_doom_b200 import synthwad
    from tests.refcheck import moves as MV
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=30, thing_pct=50, anim=True))
    a = W.Archive(data)
    tex = W.TextureDirectory(a)
    level = W.Level(a, 0)
    dyn, mv = MV.pick(level, 5, 16)
    oblob = S.compile_scene(a, tex, 0, dynamic=dyn)                  # the oracle's own scene
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0, dynamic=dyn)
    assert sc.blob == oblob
    poses = sample_poses(b2d, sc, 40, 17)
    oview = render.make_view(320, 200)
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=16)
    rest = r.render(poses)
    _assert_same(render.render(oblob, oview, poses, threads=8), rest, "at rest")
    changed = 0
    for k, (tics, seed) in enumerate(((0, 5), (9, 6), (1000, 7), (0, 8))):
        moves = mv if k == 0 else MV.state(level, dyn, seed, hole_free=False)     # any state inside the declared ranges
        r.set_time(tics)
        r.set_sector_moves(moves)
        got = r.render(poses)
        _assert_same(render.render(S.apply_moves(oblob, moves), oview, poses, threads=8, tics=tics), got, "moves %d" % k)
        changed += int((got != rest).sum())
    assert changed > 100000, "the moves never changed a pixel"
    r.set_time(0)
    r.set_sector_moves(())
    _assert_same(rest, r.render(poses), "back at rest")
    assert r.status() == 0
    # stream order: batch at rest, moves, batch moved -- no host synchronisation in between
    dp = torch.from_numpy(poses[:16].view(np.int32).reshape(-1, 4).copy()).cuda()
    out0 = torch.empty((16, 200, 320), dtype=torch.uint8, device="cuda")
    out1 = torch.empty_like(out0)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        r.render_device(dp.data_ptr(), 16, out0.data_ptr(), stream=st.cuda_stream)
        r.set_sector_moves(mv, stream=st.cuda_stream)
        r.render_device(dp.data_ptr(), 16, out1.data_ptr(), stream=st.cuda_stream)
    st.synchronize()
    _assert_same(rest[:16], out0.cpu().numpy(), "batch before the moves")
    _assert_same(render.render(S.apply_moves(oblob, mv), oview, poses[:16], threads=8), out1.cpu().numpy(), "batch after the moves")
    with pytest.raises(b2d.B2dError):
        r.set_sector_moves([(dyn[0][0], 5000, 0)])
    # 1080p, the benchmark resolution
    r2 = b2d.Renderer(sc, b2d.make_view(1920, 1080), max_batch=4)
    r2.set_sector_moves(mv)
    _assert_same(render.render(S.apply_moves(oblob, mv), render.make_view(1920, 1080), poses[:4], threads=8), r2.render(poses[:4]), "1080p moved")


def test_gpu_odd_texture_sizes(b2d):
    """Wall textures whose height is not a multiple of 4 / whose width is not a power of two (row-major pre-lit
    layout, magic floor-mod) mixed with 4-row interleaved ones."""
    from rust_doom_b200 import synthwad
    sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(4, ("E1M1",), cfg=synthwad.SynthConfig(odd_tex=True, mid_pct=20))), 0)
    poses = sample_poses(b2d, sc, 32, 61)
    for (w, h, n) in ((320, 200, 32), (1920, 1080, 6), (1000, 700, 6)):
        r = b2d.Renderer(sc, b2d.make_view(w, h), max_batch=32)
        _assert_same(render.render(sc.blob, render.make_view(w, h), poses[:n], threads=8), r.render(poses[:n]), "odd %dx%d" % (w, h))


def test_gpu_campaign_mixed_content(b2d):
    """Six more generated levels with every kind of content switched on (masked middles, sprites, animation,
    scrolling, light effects, odd texture sizes), odd resolutions, non-zero level times."""
    from rust_doom_b200 import synthwad
    sizes = ((640, 400), (1000, 700), (333, 777))
    for i, seed in enumerate(range(31, 37)):
        cfg = synthwad.SynthConfig(mid_pct=10 * (i % 4), thing_pct=15 * (i % 3), anim=bool(i & 1), odd_tex=bool(i & 2))
        sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(seed, ("MAP07",), cfg=cfg)), 0)
        poses = sample_poses(b2d, sc, 12, 300 + seed)
        w, h = sizes[i % 3]
        tics = (0, 9, 123456)[i % 3]
        r = b2d.Renderer(sc, b2d.make_view(w, h), max_batch=12)
        r.set_time(tics)
        _assert_same(render.render(sc.blob, render.make_view(w, h), poses, threads=8, tics=tics), r.render(poses),
                     "seed %d %dx%d tics %d" % (seed, w, h, tics))


def test_gpu_split_walk_raster_api_overlapped(b2d, product_scene):
    """b2d_walk_device / b2d_raster_device on two streams: batch k+1 is walked while batch k is rastered; frames
    equal the one-call path; ticket misuse is an error, not a crash."""
    import torch
    view = b2d.make_view(640, 400)
    r = b2d.Renderer(product_scene, view, max_batch=32)
    batches = [sample_poses(b2d, product_scene, 32, 500 + k) for k in range(5)]
    dps = [torch.from_numpy(p.view(np.int32).reshape(-1, 4).copy()).cuda() for p in batches]
    outs = [torch.empty((32, 400, 640), dtype=torch.uint8, device="cuda") for _ in batches]
    s_walk, s_raster = torch.cuda.Stream(priority=-1), torch.cuda.Stream()
    torch.cuda.synchronize()
    ticket = r.walk_device(dps[0].data_ptr(), 32, s_walk.cuda_stream)
    for k in range(5):
        r.raster_device(ticket, outs[k].data_ptr(), 0, s_raster.cuda_stream)
        if k + 1 < 5:
            ticket = r.walk_device(dps[k + 1].data_ptr(), 32, s_walk.cuda_stream)
    torch.cuda.synchronize()
    oview = render.make_view(640, 400)
    for k in range(5):
        _assert_same(render.render(product_scene.blob, oview, batches[k], threads=8), outs[k].cpu().numpy(), "batch %d" % k)
    with pytest.raises(b2d.B2dError):
        r.raster_device(ticket, outs[0].data_ptr())            # already rastered
    t1 = r.walk_device(dps[0].data_ptr(), 32)
    t2 = r.walk_device(dps[1].data_ptr(), 32)
    with pytest.raises(b2d.B2dError):
        r.walk_device(dps[2].data_ptr(), 32)                    # both slots pending
    r.raster_device(t1, outs[0].data_ptr())
    r.raster_device(t2, outs[1].data_ptr())
    torch.cuda.synchronize()
    _assert_same(render.render(product_scene.blob, oview, batches[1], threads=8), outs[1].cpu().numpy(), "after misuse")


def test_gpu_masked_windows_clipped_to_nothing(b2d):
    """Regression (found by tools/campaign_gpu.py): a deferred sprite / masked middle whose rows, after clipping to
    the window that was open behind it, are empty or inverted (first row below the last) must draw nothing."""
    from rust_doom_b200 import synthwad
    for seed, name, cfg, w, h, tics, fov in (
            (8802, "MAP05", synthwad.SynthConfig(rock_pct=17, sky_pct=36, door_pct=5, mid_pct=35, thing_pct=37, anim=True, odd_tex=True), 123, 746, 769541036, 77.81427875224603),
            (40250, "MAP05", synthwad.SynthConfig(rock_pct=27, sky_pct=31, door_pct=9, mid_pct=16, thing_pct=55, odd_tex=True), 701, 554, 110894393, 98.25319284638539)):
        sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(seed, (name,), cfg=cfg)), 0)
        poses = sample_poses(b2d, sc, 4, seed)
        r = b2d.Renderer(sc, b2d.make_view(w, h, fov), max_batch=4)
        r.set_time(tics)
        _assert_same(render.render(sc.blob, render.make_view(w, h, fov), poses, threads=8, tics=tics), r.render(poses), "seed %d" % seed)


def test_gpu_random_campaign_short():
    """A short run of tools/campaign_gpu.py (random levels with all content kinds, random resolution / field of view /
    level time / batch size, RGBA every fourth case) so that every GPU test tier draws fresh-ish coverage."""
    import importlib.util
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "campaign_gpu.py")
    spec = importlib.util.spec_from_file_location("campaign_gpu", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.main(cases=40, seed=2024) == 0


def test_gpu_status_is_sticky_and_reports_masked_overflow(b2d):
    """b2d_renderer_status: the device-resident entry points cannot report incomplete frames themselves; the sticky bits
    can.  Force the masked-entry arena to a single chunk (B2D_MASKED_CHUNKS=1): bit 8 must come up, be cleared by the
    read, and the frames of a normally sized renderer of the same level must be complete and exact."""
    import torch
    from rust_doom_b200 import synthwad
    sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=45, thing_pct=60))), 0)
    poses = sample_poses(b2d, sc, 16, 77)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    out = torch.empty((16, 200, 320), dtype=torch.uint8, device="cuda")
    os.environ["B2D_MASKED_CHUNKS"] = "1"
    try:
        small = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=16)
    finally:
        del os.environ["B2D_MASKED_CHUNKS"]
    assert small.status() == 0
    small.render_device(dp.data_ptr(), 16, out.data_ptr())
    assert small.status() & 8, "arena of one chunk did not overflow"
    assert small.status() == 0, "status is cleared by the read"
    with pytest.raises(b2d.B2dError):
        small.render(poses)                                   # the host path reports the same condition as an error
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=16)
    r.render_device(dp.data_ptr(), 16, out.data_ptr())
    assert r.status() == 0
    _assert_same(render.render(sc.blob, render.make_view(320, 200), poses, threads=8), out.cpu().numpy(), "arena")


def test_gpu_two_rasters_in_flight_share_the_masked_arena(b2d):
    """ADVICE r1: rasters of a level with masked content enqueued on two streams used to share one scratch list.  They
    are now ordered through an event: both batches come out exact."""
    import torch
    from rust_doom_b200 import synthwad
    sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(2, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=40, thing_pct=50))), 0)
    view = b2d.make_view(640, 400)
    r = b2d.Renderer(sc, view, max_batch=24)
    batches = [sample_poses(b2d, sc, 24, 900 + k) for k in range(4)]
    dps = [torch.from_numpy(p.view(np.int32).reshape(-1, 4).copy()).cuda() for p in batches]
    outs = [torch.empty((24, 400, 640), dtype=torch.uint8, device="cuda") for _ in batches]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for k in range(4):
        r.render_device(dps[k].data_ptr(), 24, outs[k].data_ptr(), 0, streams[k & 1].cuda_stream)
    torch.cuda.synchronize()
    assert r.status() == 0
    for k in range(4):
        _assert_same(render.render(sc.blob, render.make_view(640, 400), batches[k], threads=8), outs[k].cpu().numpy(), "batch %d" % k)


def test_gpu_set_time_async_is_stream_ordered(b2d):
    """b2d_renderer_set_time_async: no host-side synchronisation; batches enqueued before the call see the old time,
    batches after it the new one -- on the same stream and on another stream."""
    import torch
    from rust_doom_b200 import synthwad
    sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(anim=True, mid_pct=15))), 0)
    poses = sample_poses(b2d, sc, 8, 55)
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=8)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    times = [0, 8, 17, 1000, 9, 0, 123456]
    outs = [torch.empty((8, 200, 320), dtype=torch.uint8, device="cuda") for _ in times]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    for k, t in enumerate(times):
        st = (s1, s2)[k % 2]
        r.set_time_async(t, st.cuda_stream)
        r.render_device(dp.data_ptr(), 8, outs[k].data_ptr(), 0, (s2, s1)[k % 2].cuda_stream if k % 3 == 0 else st.cuda_stream)
    torch.cuda.synchronize()
    assert r.status() == 0
    oview = render.make_view(320, 200)
    for k, t in enumerate(times):
        _assert_same(render.render(sc.blob, oview, poses, threads=8, tics=t), outs[k].cpu().numpy(), "tics %d (step %d)" % (t, k))


def test_gpu_sharded_render_world1_and_checksums(b2d, product_scene, oracle_scene):
    """b2d_render_sharded through the C ABI with a one-rank NCCL communicator: chunked render into the in-place
    all-gather buffer, gather + consumer streams; every gathered frame's device checksum equals the host restatement on
    the oracle's frame (chunk not dividing the job, a short last chunk, all three modes)."""
    import torch
    from rust_doom_b200 import jobs
    poses = sample_poses(b2d, product_scene, 23, 97)
    comm = jobs.single_comm(0)
    assert comm.nccl_version >= 21900
    view = b2d.make_view(640, 400)
    r = b2d.Renderer(product_scene, view, max_batch=8)
    npix = 640 * 400
    table = jobs.ChecksumTable(1, 23, npix, torch.device("cuda", 0))
    seen = []

    def on_chunk(k, first, cnt, ptr, ranks, stream):
        seen.append((k, first, cnt, ranks))
        table.on_chunk(k, first, cnt, ptr, ranks, stream)

    st = r.render_sharded(comm, poses, 5, b2d._lib.SHARD_RENDER_GATHER, on_chunk)
    assert st["chunks"] == 5 and st["frames_local"] == 23 and st["frames_gathered"] == 23
    assert seen == [(0, 0, 5, 1), (1, 5, 5, 1), (2, 10, 5, 1), (3, 15, 5, 1), (4, 20, 3, 1)]
    assert r.status() == 0
    ofb = render.render(oracle_scene, render.make_view(640, 400), poses, threads=8)
    want = np.array([b2d.frame_checksum(ofb[i]) for i in range(23)], np.uint32)
    assert np.array_equal(table.host()[0], want)
    for mode in (b2d._lib.SHARD_RENDER_ONLY, b2d._lib.SHARD_GATHER_ONLY):
        st = r.render_sharded(comm, poses, 8, mode)
        assert st["chunks"] == 3 and st["total_ms"] > 0
    # the checksum kernel on an unaligned frame size
    odd = torch.from_numpy(ofb.reshape(-1)[:3 * 1003].copy()).cuda()
    outc = torch.zeros(3, dtype=torch.int32, device="cuda")
    b2d.frame_checksums_device(odd.data_ptr(), 3, 1003, outc.data_ptr())
    torch.cuda.synchronize()
    assert outc.cpu().numpy().view(np.uint32).tolist() == [b2d.frame_checksum(ofb.reshape(-1)[i * 1003:(i + 1) * 1003]) for i in range(3)]
    comm.close()


def test_gpu_suite_runs_on_a_supplied_iwad(tmp_path):
    """B2D_IWAD hook: with the variable set, the generic fixtures load that file instead of the generated level.  Kept
    alive with a generated IWAD written to disk (no real doom1.wad exists here): a sub-run of this suite must pass."""
    import subprocess
    import sys
    from rust_doom_b200 import synthwad
    path = tmp_path / "custom.wad"
    path.write_bytes(synthwad.build_iwad(9, ("E1M1", "E1M2"), cfg=synthwad.SynthConfig(mid_pct=10, thing_pct=10)))
    env = dict(os.environ, B2D_IWAD=str(path))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu.py", "-k",
                          "320x200 or odd_width or device_and_host or config5"], cwd=root, env=env,
                         capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "4 passed" in res.stdout


def test_gpu_per_pose_time(b2d):
    """b2d_render_timed / b2d_render_device_timed (SURVEY 8-f2 'poses (x, y, z, yaw, t)'): every pose carries its own level
    time.  A sorted timeline, an unsorted one and runs of equal tics, through the host path (small max_batch: runs are also
    cut by the batch size) and the device path; every frame equals the oracle's frame at that pose's tics."""
    import torch
    from rust_doom_b200 import synthwad
    sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(anim=True, mid_pct=15, thing_pct=20))), 0)
    poses = sample_poses(b2d, sc, 24, 66)
    oview = render.make_view(320, 200)
    timelines = [np.arange(24, dtype=np.uint32) * 3,                                   # sorted, changes every pose (light effects)
                 np.array([0, 0, 0, 9, 9, 9, 9, 17, 17, 5, 5, 5] * 2, dtype=np.uint32),    # runs, not monotone
                 np.random.default_rng(4).integers(0, 1 << 32, 24, dtype=np.uint64).astype(np.uint32)]
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=5)
    for tl in timelines:
        got = r.render_timed(poses, tl)
        for i in range(24):
            want = render.render(sc.blob, oview, poses[i:i + 1], tics=int(tl[i]))[0]
            assert np.array_equal(got[i], want), "host path: pose %d at tics %d" % (i, int(tl[i]))
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    out = torch.empty((24, 200, 320), dtype=torch.uint8, device="cuda")
    r2 = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=24)
    r2.render_device_timed(dp.data_ptr(), timelines[1], 24, out.data_ptr())
    torch.cuda.synchronize()
    assert r2.status() == 0
    g = out.cpu().numpy()
    for i in range(24):
        assert np.array_equal(g[i], render.render(sc.blob, oview, poses[i:i + 1], tics=int(timelines[1][i]))[0]), i
    # a level without time-dependent content: one launch whatever the tics say
    plain = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(light_fx=False))), 0)
    r3 = b2d.Renderer(plain, b2d.make_view(320, 200), max_batch=24)
    p3 = sample_poses(b2d, plain, 24, 67)
    got = r3.render_timed(p3, timelines[2])
    assert r3.launch_count == 2
    _assert_same(render.render(plain.blob, oview, p3, threads=8), got, "static level")
