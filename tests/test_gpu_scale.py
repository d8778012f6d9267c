"""-m gpu: the launch shapes and sizes the benchmark and large maps depend on, compared with the oracle -- the persistent
(background) walk grid where a CTA loops over several frames, the pipelined jobs.run_maps path, levels whose walk tables
need the shared-memory opt-in or do not fit at all, and subsectors crowded with decoration sprites.
tests/test_scale.py shows on the CPU that every case here is valid."""
import math
import os

import numpy as np
import pytest

from oracle import render
from tests.conftest import oracle_blob, sample_poses
from tests.test_scale import cluster_level, cluster_poses, sweep_level, walk_smem_bytes, WALK_SMEM_MAX

pytestmark = pytest.mark.gpu


def _assert_same(ofb, gfb, what=""):
    bad = [(i, int((ofb[i] != gfb[i]).sum())) for i in range(len(ofb)) if not np.array_equal(ofb[i], gfb[i])]
    assert not bad, "%s: frames differ (index, pixels): %s" % (what, bad[:6])


def _sms() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dev_poses(poses):
    import torch
    return torch.from_numpy(np.ascontiguousarray(poses).view(np.int32).reshape(-1, 4).copy()).cuda()


def _assert_worklists(r, hostcheck, blob, view, poses, what):
    counts, ids = r.worklist(len(poses))
    _, hcounts, hids = hostcheck(blob, view, poses)
    assert counts.tolist() == hcounts.tolist(), what
    for i in range(len(poses)):
        assert ids[i, :counts[i]].tolist() == hids[i, :hcounts[i]].tolist(), "%s: worklist of frame %d" % (what, i)
    return counts, ids


def _background_walk(r, poses, w, h):
    """b2d_walk_device (the background grid: one CTA per SM once n > SMs) + b2d_raster_device on a side stream."""
    import torch
    n = len(poses)
    dp = _dev_poses(poses)
    out = torch.full((n, h, w), 0xA5, dtype=torch.uint8, device="cuda")
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    ticket = r.walk_device(dp.data_ptr(), n, st.cuda_stream)
    r.raster_device(ticket, out.data_ptr(), 0, st.cuda_stream)
    st.synchronize()
    return dp, out


def _level(b2d, name):
    from rust_doom_b200 import synthwad
    data, blob = (synthwad.build_iwad(1, ("E1M1",)), None) if name == "default" else sweep_level(int(name.split("x")[0]))
    return b2d.Scene(b2d.Archive.from_bytes(data), 0), blob or oracle_blob(data)


# ---- A. persistent walk grid and the pipelined jobs path ----------------------------------------------------------------
def _states_level(b2d, name):
    """_level with per-frame state inputs: the level's scene, oracle blob and dynamic sectors (tests/refcheck/moves.py's
    declaration on the "32x32" level, which then takes the kStates walk through the shared-memory opt-in) and a pool of
    move lists (at rest only where nothing is declared)."""
    from oracle import scene as S, wad as W
    from rust_doom_b200 import synthwad
    from tests.refcheck import moves as MV
    data = synthwad.build_iwad(1, ("E1M1",)) if name == "default" else sweep_level(int(name.split("x")[0]))[0]
    a = W.Archive(data)
    level = W.Level(a, 0)
    dyn = MV.declare(level, 11, 12) if name != "default" else []
    pool = [[]] + [MV.state(level, dyn, 300 + k, hole_free=False) for k in range(3)] if dyn else [[]]
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0, dynamic=dyn)
    blob = S.compile_scene(a, W.TextureDirectory(a), 0, dynamic=dyn)
    assert sc.blob == blob
    return sc, blob, pool


@pytest.mark.parametrize("states", [False, True])
@pytest.mark.parametrize("level", ["default", "32x32"])
def test_gpu_persistent_walk_grid_matches_oracle(b2d, hostcheck, level, states):
    """n = SMs + 1 and 2 SMs + 5 frames: the background grid has one CTA per SM, so CTAs walk two or three frames each and
    every frame after a CTA's first reuses the bulk-copied tables.  Frames vs the oracle, worklists vs hostcheck, and the
    same bytes from the per-frame grid (b2d_render_device).  With `states` the batch goes through walk_device_states with
    a tic of its own for every frame (and a move list from a pool where the level declares dynamic sectors), so that each
    CTA's later frames must read their own table-set index; worklists and frames are checked at each frame's own state."""
    import torch
    from tests.test_gpu_states import _oracle
    if states:
        sc, blob, pool = _states_level(b2d, level)
    else:
        sc, blob = _level(b2d, level)
    view, oview = b2d.make_view(320, 200), render.make_view(320, 200)
    sms = _sms()
    for n in (sms + 1, 2 * sms + 5):
        poses = sample_poses(b2d, sc, n, 600 + n)
        r = b2d.Renderer(sc, view, max_batch=n)
        if not states:
            dp, out = _background_walk(r, poses, 320, 200)
            assert r.status() == 0
            _assert_worklists(r, hostcheck, blob, view, poses, "%s n=%d" % (level, n))
            _assert_same(render.render(blob, oview, poses, threads=8), out.cpu().numpy(), "%s background walk n=%d" % (level, n))
            per_frame = torch.full_like(out, 0x5A)
            r.render_device(dp.data_ptr(), n, per_frame.data_ptr())
        else:
            tics = (np.arange(n, dtype=np.uint64) * 37 + 1000).astype(np.uint32)
            moves = [pool[i % len(pool)] for i in range(n)]
            dp = _dev_poses(poses)
            out = torch.full((n, 200, 320), 0xA5, dtype=torch.uint8, device="cuda")
            st = torch.cuda.Stream()
            torch.cuda.synchronize()
            ticket = r.walk_device_states(dp.data_ptr(), tics, n, moves, st.cuda_stream)
            r.raster_device(ticket, out.data_ptr(), 0, st.cuda_stream)
            st.synchronize()
            assert r.status() == 0
            slots = r.state_slots(n)
            assert any(slots[f] != slots[f % sms] for f in range(sms, n)), "no CTA walks frames of different table sets"
            counts, ids = r.worklist(n)
            for i in range(n):
                _, hc, hids = hostcheck(blob, view, poses[i:i + 1], int(tics[i]), moves[i])
                assert counts[i] == hc[0] and ids[i, :counts[i]].tolist() == hids[0, :hc[0]].tolist(), \
                    "%s n=%d: worklist of frame %d" % (level, n, i)
            _assert_same(_oracle(blob, 320, 200, poses, tics, moves), out.cpu().numpy(), "%s background walk with states n=%d" % (level, n))
            per_frame = torch.full_like(out, 0x5A)
            r.render_device_states(dp.data_ptr(), tics, n, per_frame.data_ptr(), moves_per_pose=moves)
        torch.cuda.synchronize()
        assert r.status() == 0
        assert torch.equal(out, per_frame), "%s n=%d: persistent and per-frame walk grids disagree" % (level, n)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("interleave", [True, False])
@pytest.mark.parametrize("raster_streams", [1, 2])
def test_gpu_run_maps_matches_oracle(b2d, masked, interleave, raster_streams):
    """jobs.run_maps (bench.py's c3/c4/4k/rich path): background walks pipelined under the rasters, batches larger than the
    SM count, two plain levels (rasters alternate between two streams) or a plain one and one with masked content (then
    every raster is ordered through the masked-arena event, on one stream)."""
    from rust_doom_b200 import jobs, synthwad
    second = synthwad.SynthConfig(gx=6, gy=6, origin=(-768, -768), mid_pct=30 if masked else 0, thing_pct=40 if masked else 0)
    datas = [synthwad.build_iwad(3, ("E1M1",), cfg=synthwad.SynthConfig(gx=6, gy=5, origin=(-768, -640))),
             synthwad.build_iwad(4, ("E1M1",), cfg=second)]
    scenes = [b2d.Scene(b2d.Archive.from_bytes(d), 0) for d in datas]
    assert scenes[0].info.n_masked_mids + scenes[0].info.n_sprites == 0
    assert (scenes[1].info.n_masked_mids > 0) == masked
    batch = _sms() + 7
    poses = [sample_poses(b2d, scenes[0], 2 * batch + 3, 71), sample_poses(b2d, scenes[1], batch + 40, 72)]
    res = jobs.run_maps(scenes, poses, 320, 200, 0, batch, steps=1, warmup=0, interleave=interleave, raster_streams=raster_streams)
    assert res["status_bits"] == 0
    assert res["raster_streams"] == (2 if raster_streams == 2 and not masked else 1)
    for m, d in enumerate(datas):
        _assert_same(render.render(oracle_blob(d), render.make_view(320, 200), poses[m], threads=8), res["outs"][m].cpu().numpy(),
                     "map %d interleave=%s streams=%d" % (m, interleave, raster_streams))


# ---- B. level size sweep ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", [16, 24, 32])
def test_gpu_large_levels_match_oracle(b2d, hostcheck, g):
    """49 KB (just over the opt-in), 119 KB and 207 KB of walk shared memory: the foreground walk (b2d_render) and the
    background grid at 320x200, the foreground walk at 1080p; worklists vs hostcheck."""
    sc, blob = _level(b2d, "%dx%d" % (g, g))
    assert walk_smem_bytes(blob) > 48 * 1024
    view, oview = b2d.make_view(320, 200), render.make_view(320, 200)
    poses = sample_poses(b2d, sc, 48, 700 + g)
    r = b2d.Renderer(sc, view, max_batch=48)
    ofb = render.render(blob, oview, poses, threads=8)
    _assert_same(ofb, r.render(poses), "%dx%d foreground 320x200" % (g, g))
    _assert_worklists(r, hostcheck, blob, view, poses, "%dx%d foreground" % (g, g))
    n = _sms() + 1
    more = np.concatenate([poses, sample_poses(b2d, sc, n - 48, 800 + g)])
    rb = b2d.Renderer(sc, view, max_batch=n)
    _, out = _background_walk(rb, more, 320, 200)
    assert rb.status() == 0
    counts, ids = _assert_worklists(rb, hostcheck, blob, view, more, "%dx%d background" % (g, g))
    _assert_same(np.concatenate([ofb, render.render(blob, oview, more[48:], threads=8)]), out.cpu().numpy(), "%dx%d background" % (g, g))
    assert max(int(ids[i, :counts[i]].max()) for i in range(n)) > sc.info.n_segs // 2, "no high seg index in any worklist"
    r2 = b2d.Renderer(sc, b2d.make_view(1920, 1080), max_batch=4)
    _assert_same(render.render(blob, render.make_view(1920, 1080), poses[:4], threads=8), r2.render(poses[:4]), "%dx%d 1080p" % (g, g))
    assert r2.status() == 0


def test_gpu_level_over_the_shared_memory_limit_is_refused(b2d):
    sc, blob = _level(b2d, "34x34")
    assert walk_smem_bytes(blob) > WALK_SMEM_MAX
    with pytest.raises(b2d.B2dError, match="shared memory") as e:
        b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=4)
    assert e.value.code == b2d.ERR_INVALID_ARG


# ---- C. dense sprite clusters -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("total,layout", [(33, "ties"), (64, "ties"), (255, "ring")])
def test_gpu_sprite_clusters_match_oracle(b2d, hostcheck, total, layout):
    """One subsector with 33 / 64 / 255 sprites, exact depth ties (angle 0, shared x, shared positions) within and across
    the walk's 32-wide ranking chunks: frames at 320x200 and 1080p vs the oracle, worklists (sprite entries included)
    vs hostcheck."""
    import torch
    data, blob, _, _ = cluster_level(total, layout)
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    poses = cluster_poses(b2d, total, layout)
    view, oview = b2d.make_view(320, 200), render.make_view(320, 200)
    r = b2d.Renderer(sc, view, max_batch=len(poses))
    dp = _dev_poses(poses)
    out = torch.empty((len(poses), 200, 320), dtype=torch.uint8, device="cuda")
    r.render_device(dp.data_ptr(), len(poses), out.data_ptr())
    torch.cuda.synchronize()
    assert r.status() == 0
    _assert_same(render.render(blob, oview, poses, threads=8), out.cpu().numpy(), "%d sprites (%s) 320x200" % (total, layout))
    counts, ids = _assert_worklists(r, hostcheck, blob, view, poses, "%d sprites (%s)" % (total, layout))
    assert max(int((ids[i, :counts[i]] < 0).sum()) for i in range(len(poses))) > min(total, 40), "too few sprite entries"
    r2 = b2d.Renderer(sc, b2d.make_view(1920, 1080), max_batch=4)
    _assert_same(render.render(blob, render.make_view(1920, 1080), poses[:4], threads=8), r2.render(poses[:4]),
                 "%d sprites (%s) 1080p" % (total, layout))


def test_gpu_sprite_pile_over_the_strip_cap_is_reported(b2d):
    """255 sprites that fall into the same strips defer more than the per-strip cap of 128 entries: status bit 8 on the
    device path, B2dError on the host path -- while the ring of 255 (under the cap) above renders exactly."""
    import torch
    data, blob, _, _ = cluster_level(255, "pile")
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    poses = cluster_poses(b2d, 255, "pile")
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=len(poses))
    dp = _dev_poses(poses)
    out = torch.empty((len(poses), 200, 320), dtype=torch.uint8, device="cuda")
    r.render_device(dp.data_ptr(), len(poses), out.data_ptr())
    assert r.status() & 8
    with pytest.raises(b2d.B2dError, match="strip"):
        r.render(poses)


def test_gpu_masked_arena_holds_a_crowded_full_batch(b2d):
    """The 255-sprite ring at 1920x1080 with max_batch=64: a renderer whose arena is forced to the worst case (every strip
    of every frame at strip_masked_cap) is exact, and the default arena renders the same bytes without overflowing."""
    import torch
    from oracle import scene as S
    data, blob, (cx, cy), _ = cluster_level(255, "ring")
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    _, floor, _ = sc.sector_at(cx, cy)
    poses = np.concatenate([b2d.make_pose(cx + (k % 3) * 5, cy - (k % 5) * 4, floor + 41, 360.0 * k / 64) for k in range(64)])
    h = S.header(blob)
    cap = min(max(h[S.H_NMIDS] + h[S.H_NSPRITES], 8), 128)             # strip_masked_cap
    worst = (1920 // 32) * 64 * math.ceil(cap / 4)
    dp = _dev_poses(poses)
    outs = []
    for chunks in (None, worst):
        if chunks:
            os.environ["B2D_MASKED_CHUNKS"] = str(chunks)
        try:
            r = b2d.Renderer(sc, b2d.make_view(1920, 1080), max_batch=64)
        finally:
            os.environ.pop("B2D_MASKED_CHUNKS", None)
        out = torch.empty((64, 1080, 1920), dtype=torch.uint8, device="cuda")
        r.render_device(dp.data_ptr(), 64, out.data_ptr())
        outs.append((r.status(), out))
        del r
    (st_default, out_default), (st_worst, out_worst) = outs
    assert st_worst == 0
    _assert_same(render.render(blob, render.make_view(1920, 1080), poses[::8], threads=8), out_worst[::8].cpu().numpy(),
                 "worst-case arena")
    assert st_default == 0, "the default arena overflowed (status %d) on a batch whose strips are all within the cap" % st_default
    assert torch.equal(out_default, out_worst)
