"""-m gpu: level sets (b2d_renderer_create_levels, b2d_render_levels & co.).  Four generated levels in one renderer -- the
benchmark's c2 level, the content-rich level (masked middles, sprites, animated, scrolling and flashing content) with
declared dynamic sectors, a small static level from a WAD with another palette (its PLAYPAL inverted) and a large map whose
walk tables need the shared-memory opt-in -- and seeded, interleaved mixes of their poses.  Every frame is compared with the oracle's frame of that pose on its own level,
and with a b2d_renderer_create renderer of that level."""
import ctypes
import os

import numpy as np
import pytest

from oracle import render
from tests.conftest import oracle_blob, sample_poses
from tests.test_scale import sweep_level

pytestmark = pytest.mark.gpu

RICH_CFG = dict(mid_pct=30, thing_pct=40, anim=True)       # bench.py --config rich
C2, RICH, SMALL, LARGE = range(4)


def _other_palette(data: bytes) -> bytes:
    """the WAD with every byte of its PLAYPAL lump inverted (255 - v): a level set whose levels come from different WADs"""
    buf = bytearray(data)
    n, diro = np.frombuffer(bytes(buf[4:12]), "<i4")
    for k in range(int(n)):
        pos, size = np.frombuffer(bytes(buf[diro + 16 * k:diro + 16 * k + 8]), "<i4")
        if bytes(buf[diro + 16 * k + 8:diro + 16 * k + 16]).rstrip(b"\0") == b"PLAYPAL":
            buf[pos:pos + size] = bytes(255 - v for v in buf[pos:pos + size])
            return bytes(buf)
    raise AssertionError("no PLAYPAL lump")


@pytest.fixture(scope="module")
def levels(b2d):
    return make_levels(b2d)


def make_levels(b2d):
    """[{scene, blob (oracle), data, dyn}] of the four levels; RICH declares dynamic sectors (refcheck moves.pick) and
    carries one moved state of them (moves)"""
    from oracle import scene as S, wad as W
    from rust_doom_b200 import synthwad
    from tests.refcheck import moves as MV
    out = []
    data = synthwad.build_iwad(1, ("E1M1",))
    out.append(dict(data=data, dyn=[], blob=oracle_blob(data)))
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(**RICH_CFG))
    a = W.Archive(data)
    level = W.Level(a, 0)
    dyn, moves = MV.pick(level, 5)
    out.append(dict(data=data, dyn=dyn, moves=moves, blob=S.compile_scene(a, W.TextureDirectory(a), 0, dynamic=dyn)))
    data = _other_palette(synthwad.build_iwad(7, ("E1M1",), cfg=synthwad.SynthConfig(gx=3, gy=3, origin=(-384, -384), light_fx=False)))
    out.append(dict(data=data, dyn=[], blob=oracle_blob(data)))
    data, blob = sweep_level(16)
    out.append(dict(data=data, dyn=[], blob=blob))
    for lv in out:
        lv["scene"] = b2d.Scene(b2d.Archive.from_bytes(lv["data"]), 0, dynamic=lv["dyn"])
        assert lv["scene"].blob == lv["blob"]
    info = out[RICH]["scene"].info
    assert info.n_masked_mids > 0 and info.n_sprites > 0 and info.n_dynamic > 0
    assert out[LARGE]["scene"].info.n_segs > 2 * out[C2]["scene"].info.n_segs
    pal = [_palette(lv["scene"]) for lv in out]
    assert np.array_equal(pal[C2], pal[RICH]) and np.array_equal(pal[C2], pal[LARGE])
    assert (pal[SMALL] != pal[C2]).all()
    return out


def _mix(b2d, levels, per_level, seed, spread=None):
    """(poses, frame levels): per_level poses of every level in a seeded interleaved order.  `spread`: frame f + spread is
    never on the level of frame f (the background walk's CTA that draws frame f draws frame f + spread next)."""
    rng = np.random.default_rng(seed)
    lv = rng.permutation(np.repeat(np.arange(len(levels)), per_level))
    if spread:
        for f in range(spread, len(lv)):
            if lv[f] == lv[f - spread]:
                lv[f] = (lv[f] + 1) % len(levels)
    pools = [sample_poses(b2d, levels[k]["scene"], int((lv == k).sum()) or 1, seed + 10 * k) for k in range(len(levels))]
    used = [0] * len(levels)
    poses = np.empty(len(lv), dtype=pools[0].dtype)
    for i, k in enumerate(lv):
        poses[i] = pools[k][used[k]]
        used[k] += 1
    return poses, lv.astype(np.uint32)


def _oracle(levels, w, h, poses, lv, tics=0, moved=None):
    """the oracle's frame of every pose on its own level; moved = {level: moves}"""
    from concurrent.futures import ThreadPoolExecutor
    from oracle import scene as S
    view = render.make_view(w, h)
    blobs = [S.apply_moves(L["blob"], moved[k]) if moved and k in moved else L["blob"] for k, L in enumerate(levels)]
    out = np.empty((len(poses), h, w), np.uint8)

    def one(i):
        render.render(blobs[int(lv[i])], view, poses[i:i + 1], tics=int(tics), out=out[i:i + 1])

    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        list(ex.map(one, range(len(poses))))
    return out


def _palette(scene):
    return np.frombuffer(scene.blob, "<u4", 256, int(np.frombuffer(scene.blob, "<u4", 21)[20]))


def _assert_same(want, got, what):
    bad = [(i, int((want[i] != got[i]).sum())) for i in range(len(want)) if not np.array_equal(want[i], got[i])]
    assert not bad, "%s: frames differ (index, pixels): %s" % (what, bad[:6])


def _dev(poses):
    import torch
    return torch.from_numpy(np.ascontiguousarray(poses).view(np.int32).reshape(-1, 4).copy()).cuda()


@pytest.mark.parametrize("w,h", [(1920, 1080), (900, 600)])
def test_levels_match_oracle_and_single_level_renderers(b2d, levels, w, h):
    """Index and RGBA frames of a mixed batch (host path, batches split at max_batch; device path) equal the oracle's frame
    on the pose's level, each RGBA frame through its own level's palette (the small level's WAD has another palette; at 900
    columns, 29 strips, raster CTAs straddle frames of different levels), and are byte-identical to b2d_renderer_create
    renderers of each level."""
    import torch
    poses, lv = _mix(b2d, levels, 4, 101)
    view = b2d.make_view(w, h)
    r = b2d.Renderer.from_levels([L["scene"] for L in levels], view, max_batch=7)
    idx, rgba = r.render_levels(poses, lv, rgba=True)
    assert r.status() == 0
    _assert_same(_oracle(levels, w, h, poses, lv), idx, "%dx%d index" % (w, h))
    level0 = _palette(levels[0]["scene"])
    for i in range(len(poses)):
        assert np.array_equal(rgba[i], _palette(levels[lv[i]]["scene"])[idx[i]]), "frame %d: RGBA is not its level's palette" % i
        if lv[i] == SMALL:
            assert (rgba[i] != level0[idx[i]]).all(), "frame %d: RGBA of the other WAD's level through level 0's palette" % i
    for k, L in enumerate(levels):                              # the oracle's RGBA frames, from each level's own blob
        sel = np.nonzero(lv == k)[0]
        _, orgba = render.render(L["blob"], render.make_view(w, h), poses[sel], rgba=True, threads=8)
        _assert_same(orgba, rgba[sel], "level %d RGBA vs the oracle" % k)
    for k, L in enumerate(levels):
        sel = np.nonzero(lv == k)[0]
        one = b2d.Renderer(L["scene"], view, max_batch=7)
        i1, r1 = one.render(poses[sel], rgba=True)
        _assert_same(i1, idx[sel], "level %d vs its own renderer (index)" % k)
        _assert_same(r1, rgba[sel], "level %d vs its own renderer (RGBA)" % k)
    n = len(poses)
    out = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
    out_rgba = torch.empty((n, h, w), dtype=torch.int32, device="cuda")
    r.render_device_levels(_dev(poses).data_ptr(), lv, n, out.data_ptr(), out_rgba.data_ptr())
    torch.cuda.synchronize()
    _assert_same(idx, out.cpu().numpy(), "device path (index)")
    _assert_same(rgba, out_rgba.cpu().numpy().view(np.uint32), "device path (RGBA)")
    assert r.status() == 0


def test_levels_pipelined_walk_and_two_raster_streams(b2d, levels):
    """walk_device_levels of batch k+1 under the raster of batch k, rasters alternating between two streams and output
    buffers, batches larger than the SM count: the background walk's CTAs change level between the frames they loop over."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    batch = sms + 9
    r = b2d.Renderer.from_levels([L["scene"] for L in levels], b2d.make_view(320, 200), max_batch=batch)
    mixes = [_mix(b2d, levels, (batch + 3) // 4, 200 + k, spread=sms) for k in range(3)]
    mixes = [(p[:batch], lv[:batch]) for p, lv in mixes]
    dps = [_dev(p) for p, _ in mixes]
    outs = [torch.empty((batch, 200, 320), dtype=torch.uint8, device="cuda") for _ in mixes]
    s_walk, s_r = torch.cuda.Stream(priority=-1), (torch.cuda.Stream(), torch.cuda.Stream())
    torch.cuda.synchronize()
    ticket = r.walk_device_levels(dps[0].data_ptr(), mixes[0][1], batch, s_walk.cuda_stream)
    for k in range(3):
        r.raster_device(ticket, outs[k].data_ptr(), 0, s_r[k % 2].cuda_stream)
        if k + 1 < 3:
            ticket = r.walk_device_levels(dps[k + 1].data_ptr(), mixes[k + 1][1], batch, s_walk.cuda_stream)
    torch.cuda.synchronize()
    assert r.status() == 0
    for k, (p, lv) in enumerate(mixes):
        assert any(lv[f] != lv[f + sms] for f in range(batch - sms))
        _assert_same(_oracle(levels, 320, 200, p, lv), outs[k].cpu().numpy(), "batch %d" % k)


def test_levels_time_and_walked_tickets(b2d, levels):
    """set_time applies to every level; a ticket walked before set_time and rastered after it shows the old time."""
    import torch
    r = b2d.Renderer.from_levels([L["scene"] for L in levels], b2d.make_view(320, 200), max_batch=12)
    poses, lv = _mix(b2d, levels, 3, 300)
    r.set_time(1234)
    _assert_same(_oracle(levels, 320, 200, poses, lv, tics=1234), r.render_levels(poses, lv), "at tic 1234")
    out = torch.empty((12, 200, 320), dtype=torch.uint8, device="cuda")
    dp = _dev(poses)
    torch.cuda.synchronize()
    ticket = r.walk_device_levels(dp.data_ptr(), lv, 12)
    r.set_time(77777)
    r.raster_device(ticket, out.data_ptr())
    torch.cuda.synchronize()
    _assert_same(_oracle(levels, 320, 200, poses, lv, tics=1234), out.cpu().numpy(), "ticket walked at tic 1234")
    _assert_same(_oracle(levels, 320, 200, poses, lv, tics=77777), r.render_levels(poses, lv), "at tic 77777")
    assert r.status() == 0


def test_level_sector_moves(b2d, levels):
    """set_level_sector_moves moves one level's sectors; the other levels stay at rest; moves of a level without dynamic
    sectors and level indices out of range are refused."""
    r = b2d.Renderer.from_levels([L["scene"] for L in levels], b2d.make_view(320, 200), max_batch=16)
    poses, lv = _mix(b2d, levels, 4, 400)
    moves = levels[RICH]["moves"]
    r.set_level_sector_moves(RICH, moves)
    _assert_same(_oracle(levels, 320, 200, poses, lv, moved={RICH: moves}), r.render_levels(poses, lv), "moved")
    with pytest.raises(b2d.B2dError) as e:
        r.set_sector_moves(moves)                                   # level 0 declares no dynamic sectors
    assert e.value.code == b2d.ERR_INVALID_ARG
    for bad in (-1, 4):
        with pytest.raises(b2d.B2dError):
            r.set_level_sector_moves(bad, [])
    r.set_level_sector_moves(RICH, [])
    _assert_same(_oracle(levels, 320, 200, poses, lv), r.render_levels(poses, lv), "back at rest")
    assert r.status() == 0


def test_levels_launch_counts(b2d, levels):
    """Two launches per batch at a fixed state whatever the levels it mixes; after a change of the time, one more launch per
    timed level the batch uses whose table set of the batch's worklist slot is stale."""
    import torch
    view = b2d.make_view(320, 200)
    timed = []
    for L in levels:
        one = b2d.Renderer(L["scene"], view, max_batch=1)
        l0 = one.launch_count
        one.render_timed(sample_poses(b2d, L["scene"], 1, 5), [9])
        timed.append(one.launch_count - l0 == 3)
    assert timed[C2] and timed[RICH] and not timed[SMALL]
    r = b2d.Renderer.from_levels([L["scene"] for L in levels], view, max_batch=16)
    poses, _ = _mix(b2d, levels, 4, 500)
    dp = _dev(poses)
    out = torch.empty((16, 200, 320), dtype=torch.uint8, device="cuda")
    stale = [set(), set()]               # per worklist slot (batches alternate): timed levels whose table set is stale
    ticket = [0]

    def batch(lv):
        """-> (launches of the batch, launches expected: 2 + one per stale timed level the batch uses)"""
        slot = ticket[0] & 1
        want = 2 + len(stale[slot] & set(lv))
        stale[slot] -= set(lv)
        ticket[0] += 1
        l0 = r.launch_count
        r.render_device_levels(dp.data_ptr(), np.array(lv, np.uint32), len(lv), out.data_ptr())
        return r.launch_count - l0, want

    mix = [0, 1, 2, 3] * 4
    assert [batch(mix)[0] for _ in range(4)] == [2, 2, 2, 2]
    r.set_time(500)
    stale = [{k for k in range(4) if timed[k]} for _ in range(2)]
    got = [batch([0, 2] * 8), batch(mix), batch([1, 3] * 8), batch(mix), batch(mix)]
    assert [g for g, _ in got] == [w for _, w in got]
    assert got[0][0] == 3 and got[1][0] == 2 + sum(timed) and got[3][0] == got[4][0] == 2
    r.set_level_sector_moves(RICH, levels[RICH]["moves"])
    stale = [{RICH}, {RICH}]
    got = [batch([0, 2] * 8), batch([1] * 16), batch(mix), batch(mix)]
    assert [g for g, _ in got] == [2, 3, 3, 2] == [w for _, w in got]
    torch.cuda.synchronize()
    assert r.status() == 0


def test_set_of_one_and_level_zero(b2d, levels):
    """A set of one renders what b2d_renderer_create's renderer renders, through every pre-existing entry point tried here;
    on a set of four, those entry points act on level 0."""
    view = b2d.make_view(320, 200)
    L = levels[RICH]
    poses = sample_poses(b2d, L["scene"], 10, 600)
    a, b = b2d.Renderer(L["scene"], view, max_batch=4), b2d.Renderer.from_levels([L["scene"]], view, max_batch=4)
    for r in (a, b):
        r.set_time(4321)
        r.set_sector_moves(L["moves"])
    _assert_same(a.render(poses), b.render(poses), "render")
    tics = np.arange(10, dtype=np.uint32) * 13
    _assert_same(a.render_timed(poses, tics), b.render_timed(poses, tics), "render_timed")
    _assert_same(a.render_states(poses, tics), b.render_states(poses, tics), "render_states")
    assert a.launch_count == b.launch_count
    _assert_same(a.render(poses), b.render_levels(poses, np.zeros(10, np.uint32)), "render_levels")
    r4 = b2d.Renderer.from_levels([levels[k]["scene"] for k in (RICH, C2, SMALL, LARGE)], view, max_batch=4)
    r4.set_time(4321)
    r4.set_sector_moves(L["moves"])
    want = _oracle([levels[RICH]], 320, 200, poses, np.zeros(10, np.uint32), tics=4321, moved={0: L["moves"]})
    _assert_same(want, r4.render(poses), "render on a set of four")
    _assert_same(want, r4.render_levels(poses, np.zeros(10, np.uint32)), "render_levels, level 0")
    _assert_same(b.render_states(poses, tics), r4.render_states(poses, tics), "render_states on a set of four")
    assert a.status() == b.status() == r4.status() == 0


def test_levels_invalid_inputs_enqueue_nothing(b2d, levels):
    """A level index >= n_levels, a NULL level array, a NULL scene and n_levels outside 1..64 are B2D_ERR_INVALID_ARG;
    nothing is launched and the status word stays clear."""
    from rust_doom_b200 import _lib
    L = _lib.load()
    view = b2d.make_view(320, 200)
    scenes = [lv["scene"] for lv in levels]
    r = b2d.Renderer.from_levels(scenes, view, max_batch=4)
    poses, lv = _mix(b2d, levels, 1, 700)
    out = np.empty((4, 200, 320), np.uint8)
    l0 = r.launch_count
    for bad in ([0, 1, 4, 2], [0, 0xFFFFFFFF, 1, 2]):
        with pytest.raises(b2d.B2dError) as e:
            r.render_levels(poses, bad)
        assert e.value.code == b2d.ERR_INVALID_ARG
        with pytest.raises(b2d.B2dError):
            r.render_device_levels(0x1000, bad, 4, 0x2000)
        with pytest.raises(b2d.B2dError):
            r.walk_device_levels(0x1000, bad, 4)
    t = ctypes.c_int64(-1)
    assert L.b2d_render_levels(r._h, poses.ctypes.data, None, 4, out.ctypes.data, None) == b2d.ERR_INVALID_ARG
    assert L.b2d_render_device_levels(r._h, 0x1000, None, 4, 0x2000, None, None) == b2d.ERR_INVALID_ARG
    assert L.b2d_walk_device_levels(r._h, 0x1000, None, 4, None, ctypes.byref(t)) == b2d.ERR_INVALID_ARG
    assert r.launch_count == l0
    assert r.status() == 0
    h = ctypes.c_void_p()
    for arr, n in (((ctypes.c_void_p * 2)(scenes[0]._h, None), 2), ((ctypes.c_void_p * 1)(scenes[0]._h), 0),
                   ((ctypes.c_void_p * 65)(*([scenes[2]._h] * 65)), 65)):
        assert L.b2d_renderer_create_levels(arr, n, ctypes.byref(view), 0, 4, ctypes.byref(h)) == b2d.ERR_INVALID_ARG
    assert L.b2d_renderer_create_levels(None, 1, ctypes.byref(view), 0, 4, ctypes.byref(h)) == b2d.ERR_INVALID_ARG
    _assert_same(_oracle(levels, 320, 200, poses, lv), r.render_levels(poses, lv), "after the refusals")
    assert r.status() == 0


def test_level_set_worklists(b2d, levels):
    """Renderer.worklist after a level batch: sized by the set's stride (the largest level's), and every frame's worklist
    equals that of its own level's renderer, the large level's included."""
    view = b2d.make_view(320, 200)
    r = b2d.Renderer.from_levels([levels[k]["scene"] for k in (C2, LARGE)], view, max_batch=12)
    big = levels[LARGE]["scene"].info
    assert r.worklist_stride == big.n_segs + big.n_sprites > levels[C2]["scene"].info.n_segs
    poses, lv = _mix(b2d, [levels[C2], levels[LARGE]], 6, 800)
    r.render_levels(poses, lv)
    counts, ids = r.worklist(12)
    for k, L in enumerate((levels[C2], levels[LARGE])):
        sel = np.nonzero(lv == k)[0]
        one = b2d.Renderer(L["scene"], view, max_batch=12)
        one.render(poses[sel])
        c1, i1 = one.worklist(len(sel))
        assert counts[sel].tolist() == c1.tolist()
        for j, f in enumerate(sel):
            assert ids[f, :counts[f]].tolist() == i1[j, :c1[j]].tolist(), "frame %d" % f
    assert r.status() == 0
