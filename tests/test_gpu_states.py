"""-m gpu: per-frame states (b2d_render_states, b2d_render_device_states, b2d_walk_device_states).  Every frame is compared
with the oracle's frame at that pose's state: its own scene with the pose's moves applied (oracle/scene.py apply_moves),
rendered at the pose's tics."""
import ctypes

import numpy as np
import pytest

from oracle import render
from tests.conftest import sample_poses

pytestmark = pytest.mark.gpu


def _level(b2d, seed=1, doors=True, **cfg):
    """A generated level with animation, scrolling walls and light effects (+ cfg), its oracle blob and dynamic sectors:
    tests/refcheck/moves.py's declaration, with the ceilings of the first few non-sky sectors allowed down to their floor
    (closed doors)."""
    from oracle import scene as S, wad as W
    from rust_doom_b200 import synthwad
    from tests.refcheck import moves as MV
    data = synthwad.build_iwad(seed, ("E1M1",), cfg=synthwad.SynthConfig(anim=True, **cfg))
    a = W.Archive(data)
    level = W.Level(a, 0)
    dyn = MV.declare(level, 5, 16) if doors else []
    doors_ = []
    for k, (s, fmin, fmax, cmin, cmax) in enumerate(dyn):
        f0, c0 = int(level.sectors[s]["floor"]), int(level.sectors[s]["ceil"])
        if cmin != cmax and len(doors_) < 4:
            dyn[k] = (s, fmin, fmax, min(cmin, f0), cmax)
            doors_.append((s, f0, c0))
    oblob = S.compile_scene(a, W.TextureDirectory(a), 0, dynamic=dyn)
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0, dynamic=dyn)
    assert sc.blob == oblob
    return sc, oblob, level, dyn, doors_


def _states(level, dyn, doors, n, seed):
    """n move states: at rest, closed doors, and random states inside the declared ranges"""
    from tests.refcheck import moves as MV
    out = []
    for i in range(n):
        if i % 4 == 0:
            out.append([])
        elif i % 4 == 1:
            out.append([(s, 0, f0 - c0) for (s, f0, c0) in doors])          # ceiling down on the floor
        else:
            out.append(MV.state(level, dyn, seed + i, hole_free=False))
    return out


def _oracle(oblob, w, h, poses, tics, moves):
    from oracle import scene as S
    view = render.make_view(w, h)
    return np.stack([render.render(S.apply_moves(oblob, moves[i]) if moves[i] else oblob, view, poses[i:i + 1], threads=8,
                                   tics=int(tics[i]))[0] for i in range(len(poses))])


def _assert_same(want, got, what):
    bad = [(i, int((want[i] != got[i]).sum())) for i in range(len(want)) if not np.array_equal(want[i], got[i])]
    assert not bad, "%s: frames differ (index, pixels): %s" % (what, bad[:6])


def test_states_match_oracle_both_entry_points(b2d):
    """Timelines that change every tic, random 32-bit tics (2^32-1 included) and a different move state per frame, through
    the host path with a small max_batch (batches split) and the device path; the renderer's own time and moves stay."""
    import torch
    sc, oblob, level, dyn, doors = _level(b2d, mid_pct=30, thing_pct=50)
    assert doors and sc.info.n_masked_mids > 0 and sc.info.n_sprites > 0
    n = 24
    poses = sample_poses(b2d, sc, n, 71)
    moves = _states(level, dyn, doors, n, 900)
    timelines = [np.arange(n, dtype=np.uint32) + 1000,
                 np.concatenate([[0xFFFFFFFF], np.random.default_rng(3).integers(0, 1 << 32, n - 1, dtype=np.uint64)]).astype(np.uint32)]
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=5)
    rest = r.render(poses)
    for tl in timelines:
        want = _oracle(oblob, 320, 200, poses, tl, moves)
        _assert_same(want, r.render_states(poses, tl, moves), "host path")
        dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
        out = torch.empty((n, 200, 320), dtype=torch.uint8, device="cuda")
        r.render_device_states(dp.data_ptr(), tl, n, out.data_ptr(), moves_per_pose=moves)
        torch.cuda.synchronize()
        _assert_same(want, out.cpu().numpy(), "device path")
    assert r.status() == 0
    _assert_same(rest, r.render(poses), "the renderer's own time and moves")


def test_states_share_slots_and_launch_counts(b2d):
    """Frames with equal states share one table set wherever they are in the batch; a batch costs walk + expansion +
    raster; a level without time-dependent content keeps two launches per batch."""
    sc, oblob, level, dyn, doors = _level(b2d, mid_pct=15, thing_pct=20)
    poses = sample_poses(b2d, sc, 12, 72)
    st = _states(level, dyn, doors, 3, 950)
    tics = np.array([5, 900, 5, 17, 5, 900, 17, 17, 5, 900, 5, 17], np.uint32)
    moves = [st[[0, 1, 0, 2, 0, 1, 2, 2, 0, 1, 0, 2][i]] for i in range(12)]     # the same three states, interleaved
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=12)
    l0 = r.launch_count
    got = r.render_states(poses, tics, moves)
    assert r.launch_count - l0 == 3
    slots = r.state_slots(12).tolist()
    assert slots == [0, 1, 0, 2, 0, 1, 2, 2, 0, 1, 0, 2], slots
    _assert_same(_oracle(oblob, 320, 200, poses, tics, moves), got, "shared slots")
    r2 = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=5)
    l0 = r2.launch_count
    r2.render_states(poses, tics, moves)
    assert r2.launch_count - l0 == 9                           # 3 batches
    from rust_doom_b200 import synthwad
    plain = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(light_fx=False))), 0)
    r3 = b2d.Renderer(plain, b2d.make_view(320, 200), max_batch=12)
    p3 = sample_poses(b2d, plain, 12, 73)
    got = r3.render_states(p3, np.arange(12) * 7)
    assert r3.launch_count == 2
    _assert_same(render.render(plain.blob, render.make_view(320, 200), p3, threads=8), got, "static level")


def test_states_pipelined_walk_and_two_raster_streams(b2d):
    """walk_device_states of batch k+1 on its own stream under raster_device of batch k, rasters alternating between two
    streams, a different state per batch and per frame; afterwards a plain render still shows the renderer's own time
    and moves."""
    import torch
    sc, oblob, level, dyn, doors = _level(b2d, mid_pct=20, thing_pct=30)
    view = b2d.make_view(640, 400)
    r = b2d.Renderer(sc, view, max_batch=8)
    own = _states(level, dyn, doors, 3, 970)[2]
    r.set_time(77)
    r.set_sector_moves(own)
    batches = [sample_poses(b2d, sc, 8, 600 + k) for k in range(4)]
    tics = [np.arange(8, dtype=np.uint32) + 40 * k for k in range(4)]
    moves = [_states(level, dyn, doors, 8, 1000 + 10 * k) for k in range(4)]
    dps = [torch.from_numpy(p.view(np.int32).reshape(-1, 4).copy()).cuda() for p in batches]
    outs = [torch.empty((8, 400, 640), dtype=torch.uint8, device="cuda") for _ in batches]
    s_walk, s_r = torch.cuda.Stream(priority=-1), (torch.cuda.Stream(), torch.cuda.Stream())
    torch.cuda.synchronize()
    ticket = r.walk_device_states(dps[0].data_ptr(), tics[0], 8, moves[0], s_walk.cuda_stream)
    for k in range(4):
        r.raster_device(ticket, outs[k].data_ptr(), 0, s_r[k % 2].cuda_stream)
        if k + 1 < 4:
            ticket = r.walk_device_states(dps[k + 1].data_ptr(), tics[k + 1], 8, moves[k + 1], s_walk.cuda_stream)
    torch.cuda.synchronize()
    assert r.status() == 0
    for k in range(4):
        _assert_same(_oracle(oblob, 640, 400, batches[k], tics[k], moves[k]), outs[k].cpu().numpy(), "batch %d" % k)
    p = batches[0][:4]
    _assert_same(_oracle(oblob, 640, 400, p, [77] * 4, [own] * 4), r.render(p), "the renderer's own state")


@pytest.mark.parametrize("masked", [False, True])
def test_states_every_raster_variant(b2d, masked):
    """Each kStates instantiation launch_raster dispatches: 1080p index and RGBA, 4K index, the generic width (index and
    RGBA), on a level with and one without masked content; two sampled frames each, at different states."""
    cfg = dict(mid_pct=30, thing_pct=50) if masked else dict(mid_pct=0, thing_pct=0)
    sc, oblob, level, dyn, doors = _level(b2d, **cfg)
    assert (sc.info.n_masked_mids + sc.info.n_sprites > 0) == masked
    poses = sample_poses(b2d, sc, 2, 74)
    moves = _states(level, dyn, doors, 3, 990)[1:]
    tics = np.array([123457, 0xFFFFFFF0], np.uint32)
    for (w, h, rgba) in ((1920, 1080, False), (1920, 1080, True), (3840, 2160, False), (1000, 700, False), (1000, 700, True)):
        r = b2d.Renderer(sc, b2d.make_view(w, h), max_batch=2)
        got = r.render_states(poses, tics, moves, rgba=rgba)
        want = _oracle(oblob, w, h, poses, tics, moves)
        if rgba:
            pal = np.frombuffer(sc.blob, "<u4", 256, int(np.frombuffer(sc.blob, "<u4", 21)[20]))
            assert np.array_equal(got[1], pal[got[0]])
            got = got[0]
        _assert_same(want, got, "%dx%d rgba=%s masked=%s" % (w, h, rgba, masked))
        assert r.status() == 0


def test_states_invalid_inputs_enqueue_nothing(b2d):
    """Moves of undeclared sectors, moves outside a declared range, move ranges past the list and a NULL state array are
    refused before anything is enqueued; the next valid call renders correctly."""
    from rust_doom_b200 import _lib
    sc, oblob, level, dyn, doors = _level(b2d, mid_pct=10, thing_pct=10)
    poses = sample_poses(b2d, sc, 4, 75)
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=4)
    declared = {d[0] for d in dyn}
    undeclared = next(s for s in range(len(level.sectors)) if s not in declared)
    good = _states(level, dyn, doors, 3, 995)
    tics = [1, 2, 3, 4]
    bad_moves = [[(undeclared, 1, 0)], [(dyn[0][0], 5000, 0)]]
    for bad in bad_moves:
        l0 = r.launch_count
        with pytest.raises(b2d.B2dError) as e:
            r.render_states(poses, tics, [good[0], bad, good[1], good[2]])
        assert e.value.code == b2d.ERR_INVALID_ARG and r.launch_count == l0
        with pytest.raises(b2d.B2dError):
            r.walk_device_states(0x1000, tics, 4, [good[0], good[1], bad, good[2]])
        assert r.launch_count == l0
    L = _lib.load()
    arr = (_lib.SectorMove * 3)(*[_lib.SectorMove(*m) for m in (good[2] + good[2])[:3]])
    states = (_lib.FrameState * 4)(*[_lib.FrameState(t, 2, 5) for t in tics])          # moves [2, 7) of a 3-move list
    out = np.empty((4, 200, 320), np.uint8)
    l0 = r.launch_count
    assert L.b2d_render_states(r._h, poses.ctypes.data, states, 4, arr, 3, out.ctypes.data, None) == b2d.ERR_INVALID_ARG
    assert L.b2d_render_states(r._h, poses.ctypes.data, None, 4, arr, 3, out.ctypes.data, None) == b2d.ERR_INVALID_ARG
    t = ctypes.c_int64(-1)
    assert L.b2d_walk_device_states(r._h, 0x1000, None, 4, arr, 3, None, ctypes.byref(t)) == b2d.ERR_INVALID_ARG
    assert r.launch_count == l0
    assert r.status() == 0
    moves = [good[0], good[1], good[2], []]
    _assert_same(_oracle(oblob, 320, 200, poses, tics, moves), r.render_states(poses, tics, moves), "after the refusals")
    assert r.status() == 0
    from rust_doom_b200 import synthwad
    plain = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(light_fx=False))), 0)
    with pytest.raises(b2d.B2dError):
        b2d.Renderer(plain, b2d.make_view(320, 200), max_batch=4).render_states(poses[:1], [0], [[(0, 1, 0)]])
