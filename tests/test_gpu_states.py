"""-m gpu: per-frame states (b2d_render_states, b2d_render_device_states, b2d_walk_device_states).  Every frame is compared
with the oracle's frame at that pose's state: its own scene with the pose's moves applied (oracle/scene.py apply_moves),
rendered at the pose's tics."""
import ctypes
import os

import numpy as np
import pytest

from oracle import render
from tests.conftest import sample_poses
from tests.test_scene import EDGE_TICS, STATE_KINDS, assert_kind, declare_doors, state_level, state_moves

pytestmark = pytest.mark.gpu


def _level(b2d, seed=1, doors=True, **cfg):
    """A generated level with animation, scrolling walls and light effects (+ cfg), its oracle blob and dynamic sectors:
    tests/refcheck/moves.py's declaration, with the ceilings of the first few non-sky sectors allowed down to their floor
    (closed doors)."""
    from oracle import scene as S, wad as W
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(seed, ("E1M1",), cfg=synthwad.SynthConfig(anim=True, **cfg))
    a = W.Archive(data)
    level = W.Level(a, 0)
    dyn, doors_ = declare_doors(level) if doors else ([], [])
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
    """The oracle's frame of every pose at its own (tics, moves): apply_moves once per distinct move list, the frames on a
    thread pool (the oracle's ctypes calls release the GIL)."""
    from concurrent.futures import ThreadPoolExecutor
    from oracle import scene as S
    view = render.make_view(w, h)
    blobs = {}
    for m in moves:
        key = tuple(map(tuple, m))
        if key not in blobs:
            blobs[key] = S.apply_moves(oblob, m) if m else oblob
    out = np.empty((len(poses), h, w), np.uint8)

    def one(i):
        render.render(blobs[tuple(map(tuple, moves[i]))], view, poses[i:i + 1], tics=int(tics[i]), out=out[i:i + 1])

    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        list(ex.map(one, range(len(poses))))
    return out


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


def check_state_sets(r, oblob, tics, moves, n):
    """The table sets of the last batch r walked with per-frame states, read back: each equals oracle/scene.py tables_at of
    the frames that read it, so frames that share a set have equal oracle tables.  -> (set index per frame, oracle tables
    per frame)."""
    from oracle import scene as S
    from rust_doom_b200 import B2dError
    slots = r.state_slots(n)
    nsets = int(slots.max()) + 1
    assert set(slots.tolist()) == set(range(nsets)), "set indices are not 0 .. n_sets-1"
    cache = {}
    want = []
    for i in range(n):
        key = (int(tics[i]), tuple(map(tuple, moves[i])))
        if key not in cache:
            cache[key] = S.tables_at(oblob, key[0], moves[i])
        want.append(cache[key])
    got = [r.state_tables(k) for k in range(nsets)]
    for i in range(n):
        if got[slots[i]] != want[i]:
            g, w = np.frombuffer(got[slots[i]], np.int32), np.frombuffer(want[i], np.int32)
            pytest.fail("frame %d (tics %d): table set %d differs from the oracle's tables at words %s" % (
                i, int(tics[i]), slots[i], np.nonzero(g != w)[0][:8]))
    with pytest.raises(B2dError):
        r.state_tables(nsets)
    return slots, want


@pytest.mark.parametrize("kind", STATE_KINDS)
def test_states_level_kinds_at_edge_tics(b2d, kind):
    """One batch per level kind (tests/test_scene.py state_level: light effects only, animation only, scrolling only,
    dynamic sectors only, everything) through render_device_states, every edge tic with every move list of the kind (at
    rest, all offsets zero, doors shut, random): frames equal the oracle, every expanded table set equals the oracle's
    tables_at, and the number of sets is what the compact state makes of the kind -- one per distinct tables where the
    state keeps exactly what the tables depend on, one per (tics >> 3, moves) where the level only animates (its frames
    repeat every n steps, the state does not know n), and a move list of zeros is the rest state."""
    import torch
    from oracle import scene as S, wad as W
    data, dyn, doors, level = state_level(kind)
    a = W.Archive(data)
    oblob = S.compile_scene(a, W.TextureDirectory(a), 0, dynamic=dyn)
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0, dynamic=dyn)
    assert sc.blob == oblob
    assert_kind(oblob, kind)
    lists = state_moves(level, dyn, doors, 40)
    pairs = [(t, m) for t in EDGE_TICS for m in range(len(lists))]
    n = len(pairs)
    tics = np.array([t for t, _ in pairs], np.uint64).astype(np.uint32)
    moves = [lists[m] for _, m in pairs]
    poses = sample_poses(b2d, sc, n, 76)
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=n)
    with pytest.raises(b2d.B2dError):
        r.state_tables(0)                                           # nothing walked yet
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    out = torch.empty((n, 200, 320), dtype=torch.uint8, device="cuda")
    r.render_device_states(dp.data_ptr(), tics, n, out.data_ptr(), moves_per_pose=moves)
    torch.cuda.synchronize()
    assert r.status() == 0
    _assert_same(_oracle(oblob, 320, 200, poses, tics, moves), out.cpu().numpy(), kind)
    slots, want = check_state_sets(r, oblob, tics, moves, n)
    nsets = int(slots.max()) + 1
    if kind == "anim":
        assert nsets == len({(int(t) >> 3, m) for t, m in pairs})
    elif kind != "all":
        assert nsets == len(set(want)), "same set if and only if same tables"
    if kind == "moves":
        for k in range(len(EDGE_TICS)):                             # [] and the all-zero list: one set, at every tic
            assert slots[len(lists) * k] == slots[len(lists) * k + 1] == slots[0]
