"""-m gpu: per-frame states with per-frame levels (b2d_render_levels_states, b2d_render_device_levels_states,
b2d_walk_device_levels_states).  The four levels of tests/test_gpu_levels.py in one renderer; every frame carries its own
level, level time and (on the level with declared dynamic sectors) move slice.  Every frame is compared with the oracle's
frame of that pose on its own level at its own state, and with a b2d_renderer_create renderer of that level through
render_states; every expanded table set, read back, with oracle/scene.py tables_at of its level."""
import ctypes
import os

import numpy as np
import pytest

from oracle import render
from tests.conftest import sample_poses
from tests.test_gpu_levels import C2, LARGE, RICH, SMALL, _assert_same, _dev, _mix, _oracle, _palette, levels  # noqa: F401

pytestmark = pytest.mark.gpu


def _rich_states(levels, n, seed):
    """n move lists of the rich level: at rest, moves.pick's state, its doors down (every declared ceiling at the lowest
    height its range and its floor allow) and random states inside the declared ranges"""
    from oracle import wad as W
    from tests.refcheck import moves as MV
    L = levels[RICH]
    level = W.Level(W.Archive(L["data"]), 0)
    secs = level.sectors
    down = [(s, 0, max(cmin, int(secs[s]["floor"])) - int(secs[s]["ceil"])) for (s, _, _, cmin, _) in L["dyn"]]
    assert any(m[2] for m in down)
    out = []
    for i in range(n):
        k = i % 4
        out.append([] if k == 0 else L["moves"] if k == 1 else down if k == 2 else MV.state(level, L["dyn"], seed + i, hole_free=False))
    return out


def _per_frame(levels, lv, seed, tic0=0):
    """(tics, moves) of a batch: a distinct tic per frame (consecutive from tic0, a few random 32-bit ones mixed in) and a
    move list per frame on the rich level"""
    rng = np.random.default_rng(seed)
    n = len(lv)
    tics = (np.arange(n, dtype=np.uint64) * 7 + tic0)
    tics[rng.choice(n, size=max(1, n // 5), replace=False)] = rng.integers(0, 1 << 32, max(1, n // 5), dtype=np.uint64)
    rich = _rich_states(levels, n, seed)
    moves = [rich[i] if lv[i] == RICH else [] for i in range(n)]
    return tics.astype(np.uint32), moves


def _oracle_states(levels, w, h, poses, lv, tics, moves):
    """the oracle's frame of every pose on its own level at its own (tics, moves)"""
    from concurrent.futures import ThreadPoolExecutor
    from oracle import scene as S
    view = render.make_view(w, h)
    blobs = {}
    for k, m in zip(lv, moves):
        key = (int(k), tuple(map(tuple, m)))
        if key not in blobs:
            blobs[key] = S.apply_moves(levels[int(k)]["blob"], m) if m else levels[int(k)]["blob"]
    out = np.empty((len(poses), h, w), np.uint8)

    def one(i):
        render.render(blobs[(int(lv[i]), tuple(map(tuple, moves[i])))], view, poses[i:i + 1], tics=int(tics[i]), out=out[i:i + 1])

    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        list(ex.map(one, range(len(poses))))
    return out


def _timed(b2d, levels):
    """per level: it has time-dependent content or dynamic sectors (a timed batch on its own renderer costs 3 launches)"""
    out = []
    for L in levels:
        one = b2d.Renderer(L["scene"], b2d.make_view(64, 40), max_batch=1)
        l0 = one.launch_count
        one.render_timed(sample_poses(b2d, L["scene"], 1, 5), [9])
        out.append(one.launch_count - l0 == 3)
    return out


def check_level_sets(r, levels, timed, lv, tics, moves, n):
    """The table sets of the last batch r walked with per-frame states and levels, read back: frames share a set exactly
    when their (level, oracle tables) are equal, sets are numbered in order of first appearance, frames on levels without
    a table set have none (0xFFFFFFFF), and each set equals oracle/scene.py tables_at of its level.  -> set per frame."""
    from oracle import scene as S
    from rust_doom_b200 import B2dError
    slots = r.state_slots(n)
    has = [timed[int(lv[i])] for i in range(n)]
    assert all((slots[i] != 0xFFFFFFFF) == has[i] for i in range(n)), slots.tolist()
    order = [int(s) for i, s in enumerate(slots) if has[i]]
    first = list(dict.fromkeys(order))
    assert first == list(range(len(first))), "sets not numbered in order of first appearance: %s" % first[:10]
    cache, want, seen = {}, {}, {}
    for i in range(n):
        if not has[i]:
            continue
        key = (int(lv[i]), int(tics[i]), tuple(map(tuple, moves[i])))
        if key not in cache:
            cache[key] = S.tables_at(levels[key[0]]["blob"], key[1], moves[i])
        s = int(slots[i])
        if s in want:
            assert want[s] == cache[key] and seen[s] == key[0], "frame %d shares set %d with a frame of other tables" % (i, s)
        else:
            want[s], seen[s] = cache[key], key[0]
    for s in sorted(want):
        got = r.state_tables(s)
        assert len(got) == len(want[s]), "set %d: size of another level's tables" % s
        if got != want[s]:
            g, w = np.frombuffer(got, np.int32), np.frombuffer(want[s], np.int32)
            pytest.fail("set %d (level %d) differs from the oracle's tables at words %s" % (s, seen[s], np.nonzero(g != w)[0][:8]))
    with pytest.raises(B2dError):
        r.state_tables(len(want))
    return slots


@pytest.mark.parametrize("w,h", [(1920, 1080), (900, 600)])
def test_levels_states_match_oracle_and_single_level_renderers(b2d, levels, w, h):
    """Index and RGBA frames of a mixed batch with a tic per frame and a move slice per rich-level frame (closed doors among
    them), through the host path with n > max_batch and through the device path: each equals the oracle's frame on its
    level at its state (RGBA through its level's palette; at 900 columns raster CTAs straddle frames of different levels)
    and a b2d_renderer_create renderer of the level through render_states."""
    import torch
    poses, lv = _mix(b2d, levels, 4, 1101)
    tics, moves = _per_frame(levels, lv, 1102, tic0=300)
    view = b2d.make_view(w, h)
    r = b2d.Renderer.from_levels([L["scene"] for L in levels], view, max_batch=7)
    rest = r.render_levels(poses, lv)
    idx, rgba = r.render_levels_states(poses, lv, tics, moves, rgba=True)
    assert r.status() == 0
    _assert_same(_oracle_states(levels, w, h, poses, lv, tics, moves), idx, "%dx%d index" % (w, h))
    for i in range(len(poses)):
        assert np.array_equal(rgba[i], _palette(levels[lv[i]]["scene"])[idx[i]]), "frame %d: RGBA is not its level's palette" % i
    for k, L in enumerate(levels):
        sel = np.nonzero(lv == k)[0]
        one = b2d.Renderer(L["scene"], view, max_batch=7)
        i1, r1 = one.render_states(poses[sel], tics[sel], [moves[i] for i in sel], rgba=True)
        _assert_same(i1, idx[sel], "level %d vs its own renderer (index)" % k)
        _assert_same(r1, rgba[sel], "level %d vs its own renderer (RGBA)" % k)
    n = len(poses)
    out = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
    out_rgba = torch.empty((n, h, w), dtype=torch.int32, device="cuda")
    r.render_device_levels_states(_dev(poses).data_ptr(), lv, tics, n, out.data_ptr(), out_rgba.data_ptr(), moves_per_pose=moves)
    torch.cuda.synchronize()
    _assert_same(idx, out.cpu().numpy(), "device path (index)")
    _assert_same(rgba, out_rgba.cpu().numpy().view(np.uint32), "device path (RGBA)")
    assert r.status() == 0
    _assert_same(rest, r.render_levels(poses, lv), "the renderer's own time and moves")


def test_levels_states_sets_and_launch_counts(b2d, levels):
    """Equal (level, state) pairs share one set wherever they are in the batch; the same tic on c2 and on the rich level is
    two sets; a batch only on the untimed levels costs 2 launches, any other 3, whatever it mixes; every set read back
    equals the oracle's tables of its level."""
    import torch
    timed = _timed(b2d, levels)
    assert timed[C2] and timed[RICH] and not timed[SMALL]
    untimed = [k for k in range(4) if not timed[k]]
    view = b2d.make_view(320, 200)
    r = b2d.Renderer.from_levels([L["scene"] for L in levels], view, max_batch=16)
    poses, _ = _mix(b2d, levels, 4, 1200)
    dp = _dev(poses)
    out = torch.empty((16, 200, 320), dtype=torch.uint8, device="cuda")
    mv = levels[RICH]["moves"]

    def batch(lv, tics, moves):
        l0 = r.launch_count
        r.render_device_levels_states(dp.data_ptr(), np.array(lv, np.uint32), np.array(tics, np.uint32), len(lv), out.data_ptr(),
                                      moves_per_pose=moves)
        torch.cuda.synchronize()
        return r.launch_count - l0

    lv = [C2, RICH, SMALL, RICH, C2, LARGE, RICH, C2] * 2
    tics = [40] * 16
    moves = [mv if (k == RICH and i % 4 == 3) else [] for i, k in enumerate(lv)]
    assert batch(lv, tics, moves) == 3
    slots = check_level_sets(r, levels, timed, lv, tics, moves, 16).tolist()
    # c2 @40 -> set 0; rich @40 (the same tic) at rest -> set 1, moved -> set 2; frames of untimed levels have none
    want, keys = [], {}
    for i, k in enumerate(lv):
        want.append(keys.setdefault((k, bool(moves[i])), len(keys)) if timed[k] else 0xFFFFFFFF)
    assert slots == want and want[:2] == [0, 1] and want[3] == 2, slots
    assert batch(untimed * (16 // len(untimed)), list(range(16)), None) == 2
    assert r.state_slots(16).tolist() == [0xFFFFFFFF] * 16
    assert batch([SMALL] * 15 + [C2], [7] * 16, None) == 3
    mix = list(range(4)) * 4
    mix_moves = [mv if k == RICH else [] for k in mix]
    assert batch(mix, list(range(100, 116)), mix_moves) == 3
    check_level_sets(r, levels, timed, mix, list(range(100, 116)), mix_moves, 16)
    assert batch([RICH] * 16, [9] * 16, [mv] * 16) == 3
    assert r.state_slots(16).tolist() == [0] * 16
    assert r.status() == 0


def test_levels_states_pipelined_tickets(b2d, levels):
    """walk_device_levels_states of batch k+1 on a walk stream under the raster of batch k, rasters alternating between two
    streams, plain walk_device_levels batches interleaved and set_time / set_level_sector_moves calls between them: the
    per-frame batches equal the oracle at their own states, the plain ones at the renderer's state, which the per-frame
    calls leave as it is."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    batch = sms + 9
    r = b2d.Renderer.from_levels([L["scene"] for L in levels], b2d.make_view(320, 200), max_batch=batch)
    mixes = [_mix(b2d, levels, (batch + 3) // 4, 1300 + k, spread=sms) for k in range(5)]
    mixes = [(p[:batch], lv[:batch]) for p, lv in mixes]
    dps = [_dev(p) for p, _ in mixes]
    outs = [torch.empty((batch, 200, 320), dtype=torch.uint8, device="cuda") for _ in mixes]
    s_walk, s_r = torch.cuda.Stream(priority=-1), (torch.cuda.Stream(), torch.cuda.Stream())
    mv = levels[RICH]["moves"]
    # (per-frame?, renderer time and rich-level moves set before the walk)
    plan = [(True, 10, None), (False, 2000, mv), (True, 2001, None), (False, 35 * 60, []), (True, 5, mv)]
    states = [_per_frame(levels, lv, 1310 + k, tic0=50 * k) if pf else None for k, ((_, lv), (pf, _, _)) in enumerate(zip(mixes, plan))]
    renderer_state = []
    torch.cuda.synchronize()

    def walk(k):
        pf, t, m = plan[k]
        r.set_time(t)
        if m is not None:
            r.set_level_sector_moves(RICH, m)
        renderer_state.append((t, m if m is not None else (renderer_state[-1][1] if renderer_state else [])))
        if pf:
            tics, moves = states[k]
            return r.walk_device_levels_states(dps[k].data_ptr(), mixes[k][1], tics, batch, moves, s_walk.cuda_stream)
        return r.walk_device_levels(dps[k].data_ptr(), mixes[k][1], batch, s_walk.cuda_stream)

    ticket = walk(0)
    for k in range(len(plan)):
        r.raster_device(ticket, outs[k].data_ptr(), 0, s_r[k % 2].cuda_stream)
        if k + 1 < len(plan):
            ticket = walk(k + 1)
    torch.cuda.synchronize()
    assert r.status() == 0
    for k, (p, lv) in enumerate(mixes):
        if plan[k][0]:
            tics, moves = states[k]
            _assert_same(_oracle_states(levels, 320, 200, p, lv, tics, moves), outs[k].cpu().numpy(), "per-frame batch %d" % k)
        else:
            t, m = renderer_state[k]
            _assert_same(_oracle(levels, 320, 200, p, lv, tics=t, moved={RICH: m} if m else None), outs[k].cpu().numpy(),
                         "plain batch %d" % k)
    t, m = renderer_state[-1]
    p, lv = mixes[0]
    _assert_same(_oracle(levels, 320, 200, p, lv, tics=t, moved={RICH: m} if m else None), r.render_levels(p, lv),
                 "the renderer's own state after the per-frame batches")


def test_levels_states_1000_frame_batch(b2d, levels):
    """A 1000-frame 1080p batch on the rich and c2 levels, nearly every frame at its own state: the expansion's records
    outnumber its grid's threads (more than one pass of the grid-stride loop) and the masked-entry arena is at its sizing
    limit (max_batch 1000 at 1080p).  Sampled frames equal the oracle's, and every set read back equals the oracle's tables."""
    import torch
    from rust_doom_b200 import poses as P
    N, W, H = 1000, 1920, 1080
    two = [levels[C2], levels[RICH]]
    rng = np.random.default_rng(1400)
    lv = rng.integers(0, 2, N).astype(np.uint32)
    pools = [P.flythrough_poses(L["scene"], N, 2) for L in two]
    poses = np.empty(N, dtype=pools[0].dtype)
    for i in range(N):
        poses[i] = pools[lv[i]][i]
    tics = (np.arange(N, dtype=np.uint32) * 3 + 9000)
    rich = _rich_states(levels, N, 1401)
    moves = [rich[i] if lv[i] == 1 else [] for i in range(N)]
    r = b2d.Renderer.from_levels([L["scene"] for L in two], b2d.make_view(W, H), max_batch=N)
    out = torch.empty((N, H, W), dtype=torch.uint8, device="cuda")
    dp = _dev(poses)
    l0 = r.launch_count
    ticket = r.walk_device_levels_states(dp.data_ptr(), lv, tics, N, moves)
    r.raster_device(ticket, out.data_ptr())
    torch.cuda.synchronize()
    assert r.launch_count - l0 == 3
    assert r.status() == 0
    slots = check_level_sets(r, two, [True, True], lv, tics, moves, N)
    nsets = int(slots.max()) + 1
    assert nsets > 0.8 * N                      # c2's light effects repeat some states
    from oracle import scene as S
    recs = sum(int(sum(S.header(two[int(lv[i])]["blob"])[k] for k in (S.H_NTEX, S.H_NSECTORS, S.H_NSEGS, S.H_NSPRITES, S.H_NMIDS)))
               for i in dict((int(s), i) for i, s in enumerate(slots)).values())
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert recs > sms * 16 * 256, "one pass of the expansion grid"
    sample = np.arange(0, N, 20)
    _assert_same(_oracle_states(two, W, H, poses[sample], lv[sample], tics[sample], [moves[i] for i in sample]),
                 out[torch.from_numpy(sample).cuda()].cpu().numpy(), "sampled frames")


def test_levels_states_invalid_inputs_enqueue_nothing(b2d, levels):
    """A level >= n_levels, a NULL level or state array, a move range past n_moves, a move of a sector that is not declared
    dynamic on the frame's level (a rich-level move on a c2 frame) or outside its range: B2D_ERR_INVALID_ARG, and nothing
    launched."""
    from rust_doom_b200 import _lib
    L = _lib.load()
    r = b2d.Renderer.from_levels([lv["scene"] for lv in levels], b2d.make_view(320, 200), max_batch=4)
    lv = np.array([C2, RICH, SMALL, LARGE], np.uint32)
    poses = np.concatenate([sample_poses(b2d, levels[int(k)]["scene"], 1, 1500 + int(k)) for k in lv])
    mv = levels[RICH]["moves"]
    s0 = levels[RICH]["dyn"][0][0]
    out = np.empty((4, 200, 320), np.uint8)
    l0 = r.launch_count
    bad_calls = [
        ([C2, RICH, 4, LARGE], [[]] * 4),                                   # level >= n_levels
        ([C2, RICH, SMALL, 0xFFFFFFFF], [[]] * 4),
        (lv, [mv, [], [], []]),                                             # a rich-level move on a c2 frame
        (lv, [[], [], mv, []]),                                             # ... on a level without dynamic sectors
        (lv, [[], [(s0, 0, 1 << 20)], [], []]),                             # outside its range
    ]
    for levs, moves in bad_calls:
        with pytest.raises(b2d.B2dError) as e:
            r.render_levels_states(poses, levs, [1, 2, 3, 4], moves)
        assert e.value.code == b2d.ERR_INVALID_ARG
        with pytest.raises(b2d.B2dError):
            r.render_device_levels_states(0x1000, levs, [1, 2, 3, 4], 4, 0x2000, moves_per_pose=moves)
        with pytest.raises(b2d.B2dError):
            r.walk_device_levels_states(0x1000, levs, [1, 2, 3, 4], 4, moves)
    t = ctypes.c_int64(-1)
    st = (_lib.FrameState * 4)(*[_lib.FrameState(1, 0, 0) for _ in range(4)])
    past = (_lib.FrameState * 4)(_lib.FrameState(1, 0, 0), _lib.FrameState(1, 0, 2), _lib.FrameState(1, 0, 0), _lib.FrameState(1, 0, 0))
    one = (_lib.SectorMove * 1)(_lib.SectorMove(s0, 0, 0))
    lvp = lv.ctypes.data
    for levs, states, moves, nm in ((None, st, None, 0), (lvp, None, None, 0), (lvp, past, one, 1)):
        assert L.b2d_render_levels_states(r._h, poses.ctypes.data, levs, states, 4, moves, nm, out.ctypes.data, None) == b2d.ERR_INVALID_ARG
        assert L.b2d_render_device_levels_states(r._h, 0x1000, levs, states, 4, moves, nm, 0x2000, None, None) == b2d.ERR_INVALID_ARG
        assert L.b2d_walk_device_levels_states(r._h, 0x1000, levs, states, 4, moves, nm, None, ctypes.byref(t)) == b2d.ERR_INVALID_ARG
    assert r.launch_count == l0
    assert r.status() == 0
    tics = np.array([1, 2, 3, 4], np.uint32)
    moves = [[], mv, [], []]
    _assert_same(_oracle_states(levels, 320, 200, poses, lv, tics, moves), r.render_levels_states(poses, lv, tics, moves),
                 "after the refusals")
    assert r.status() == 0
