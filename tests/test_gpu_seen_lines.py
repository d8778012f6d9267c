"""-m gpu: seen lines (b2d_raster_device_seen, DESIGN.md C20).  For every walk form -- plain, per-frame states, per-frame
levels, both, and both with fixed colormaps and extra light -- on a level with doors and one with masked middles and
sprites, at 320x200 and 1920x1080, the index frames equal the ordinary raster's and each frame's row equals the oracle's
seen set at that frame's level and state (oracle/seen.py).  Rows are OR-ed into, rows past the batch are untouched, an
agent's fly-through accumulates into its rows, refusals enqueue nothing, a seen raster is one launch, and the first
call's table upload orders later calls on other streams.  The seen automap (b2d_automap_seen_device) against
oracle/automap_seen.py for every flag on one level and a level set, its refusals, the fly-through's automap, and both CLIs'
--automap-flags seen,allmap."""
import numpy as np
import pytest

from oracle import render
from oracle import scene as S
from oracle import seen as O
from tests.conftest import sample_poses
from tests.test_gpu_resolve import clock, mark, must_wait, pending  # noqa: F401
from tests.test_gpu_states import _level, _states

pytestmark = pytest.mark.gpu

FORMS = ["plain", "states", "levels", "levels_states", "lights"]


@pytest.fixture(scope="module")
def lset(b2d):
    """[(scene, oracle blob, oracle level, dynamic sectors, doors)]: a generated level with doors, and one with masked
    middles and sprites as well"""
    return [_level(b2d, seed=1), _level(b2d, seed=3, mid_pct=30, thing_pct=40)]


def _oracle_rows(entries, view, poses, levels, moves, words):
    """uint32 [n, words]: the oracle's seen lines of each pose at its level and move state"""
    out = np.zeros((len(poses), words), np.uint32)
    for i in range(len(poses)):
        _, oblob, level, _, _ = entries[levels[i]]
        blob = S.apply_moves(oblob, moves[i]) if moves[i] else oblob
        out[i] = O.seen_lines(level, O.seg_owned(blob, view, poses[i:i + 1]), words)[0]
    return out


def _batch(b2d, lset, form, which, w, h, n, seed):
    """(renderer, poses, per-frame kwargs of render_seen, levels, moves, entries) of one walk form"""
    from rust_doom_b200 import poses as P
    per_level = form in ("levels", "levels_states", "lights")
    entries = [lset[which], lset[1 - which]] if per_level else [lset[which]]
    view = b2d.make_view(w, h)
    r = (b2d.Renderer.from_levels([e[0] for e in entries], view, max_batch=n) if per_level
         else b2d.Renderer(entries[0][0], view, max_batch=n))
    rng = np.random.default_rng(seed)
    levels = [int(v) for v in rng.integers(0, len(entries), n)] if per_level else [0] * n
    poses = np.concatenate([P.random_poses(entries[lv][0], 1, seed + 7 * i) for i, lv in enumerate(levels)])
    moves = [[] for _ in range(n)]
    kw = {}
    if form in ("states", "levels_states", "lights"):
        moves = []
        for i, lv in enumerate(levels):
            _, _, level, dyn, doors = entries[lv]
            moves.append(_states(level, dyn, doors, 4, seed + i)[i % 4])
        kw["tics"] = [int(t) for t in rng.integers(0, 1 << 20, n)]
        kw["moves_per_pose"] = moves
    if per_level:
        kw["levels"] = levels
    if form == "lights":
        kw["lights"] = [((-1, 0, 32, 5)[i % 4], i % 3) for i in range(n)]
    return r, poses, kw, levels, moves, entries


def _plain_render(r, poses, kw):
    """the ordinary raster of a re-walk of the same batch (the one-call render of the same form)"""
    if "levels" in kw:
        if "tics" in kw:
            return r.render_levels_states(poses, kw["levels"], kw["tics"], kw["moves_per_pose"], lights=kw.get("lights"))
        return r.render_levels(poses, kw["levels"])
    if "tics" in kw:
        return r.render_states(poses, kw["tics"], kw["moves_per_pose"])
    return r.render(poses)


@pytest.mark.parametrize("w,h", [(320, 200), (1920, 1080)])
@pytest.mark.parametrize("which", [0, 1], ids=["doors", "masked"])
@pytest.mark.parametrize("form", FORMS)
def test_every_walk_form(b2d, lset, form, which, w, h):
    import torch
    n = 8 if w == 320 else 4
    r, poses, kw, levels, moves, entries = _batch(b2d, lset, form, which, w, h, n, 11 * FORMS.index(form) + which)
    words = r.seen_words
    assert words == O.words_for([e[2] for e in entries])
    idx, seen = r.render_seen(poses, **kw)
    torch.cuda.synchronize()
    assert r.status() == 0
    assert np.array_equal(idx.cpu().numpy(), _plain_render(r, poses, kw)), "index frames differ from the ordinary raster"
    got = seen.cpu().numpy().view(np.uint32)
    want = _oracle_rows(entries, render.make_view(w, h), poses, levels, moves, words)
    bad = [i for i in range(n) if not np.array_equal(got[i], want[i])]
    assert not bad, [(i, sorted(set(b2d.seen_lines(got[i])) ^ set(b2d.seen_lines(want[i])))) for i in bad[:4]]
    assert any(len(b2d.seen_lines(want[i])) > 0 for i in range(n))


def test_rows_are_or_ed_into(b2d, lset):
    """Rows pre-filled with a pattern keep it plus the frames' lines (bits past a level's line count included); the rows
    after the batch's are untouched."""
    import torch
    n = 6
    r, poses, kw, levels, moves, entries = _batch(b2d, lset, "levels", 0, 320, 200, n, 5)
    words = r.seen_words
    rng = np.random.default_rng(2)
    pattern = rng.integers(0, 1 << 32, (n + 3, words), dtype=np.uint64).astype(np.uint32)
    buf = torch.from_numpy(pattern.view(np.int32).copy()).cuda()
    _, back = r.render_seen(poses, seen=buf[:n], **kw)
    torch.cuda.synchronize()
    got = buf.cpu().numpy().view(np.uint32)
    want = _oracle_rows(entries, render.make_view(320, 200), poses, levels, moves, words)
    assert back.data_ptr() == buf.data_ptr()
    assert np.array_equal(got[:n], pattern[:n] | want)
    assert np.array_equal(got[n:], pattern[n:])


def test_agent_fly_through_accumulates(b2d, lset):
    """a 200-pose fly-through in batches of 32 into 32 persistent rows: their OR is the OR of the oracle's sets"""
    import torch
    from rust_doom_b200 import poses as P
    sc, oblob, level, _, _ = lset[1]
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=32)
    poses = P.flythrough_poses(sc, 200, 21)
    words = r.seen_words
    rows = torch.zeros((32, words), dtype=torch.int32, device="cuda")
    for i in range(0, 200, 32):
        k = min(32, 200 - i)
        r.render_seen(poses[i:i + k], seen=rows[:k])
    torch.cuda.synchronize()
    got = np.bitwise_or.reduce(rows.cpu().numpy().view(np.uint32), axis=0)
    want = np.bitwise_or.reduce(O.seen_lines(level, O.seg_owned(oblob, render.make_view(320, 200), poses), words), axis=0)
    assert np.array_equal(got, want)
    assert len(b2d.seen_lines(want)) > 10


def test_refusals_enqueue_nothing_and_a_seen_raster_is_one_launch(b2d, lset):
    import torch
    from rust_doom_b200 import B2dError
    sc = lset[0][0]
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=4)
    poses = sample_poses(b2d, sc, 4, 3)
    dp = torch.from_numpy(np.ascontiguousarray(poses).view(np.uint8).reshape(-1)).cuda()
    idx = torch.full((4, 200, 320), 0xEE, dtype=torch.uint8, device="cuda")
    seen = torch.zeros((4, r.seen_words), dtype=torch.int32, device="cuda")
    ticket = r.walk_device(dp.data_ptr(), 4)
    torch.cuda.synchronize()
    l0 = r.launch_count
    for args in ((ticket, idx.data_ptr(), 0), (ticket, 0, seen.data_ptr()), (ticket + 1, idx.data_ptr(), seen.data_ptr()),
                 (-1, idx.data_ptr(), seen.data_ptr())):
        with pytest.raises(B2dError):
            r.raster_device_seen(*args)
    torch.cuda.synchronize()
    assert r.launch_count == l0 and (idx.cpu().numpy() == 0xEE).all() and not seen.cpu().numpy().any()
    r.raster_device_seen(ticket, idx.data_ptr(), seen.data_ptr())
    torch.cuda.synchronize()
    assert r.launch_count == l0 + 1 and r.status() == 0
    with pytest.raises(B2dError):                                      # a ticket is rastered once
        r.raster_device_seen(ticket, idx.data_ptr(), seen.data_ptr())
    assert r.launch_count == l0 + 1
    assert np.array_equal(idx.cpu().numpy(), r.render(poses))


def test_first_call_on_a_held_stream_orders_later_calls(b2d, clock):
    """the first seen raster uploads the seg -> linedef tables on its own stream: it returns while that stream is held,
    and a seen raster on another stream right after it waits for the upload"""
    import torch
    from rust_doom_b200 import synthwad
    sc = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",))), 0)
    view = b2d.make_view(320, 200)
    poses = sample_poses(b2d, sc, 4, 9)
    dp = torch.from_numpy(np.ascontiguousarray(poses).view(np.uint8).reshape(-1)).cuda()
    a, b = (torch.empty((4, 200, 320), dtype=torch.uint8, device="cuda") for _ in range(2))
    sa, sb = (torch.zeros((4, 64), dtype=torch.int32, device="cuda") for _ in range(2))
    warm = b2d.Renderer(sc, view, max_batch=4)                          # the kernel's module loaded outside the hold
    warm.raster_device_seen(warm.walk_device(dp.data_ptr(), 4), a.data_ptr(), sa.data_ptr())
    r = b2d.Renderer(sc, view, max_batch=4)
    assert r.seen_words <= 64
    t1 = r.walk_device(dp.data_ptr(), 4)
    t2 = r.walk_device(dp.data_ptr(), 4)
    torch.cuda.synchronize()
    sa.zero_()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    hold = clock.hold(s1)
    r.raster_device_seen(t1, a.data_ptr(), sa.data_ptr(), s1.cuda_stream)
    pending(hold, "the first call")
    r.raster_device_seen(t2, b.data_ptr(), sb.data_ptr(), s2.cuda_stream)
    pending(hold, "a call on another stream")
    must_wait(mark(s2), hold, "the second call behind the first call's held upload")
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(sa, sb) and sa.any()


# ---- the seen automap (b2d_automap_seen_device) ----------------------------------------------------------------------
def _automap_items(entry):
    from oracle import automap as A
    from oracle import automap_seen as AS
    sc, _, level, _, _ = entry
    return A.lines(level), AS.dontdraw(level), A.things(sc.blob)


def _oracle_automap(items, poses, levels, w, h, scale, flags, mapped):
    from oracle import automap_seen as AS
    out = np.empty((len(poses), h, w), np.uint8)
    for i in range(len(poses)):
        table, hidden, things = items[levels[i]]
        out[i:i + 1] = AS.automap(table, hidden, things, w, h, poses[i:i + 1], scale, flags,
                                  None if mapped is None else mapped[i:i + 1])
    return out


@pytest.mark.parametrize("w,h", [(320, 200), (1920, 1080)])
@pytest.mark.parametrize("per_level", [False, True], ids=["one_level", "level_set"])
def test_seen_automap_every_flag(b2d, lset, w, h, per_level):
    import torch
    from tests.test_automap import random_poses
    entries = [lset[0], lset[1]] if per_level else [lset[1]]
    view = b2d.make_view(w, h)
    r = b2d.Renderer.from_levels([e[0] for e in entries], view, max_batch=4) if per_level else b2d.Renderer(entries[0][0], view, max_batch=4)
    items = [_automap_items(e) for e in entries]
    words = r.seen_words
    rng = np.random.default_rng(w + per_level)
    n = 3 if w == 320 else 2
    for flags in range(16):
        levels = [int(v) for v in rng.integers(0, len(entries), n)]
        poses = np.concatenate([random_poses(items[lv][0], 1, 31 * flags + i) for i, lv in enumerate(levels)])
        mapped = rng.integers(0, 1 << 32, (n, words), dtype=np.uint64).astype(np.uint32)
        seen = torch.from_numpy(mapped.view(np.int32).copy()).cuda()
        got = r.automap(poses, levels if per_level else None, 0.2, flags, seen=seen).cpu().numpy()
        want = _oracle_automap(items, poses, levels, w, h, 13107, flags, mapped)
        assert np.array_equal(got, want), (flags, np.argwhere(got != want)[:5])
        if flags < 8:                                      # d_seen NULL: b2d_automap_device's frames
            dp = torch.from_numpy(np.ascontiguousarray(poses).view(np.uint8).reshape(-1)).cuda()
            a, b = (torch.full((n, h, w), 0xEE, dtype=torch.uint8, device="cuda") for _ in range(2))
            lvs = levels if per_level else None
            r.automap_device(dp.data_ptr(), n, a.data_ptr(), 13107, flags, lvs)
            _lib_seen_automap(r, dp.data_ptr(), lvs, 0, n, flags, b.data_ptr())
            torch.cuda.synchronize()
            assert torch.equal(a, b)


def _lib_seen_automap(r, poses_ptr, levels, seen_ptr, n, flags, out_ptr, scale=13107):
    from rust_doom_b200 import _check, _levels_array, _lib
    lv = None if levels is None else _levels_array(levels, n)
    _check(_lib.load().b2d_automap_seen_device(r._h, poses_ptr, None if lv is None else lv.ctypes.data, seen_ptr or None, n,
                                               scale, flags, out_ptr, None))


def test_seen_automap_refusals(b2d, lset):
    import torch
    from rust_doom_b200 import B2dError
    r = b2d.Renderer(lset[0][0], b2d.make_view(320, 200), max_batch=4)
    poses = sample_poses(b2d, lset[0][0], 2, 4)
    dp = torch.from_numpy(np.ascontiguousarray(poses).view(np.uint8).reshape(-1)).cuda()
    out = torch.full((2, 200, 320), 0xEE, dtype=torch.uint8, device="cuda")
    seen = torch.zeros((2, r.seen_words + 1), dtype=torch.int32, device="cuda")
    l0 = r.launch_count
    for args in ((dp.data_ptr(), None, seen.data_ptr(), 2, 16, out.data_ptr()),
                 (dp.data_ptr(), None, seen.data_ptr() + 2, 2, 0, out.data_ptr()),
                 (dp.data_ptr(), [1, 0], seen.data_ptr(), 2, 8, out.data_ptr()),
                 (0, None, seen.data_ptr(), 2, 8, out.data_ptr()),
                 (dp.data_ptr(), None, seen.data_ptr(), 2, 8, 0)):
        with pytest.raises(B2dError):
            _lib_seen_automap(r, *args)
    with pytest.raises(B2dError):
        _lib_seen_automap(r, dp.data_ptr(), None, seen.data_ptr(), 2, 8, out.data_ptr(), scale=255)
    with pytest.raises(B2dError):                          # b2d_automap_device still refuses ALLMAP
        from rust_doom_b200 import _check, _lib
        _check(_lib.load().b2d_automap_device(r._h, dp.data_ptr(), None, 2, 13107, 8, out.data_ptr(), None))
    torch.cuda.synchronize()
    assert r.launch_count == l0 and (out.cpu().numpy() == 0xEE).all()


def test_fly_through_automap_shows_what_it_saw(b2d, lset):
    """the 200-pose fly-through's OR-ed row drawn by the seen automap equals the oracle automap with that row"""
    import torch
    from rust_doom_b200 import poses as P
    sc, oblob, level, _, _ = lset[1]
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=32)
    poses = P.flythrough_poses(sc, 200, 21)
    rows = torch.zeros((32, r.seen_words), dtype=torch.int32, device="cuda")
    for i in range(0, 200, 32):
        k = min(32, 200 - i)
        r.render_seen(poses[i:i + k], seen=rows[:k])
    row = np.bitwise_or.reduce(rows.cpu().numpy().view(np.uint32), axis=0)[None]
    items = [_automap_items(lset[1])]
    for flags in (0, 1, 8, 13):
        got = r.automap(poses[-1:], None, 0.2, flags, seen=torch.from_numpy(row.view(np.int32).copy()).cuda()).cpu().numpy()
        assert np.array_equal(got, _oracle_automap(items, poses[-1:], [0], 320, 200, 13107, flags, row)), flags


@pytest.mark.parametrize("which", ["python", "native"])
def test_clis_write_the_seen_automap(b2d, tmp_path, which):
    """--automap-flags seen,allmap with --levels: each level's automap of its first pose shows the lines all the run's frames
    of that level saw, and the unseen ones in grey"""
    import subprocess
    from oracle import automap as A
    from oracle import automap_seen as AS
    from oracle import resolve as R
    from oracle import wad as W
    from rust_doom_b200 import cli, synthwad
    from tests.test_cli import _b2d_binary
    data = synthwad.build_iwad(1, ("E1M1", "E1M2"))
    wad = tmp_path / "syn.wad"
    wad.write_bytes(data)
    dump = tmp_path / "d.ppm"
    per = 3
    args = ["-r", "160x100", "--levels", "0,1", "--poses", str(per), "--dump", str(dump), "--automap", "0.25",
            "--automap-flags", "seen,allmap"]
    arch = b2d.Archive.from_bytes(data)
    scenes = [b2d.Scene(arch, i) for i in (0, 1)]
    if which == "python":
        assert cli.main(["--iwad", str(wad)] + args) == 0
        poses = cli.level_set_job(b2d, scenes, per, 0)[0]
        assert cli.main(["--iwad", str(wad), "--dump", str(dump), "--automap", "0.2", "--automap-flags", "seen,bogus"]) == 2
    else:
        out = subprocess.run([_b2d_binary(), "-i", str(wad)] + args, capture_output=True, text=True)
        assert out.returncode == 0, out.stderr
        poses = np.concatenate([np.repeat(sc.start_pose, per) for sc in scenes])
        for k, sc in enumerate(scenes):
            for i in range(per):
                poses["angle"][k * per + i] = (int(sc.start_pose["angle"][0]) + ((i << 32) // per)) & 0xFFFFFFFF
        bad = subprocess.run([_b2d_binary(), "-i", str(wad), "--dump", str(dump), "--automap", "0.2", "--automap-flags", "seen,bogus"],
                             capture_output=True, text=True)
        assert bad.returncode == 2
    pal = W.TextureDirectory(W.Archive(data)).palettes[0]
    view = render.make_view(160, 100)
    for lvl in (0, 1):
        level, sc = W.Level(W.Archive(data), lvl), scenes[lvl]
        mine = poses[lvl * per:(lvl + 1) * per]
        row = np.bitwise_or.reduce(O.seen_lines(level, O.seg_owned(sc.blob, view, mine), O.words_for([level])), axis=0)
        words = max(O.words_for([W.Level(W.Archive(data), k)]) for k in (0, 1))
        row = np.concatenate([row, np.zeros(words - len(row), np.uint32)])[None]
        idx = AS.automap(A.lines(level), AS.dontdraw(level), A.things(sc.blob), 160, 100, mine[:1], 16384, AS.ALLMAP, row)
        assert (idx == AS.ALLMAP_COLOUR).any()
        want = R.resolve(idx, [pal], 1, "rgb")[0]
        assert (tmp_path / ("d.automap.%d.ppm" % lvl)).read_bytes() == cli.encode_ppm(want), lvl
