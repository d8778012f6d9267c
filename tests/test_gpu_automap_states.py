"""-m gpu: the state automap (b2d_automap_states_device, DESIGN.md C21) bit for bit against oracle/automap_states.py on a level with
doors, the content-rich level and a three-level set with per-frame levels, at 320x200, 1920x1080 and an odd size into an
unaligned output, for every flag, with a different random state per frame, random arrows and the seen rows that
b2d_raster_device_seen gives for the same poses and states; its identities with b2d_automap_seen_device and
b2d_automap_device; a shut door that changes a frame; refusals that enqueue nothing; its staging's stream order; and both
CLIs' --automap-flags others."""
import subprocess

import numpy as np
import pytest

from oracle import automap as A
from oracle import automap_states as AST
from oracle import resolve as R
from oracle import wad as W
from tests.test_automap import random_poses
from tests.test_automap_states import _random_arrows, oracle
from tests.test_gpu_resolve import clock, mark, must_wait, pending  # noqa: F401
from tests.test_gpu_states import _level, _states

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lset(b2d):
    """[(scene, oracle blob, oracle level, dynamic sectors, doors)]: generated levels with doors, the second with masked
    middles and sprites (the content-rich configuration), the third another seed"""
    return [_level(b2d, seed=1), _level(b2d, seed=3, mid_pct=30, thing_pct=40), _level(b2d, seed=5)]


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()


def _case(lset, entries, n, seed):
    """(levels, poses, moves, arrows) of n frames over `entries` (indices into lset)"""
    rng = np.random.default_rng(seed)
    levels = [int(v) for v in rng.integers(0, len(entries), n)]
    poses, moves, arrows = [], [], []
    for i, lv in enumerate(levels):
        _, _, level, dyn, doors = lset[entries[lv]]
        table = A.lines(level)
        poses.append(random_poses(table, 1, seed * 31 + i, margin=64))
        moves.append(_states(level, dyn, doors, 4, seed + i)[(seed + i) % 4])
        arrows.append(_random_arrows(rng, table, int(rng.integers(0, 9))))
    return levels, np.concatenate(poses), moves, arrows


def _oracle(lset, entries, levels, poses, w, h, scale, flags, mapped, moves, arrows):
    out = np.empty((len(poses), h, w), np.uint8)
    for i, lv in enumerate(levels):
        sc, _, level, _, _ = lset[entries[lv]]
        out[i:i + 1] = oracle(level, A.things(sc.blob), w, h, poses[i:i + 1], scale, flags,
                              None if mapped is None else mapped[i:i + 1], [moves[i]], [arrows[i]])
    return out


@pytest.mark.parametrize("w,h", [(320, 200), (1920, 1080), (333, 187)])
@pytest.mark.parametrize("entries", [(0,), (1,), (0, 1, 2)], ids=["doors", "rich", "level_set"])
def test_equals_the_oracle(b2d, lset, entries, w, h):
    import torch
    per_level = len(entries) > 1
    view = b2d.make_view(w, h)
    scenes = [lset[e][0] for e in entries]
    r = b2d.Renderer.from_levels(scenes, view, max_batch=4) if per_level else b2d.Renderer(scenes[0], view, max_batch=4)
    n = 3 if w * h < 10 ** 6 else 2
    unaligned = (w, h) == (333, 187)
    for flags in range(16):
        if w * h > 10 ** 6 and flags % 3:
            continue                                       # 1080p: flags 0, 3, 6, 9, 12, 15
        levels, poses, moves, arrows = _case(lset, entries, n, 7 * flags + w)
        lv = levels if per_level else None
        kw = {"tics": [0] * n, "moves_per_pose": moves}
        if per_level:
            kw["levels"] = levels
        seen = r.render_seen(poses, **kw)[1] if flags % 2 == 0 else None
        mapped = None if seen is None else seen.cpu().numpy().view(np.uint32)
        buf = torch.full((n * h * w + 8,), 0xEE, dtype=torch.uint8, device="cuda")
        off = 3 if unaligned else 0
        dp = _dev(poses)
        r.automap_device(dp.data_ptr(), n, buf.data_ptr() + off, 13107, flags, lv, 0, None if seen is None else seen.data_ptr(),
                         moves, arrows)
        torch.cuda.synchronize()
        got = buf.cpu().numpy()
        assert (got[:off] == 0xEE).all() and (got[off + n * h * w:] == 0xEE).all()
        got = got[off:off + n * h * w].reshape(n, h, w)
        want = _oracle(lset, entries, levels, poses, w, h, 13107, flags, mapped, moves, arrows)
        assert np.array_equal(got, want), (flags, np.argwhere(got != want)[:5])


def _lib_states(r, dp, n, out_ptr, flags, levels=None, states=None, moves=(), ranges=None, arrows=None, seen_ptr=0, scale=13107,
                n_moves=None, n_arrows=None, stream=0):
    """b2d_automap_states_device with ctypes arrays built here (each None for NULL)"""
    import ctypes
    from rust_doom_b200 import _levels_array, _lib
    lv = None if levels is None else _levels_array(levels, n)
    st = None
    if states is not None:
        st = (_lib.FrameState * max(len(states), 1))(*[_lib.FrameState(*s) for s in states])
    mv = (_lib.SectorMove * max(len(moves), 1))(*[_lib.SectorMove(*m) for m in moves]) if moves else None
    rg = None if ranges is None else (_lib.ArrowRange * max(len(ranges), 1))(*[_lib.ArrowRange(*g) for g in ranges])
    ar = arrows
    if isinstance(arrows, list):
        ar = (_lib.AutomapArrow * max(len(arrows), 1))(*[_lib.AutomapArrow(*a) for a in arrows])
    elif isinstance(arrows, np.ndarray):
        ar = ctypes.cast(arrows.ctypes.data, ctypes.POINTER(_lib.AutomapArrow))
    return _lib.load().b2d_automap_states_device(
        r._h, dp, None if lv is None else lv.ctypes.data, st, mv, len(moves) if n_moves is None else n_moves, rg, ar,
        (len(arrows) if arrows is not None else 0) if n_arrows is None else n_arrows, seen_ptr or None, n, scale, flags,
        out_ptr, stream or None)


@pytest.mark.parametrize("per_level", [False, True], ids=["one_level", "level_set"])
def test_identities(b2d, lset, per_level):
    """every frame at rest and no arrows: b2d_automap_seen_device's frames; with d_seen NULL and flags below ALLMAP,
    b2d_automap_device's"""
    import torch
    from rust_doom_b200 import _check, _levels_array, _lib
    entries = (0, 1, 2) if per_level else (1,)
    view = b2d.make_view(320, 200)
    scenes = [lset[e][0] for e in entries]
    r = b2d.Renderer.from_levels(scenes, view, max_batch=4) if per_level else b2d.Renderer(scenes[0], view, max_batch=4)
    n = 4
    for flags in range(16):
        levels, poses, _, _ = _case(lset, entries, n, 90 + flags)
        lv = levels if per_level else None
        dp = _dev(poses)
        rows = torch.from_numpy(np.random.default_rng(flags).integers(0, 1 << 32, (n, r.seen_words), dtype=np.uint64)
                                .astype(np.uint32).view(np.int32)).cuda()
        outs = [torch.full((n, 200, 320), 0xEE, dtype=torch.uint8, device="cuda") for _ in range(4)]
        lva = None if lv is None else _levels_array(lv, n)
        _check(_lib.load().b2d_automap_seen_device(r._h, dp.data_ptr(), None if lva is None else lva.ctypes.data, rows.data_ptr(),
                                                   n, 13107, flags, outs[0].data_ptr(), None))
        _check(_lib_states(r, dp.data_ptr(), n, outs[1].data_ptr(), flags, lv, seen_ptr=rows.data_ptr()))
        _check(_lib_states(r, dp.data_ptr(), n, outs[2].data_ptr(), flags, lv, [(5, 0, 0)] * n, [], [(0, 0)] * n, [],
                           seen_ptr=rows.data_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), flags
        if flags < 8:
            r.automap_device(dp.data_ptr(), n, outs[0].data_ptr(), 13107, flags, lv)
            _check(_lib_states(r, dp.data_ptr(), n, outs[3].data_ptr(), flags, lv))
            torch.cuda.synchronize()
            assert torch.equal(outs[0], outs[3]), flags


def test_an_open_door_changes_the_frame(b2d):
    """the door micro level (tests/test_scene.py): room A and a door B (ceiling 0, dynamic up to 128) share linedef 6.
    From A facing the door, raised by 72 the line is yellow as when shut; raised by 128 it is gone, so the frame differs
    from the rest state's; every frame equals the oracle's"""
    import torch
    from tests.test_scene import _micro_level
    data = _micro_level(two_sided_flags=0x0004, front=(0, 128), back=(0, 0))
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0, dynamic=[(1, 0, 0, 0, 128)])
    level = W.Level(W.Archive(data), 0)
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=4)
    poses = np.repeat(sc.start_pose, 3)
    poses["x"], poses["y"], poses["angle"] = -128 << 16, 128 << 16, 0
    dp = _dev(poses)
    moves = [[], [(1, 0, 72)], [(1, 0, 128)]]
    for flags in (0, A.ALL_LINES | A.THINGS):
        out = torch.empty((3, 200, 320), dtype=torch.uint8, device="cuda")
        r.automap_device(dp.data_ptr(), 3, out.data_ptr(), 1 << 16, flags, moves_per_pose=moves)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert np.array_equal(got, oracle(level, A.things(sc.blob), 320, 200, poses, 1 << 16, flags, None, moves)), flags
        assert np.array_equal(got[0], got[1]) and not np.array_equal(got[0], got[2]), flags
        assert (got[0] == 231).any() and not (got[2] == 231).any(), flags


def test_refusals_enqueue_nothing(b2d, lset):
    import torch
    from rust_doom_b200 import synthwad
    plain = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",))), 0)
    sc, _, level, dyn, _ = lset[0]
    r = b2d.Renderer.from_levels([sc, plain], b2d.make_view(320, 200), max_batch=4)
    poses = random_poses(A.lines(level), 2, 4)
    dp = _dev(poses).data_ptr()
    out = torch.full((2, 200, 320), 0xEE, dtype=torch.uint8, device="cuda")
    o = out.data_ptr()
    seen = torch.zeros((2, r.seen_words + 1), dtype=torch.int32, device="cuda")
    s0 = dyn[0][0]
    arrows = [(0, 0, 0, 112), (1 << 16, 0, 0, 96)]
    r.automap_device(dp, 2, o, 13107, 0, [0, 1], 0, None, [[], []], [[(0, 0, 0, 1)], []])      # tables and staging exist
    torch.cuda.synchronize()
    out.fill_(0xEE)
    torch.cuda.synchronize()
    l0 = r.launch_count
    ok = dict(levels=[0, 1], states=[(0, 0, 0), (0, 0, 0)], moves=[], ranges=[(0, 1), (1, 1)], arrows=arrows)
    cases = [
        dict(flags=16), dict(seen_ptr=seen.data_ptr() + 2), dict(scale=255), dict(scale=(64 << 16) + 1), dict(levels=[0, 2]),
        dict(dp=0), dict(out_ptr=0),
        dict(states=[(0, 0, 1), (0, 0, 0)]),                                     # a move range past n_moves
        dict(states=[(0, 0, 1), (0, 0, 0)], moves=[(s0, 0, 0)], n_moves=0),      # ... and the count it is checked against
        dict(states=[(0, 0, 1), (0, 0, 0)], moves=[(len(level.sectors) + 5, 0, 0)]),                 # an undeclared sector
        dict(states=[(0, 0, 1), (0, 0, 0)], moves=[(s0, 0, 100000)]),                                # outside its range
        dict(states=[(0, 0, 0), (0, 0, 1)], moves=[(s0, 0, 0)]),                 # moves on the level without dynamic sectors
        dict(states=[(0, 0, 1), (0, 0, 0)], moves=[(s0, 0, 0)], n_moves=1, moves_null=True),
        dict(ranges=[(0, 1), (1, 2)]),                                            # an arrow range past n_arrows
        dict(ranges=[(3, 0), (0, 1)]),
        dict(arrows=[(0, 0, 0, 0), (0, 0, 0, 96)]),                               # colour 0
        dict(arrows=[(0, 0, 0, 112), (0, 0, 0, 256)]),
        dict(arrows=None, n_arrows=2),
    ]
    from rust_doom_b200 import ERR_INVALID_ARG
    for c in cases:
        a = dict(ok)
        a.update(c)
        if a.pop("moves_null", False):
            a["moves"] = ()
        args = dict(levels=a["levels"], states=a["states"], moves=a["moves"], ranges=a["ranges"], arrows=a["arrows"],
                    seen_ptr=a.get("seen_ptr", 0), scale=a.get("scale", 13107), n_moves=a.get("n_moves"), n_arrows=a.get("n_arrows"))
        assert _lib_states(r, a.get("dp", dp), 2, a.get("out_ptr", o), a.get("flags", 0), **args) == ERR_INVALID_ARG, c
    torch.cuda.synchronize()
    assert r.launch_count == l0 and (out.cpu().numpy() == 0xEE).all()
    # a frame whose items reach 2^24: lines + 7 + 7 * arrows + 3 * things
    nl, nt = len(A.lines(level)), len(A.things(sc.blob))
    k = ((1 << 24) - nl - 7 - 3 * nt + 6) // 7
    many = np.zeros(k, np.dtype([("x", "<i4"), ("y", "<i4"), ("angle", "<u4"), ("colour", "<u4")]))
    many["x"], many["colour"] = 0x7FFF0000, 112                                  # off every frame
    assert _lib_states(r, dp, 2, o, 0, [0, 0], ranges=[(0, k), (0, 0)], arrows=many, n_arrows=k) == ERR_INVALID_ARG
    assert _lib_states(r, dp, 2, o, 0, [0, 0], ranges=[(0, k - 1), (0, 0)], arrows=many, n_arrows=k) == 0
    torch.cuda.synchronize()
    assert r.launch_count == l0 + 1
    out.fill_(0xEE)
    assert _lib_states(r, dp, 2, o, 0, **{key: ok[key] for key in ("levels", "states", "moves", "ranges", "arrows")}) == 0
    torch.cuda.synchronize()
    assert r.launch_count == l0 + 2 and not (out.cpu().numpy() == 0xEE).all()


def test_second_call_waits_for_the_first_calls_staging_copy(b2d, lset, clock):
    """the call's staging is rewritten only after the previous call's copy has read it; a call with no per-frame input
    stages nothing and does not wait; the frames are the oracle's"""
    import torch
    entries = (0, 1, 2)
    r = b2d.Renderer.from_levels([lset[e][0] for e in entries], b2d.make_view(320, 200), max_batch=4)
    la, pa, ma, aa = _case(lset, entries, 6, 41)
    lb, _, mb, ab = _case(lset, entries, 6, 42)
    dp = _dev(pa)
    a, b, c = (torch.empty((6, 200, 320), dtype=torch.uint8, device="cuda") for _ in range(3))
    r.automap_device(dp.data_ptr(), 6, a.data_ptr(), 13107, 7, la, 0, None, ma, aa)          # staging grown outside the hold
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    hold = clock.hold(s)
    r.automap_device(dp.data_ptr(), 6, a.data_ptr(), 13107, 7, la, s.cuda_stream, None, ma, aa)
    pending(hold, "first call")
    from rust_doom_b200 import _check
    _check(_lib_states(r, dp.data_ptr(), 6, c.data_ptr(), 5, stream=s.cuda_stream))
    pending(hold, "a call without per-frame inputs")
    r.automap_device(dp.data_ptr(), 6, b.data_ptr(), 13107, 7, lb, s.cuda_stream, None, mb, ab)
    assert hold.query(), "the second call rewrote the staging the first call's held copy reads"
    torch.cuda.synchronize()
    assert np.array_equal(a.cpu().numpy(), _oracle(lset, entries, la, pa, 320, 200, 13107, 7, None, ma, aa))
    assert np.array_equal(b.cpu().numpy(), _oracle(lset, entries, lb, pa, 320, 200, 13107, 7, None, mb, ab))


def test_first_call_on_a_held_stream_orders_later_calls(b2d, lset, clock):
    """the first automap call of a renderer uploads the tables (the state variant's included) on its own stream; a state
    automap on another stream right after it (one that stages nothing) waits for that upload"""
    import torch
    entries = (0, 1)
    levels, poses, moves, arrows = _case(lset, entries, 4, 77)
    dp = _dev(poses)
    a, b = (torch.full((4, 200, 320), 0xEE, dtype=torch.uint8, device="cuda") for _ in range(2))
    warm = b2d.Renderer(lset[2][0], b2d.make_view(320, 200), max_batch=4)
    warm.automap_device(dp.data_ptr(), 4, a.data_ptr(), 13107, 7, None, 0, None, [[]] * 4, [[]] * 4)   # the module loaded
    r = b2d.Renderer.from_levels([lset[e][0] for e in entries], b2d.make_view(320, 200), max_batch=4)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    hold = clock.hold(s1)
    r.automap_device(dp.data_ptr(), 4, a.data_ptr(), 13107, 7, levels, s1.cuda_stream)
    pending(hold, "the first call")
    from rust_doom_b200 import _check
    _check(_lib_states(r, dp.data_ptr(), 4, b.data_ptr(), 7, stream=s2.cuda_stream))          # stages nothing
    pending(hold, "a state call on another stream")
    must_wait(mark(s2), hold, "the state call behind the first call's held upload")
    torch.cuda.synchronize()
    rest = [[]] * 4, [[]] * 4
    assert np.array_equal(b.cpu().numpy(), _oracle(lset, entries, [0] * 4, poses, 320, 200, 13107, 7, None, *rest))


# ---- CLIs ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["python", "native"])
def test_clis_write_the_others_automap(b2d, tmp_path, which):
    """--automap-flags others with --levels: each level's automap of its first pose shows that pose's arrow in green 112
    and the next three poses' in 96, 64 and 176"""
    from rust_doom_b200 import cli, synthwad
    from tests.test_cli import _b2d_binary
    data = synthwad.build_iwad(1, ("E1M1", "E1M2"))
    wad = tmp_path / "syn.wad"
    wad.write_bytes(data)
    dump = tmp_path / "d.ppm"
    per = 4
    args = ["-r", "160x100", "--levels", "0,1", "--poses", str(per), "--dump", str(dump), "--automap", "1.0",
            "--automap-flags", "rotate,others"]
    arch = b2d.Archive.from_bytes(data)
    scenes = [b2d.Scene(arch, i) for i in (0, 1)]
    if which == "python":
        assert cli.main(["--iwad", str(wad)] + args) == 0
        poses = cli.level_set_job(b2d, scenes, per, 0)[0]
        assert cli.main(["--iwad", str(wad), "--dump", str(dump), "--automap", "0.2", "--automap-flags", "others,bogus"]) == 2
    else:
        out = subprocess.run([_b2d_binary(), "-i", str(wad)] + args, capture_output=True, text=True)
        assert out.returncode == 0, out.stderr
        poses = np.concatenate([np.repeat(sc.start_pose, per) for sc in scenes])
        for k, sc in enumerate(scenes):
            for i in range(per):
                poses["angle"][k * per + i] = (int(sc.start_pose["angle"][0]) + ((i << 32) // per)) & 0xFFFFFFFF
    pal = W.TextureDirectory(W.Archive(data)).palettes[0]
    for lvl in (0, 1):
        level, sc = W.Level(W.Archive(data), lvl), scenes[lvl]
        mine = poses[lvl * per:(lvl + 1) * per]
        arrows = [[(int(p["x"]), int(p["y"]), int(p["angle"]), c) for p, c in zip(mine, cli.OTHER_COLOURS)]]
        idx = AST.automap(A.lines(level), A.things(sc.blob), 160, 100, mine[:1], 65536, A.ROTATE, arrows)
        assert (idx == 96).any(), lvl                     # the second pose's arrow, a colour no line of the map has
        want = R.resolve(idx, [pal], 1, "rgb")[0]
        assert (tmp_path / ("d.automap.%d.ppm" % lvl)).read_bytes() == cli.encode_ppm(want), lvl
