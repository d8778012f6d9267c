"""-m gpu: the automap's grid and marks (b2d_automap_marks_device, DESIGN.md C22) bit for bit against
oracle/automap_marks.py on one level and on a three-level set whose levels have different grid origins (one set through
b2d_scene_set_automap_grid_origin) and digit sets (one level without digits), at 320x200 and 1920x1080, for every flag,
with and without marks, random states, arrows and seen rows; its identity with b2d_automap_states_device in frames and
launches; refusals that enqueue nothing, and the other automap calls' refusal of the grid flag; the table upload's
stream order; Renderer.automap's routing; and both CLIs' --automap-flags grid."""
import subprocess

import numpy as np
import pytest

from oracle import automap as A
from oracle import automap_marks as AM
from oracle import resolve as R
from oracle import wad as W
from tests.test_automap import random_poses
from tests.test_automap_marks import _random_marks, digit_images, digit_pwad, oracle
from tests.test_automap_states import _random_arrows
from tests.test_gpu_automap_states import _dev, _lib_states
from tests.test_gpu_resolve import clock, mark, must_wait, pending  # noqa: F401
from tests.test_gpu_states import _states
from tests.test_scene import declare_doors

pytestmark = pytest.mark.gpu


def _mlevel(b2d, seed, origin, digit_seed, set_origin=None, **cfg):
    """(scene, level, dynamic sectors, doors, grid origin, oracle digits): a generated level with doors whose BLOCKMAP
    header is `origin`, with the digits of digit_images(digit_seed) from a PWAD overlay (None: no digits); set_origin:
    the origin given to the scene afterwards instead"""
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(seed, ("E1M1",), cfg=synthwad.SynthConfig(anim=True, origin=origin, **cfg))
    overlays = () if digit_seed is None else (digit_pwad(digit_images(digit_seed)),)
    a = W.Archive(data, overlays=overlays)
    level = W.Level(a, 0)
    dyn, doors = declare_doors(level)
    sc = b2d.Scene(b2d.Archive.from_bytes(data, overlays=overlays), 0, dynamic=dyn)
    assert sc.automap_grid_origin == AM.grid_origin(a, 0) == tuple(origin)
    if set_origin is not None:
        sc.set_automap_grid_origin(*set_origin)
        origin = set_origin
    digits = AM.archive_digits(a)
    assert digits == [None] * 10 if digit_seed is None else all(d is not None for d in digits)
    return sc, level, dyn, doors, tuple(origin), digits


@pytest.fixture(scope="module")
def mset(b2d):
    return [_mlevel(b2d, 1, (-1280, -1152), 11), _mlevel(b2d, 3, (-512, 640), 12, mid_pct=30, thing_pct=40),
            _mlevel(b2d, 5, (1024, -2048), None, set_origin=(32767, -32767))]


def _case(mset, entries, n, seed, w, h, scale, with_marks=True):
    """(levels, poses, moves, arrows, marks) of n frames over `entries` (indices into mset)"""
    rng = np.random.default_rng(seed)
    levels = [int(v) for v in rng.integers(0, len(entries), n)]
    poses, moves, arrows, marks = [], [], [], []
    for i, lv in enumerate(levels):
        _, level, dyn, doors, _, _ = mset[entries[lv]]
        table = A.lines(level)
        p = random_poses(table, 1, seed * 31 + i, margin=64)
        poses.append(p)
        moves.append(_states(level, dyn, doors, 4, seed + i)[(seed + i) % 4])
        arrows.append(_random_arrows(rng, table, int(rng.integers(0, 5))))
        marks.append(_random_marks(rng, table, p[0], int(rng.integers(0, 13)), w, h, scale) if with_marks else None)
    return levels, np.concatenate(poses), moves, arrows, marks


def _oracle(mset, entries, levels, poses, w, h, scale, flags, mapped, moves, arrows, marks):
    out = np.empty((len(poses), h, w), np.uint8)
    for i, lv in enumerate(levels):
        sc, level, _, _, origin, digits = mset[entries[lv]]
        out[i:i + 1] = oracle(level, A.things(sc.blob), w, h, poses[i:i + 1], scale, flags,
                              None if mapped is None else mapped[i:i + 1], [moves[i]], [arrows[i]], origin, digits,
                              None if marks is None else [marks[i]])
    return out


def _renderer(b2d, mset, entries, w, h):
    view = b2d.make_view(w, h)
    scenes = [mset[e][0] for e in entries]
    return b2d.Renderer.from_levels(scenes, view, max_batch=4) if len(entries) > 1 else b2d.Renderer(scenes[0], view, max_batch=4)


@pytest.mark.parametrize("w,h", [(320, 200), (1920, 1080)])
@pytest.mark.parametrize("entries", [(0,), (0, 1, 2)], ids=["one_level", "level_set"])
def test_equals_the_oracle(b2d, mset, entries, w, h):
    import torch
    per_level = len(entries) > 1
    r = _renderer(b2d, mset, entries, w, h)
    n = 3 if w * h < 10 ** 6 else 1
    for flags in range(32):
        scale = (A.SCALE_MIN, 13107, 65536, 13107 * 3)[flags % 4]
        levels, poses, moves, arrows, marks = _case(mset, entries, n, 5 * flags + w, w, h, scale, with_marks=flags % 3 != 0)
        lv = levels if per_level else None
        kw = {"tics": [0] * n, "moves_per_pose": moves}
        if per_level:
            kw["levels"] = levels
        seen = r.render_seen(poses, **kw)[1] if flags % 2 == 0 else None
        mapped = None if seen is None else seen.cpu().numpy().view(np.uint32)
        buf = torch.full((n * h * w + 8,), 0xEE, dtype=torch.uint8, device="cuda")
        dp = _dev(poses)
        r.automap_marks_device(dp.data_ptr(), n, buf.data_ptr(), scale, flags, lv, 0, None if seen is None else seen.data_ptr(),
                               moves, arrows, None if flags % 3 == 0 else marks)
        torch.cuda.synchronize()
        got = buf.cpu().numpy()
        assert (got[n * h * w:] == 0xEE).all()
        got = got[:n * h * w].reshape(n, h, w)
        want = _oracle(mset, entries, levels, poses, w, h, scale, flags, mapped, moves, arrows, None if flags % 3 == 0 else marks)
        assert np.array_equal(got, want), (flags, np.argwhere(got != want)[:5])
        if flags & AM.GRID:
            assert (got == AM.GRID_COLOUR).any(), flags


def _lib_marks(r, dp, n, out_ptr, flags, levels=None, mark_ranges=None, marks=None, n_marks=None, stream=0, scale=13107):
    """b2d_automap_marks_device at rest, without arrows or seen rows, with ctypes arrays built here (each None for NULL)"""
    import ctypes
    from rust_doom_b200 import _levels_array, _lib
    lv = None if levels is None else _levels_array(levels, n)
    rg = None if mark_ranges is None else (_lib.ArrowRange * max(len(mark_ranges), 1))(*[_lib.ArrowRange(*g) for g in mark_ranges])
    mk = marks
    if isinstance(marks, list):
        mk = (_lib.AutomapMark * max(len(marks), 1))(*[_lib.AutomapMark(*m) for m in marks])
    elif isinstance(marks, np.ndarray):
        mk = ctypes.cast(marks.ctypes.data, ctypes.POINTER(_lib.AutomapMark))
    return _lib.load().b2d_automap_marks_device(
        r._h, dp, None if lv is None else lv.ctypes.data, None, None, 0, None, None, 0, None, n, scale, flags, out_ptr,
        stream or None, rg, mk, (len(marks) if marks is not None else 0) if n_marks is None else n_marks)


@pytest.mark.parametrize("entries", [(1,), (0, 1, 2)], ids=["one_level", "level_set"])
def test_without_grid_and_marks_the_states_call(b2d, mset, entries):
    """flags below GRID and no marks: b2d_automap_states_device's frames, in one launch each"""
    import torch
    r = _renderer(b2d, mset, entries, 320, 200)
    n = 4
    for flags in range(16):
        levels, poses, moves, arrows, _ = _case(mset, entries, n, 70 + flags, 320, 200, 13107)
        lv = levels if len(entries) > 1 else None
        dp = _dev(poses)
        a, b, c = (torch.full((n, 200, 320), 0xEE, dtype=torch.uint8, device="cuda") for _ in range(3))
        l0 = r.launch_count
        r.automap_device(dp.data_ptr(), n, a.data_ptr(), 13107, flags, lv, 0, None, moves, arrows)
        l1 = r.launch_count
        r.automap_marks_device(dp.data_ptr(), n, b.data_ptr(), 13107, flags, lv, 0, None, moves, arrows)
        l2 = r.launch_count
        r.automap_marks_device(dp.data_ptr(), n, c.data_ptr(), 13107, flags, lv, 0, None, moves, arrows, [[]] * n)
        torch.cuda.synchronize()
        assert torch.equal(a, b) and torch.equal(a, c), flags
        assert l1 - l0 == l2 - l1 == r.launch_count - l2 == 1


def test_refusals_enqueue_nothing(b2d, mset):
    import torch
    from rust_doom_b200 import ERR_INVALID_ARG, _check, _lib
    sc, level, _, _, _, _ = mset[0]
    r = b2d.Renderer.from_levels([sc, mset[2][0]], b2d.make_view(320, 200), max_batch=4)
    poses = random_poses(A.lines(level), 2, 4)
    dp = _dev(poses).data_ptr()
    out = torch.full((2, 200, 320), 0xEE, dtype=torch.uint8, device="cuda")
    o = out.data_ptr()
    _check(_lib_marks(r, dp, 2, o, AM.GRID, [0, 1], [(0, 1), (1, 1)], [(0, 0, 1), (0, 0, 2)]))     # tables and staging exist
    torch.cuda.synchronize()
    out.fill_(0xEE)
    torch.cuda.synchronize()
    l0 = r.launch_count
    ok = dict(levels=[0, 1], mark_ranges=[(0, 1), (1, 1)], marks=[(0, 0, 1), (0, 0, 2)])
    cases = [dict(flags=32), dict(flags=AM.GRID | 64), dict(scale=255), dict(levels=[0, 2]), dict(dp=0), dict(out_ptr=0),
             dict(marks=[(0, 0, 10), (0, 0, 2)]), dict(marks=[(0, 0, 1), (0, 0, 0xFFFFFFFF)]),
             dict(mark_ranges=[(0, 1), (1, 2)]), dict(mark_ranges=[(3, 0), (0, 1)]), dict(marks=None, n_marks=2)]
    for c in cases:
        a = dict(ok)
        a.update(c)
        assert _lib_marks(r, a.get("dp", dp), 2, a.get("out_ptr", o), a.get("flags", AM.GRID), a["levels"], a["mark_ranges"],
                          a["marks"], a.get("n_marks"), scale=a.get("scale", 13107)) == ERR_INVALID_ARG, c
    # every refusal of the states call (a bad arrow here) through the marks call
    arrow = (_lib.AutomapArrow * 1)(_lib.AutomapArrow(0, 0, 0, 0))
    rg = (_lib.ArrowRange * 2)(_lib.ArrowRange(0, 1), _lib.ArrowRange(0, 0))
    assert _lib.load().b2d_automap_marks_device(r._h, dp, None, None, None, 0, rg, arrow, 1, None, 2, 13107, AM.GRID, o, None,
                                                None, None, 0) == ERR_INVALID_ARG
    # the other automap calls refuse the grid flag
    for flags in (AM.GRID, AM.GRID | A.ROTATE):
        assert _lib.load().b2d_automap_device(r._h, dp, None, 2, 13107, flags, o, None) == ERR_INVALID_ARG
        assert _lib.load().b2d_automap_seen_device(r._h, dp, None, None, 2, 13107, flags, o, None) == ERR_INVALID_ARG
        assert _lib_states(r, dp, 2, o, flags) == ERR_INVALID_ARG
    with pytest.raises(b2d.B2dError):
        r.automap_device(dp, 2, o, 13107, AM.GRID)
    torch.cuda.synchronize()
    assert r.launch_count == l0 and (out.cpu().numpy() == 0xEE).all()
    # a frame whose items reach 2^24: lines + 7 + 7 * arrows + 3 * things + marks, the last 1 .. 7 of them marks
    import ctypes
    nl, nt = len(A.lines(level)), len(A.things(sc.blob))
    base = (1 << 24) - nl - 7 - 3 * nt
    ka = (base - 1) // 7
    km = base - 7 * ka
    many = np.zeros(ka, np.dtype([("x", "<i4"), ("y", "<i4"), ("angle", "<u4"), ("colour", "<u4")]))
    many["x"], many["colour"] = 0x7FFF0000, 112                                  # off every frame
    arrows = ctypes.cast(many.ctypes.data, ctypes.POINTER(_lib.AutomapArrow))
    rg = (_lib.ArrowRange * 2)(_lib.ArrowRange(0, ka), _lib.ArrowRange(0, 0))
    marks = (_lib.AutomapMark * km)(*[_lib.AutomapMark(0x7FFF0000, 0, 1)] * km)

    def reach(n_marks):
        mr = (_lib.ArrowRange * 2)(_lib.ArrowRange(0, n_marks), _lib.ArrowRange(0, 0))
        return _lib.load().b2d_automap_marks_device(r._h, dp, None, None, None, 0, rg, arrows, ka, None, 2, 13107, AM.GRID, o,
                                                    None, mr, marks, km)
    assert reach(km) == ERR_INVALID_ARG
    assert reach(km - 1) == 0
    torch.cuda.synchronize()
    assert r.launch_count == l0 + 1


def test_first_call_on_a_held_stream_orders_later_calls(b2d, mset, clock):
    """the first automap call of a renderer uploads the tables (the grid origins and digits included) on its own stream;
    a marks call on another stream right after it (one that stages nothing) waits for that upload"""
    import torch
    entries = (0, 1)
    levels, poses, moves, arrows, marks = _case(mset, entries, 4, 77, 320, 200, 13107)
    dp = _dev(poses)
    a, b, c = (torch.full((4, 200, 320), 0xEE, dtype=torch.uint8, device="cuda") for _ in range(3))
    warm = b2d.Renderer(mset[2][0], b2d.make_view(320, 200), max_batch=4)
    warm.automap_marks_device(dp.data_ptr(), 4, a.data_ptr(), 13107, 23, None, 0, None, None, None, [[]] * 4)   # module loaded
    for first in ("plain", "marks"):
        r = b2d.Renderer.from_levels([mset[e][0] for e in entries], b2d.make_view(320, 200), max_batch=4)
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        torch.cuda.synchronize()
        hold = clock.hold(s1)
        if first == "plain":
            r.automap_device(dp.data_ptr(), 4, a.data_ptr(), 13107, 7, levels, s1.cuda_stream)
        else:
            r.automap_marks_device(dp.data_ptr(), 4, c.data_ptr(), 13107, 23, levels, s1.cuda_stream, None, moves, arrows, marks)
        pending(hold, "the first call")
        from rust_doom_b200 import _check
        _check(_lib_marks(r, dp.data_ptr(), 4, b.data_ptr(), AM.GRID | 7, stream=s2.cuda_stream))          # stages nothing
        pending(hold, "a marks call on another stream")
        must_wait(mark(s2), hold, "the marks call behind the first call's held upload")
        torch.cuda.synchronize()
        rest = [[]] * 4, [[]] * 4, None
        assert np.array_equal(b.cpu().numpy(), _oracle(mset, entries, [0] * 4, poses, 320, 200, 13107, AM.GRID | 7, None, *rest))
        if first == "marks":
            assert np.array_equal(c.cpu().numpy(), _oracle(mset, entries, levels, poses, 320, 200, 13107, 23, None, moves, arrows,
                                                           marks))


def test_renderer_automap_routes_grid_and_marks(b2d, mset):
    """Renderer.automap with "grid" or marks calls b2d_automap_marks_device; without them it is the C21 call"""
    import torch
    r = _renderer(b2d, mset, (0,), 320, 200)
    levels, poses, moves, arrows, marks = _case(mset, (0,), 3, 5, 320, 200, 13107)
    for flags, mk in (("rotate,grid", None), ("things", marks), ("grid,all", marks), ("things", None)):
        got = r.automap(poses, None, 0.2, flags, None, moves, arrows, mk).cpu().numpy()
        bits = b2d.automap_flags(flags)
        assert np.array_equal(got, _oracle(mset, (0,), levels, poses, 320, 200, 13107, bits, None, moves, arrows, mk)), flags
    torch.cuda.synchronize()


# ---- CLIs ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["python", "native"])
def test_clis_write_the_grid_automap(b2d, tmp_path, which):
    """--automap-flags grid with --levels: each level's automap of its first pose shows the grid at the level's BLOCKMAP
    origin under the map"""
    from oracle import scene as S
    from rust_doom_b200 import cli, synthwad
    from tests.test_cli import _b2d_binary
    cfg = synthwad.SynthConfig(origin=(-1000, -900))
    data = synthwad.build_iwad(1, ("E1M1", "E1M2"), cfg)
    wad = tmp_path / "syn.wad"
    wad.write_bytes(data)
    dump = tmp_path / "d.ppm"
    per = 2
    args = ["-r", "160x100", "--levels", "0,1", "--poses", str(per), "--dump", str(dump), "--automap", "0.5",
            "--automap-flags", "rotate,grid"]
    arch = b2d.Archive.from_bytes(data)
    scenes = [b2d.Scene(arch, i) for i in (0, 1)]
    if which == "python":
        assert cli.main(["--iwad", str(wad)] + args) == 0
        poses = cli.level_set_job(b2d, scenes, per, 0)[0]
    else:
        out = subprocess.run([_b2d_binary(), "-i", str(wad)] + args, capture_output=True, text=True)
        assert out.returncode == 0, out.stderr
        poses = np.concatenate([np.repeat(sc.start_pose, per) for sc in scenes])
        for k, sc in enumerate(scenes):
            for i in range(per):
                poses["angle"][k * per + i] = (int(sc.start_pose["angle"][0]) + ((i << 32) // per)) & 0xFFFFFFFF
    a = W.Archive(data)
    pal = W.TextureDirectory(a).palettes[0]
    for lvl in (0, 1):
        level = W.Level(a, lvl)
        things = A.things(S.compile_scene(a, W.TextureDirectory(a), lvl))
        idx = AM.automap(A.lines(level), things, 160, 100, poses[lvl * per:lvl * per + 1], 32768, A.ROTATE | AM.GRID, None,
                         AM.grid_origin(a, lvl))
        assert (idx == AM.GRID_COLOUR).any(), lvl
        want = R.resolve(idx, [pal], 1, "rgb")[0]
        assert (tmp_path / ("d.automap.%d.ppm" % lvl)).read_bytes() == cli.encode_ppm(want), lvl
