"""The automap's grid and numbered marks (DESIGN.md C22) on the CPU: the grid origin of archive and lump scenes, the digit
patches' loaders, the oracle's grid, draw order, digit blits, fit rule and rotation by hand, and the kernel's tile code
(b2d_math.cuh automap_grid_range & co., run by tests/hostcheck/automap_marks.cpp) against oracle/automap_marks.py with
random states, seen rows, arrows and marks on the generated levels at odd and extreme sizes, every flag, both scale
limits, poses and grid origins at the map's edges; and the --automap-flags name `grid` in both CLIs."""
import ctypes
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import automap as A
from oracle import automap_marks as AM
from oracle import automap_seen as AS
from oracle import automap_states as AST
from oracle import render
from oracle import wad as W
from tests.test_automap import random_poses
from tests.test_automap_states import (ARROW, _c2, _levels, _random_arrows, device_tables, offsets, per_sector)

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostcheck", "automap_marks.cpp")
DIGIT = np.dtype([("px", "<u8"), ("w", "<i4"), ("h", "<i4"), ("left", "<i4"), ("top", "<i4")])
MARK = np.dtype([("x", "<i4"), ("y", "<i4"), ("number", "<u4")])
GRID = AM.GRID


@functools.lru_cache(maxsize=None)
def mirror():
    """the kernel's algorithm, compiled into a temporary directory (the source tree may be read-only)"""
    out = os.path.join(tempfile.mkdtemp(prefix="b2d_ammarks_"), "libb2d_automap_marks.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out, SRC])
    return ctypes.CDLL(out)


# ---- digit patches ---------------------------------------------------------------------------------------------------
def digit_images(seed: int):
    """ten small digit pictures as encode_picture takes them (-1: transparent), each with palette index 0 somewhere and
    a hole, and their (leftoffset, topoffset), some negative"""
    rng = np.random.default_rng(seed)
    out = []
    for d in range(10):
        w, h = 3 + d % 3, 5 + d % 2
        img = rng.integers(1, 256, (h, w)).astype(np.int16)
        img[rng.integers(0, h), rng.integers(0, w)] = 0
        img[(d + 1) % h, (d + 2) % w] = -1
        out.append((img, (d % 4) - 1, (d % 3) * 2 - 1))
    return out


def digit_pwad(images, names=None) -> bytes:
    from rust_doom_b200 import synthwad
    lumps = [(("AMMNUM%d" % d) if names is None else names[d], synthwad.encode_picture(img, xo, yo))
             for d, (img, xo, yo) in enumerate(images)]
    return synthwad.assemble_wad(lumps, ident=b"PWAD")


def digits_array(digits):
    """the AutomapDigit table of an oracle digit list (host texel pointers into the returned keep-alive list)"""
    arr, keep = np.zeros(10, DIGIT), []
    for d, dg in enumerate(digits or [None] * 10):
        if dg is None:
            continue
        px = np.ascontiguousarray(dg[0], np.uint16)
        keep.append(px)
        arr[d] = (px.ctypes.data, px.shape[1], px.shape[0], dg[1], dg[2])
    return arr, keep


# ---- the kernel's tiles and the oracle -------------------------------------------------------------------------------
def hostcheck(lines, dyn, things, w, h, poses, scale, flags, mapped=None, words=1, offs=None, arrows=None, origin=(0, 0),
              digits=None, marks=None, stats=None):
    n = len(poses)
    pool, off_at = [], np.full(max(n, 1), -1, np.int32)
    for f in range(n):
        if offs is not None and offs[f] is not None:
            off_at[f] = len(pool)
            pool += [int(v) for v in offs[f]]
    pool = np.array(pool + [0], np.int32)

    def flatten(per, dtype, conv):
        flat, ranges = [], np.zeros(2 * max(n, 1), np.uint32)
        for f in range(n):
            mine = [] if per is None or per[f] is None else list(per[f])
            ranges[2 * f], ranges[2 * f + 1] = len(flat), len(mine)
            flat += mine
        arr = np.zeros(max(len(flat), 1), dtype)
        for k, a in enumerate(flat):
            arr[k] = conv(a)
        return ranges, arr
    ranges, arr = flatten(arrows, ARROW, lambda a: (int(a[0]), int(a[1]), int(a[2]) & 0xFFFFFFFF, int(a[3])))
    mranges, marr = flatten(marks, MARK, lambda m: (int(m[0]), int(m[1]), int(m[2])))
    dig, keep = digits_array(digits)
    th = np.ascontiguousarray(np.array(things, np.int32).reshape(-1, 2))
    poses = np.ascontiguousarray(poses)
    out = np.empty((n, h, w), np.uint8)
    mp = None if mapped is None else np.ascontiguousarray(mapped, np.uint32)
    st = np.zeros(2, np.int64)
    rc = mirror().hostcheck_automap_marks(
        ctypes.c_void_p(lines.ctypes.data), len(lines), ctypes.c_void_p(dyn.ctypes.data), ctypes.c_void_p(th.ctypes.data),
        len(th), ctypes.byref(render.make_view(w, h)), ctypes.c_void_p(poses.ctypes.data), n, ctypes.c_int32(scale), flags,
        None if mp is None else ctypes.c_void_p(mp.ctypes.data), words, ctypes.c_void_p(pool.ctypes.data),
        ctypes.c_void_p(off_at.ctypes.data), ctypes.c_void_p(ranges.ctypes.data), ctypes.c_void_p(arr.ctypes.data),
        ctypes.c_int32(origin[0]), ctypes.c_int32(origin[1]), ctypes.c_void_p(dig.ctypes.data),
        None if marks is None else ctypes.c_void_p(mranges.ctypes.data), ctypes.c_void_p(marr.ctypes.data),
        ctypes.c_void_p(out.ctypes.data), ctypes.c_void_p(st.ctypes.data))
    assert rc == 0, rc
    del keep
    if stats is not None:
        stats += st
    return out


def oracle(level, things, w, h, poses, scale, flags, mapped=None, moves=None, arrows=None, origin=(0, 0), digits=None,
           marks=None):
    """oracle/automap_marks.py at each frame's moves, with the lines coloured by oracle/automap_seen.py's rule and the
    frame's row of seen lines"""
    hidden = AS.dontdraw(level)
    out = np.empty((len(poses), h, w), np.uint8)
    for f in range(len(poses)):
        m = [] if moves is None or moves[f] is None else moves[f]
        table = AST.lines(level, *per_sector(m))
        row = None if mapped is None else np.asarray(mapped[f], np.uint32)
        t = []
        for line in table:
            ld = line[6]
            c = AS.line_colour(line, hidden[ld], row is None or bool((int(row[ld >> 5]) >> (ld & 31)) & 1), flags)
            t.append(line[:4] + (c, c, ld))
        out[f:f + 1] = AM.automap(t, things, w, h, poses[f:f + 1], scale, flags & (A.ROTATE | A.THINGS | GRID),
                                  None if arrows is None else [arrows[f]], origin, digits,
                                  None if marks is None else [marks[f]])
    return out


def _empty_level():
    """the device tables of a level without lines or things: only the arrow and what a test adds is drawn"""
    from tests.test_automap import table_array
    level, _ = _c2()
    _, dyn, _ = device_tables(level, [])
    return table_array([(0, 0, 0, 0, 0, 0, 0)])[:0].copy(), dyn


def _both_empty(w, h, poses, scale, flags, origin=(0, 0)):
    """the oracle's and the tiles' frames of the empty level"""
    lines, dyn = _empty_level()
    return [AM.automap([], [], w, h, poses, scale, flags, None, origin),
            hostcheck(lines, dyn, [], w, h, poses, scale, flags, origin=origin)]


# ---- grid origin and digit loaders -----------------------------------------------------------------------------------
def _relumped(data: bytes, level: int, blockmap):
    """the WAD with level `level`'s lump at marker + 10 replaced by (name, bytes), or removed when blockmap is None"""
    from rust_doom_b200 import synthwad
    a = W.Archive(data)
    at = a.levels[level] + 10
    lumps = []
    for i, (name, _, _) in enumerate(a.lumps):
        if i == at:
            if blockmap is not None:
                lumps.append(blockmap)
            continue
        lumps.append((name.rstrip(b"\0").decode(), a.read(i)))
    return synthwad.assemble_wad(lumps)


def test_grid_origin_of_generated_levels(b2d):
    from rust_doom_b200 import synthwad
    for cfg in (synthwad.SynthConfig(), synthwad.SynthConfig(origin=(3000, -7))):
        data = synthwad.build_iwad(2, ("E1M1", "E1M2"), cfg)
        for lv in range(2):
            assert AM.grid_origin(W.Archive(data), lv) == tuple(cfg.origin)
            assert b2d.Scene(b2d.Archive.from_bytes(data), lv).automap_grid_origin == tuple(cfg.origin)


@pytest.mark.parametrize("blockmap", [None, ("BLOCKMAP", b"\x05\x00\x06\x00\x00\x00"), ("REJECTX", b"\x05\x00\x06\x00\0\0\0\0")])
def test_grid_origin_is_zero_without_a_blockmap_header(b2d, synth_wad, blockmap):
    """no lump at marker + 10, a 6-byte BLOCKMAP, an 8-byte lump of another name: (0, 0)"""
    data = _relumped(synth_wad, 0, blockmap)
    assert AM.grid_origin(W.Archive(data), 0) == (0, 0)
    assert b2d.Scene(b2d.Archive.from_bytes(data), 0).automap_grid_origin == (0, 0)
    ok = _relumped(synth_wad, 0, ("BLOCKMAP", b"\xfb\xff\x06\x80\0\0\0\0"))
    assert AM.grid_origin(W.Archive(ok), 0) == (-5, -32762)
    assert b2d.Scene(b2d.Archive.from_bytes(ok), 0).automap_grid_origin == (-5, -32762)


def test_grid_origin_of_a_lump_scene_and_the_setter(b2d, synth_wad):
    from tests.test_palettes import lump_scene
    sc = lump_scene(b2d, synth_wad)
    assert sc.automap_grid_origin == (0, 0)
    for xy in ((-1280, -1152), (2 ** 31 - 1, -2 ** 31), (0, 0)):
        sc.set_automap_grid_origin(*xy)
        assert sc.automap_grid_origin == xy
    with pytest.raises(ValueError):
        sc.set_automap_grid_origin(2 ** 31, 0)


def test_digits_load_from_an_overlay_and_from_textures(synth_wad):
    """a PWAD's AMMNUM lumps decode with their offsets; a second overlay's lump of the same name wins; a lump that is not
    a picture is a missing digit; a lump scene takes textures of those names at offsets 0"""
    images = digit_images(5)
    a = W.Archive(synth_wad)
    assert AM.archive_digits(a) == [None] * 10
    a = W.Archive(synth_wad, overlays=(digit_pwad(images),))
    got = AM.archive_digits(a)
    for d, (img, xo, yo) in enumerate(images):
        px, gx, gy = got[d]
        assert (gx, gy) == (xo, yo)
        assert np.array_equal(np.where(img < 0, -1, px.astype(np.int32)), img.astype(np.int32))
        assert ((px >> 8) != 0).sum() == (img < 0).sum()
    later = [(np.full((2, 2), 7, np.int16), 4, 4)] + images[1:]
    from rust_doom_b200 import synthwad
    broken = synthwad.assemble_wad([("AMMNUM9", b"\x01\x00")], ident=b"PWAD")
    got = AM.archive_digits(W.Archive(synth_wad, overlays=(digit_pwad(images), digit_pwad(later[:1]), broken)))
    assert got[0][1:] == (4, 4) and (got[0][0] == 7).all()
    assert got[9] is None and got[1][1:] == images[1][1:]
    tex = {b"AMMNUM3": np.full((5, 3), 9, np.uint16), b"OTHER": np.zeros((1, 1), np.uint16)}
    got = AM.image_digits(tex)
    assert got[3][1:] == (0, 0) and (got[3][0] == 9).all() and sum(g is not None for g in got) == 1


# ---- the oracle by hand ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("origin,cols,rows", [((-1280 + 37, -1152 + 5), (69, 197), (95,)),
                                              ((-300, -7), (116, 244), (107,)),
                                              ((32767, 32767), (31, 159, 287), (101,)),
                                              ((0, 0), (32, 160, 288), (100,))])
def test_grid_rows_and_columns(origin, cols, rows):
    """320x200 at one pixel per map unit, the pose at (0, 0): map x is column 160 + x, map y row 100 - y, so the lines
    x = ox + 128 j and y = oy + 128 j land on these columns and rows; every pixel off them and off the arrow is 0"""
    pose = np.zeros(1, render.POSE)
    want = np.zeros((200, 320), np.uint8)
    want[:, list(cols)] = AM.GRID_COLOUR
    want[list(rows), :] = AM.GRID_COLOUR
    for frame, plain in zip(_both_empty(320, 200, pose, 65536, GRID, origin), _both_empty(320, 200, pose, 65536, 0, origin)):
        arrow = frame[0] == A.ARROW
        assert arrow.any() and np.array_equal(np.where(arrow, want, frame[0]), want)
        assert np.array_equal(plain[0] == A.ARROW, arrow) and not plain[0][~arrow].any()


def test_lattice_spans_the_whole_map_range():
    assert AM.lattice(0) == (-256, 255)
    assert AM.lattice(-32768) == (0, 511) and AM.lattice(32767) == (-511, 0)
    assert AM.lattice(100) == (-256, 255) and AM.lattice(-100) == (-255, 256)


def test_a_linedef_is_drawn_over_the_grid():
    """a line along the grid column x = 0 from y = -50 to 50 covers that column's rows 50..149 (the pixel centres
    between Q8 rows 12800 and 38400) with its colour; the rest of the column is grid"""
    from tests.test_automap import table_array
    _, dyn = _empty_level()
    table = [(0, -50, 0, 50, 176, 176, 0)]
    lines = table_array(table)
    pose = np.zeros(1, render.POSE)
    pose["x"], pose["y"] = 40 << 16, 0                     # the arrow away from the column
    want_rows = np.arange(50, 150)
    got_o = AM.automap(table, [], 320, 200, pose, 65536, GRID)[0]
    got_h = hostcheck(lines, dyn[:1], [], 320, 200, pose, 65536, GRID)[0]
    for frame in (got_o, got_h):
        col = frame[:, 120]
        assert (col[want_rows] == 176).all() and (col[:50] == AM.GRID_COLOUR).all() and (col[150:] == AM.GRID_COLOUR).all()


def _mark_frames(w, h, flags, marks, images, table=None, pose=None):
    from tests.test_automap import table_array
    empty, dyn = _empty_level()
    table = table or []
    lines = table_array(table) if table else empty
    digits = [(np.where(img < 0, 0xFFFF, img).astype(np.uint16), xo, yo) for img, xo, yo in images]
    pose = np.zeros(1, render.POSE) if pose is None else pose
    return (AM.automap(table, [], w, h, pose, 65536, flags, None, (0, 0), digits, [marks])[0],
            hostcheck(lines, dyn[:max(len(table), 1)], [], w, h, pose, 65536, flags, digits=digits, marks=[marks])[0])


@pytest.mark.parametrize("w,h,k", [(320, 200, 1), (1920, 1080, 5)])
def test_digit_blit(w, h, k):
    """digit 4 (5 wide, 5 tall, offsets (-1, 1) from digit_images) at map (10, -20): pixel (W/2 + 10, H/2 + 20), top-left
    that minus k (left, top), each texel a k x k block; transparent texels keep the background"""
    images = digit_images(3)
    img, xo, yo = images[4]
    for frame in _mark_frames(w, h, 0, [(10 << 16, -20 << 16, 4)], images):
        left, top = w // 2 + 10 - k * xo, h // 2 + 20 - k * yo
        block = frame[top:top + k * img.shape[0], left:left + k * img.shape[1]]
        want = np.repeat(np.repeat(np.where(img < 0, 0, img), k, 0), k, 1).astype(np.uint8)
        assert np.array_equal(block, want)
        outside = frame.copy()
        outside[top:top + k * img.shape[0], left:left + k * img.shape[1]] = 0
        assert set(np.unique(outside)) <= {0, A.ARROW}


@pytest.mark.parametrize("edge", ["left", "right", "top", "bottom"])
def test_fit_rule_at_each_edge(edge):
    """a mark whose rectangle touches an edge of the 320x200 frame is drawn; one pixel further out it is not drawn at all"""
    images = [(np.full((6, 4), 50, np.int16), 0, 0)] * 10
    at = {"left": (-160, 0), "right": (320 - 4 - 160, 0), "top": (0, 100), "bottom": (0, 100 - 194)}[edge]
    out = {"left": (-1, 0), "right": (1, 0), "top": (0, 1), "bottom": (0, -1)}[edge]
    fits = [(at[0] << 16, at[1] << 16, 2)]
    beyond = [((at[0] + out[0]) << 16, (at[1] + out[1]) << 16, 2)]
    for frame in _mark_frames(320, 200, 0, fits, images):
        assert (frame == 50).sum() == 24
    for frame in _mark_frames(320, 200, 0, beyond, images):
        assert (frame == 50).sum() == 0


def test_rotated_mark_position_and_upright_patch():
    """ROTATE with the pose facing east turns map (40, 20) to screen offset (-20, 40): pixel (140, 60); the patch is not
    turned"""
    img = np.arange(1, 16, dtype=np.int16).reshape(5, 3)
    images = [(img, 0, 0)] * 10
    for frame in _mark_frames(320, 200, A.ROTATE, [(40 << 16, 20 << 16, 7)], images):
        assert np.array_equal(frame[60:65, 140:143], img.astype(np.uint8))


def test_index_zero_texel_covers_a_line():
    """a mark over a horizontal wall: its index-0 texel leaves 0 where the wall was, its transparent texel keeps the wall"""
    img = np.array([[0, -1, 9]], np.int16)
    images = [(img, 0, 0)] * 10
    table = [(-100, 30, 100, 30, 176, 176, 0)]             # row 70
    for frame in _mark_frames(320, 200, 0, [(-10 << 16, 30 << 16, 1)], images, table):
        assert list(frame[70, 150:153]) == [0, 176, 9] and frame[70, 149] == 176 and frame[70, 153] == 176


def test_marks_draw_in_list_order_past_ten():
    """eleven marks at one point: the last one's digit wins; the number only picks the digit"""
    images = [(np.full((2, 2), 10 + d, np.int16), 0, 0) for d in range(10)]
    marks = [(0, 0, d % 10) for d in range(11)]
    for frame in _mark_frames(320, 200, 0, marks, images):
        assert (frame[100:102, 160:162] == 10).all()


def test_without_grid_and_marks_the_states_oracle():
    level, blob = _c2()
    table, things = A.lines(level), A.things(blob)
    poses = random_poses(table, 2, 9)
    for flags in range(8):
        assert np.array_equal(AM.automap(table, things, 160, 100, poses, 13107, flags, origin=(5, 5), marks=[[], None]),
                              AST.automap(table, things, 160, 100, poses, 13107, flags))


# ---- the rule against the oracle -------------------------------------------------------------------------------------
def _digit_set(seed, missing=()):
    return [None if d in missing else (np.where(img < 0, 0xFFFF, img).astype(np.uint16), xo, yo)
            for d, (img, xo, yo) in enumerate(digit_images(seed))]


def _random_marks(rng, table, pose, n, w, h, scale):
    """n marks: most near the pose (on screen), some at far points and the map's corners"""
    out = []
    for _ in range(n):
        kind = rng.integers(0, 6)
        if kind == 0:
            x, y = int(rng.choice([-32767, 32767])) << 16, int(rng.choice([-32767, 32767])) << 16
        elif kind == 1:
            x, y = int(rng.integers(-2 ** 31, 2 ** 31)), int(rng.integers(-2 ** 31, 2 ** 31))
        else:                                              # within the frame's half-extent of the pose, and a bit past it
            rx, ry = (w * 2 ** 31) // scale + 65536, (h * 2 ** 31) // scale + 65536
            x = int(np.clip(int(pose["x"]) + int(rng.integers(-rx, rx + 1)), -2 ** 31, 2 ** 31 - 1))
            y = int(np.clip(int(pose["y"]) + int(rng.integers(-ry, ry + 1)), -2 ** 31, 2 ** 31 - 1))
        out.append((x, y, int(rng.integers(0, 10))))
    return out


@pytest.mark.parametrize("w,h", [(320, 200), (333, 187), (1, 2), (4096, 24), (1920, 1080)])
@pytest.mark.parametrize("which", ["c2", "rich", "dyn"])
def test_hostcheck_equals_the_oracle(which, w, h):
    from tests.refcheck import moves as MV
    level, blob, dynamic = _levels()[which]
    lines, dyn, slots = device_tables(level, dynamic)
    table, things = A.lines(level), A.things(blob)
    words = (len(level.linedefs) + 31) // 32
    rng = np.random.default_rng(w * 11 + h + len(which))
    digits = _digit_set(w + h, missing=(3,) if which == "rich" else ())
    n = 1 if w * h > 10 ** 6 else 2
    for flags in range(32):
        poses = random_poses(table, n, 17 * flags + w + h, margin=64)
        if flags % 8 == 5:
            poses["x"][0], poses["y"][0] = 32767 << 16, -(32767 << 16)
        scale = (A.SCALE_MIN, A.SCALE_MAX, 13107, 65536)[flags % 4] if flags % 16 >= 12 else 13107
        origin = [(-32767, 32767), (32767, -32767), (-1280, -1152), (37, -5)][flags % 4]
        moves = [MV.state(level, dynamic, 100 * flags + f, hole_free=False) if (flags + f) % 3 else [] for f in range(n)]
        offs = [offsets(slots, m) if m else None for m in moves]
        arrows = [_random_arrows(rng, table, int(rng.integers(0, 5))) for _ in range(n)]
        marks = [_random_marks(rng, table, poses[f], int(rng.integers(0, 13)), w, h, scale) for f in range(n)]
        mapped = rng.integers(0, 1 << 32, (n, words), dtype=np.uint64).astype(np.uint32) if flags % 2 == 0 else None
        want = oracle(level, things, w, h, poses, scale, flags, mapped, moves, arrows, origin, digits, marks)
        got = hostcheck(lines, dyn, things, w, h, poses, scale, flags, mapped, words, offs, arrows, origin, digits, marks)
        assert np.array_equal(got, want), (flags, np.argwhere(got != want)[:5])
        if flags < 16:                                     # no grid, no marks: the state automap's frames
            from tests.test_automap_states import hostcheck as states_hostcheck
            assert np.array_equal(hostcheck(lines, dyn, things, w, h, poses, scale, flags, mapped, words, offs, arrows, origin,
                                            digits),
                                  states_hostcheck(lines, dyn, things, w, h, poses, scale, flags, mapped, words, offs, arrows))


def test_grid_range_culls_most_lines_per_tile():
    """at 1920x1080, Doom's default scale, each tile draws a few grid lines instead of the lattice's 1024, north-up and
    rotated"""
    level, blob, _ = _levels()["c2"]
    lines, dyn, _ = device_tables(level, [])
    poses = random_poses(A.lines(level), 2, 4)
    for flags in (GRID, GRID | A.ROTATE):
        st = np.zeros(2, np.int64)
        hostcheck(lines, dyn, [], 1920, 1080, poses, 13107, flags, origin=(-1280, -1152), stats=st)
        tiles = 2 * 15 * 34
        assert st[1] == tiles * 1024 and st[0] < tiles * 8, st


@pytest.mark.parametrize("flags", [0, A.ROTATE])
@pytest.mark.parametrize("scale", [A.SCALE_MIN, 13107, A.SCALE_MAX])
def test_grid_range_holds_every_line_that_draws(flags, scale):
    """every lattice line that draws a pixel in a rectangle lies in the rectangle's range: checked per 16 x 8 rectangle
    of a 320 x 200 frame over random poses"""
    rng = np.random.default_rng(scale + flags)
    view = render.make_view(320, 200)
    for _ in range(3):
        pose = np.zeros(1, render.POSE)
        pose["x"], pose["y"] = int(rng.integers(-2 ** 31, 2 ** 31)), int(rng.integers(-2 ** 31, 2 ** 31))
        pose["angle"] = int(rng.integers(0, 2 ** 32))
        o = int(rng.integers(-32768, 32768))
        px, py, angle = int(pose["x"][0]), int(pose["y"][0]), int(pose["angle"][0])
        c, s = render.sincos_q30((0x40000000 - angle) & 0xFFFFFFFF)
        jlo, jhi = AM.lattice(o)
        hits = {}
        for j in range(jlo, jhi + 1):
            at = (o + 128 * j) << 16
            P = A._screen(at - px, (-32768 << 16) - py, bool(flags), c, s, scale, 320, 200)
            Q = A._screen(at - px, (32767 << 16) - py, bool(flags), c, s, scale, 320, 200)
            for (x, y) in AM._frame_line_pixels(P[0], P[1], Q[0], Q[1], 320, 200):
                hits.setdefault((x // 16, y // 8), set()).add(j)
        out = np.zeros(2, np.int64)
        for (bx, by), js in hits.items():
            mirror().hostcheck_grid_range(ctypes.byref(view), ctypes.c_void_p(pose.ctypes.data), ctypes.c_int32(scale), flags,
                                          ctypes.c_int32(o), 1, 16 * bx, 8 * by, 16 * bx + 16, 8 * by + 8,
                                          ctypes.c_void_p(out.ctypes.data))
            assert out[0] <= min(js) and max(js) <= out[1], (bx, by, js, out)


# ---- the CLIs' flag name ---------------------------------------------------------------------------------------------
def test_flag_parsing():
    import rust_doom_b200 as b2d
    from rust_doom_b200 import cli
    assert b2d.automap_flags("grid") == 16 and b2d.automap_flags("rotate,grid") == 17
    assert cli.automap_flag_options("grid,seen,others") == ("grid", True, True)
    with pytest.raises(ValueError):
        cli.automap_flag_options("grids")


def test_compiled_cli_parses_grid(tmp_path):
    """the compiled CLI takes `grid` and refuses a misspelling as a usage error, before it opens any device"""
    from rust_doom_b200 import synthwad
    from tests.test_cli import _b2d_binary
    wad = tmp_path / "syn.wad"
    wad.write_bytes(synthwad.build_iwad(1, ("E1M1",)))
    bad = subprocess.run([_b2d_binary(), "-i", str(wad), "--dump", str(tmp_path / "d.ppm"), "--automap", "0.2",
                          "--automap-flags", "grid,bogus"], capture_output=True, text=True)
    assert bad.returncode == 2 and "grid" in bad.stderr
    assert not (tmp_path / "d.ppm").exists()
