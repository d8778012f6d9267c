"""Seen lines (DESIGN.md C20) on the CPU: the oracle's seen set (oracle/seen.py) by hand on the micro level with a door,
tied to the oracle rasteriser's own drawing on the generated levels at odd and extreme sizes, and the rows of linedef bits
it makes, with the Python helper that unpacks a row.  The product's rules on the CPU (tests/hostcheck/seen_lines.cpp): the
raster's strip clip loop with the marking against the oracle's rows on the generated levels and level-shape fixtures at odd
and extreme sizes, and the seen automap's tiles against oracle/automap_seen.py for every flag with random mapped rows; and
the --automap-flags names."""
import ctypes
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import render
from oracle import scene as S
from oracle import seen as O
from oracle import wad as W
from tests.test_automap import random_poses
from tests.test_scene import _micro_level

SIZES = [(320, 200), (333, 187), (1, 2), (1920, 1080), (4096, 24)]
SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostcheck", "seen_lines.cpp")


def _door():
    data = _micro_level(two_sided_flags=0x0004, front=(0, 128), back=(0, 0))
    a = W.Archive(data)
    return W.Level(a, 0), S.compile_scene(a, W.TextureDirectory(a), 0, dynamic=[(1, 0, 0, 0, 124)])


def _lines(level, blob, view, poses):
    rows = O.seen_lines(level, O.seg_owned(blob, view, poses), O.words_for([level]))
    return [np.flatnonzero(np.unpackbits(r.view(np.uint8), bitorder="little")).tolist() for r in rows]


def test_door_hides_room_b_until_it_opens():
    """Room A (x < 0): linedefs 0 west, 1 north, 2 south; room B (x > 0): 3 north, 4 east, 5 south; 6 the door between
    them.  From (-128, 128) facing east at 320x200 the view spans about +-51 degrees: A's north and south walls at the
    edges, the door in the middle, A's west wall behind.  Shut, the door closes every column it covers; raised by 72 its
    opening (72..0, the eye at 60) shows B's east wall and, at the door's edges, B's north and south walls."""
    level, blob = _door()
    v = render.make_view(320, 200)
    pose = render.make_pose(-128, 128, 60, 0)
    assert _lines(level, blob, v, pose) == [[1, 2, 6]]
    assert _lines(level, S.apply_moves(blob, [(1, 0, 72)]), v, pose) == [[1, 2, 3, 4, 5, 6]]
    # facing west: the west wall only (the view spans y = 128 +- 156 at x = -256, beyond the room's north and south walls
    # only at the edges)
    assert _lines(level, blob, v, render.make_pose(-128, 128, 60, 180)) == [[0, 1, 2]]


def _level_blob(data, lv=0):
    a = W.Archive(data)
    return W.Level(a, lv), S.compile_scene(a, W.TextureDirectory(a), lv)


@pytest.fixture(scope="module")
def levels():
    from rust_doom_b200 import synthwad
    from tests.test_lights import rich_wad
    return {"c2": _level_blob(synthwad.build_iwad(1, ("E1M1",))), "rich": _level_blob(rich_wad())}


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("which", ["c2", "rich"])
def test_seen_segs_cover_every_drawn_seg(levels, which, w, h):
    """Every seg the rasteriser draws a pixel for owns a column; a seg that owns a column is one the frame's walk reaches
    with the column's window open, so on a closed level at least one seg owns every column."""
    level, blob = levels[which]
    from oracle import automap as A
    poses = random_poses(A.lines(level), 3 if w * h < 10 ** 6 else 1, 2 * SIZES.index((w, h)) + (which == "rich"), margin=-64)
    poses["z"] = 41 << 16
    v = render.make_view(w, h)
    owned = O.seg_owned(blob, v, poses)
    _, hits = render.render(blob, v, poses, seg_hits=True)
    assert not ((hits > 0) & ~owned).any()
    assert owned.any(axis=1).all()


def test_rows_follow_the_segs_lump(levels):
    level, blob = levels["c2"]
    nseg, nline = len(level.segs), len(level.linedefs)
    owned = np.zeros((2, nseg), bool)
    owned[0, :] = True
    rows = O.seen_lines(level, owned, O.words_for([level]) + 1)
    want = np.zeros(nline, bool)
    want[np.asarray(level.segs["linedef"], np.int64)] = True
    got = np.unpackbits(rows[0].view(np.uint8), bitorder="little").astype(bool)
    assert np.array_equal(got[:nline], want) and not got[nline:].any()
    assert not rows[1].any()
    assert O.words_for([level]) == (nline + 31) // 32 and O.words_for([]) == 1


def test_python_helper_unpacks_a_row(b2d):
    row = np.zeros(3, np.uint32)
    for l in (0, 5, 31, 32, 95):
        row[l >> 5] |= np.uint32(1 << (l & 31))
    assert b2d.seen_lines(row).tolist() == [0, 5, 31, 32, 95]
    assert b2d.seen_lines(row.view(np.int32)).tolist() == [0, 5, 31, 32, 95]
    assert b2d.seen_lines(np.zeros(2, np.uint32)).tolist() == []


# ---- the product's marking and seen automap on the CPU (tests/hostcheck/seen_lines.cpp) --------------------------------
@functools.lru_cache(maxsize=None)
def mirror():
    """the kernels' algorithms, compiled into a temporary directory (the source tree may be read-only)"""
    out = os.path.join(tempfile.mkdtemp(prefix="b2d_seen_"), "libb2d_seen_lines.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out, SRC])
    return ctypes.CDLL(out)


def hostcheck_rows(b2d, blob, level, w, h, poses, words, moves=()):
    seg_line = np.array([int(l) if int(l) < len(level.linedefs) else -1 for l in level.segs["linedef"]], np.int32)
    rows = np.zeros((len(poses), words), np.uint32)
    mv = np.array(list(moves), np.int32).reshape(-1, 3) if moves else np.zeros((0, 3), np.int32)
    poses = np.ascontiguousarray(poses)
    rc = mirror().hostcheck_seen(ctypes.c_char_p(blob), ctypes.byref(b2d.make_view(w, h)), ctypes.c_void_p(poses.ctypes.data),
                                 len(poses), ctypes.c_void_p(seg_line.ctypes.data), words, ctypes.c_void_p(rows.ctypes.data),
                                 ctypes.c_void_p(mv.ctypes.data), len(mv))
    assert rc == 0
    return rows


def _shape_levels():
    from tests.test_level_shapes import hall_level, rotunda_level
    return {"rotundas": rotunda_level(), "hall": hall_level()}


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("which", ["c2", "rich", "rotundas", "hall"])
def test_hostcheck_rows_equal_the_oracle(b2d, levels, which, w, h):
    if which in levels:
        level, blob = levels[which]
        from oracle import automap as A
        poses = random_poses(A.lines(level), 4 if w * h < 10 ** 6 else 2, 3 * SIZES.index((w, h)) + len(which), margin=-64)
        poses["z"] = 41 << 16
    else:
        lv = _shape_levels()[which]
        level, blob = W.Level(W.Archive(lv.wad), 0), lv.blob
        poses = lv.pose_array()[:6 if w * h < 10 ** 6 else 2]
    words = O.words_for([level])
    want = O.seen_lines(level, O.seg_owned(blob, render.make_view(w, h), poses), words)
    got = hostcheck_rows(b2d, blob, level, w, h, poses, words)
    assert np.array_equal(got, want), [i for i in range(len(poses)) if not np.array_equal(got[i], want[i])]
    assert want.any()


def test_hostcheck_door_hides_room_b_until_it_opens(b2d):
    level, blob = _door()
    pose = render.make_pose(-128, 128, 60, 0)
    words = O.words_for([level])
    shut = hostcheck_rows(b2d, blob, level, 320, 200, pose, words)
    raised = hostcheck_rows(b2d, blob, level, 320, 200, pose, words, [(1, 0, 72)])
    assert b2d.seen_lines(shut[0]).tolist() == [1, 2, 6]
    assert b2d.seen_lines(raised[0]).tolist() == [1, 2, 3, 4, 5, 6]


def _patched_level():
    """the c2 WAD with teleporter, secret, don't-draw and out-of-range lines (tests/test_automap.py)"""
    from rust_doom_b200 import synthwad
    from tests.test_automap import patched_wad
    return patched_wad(synthwad.build_iwad(1, ("E1M1", "E1M2"))), 0


def hostcheck_automap_seen(table, hidden, things, w, h, poses, scale, flags, mapped, words):
    from tests.test_automap import table_array
    lines = table_array(table)
    lines["pad"] = [1 if hidden[t[6]] else 0 for t in table]           # the device copy's don't-draw bit
    th = np.ascontiguousarray(np.array(things, np.int32).reshape(-1, 2))
    poses = np.ascontiguousarray(poses)
    out = np.empty((len(poses), h, w), np.uint8)
    mp = None if mapped is None else np.ascontiguousarray(mapped, np.uint32)
    rc = mirror().hostcheck_automap_seen(ctypes.c_void_p(lines.ctypes.data), len(lines), ctypes.c_void_p(th.ctypes.data), len(th),
                                         ctypes.byref(render.make_view(w, h)), ctypes.c_void_p(poses.ctypes.data), len(poses),
                                         ctypes.c_int32(scale), flags, None if mp is None else ctypes.c_void_p(mp.ctypes.data),
                                         words, ctypes.c_void_p(out.ctypes.data))
    assert rc == 0
    return out


@pytest.mark.parametrize("w,h", [(320, 200), (333, 187), (1, 2), (4096, 24)])
def test_hostcheck_seen_automap_equals_the_oracle(b2d, w, h):
    from oracle import automap as A
    from oracle import automap_seen as AS
    data, lvi = _patched_level()
    level = W.Level(W.Archive(data), lvi)
    sc = b2d.Scene(b2d.Archive.from_bytes(data), lvi)
    table, things, hidden = A.lines(level), A.things(sc.blob), AS.dontdraw(level)
    assert any(hidden.values())
    words = O.words_for([level])
    rng = np.random.default_rng(w + h)
    for flags in range(16):
        poses = random_poses(table, 2, 7 * flags + w)
        mapped = rng.integers(0, 1 << 32, (2, words), dtype=np.uint64).astype(np.uint32)
        want = AS.automap(table, hidden, things, w, h, poses, 13107, flags, mapped)
        got = hostcheck_automap_seen(table, hidden, things, w, h, poses, 13107, flags, mapped, words)
        assert np.array_equal(got, want), (flags, np.argwhere(got != want)[:5])
        if flags < 8:                                      # every line mapped: the C19 frames
            ones = np.full((2, words), 0xFFFFFFFF, np.uint32)
            c19 = A.automap(table, things, w, h, poses, 13107, flags)
            assert np.array_equal(AS.automap(table, hidden, things, w, h, poses, 13107, flags, ones), c19)
            assert np.array_equal(hostcheck_automap_seen(table, hidden, things, w, h, poses, 13107, flags, None, words), c19)


def test_flag_parsing():
    import rust_doom_b200 as b2d
    from rust_doom_b200 import cli
    assert b2d.automap_flags("rotate,allmap") == 9 and b2d.automap_flags(["allmap"]) == b2d.AUTOMAP_ALLMAP
    assert cli.automap_flag_names("seen,allmap") == ("allmap", True)
    assert cli.automap_flag_names("rotate,things") == ("rotate,things", False)
    for bad in ("seen,bogus", "mapped", "all,seeen"):
        with pytest.raises(ValueError):
            cli.automap_flag_names(bad)
    with pytest.raises(ValueError):
        b2d.automap_flags("seen")                          # a CLI name: the library flag is the row itself
