"""The automap (DESIGN.md C19) without a GPU: b2d_scene_automap_lines against oracle/automap.py's table (generated levels,
a WAD whose LINEDEFS carry secret, don't-draw, teleporter and out-of-range entries, scenes from lumps), and the kernel's
tile algorithm on the CPU (tests/hostcheck/automap.cpp, the product's B2D_HD rule) against the oracle's frames bit for bit
at odd and extreme view sizes, every flag combination, the scale range's ends and coordinates at +-32767 map units."""
import ctypes
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import automap as A
from oracle import render
from oracle import wad as W
from tests.test_palettes import lump_scene

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostcheck", "automap.cpp")
LINE = np.dtype([("x0", "<i4"), ("y0", "<i4"), ("x1", "<i4"), ("y1", "<i4"), ("colour", "u1"), ("colour_all", "u1"),
                 ("pad", "<u2"), ("linedef", "<i4")])
POSE = render.POSE
SCALES = (A.SCALE_MIN, 13107, A.SCALE_MAX)


@functools.lru_cache(maxsize=None)
def mirror():
    """the kernel's algorithm, compiled into a temporary directory (the source tree may be read-only)"""
    out = os.path.join(tempfile.mkdtemp(prefix="b2d_automap_"), "libb2d_automap.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out, SRC])
    return ctypes.CDLL(out)


def table_array(table) -> np.ndarray:
    out = np.zeros(len(table), LINE)
    for i, t in enumerate(table):
        out[i] = (t[0], t[1], t[2], t[3], t[4], t[5], 0, t[6])
    return out


def hostcheck(table, things, w, h, poses, scale, flags) -> np.ndarray:
    lines = table_array(table)
    th = np.ascontiguousarray(np.array(things, np.int32).reshape(-1, 2))
    poses = np.ascontiguousarray(poses)
    view = render.make_view(w, h)
    out = np.empty((len(poses), h, w), np.uint8)
    rc = mirror().hostcheck_automap(ctypes.c_void_p(lines.ctypes.data), len(lines), ctypes.c_void_p(th.ctypes.data), len(th),
                                    ctypes.byref(view), ctypes.c_void_p(poses.ctypes.data), len(poses), ctypes.c_int32(scale),
                                    flags, ctypes.c_void_p(out.ctypes.data))
    assert rc == 0, "an item drew outside its tile"
    return out


def product_table(scene) -> list:
    return [tuple(int(r[k]) for k in ("x0", "y0", "x1", "y1", "colour", "colour_all", "linedef")) for r in scene.automap_lines()]


def random_poses(table, n, seed, margin=256):
    """poses anywhere in the table's bounding box and `margin` units around it, at full 16.16 and BAM resolution"""
    rng = np.random.default_rng(seed)
    xs = [t[0] for t in table] + [t[2] for t in table]
    ys = [t[1] for t in table] + [t[3] for t in table]
    out = np.zeros(n, POSE)
    out["x"] = rng.integers((min(xs) - margin) << 16, (max(xs) + margin) << 16, n)
    out["y"] = rng.integers((min(ys) - margin) << 16, (max(ys) + margin) << 16, n)
    out["angle"] = rng.integers(0, 1 << 32, n, dtype=np.uint64)
    return out


# ---- the line table ------------------------------------------------------------------------------------------------
def _find_lump(data: bytes, name: bytes, nth: int = 0):
    n, diro = np.frombuffer(data[4:12], "<i4")
    seen = 0
    for k in range(int(n)):
        pos, size = np.frombuffer(data[diro + 16 * k:diro + 16 * k + 8], "<i4")
        if data[diro + 16 * k + 8:diro + 16 * k + 16].rstrip(b"\0") == name:
            if seen == nth:
                return int(pos), int(size)
            seen += 1
    raise AssertionError("no %r lump" % name)


def patched_wad(data: bytes) -> bytes:
    """level 0's LINEDEFS with a teleporter, a secret and a don't-draw two-sided line, a secret teleporter, a don't-draw
    one-sided wall, out-of-range v1 / v2, out-of-range left and right sidedefs, and a left sidedef whose sector is out of
    range"""
    buf = bytearray(data)
    pos, size = _find_lump(data, b"LINEDEFS")
    ld = np.frombuffer(buf, W.LINEDEF, count=size // 14, offset=pos)
    two = [i for i in range(len(ld)) if ld[i]["left"] >= 0]
    one = [i for i in range(len(ld)) if ld[i]["left"] < 0]
    assert len(two) >= 8 and len(one) >= 3
    ld["special"][two[0]] = 39
    ld["flags"][two[1]] |= A.ML_SECRET
    ld["flags"][two[2]] |= A.ML_DONTDRAW
    ld["special"][two[3]] = 39
    ld["flags"][two[3]] |= A.ML_SECRET | A.ML_DONTDRAW
    ld["flags"][one[0]] |= A.ML_DONTDRAW
    ld["v1"][one[1]] = 0xFFFF
    ld["v2"][two[4]] = 0xFFF0
    ld["left"][two[5]] = 0x7FFF
    ld["right"][two[6]] = 0x7FFF
    spos, ssize = _find_lump(data, b"SIDEDEFS")
    sd = np.frombuffer(buf, W.SIDEDEF, count=ssize // 30, offset=spos)
    sd["sector"][int(ld["left"][two[7]])] = 0xFFFF
    return bytes(buf)


@pytest.fixture(scope="module")
def levels():
    """(name, wad bytes, level index): the c2 level, its second map, the content-rich level and the patched c2 level"""
    from rust_doom_b200 import synthwad
    from tests.test_lights import rich_wad
    c2 = synthwad.build_iwad(1, ("E1M1", "E1M2"))
    return [("c2", c2, 0), ("c2-E1M2", c2, 1), ("rich", rich_wad(), 0), ("patched", patched_wad(c2), 0)]


def test_line_table_matches_the_oracle(b2d, levels):
    for name, data, lv in levels:
        sc = b2d.Scene(b2d.Archive.from_bytes(data), lv)
        want = A.lines(W.Level(W.Archive(data), lv))
        assert product_table(sc) == want, name
        assert len(want) > 50, name


def test_line_table_covers_every_colour_rule(b2d, levels):
    name, data, lv = levels[3]
    level = W.Level(W.Archive(data), lv)
    table = product_table(b2d.Scene(b2d.Archive.from_bytes(data), lv))
    by_index = {t[6]: t for t in table}
    assert len(table) == len(level.linedefs) - 2                     # the two lines with an out-of-range vertex
    colours = {(t[4], t[5]) for t in table}
    for c in ((A.TELEPORT, A.TELEPORT), (A.WALL, A.WALL), (0, A.WALL), (A.FLOOR_STEP, A.FLOOR_STEP), (0, A.PLAIN), (0, A.TELEPORT)):
        assert c in colours, c
    ld = level.linedefs
    for i, t in by_index.items():
        if int(ld[i]["left"]) == 0x7FFF or int(ld[i]["right"]) == 0x7FFF:
            assert t[4:6] == (A.WALL, A.WALL), i                     # an out-of-range sidedef: a one-sided wall


def test_lump_scene_has_the_archive_scenes_table(b2d, levels):
    for name, data, lv in levels:
        assert product_table(lump_scene(b2d, data, lv)) == product_table(b2d.Scene(b2d.Archive.from_bytes(data), lv)), name


def test_automap_lines_capacity_is_checked(b2d, levels):
    import ctypes as C
    from rust_doom_b200 import _lib
    sc = b2d.Scene(b2d.Archive.from_bytes(levels[0][1]), 0)
    n = C.c_size_t()
    assert _lib.load().b2d_scene_automap_lines(sc._h, None, 0, C.byref(n)) == 0 and n.value > 0
    buf = (_lib.AutomapLine * n.value)()
    assert _lib.load().b2d_scene_automap_lines(sc._h, buf, n.value - 1, C.byref(n)) == b2d.ERR_INVALID_ARG
    assert _lib.load().b2d_scene_automap_lines(None, buf, n.value, C.byref(n)) == b2d.ERR_INVALID_ARG


# ---- the pixel rule ------------------------------------------------------------------------------------------------
def test_sincos_keeps_the_rotation_inside_int64():
    """C19's bound: |c| + |s| <= 1.4143 * 2^30 for every angle, so |dx c - dy s| < 2^63 for |dx|, |dy| <= 2^32 + 2^20"""
    rng = np.random.default_rng(3)
    angles = list(rng.integers(0, 1 << 32, 20000, dtype=np.uint64)) + [k << 29 for k in range(8)] + [(k << 29) + d for k in range(8) for d in (-1, 1)]
    worst = max(abs(c) + abs(s) for c, s in (render.sincos_q30(int(a) & 0xFFFFFFFF) for a in angles))
    assert worst <= 1.4143 * 2 ** 30
    assert worst * (2 ** 32 + 2 ** 20) < 2 ** 63


@pytest.mark.parametrize("w,h", [(320, 200), (333, 187), (1, 2), (4096, 24)])
def test_hostcheck_matches_the_oracle(b2d, levels, w, h):
    name, data, lv = levels[2]
    sc = b2d.Scene(b2d.Archive.from_bytes(data), lv)
    table, things = product_table(sc), A.things(sc.blob)
    assert things
    for flags in range(8):
        for k, scale in enumerate(SCALES):
            poses = random_poses(table, 2, 100 * flags + k)
            want = A.automap(table, things, w, h, poses, scale, flags)
            got = hostcheck(table, things, w, h, poses, scale, flags)
            assert np.array_equal(got, want), (w, h, flags, scale, np.argwhere(got != want)[:5])
            if w * h > 2:
                assert (want != 0).any()


def _extreme():
    """lines and things at the corners and edges of the map's range, poses at its far ends"""
    e = 32767
    pts = [(-e - 1, -e - 1), (e, e), (-e - 1, e), (e, -e - 1), (0, e), (e, 0), (-e - 1, 0), (0, -e - 1), (5, 7)]
    table = []
    for i, a in enumerate(pts):
        for b in pts[i + 1:]:
            table.append((a[0], a[1], b[0], b[1], 176, 176, len(table)))
    table.append((e, e, e, e, 64, 64, len(table)))                 # zero length
    things = [(e, e), (-e - 1, -e - 1), (e, -e - 1), (0, 0)]
    poses = np.zeros(8, POSE)
    poses["x"] = [2 ** 31 - 1, -2 ** 31, 2 ** 31 - 1, -2 ** 31, 0, 12345, 2 ** 31 - 1, -2 ** 31]
    poses["y"] = [2 ** 31 - 1, -2 ** 31, -2 ** 31, 2 ** 31 - 1, 0, -54321, 0, 0]
    poses["angle"] = [0x20000000, 0xA0000000, 0x60000000, 0xE0000000, 0x12345678, 0x40000000, 0x9ABCDEF0, 0xFFFFFFFF]
    return table, things, poses


@pytest.mark.parametrize("w,h", [(320, 200), (333, 187), (1, 2), (4096, 24)])
def test_hostcheck_matches_the_oracle_at_extreme_coordinates(w, h):
    table, things, poses = _extreme()
    for flags in range(8):
        for scale in SCALES + (A.SCALE_MAX - 1, 65536):
            want = A.automap(table, things, w, h, poses, scale, flags)
            got = hostcheck(table, things, w, h, poses, scale, flags)
            assert np.array_equal(got, want), (w, h, flags, scale, np.argwhere(got != want)[:5])


def test_pixel_rule_by_hand():
    """lines worked out by hand at 1 pixel per map unit on a 200 x 200 view centred on (0, 0): map point (x, y) sits at
    pixel coordinate (100 + x, 100 - y), and the arrow (within 21 units of the centre) stays clear of x >= 40"""
    p = np.zeros(1, POSE)

    def drawn(table):
        f = A.automap([(x0, y0, x1, y1, c, c, 0) for (x0, y0, x1, y1, c) in table], [], 200, 200, p, 65536, 0)[0]
        base = A.automap([], [], 200, 200, p, 65536, 0)[0]
        return {(int(y), int(x)): int(f[y, x]) for y, x in np.argwhere(f != base)}
    # x = 140 .. 144 at y = 100: pixel centres 140.5 .. 143.5 are inside, row 100
    assert drawn([(40, 0, 44, 0, 5)]) == {(100, c): 5 for c in range(140, 144)}
    # vertical, y = 102 .. 98 on column 142: centres 98.5 .. 101.5
    assert drawn([(42, -2, 42, 2, 7)]) == {(r, 142): 7 for r in range(98, 102)}
    # a point at (141, 99) has no pixel centre in its range: the pixel of its first endpoint
    assert drawn([(41, 1, 41, 1, 9)]) == {(99, 141): 9}
    # a diagonal from (140, 100) to (143, 98): X major, row floor(100 - (c - 140) * 2 / 3) at the centres c = 140.5 .. 142.5
    assert drawn([(40, 0, 43, 2, 3)]) == {(99, 140): 3, (99, 141): 3, (98, 142): 3}
    # later items win where they cross
    both = drawn([(40, 0, 44, 0, 5), (42, -2, 42, 2, 7)])
    assert both[(100, 142)] == 7 and both[(100, 141)] == 5 and len(both) == 7


def test_python_cli_refuses_automap_arguments(tmp_path, capsys):
    """scales outside 1/256 .. 64, unknown flags and --automap without --dump: usage errors before anything is rendered"""
    from rust_doom_b200 import cli
    dump = str(tmp_path / "d.ppm")
    for argv in (["--dump", dump, "--automap", "100"], ["--dump", dump, "--automap", "0.001"],
                 ["--dump", dump, "--automap", "0.2", "--automap-flags", "iddt"], ["--automap", "0.2"]):
        assert cli.main(argv) == 2, argv
        assert "--automap" in capsys.readouterr().err
    assert not os.path.exists(dump)
