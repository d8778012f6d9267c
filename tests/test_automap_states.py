"""The state automap (DESIGN.md C21) on the CPU: line colours at a frame's sector heights by hand on the micro level with a
door and with a lift step, lines that never change, the oracle at rest, other players' arrows by hand, and the kernel's
rule (b2d_math.cuh automap_state_item, run by tests/hostcheck/automap_states.cpp) against oracle/automap_states.py with random
states, seen rows and arrows on the generated levels at odd and extreme sizes, every flag and both scale limits; and the
--automap-flags name `others` in both CLIs."""
import ctypes
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import automap as A
from oracle import automap_seen as AS
from oracle import automap_states as AST
from oracle import render
from oracle import scene as S
from oracle import wad as W
from tests.test_automap import random_poses, table_array
from tests.test_scene import _micro_level

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostcheck", "automap_states.cpp")
DYN = np.dtype([("floor", "<i4", 2), ("ceil", "<i4", 2), ("slot", "<u4", 2)])
ARROW = np.dtype([("x", "<i4"), ("y", "<i4"), ("angle", "<u4"), ("colour", "<u4")])
NO_SLOT, DONTDRAW, CHANGEABLE = 0xFFFFFFFF, 1, 2


@functools.lru_cache(maxsize=None)
def mirror():
    """the kernel's algorithm, compiled into a temporary directory (the source tree may be read-only)"""
    out = os.path.join(tempfile.mkdtemp(prefix="b2d_amstates_"), "libb2d_automap_states.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out, SRC])
    return ctypes.CDLL(out)


# ---- the device tables, restated -------------------------------------------------------------------------------------
def device_tables(level, dynamic):
    """(lines, dyn, slots): the device copy of the rest table (the don't-draw and changeable bits), one AutomapDynLine per
    line, and {sector: dynamic slot} in the order of `dynamic` (a list of (sector, fmin, fmax, cmin, cmax))"""
    slots = {}
    for d in dynamic:
        slots.setdefault(int(d[0]), len(slots))
    table = A.lines(level)
    lines = table_array(table)
    dyn = np.zeros(max(len(table), 1), DYN)
    ns, nsec = len(level.sidedefs), len(level.sectors)

    def sector(side):
        if not 0 <= side < ns:
            return None
        sec = int(level.sidedefs[side]["sector"])
        return sec if sec < nsec else None
    for i, t in enumerate(table):
        ld = level.linedefs[t[6]]
        bits = DONTDRAW if int(ld["flags"]) & A.ML_DONTDRAW else 0
        front, back = sector(int(ld["right"])), sector(int(ld["left"]))
        if (front is not None and back is not None and int(ld["special"]) != 39 and not int(ld["flags"]) & A.ML_SECRET
                and (front in slots or back in slots)):
            bits |= CHANGEABLE
            dyn[i] = ((int(level.sectors[front]["floor"]), int(level.sectors[back]["floor"])),
                      (int(level.sectors[front]["ceil"]), int(level.sectors[back]["ceil"])),
                      (slots.get(front, NO_SLOT), slots.get(back, NO_SLOT)))
        lines["pad"][i] = bits
    return lines, dyn, slots


def offsets(slots, moves):
    """the compact offsets of a move list: floor, ceiling per dynamic slot"""
    off = np.zeros(2 * max(len(slots), 1), np.int32)
    for (s, fo, co) in moves:
        off[2 * slots[int(s)]], off[2 * slots[int(s)] + 1] = fo, co
    return off


def per_sector(moves):
    return {int(m[0]): int(m[1]) for m in moves}, {int(m[0]): int(m[2]) for m in moves}


def state_colours(lines, dyn, i, off):
    out = (ctypes.c_uint8 * 2)()
    mirror().hostcheck_state_colours(ctypes.c_void_p(lines[i:i + 1].ctypes.data), ctypes.c_void_p(dyn[i:i + 1].ctypes.data),
                                     ctypes.c_void_p(off.ctypes.data), out)
    return out[0], out[1]


# ---- line colours by hand --------------------------------------------------------------------------------------------
def _micro(front, back, dynamic):
    a = W.Archive(_micro_level(two_sided_flags=0x0004, front=front, back=back))
    return W.Level(a, 0), dynamic


def test_door_line_follows_the_door():
    """Room A (sector 0, floor 0, ceiling 128) and a door B (sector 1, ceiling 0, dynamic 0..128) share linedef 6: yellow
    231 while shut and while partly raised; fully raised the two ceilings meet, so it is not drawn normally and is grey 96
    under ALL_LINES."""
    level, dynamic = _micro((0, 128), (0, 0), [(1, 0, 0, 0, 128)])
    lines, dyn, slots = device_tables(level, dynamic)
    assert lines["pad"][6] == CHANGEABLE and not (lines["pad"][:6] & CHANGEABLE).any()
    for raise_by, want in ((0, (231, 231)), (72, (231, 231)), (127, (231, 231)), (128, (0, 96))):
        moves = [(1, 0, raise_by)]
        assert AST.lines(level, *per_sector(moves))[6][4:6] == want, raise_by
        assert state_colours(lines, dyn, 6, offsets(slots, moves)) == want, raise_by
    assert A.lines(level)[6][4:6] == (231, 231)


def test_floor_move_makes_a_step_line_appear_and_disappear():
    """A lift: B's floor (dynamic, heights 0..48) moved off A's height 24 shows the brown 64 step; back at 24 it is gone."""
    level, dynamic = _micro((24, 128), (24, 128), [(1, 0, 48, 128, 128)])
    lines, dyn, slots = device_tables(level, dynamic)
    for fo, want in ((0, (0, 96)), (-24, (64, 64)), (16, (64, 64)), (0, (0, 96))):
        moves = [(1, fo, 0)]
        assert AST.lines(level, *per_sector(moves))[6][4:6] == want, fo
        assert state_colours(lines, dyn, 6, offsets(slots, moves)) == want, fo


def _patched():
    from rust_doom_b200 import synthwad
    from tests.test_automap import patched_wad
    data = patched_wad(synthwad.build_iwad(1, ("E1M1", "E1M2")))
    return data, W.Level(W.Archive(data), 0)


def test_lines_that_never_change():
    """Teleporters, secret lines and one-sided walls keep their colours whatever the sectors do, and don't-draw lines stay
    undrawn normally, with every sector of the level dynamic and moved."""
    from tests.refcheck import moves as MV
    data, level = _patched()
    dynamic = MV.declare(level, 3, len(level.sectors))
    lines, dyn, slots = device_tables(level, dynamic)
    rest = A.lines(level)
    fixed = [i for i, t in enumerate(rest)
             if int(level.linedefs[t[6]]["special"]) == 39 or int(level.linedefs[t[6]]["flags"]) & A.ML_SECRET
             or int(level.linedefs[t[6]]["left"]) < 0 or int(level.linedefs[t[6]]["left"]) >= len(level.sidedefs)]
    hidden = [i for i, t in enumerate(rest) if int(level.linedefs[t[6]]["flags"]) & A.ML_DONTDRAW]
    assert len(fixed) >= 5 and hidden
    assert not (lines["pad"][fixed] & CHANGEABLE).any()
    changed = 0
    for seed in range(6):
        moves = MV.state(level, dynamic, seed, hole_free=False)
        at = AST.lines(level, *per_sector(moves))
        off = offsets(slots, moves)
        for i in fixed:
            assert at[i] == rest[i] and state_colours(lines, dyn, i, off) == rest[i][4:6]
        for i in hidden:
            assert at[i][4] == 0 and state_colours(lines, dyn, i, off)[0] == 0
        for i in range(len(rest)):
            assert state_colours(lines, dyn, i, off) == at[i][4:6], (seed, i)
        changed += sum(at[i][4:6] != rest[i][4:6] for i in range(len(rest)))
    assert changed > 0


def test_oracle_at_rest_is_the_rest_table():
    """without offsets and arrows, oracle/automap_states.py gives oracle/automap.py's table and frames"""
    from rust_doom_b200 import synthwad
    for data in (synthwad.build_iwad(1, ("E1M1",)), _patched()[0]):
        a = W.Archive(data)
        level = W.Level(a, 0)
        assert AST.lines(level) == A.lines(level)
        assert AST.lines(level, {}, {}) == A.lines(level)
        zeros = [0] * len(level.sectors)
        assert AST.lines(level, zeros, zeros) == A.lines(level)
        table, things = A.lines(level), A.things(S.compile_scene(a, W.TextureDirectory(a), 0))
        for flags in range(8):
            poses = random_poses(table, 2, 50 + flags)
            want = A.automap(table, things, 160, 100, poses, 13107, flags)
            assert np.array_equal(AST.automap(table, things, 160, 100, poses, 13107, flags), want)
            assert np.array_equal(AST.automap(table, things, 160, 100, poses, 13107, flags, [[], None]), want)


# ---- arrows by hand --------------------------------------------------------------------------------------------------
def hostcheck(lines, dyn, things, w, h, poses, scale, flags, mapped=None, words=1, offs=None, arrows=None):
    """the tile algorithm over one level: offs[f] (compact offsets or None) and arrows[f] (list of (x, y, angle, colour))"""
    n = len(poses)
    pool, off_at = [], np.full(max(n, 1), -1, np.int32)
    for f in range(n):
        if offs is not None and offs[f] is not None:
            off_at[f] = len(pool)
            pool += [int(v) for v in offs[f]]
    pool = np.array(pool + [0], np.int32)
    flat, ranges = [], np.zeros(2 * max(n, 1), np.uint32)
    for f in range(n):
        mine = [] if arrows is None else list(arrows[f])
        ranges[2 * f], ranges[2 * f + 1] = len(flat), len(mine)
        flat += mine
    arr = np.zeros(max(len(flat), 1), ARROW)
    for k, a in enumerate(flat):
        arr[k] = (int(a[0]), int(a[1]), int(a[2]) & 0xFFFFFFFF, int(a[3]))
    th = np.ascontiguousarray(np.array(things, np.int32).reshape(-1, 2))
    poses = np.ascontiguousarray(poses)
    out = np.empty((n, h, w), np.uint8)
    mp = None if mapped is None else np.ascontiguousarray(mapped, np.uint32)
    rc = mirror().hostcheck_automap_states(
        ctypes.c_void_p(lines.ctypes.data), len(lines), ctypes.c_void_p(dyn.ctypes.data), ctypes.c_void_p(th.ctypes.data),
        len(th), ctypes.byref(render.make_view(w, h)), ctypes.c_void_p(poses.ctypes.data), n, ctypes.c_int32(scale), flags,
        None if mp is None else ctypes.c_void_p(mp.ctypes.data), words, ctypes.c_void_p(pool.ctypes.data),
        ctypes.c_void_p(off_at.ctypes.data), ctypes.c_void_p(ranges.ctypes.data), ctypes.c_void_p(arr.ctypes.data),
        ctypes.c_void_p(out.ctypes.data))
    assert rc == 0, rc
    return out


def oracle(level, things, w, h, poses, scale, flags, mapped=None, moves=None, arrows=None):
    """oracle/automap_states.py at each frame's moves, through oracle/automap_seen.py's colour rule with its row of seen
    lines"""
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
        out[f:f + 1] = AST.automap(t, things, w, h, poses[f:f + 1], scale, flags & (A.ROTATE | A.THINGS),
                                 None if arrows is None else [arrows[f]])
    return out


def _c2():
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1",))
    a = W.Archive(data)
    return W.Level(a, 0), S.compile_scene(a, W.TextureDirectory(a), 0)


@pytest.mark.parametrize("flags", [0, A.ROTATE])
def test_an_arrow_at_the_pose_is_the_own_arrow(flags):
    level, blob = _c2()
    lines, dyn, _ = device_tables(level, [])
    things = A.things(blob)
    poses = random_poses(A.lines(level), 4, 17 + flags, margin=0)
    mine = [[(int(p["x"]), int(p["y"]), int(p["angle"]), 112)] for p in poses]
    for run in (lambda a: oracle(level, things, 320, 200, poses, 13107, flags, arrows=a),
                lambda a: hostcheck(lines, dyn, things, 320, 200, poses, 13107, flags, arrows=a)):
        plain, green = run(None), run(mine)
        own = plain == A.ARROW
        assert own.any(axis=(1, 2)).all()
        assert np.array_equal(green == 112, own | (plain == 112)) and np.array_equal(green[~own], plain[~own])


@pytest.mark.parametrize("flags,angle,tip", [
    (0, 0x00000000, ("x", max, 217, 80)), (0, 0x40000000, ("y", min, 62, 200)),
    (0, 0x80000000, ("x", min, 182, 80)), (0, 0xC0000000, ("y", max, 97, 200)),
    (A.ROTATE, 0x00000000, ("y", min, 42, 140)), (A.ROTATE, 0x40000000, ("x", min, 122, 60)),
    (A.ROTATE, 0x80000000, ("y", max, 77, 140)), (A.ROTATE, 0xC0000000, ("x", max, 157, 60))])
def test_arrow_tip_lands_on_its_pixel(flags, angle, tip):
    """320x200 at one pixel per map unit, the pose at (0, 0) facing east, an arrow at (+40, +20) in colour 250.  The tip is
    R = 1198372 (16.16) ahead of the centre: R * 2^16 >> 24 = 4681 Q8 steps forwards, -4682 backwards (the shift floors).
    North-up the centre is Q8 (128 * 320 + 40 * 256, 128 * 200 - 20 * 256) = (51200, 20480), pixel (200, 80):
    east X = 55881, the last pixel whose centre is not past it is 217; north Y = 15799, first row 62; west X = 46518,
    first column 182; south Y = 25162, last row 97.  Rotated, the map turns (40, 20) to (-20, 40): centre (35840, 15360),
    pixel (140, 60), and the arrow turns by the same 90 degrees: east points up to Y = 10679 (first row 42), north left to
    X = 31158 (first column 122), west down to Y = 20042 (last row 77), south right to X = 40521 (last column 157)."""
    level, blob = _c2()
    lines, dyn, _ = device_tables(level, [])
    pose = np.zeros(1, render.POSE)
    arrow = [[(40 << 16, 20 << 16, angle, 250)]]
    axis, pick, extreme, at = tip
    for frame in (oracle(level, [], 320, 200, pose, 65536, flags, arrows=arrow)[0],
                  hostcheck(lines, dyn, [], 320, 200, pose, 65536, flags, arrows=arrow)[0]):
        ys, xs = np.nonzero(frame == 250)
        major, minor = (xs, ys) if axis == "x" else (ys, xs)
        assert pick(major) == extreme and at in minor[major == extreme], (major, minor)


# ---- the rule against the oracle -------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _levels():
    """{name: (level, blob, dynamic)}: the patched c2 level and the content-rich level with random dynamic sectors
    (tests/refcheck/moves.pick), and a c2 level with many of them"""
    from rust_doom_b200 import synthwad
    from tests.refcheck import moves as MV
    from tests.test_lights import rich_wad
    out = {}
    for name, data, n in (("c2", _patched()[0], 6), ("rich", rich_wad(), 6), ("dyn", synthwad.build_iwad(5, ("E1M1",)), 40)):
        a = W.Archive(data)
        level = W.Level(a, 0)
        dynamic, _ = MV.pick(level, 11 + n, n)
        out[name] = (level, S.compile_scene(a, W.TextureDirectory(a), 0, dynamic=dynamic), dynamic)
    return out


def _random_arrows(rng, table, n):
    xs = [t[0] for t in table] + [t[2] for t in table]
    ys = [t[1] for t in table] + [t[3] for t in table]
    out = []
    for _ in range(n):
        kind = rng.integers(0, 4)
        if kind == 0:                                      # the level's corners of the coordinate range
            x, y = int(rng.choice([-32767, 32767])) << 16, int(rng.choice([-32767, 32767])) << 16
        elif kind == 1:                                    # far off-screen, at full 16.16 resolution
            x, y = int(rng.integers(-2 ** 31, 2 ** 31)), int(rng.integers(-2 ** 31, 2 ** 31))
        else:
            x = int(rng.integers((min(xs) - 64) << 16, (max(xs) + 64) << 16))
            y = int(rng.integers((min(ys) - 64) << 16, (max(ys) + 64) << 16))
        out.append((x, y, int(rng.integers(0, 1 << 32)), int(rng.integers(1, 256))))
    return out


@pytest.mark.parametrize("w,h", [(320, 200), (333, 187), (1, 2), (4096, 24)])
@pytest.mark.parametrize("which", ["c2", "rich", "dyn"])
def test_hostcheck_equals_the_oracle(which, w, h):
    from tests.refcheck import moves as MV
    level, blob, dynamic = _levels()[which]
    lines, dyn, slots = device_tables(level, dynamic)
    assert (lines["pad"] & CHANGEABLE).any()
    table, things = A.lines(level), A.things(blob)
    words = (len(level.linedefs) + 31) // 32
    rng = np.random.default_rng(w * 7 + h + len(which))
    n = 2
    for flags in range(16):
        poses = random_poses(table, n, 13 * flags + w + h, margin=64)
        if flags == 5:
            poses["x"][0], poses["y"][0] = 32767 << 16, -(32767 << 16)
        scale = (A.SCALE_MIN, A.SCALE_MAX, 13107, 65536)[flags % 4] if flags >= 12 else 13107
        moves = [MV.state(level, dynamic, 100 * flags + f, hole_free=False) if (flags + f) % 3 else [] for f in range(n)]
        offs = [offsets(slots, m) if m else None for m in moves]
        arrows = [_random_arrows(rng, table, int(rng.integers(0, 9))) for _ in range(n)]
        mapped = rng.integers(0, 1 << 32, (n, words), dtype=np.uint64).astype(np.uint32) if flags % 2 == 0 else None
        want = oracle(level, things, w, h, poses, scale, flags, mapped, moves, arrows)
        got = hostcheck(lines, dyn, things, w, h, poses, scale, flags, mapped, words, offs, arrows)
        assert np.array_equal(got, want), (flags, np.argwhere(got != want)[:5])
        if flags < 8 and mapped is None:                   # at rest, no arrows: the C19 frames
            c19 = A.automap(table, things, w, h, poses, scale, flags)
            assert np.array_equal(hostcheck(lines, dyn, things, w, h, poses, scale, flags), c19)


def test_some_frames_change_with_their_state():
    level, blob, dynamic = _levels()["dyn"]
    lines, dyn, slots = device_tables(level, dynamic)
    table, things = A.lines(level), A.things(blob)
    from tests.refcheck import moves as MV
    poses = random_poses(table, 6, 3, margin=0)
    moves = [MV.state(level, dynamic, 40 + f, hole_free=False) for f in range(6)]
    at_rest = hostcheck(lines, dyn, things, 320, 200, poses, 6554, A.ALL_LINES)
    moved = hostcheck(lines, dyn, things, 320, 200, poses, 6554, A.ALL_LINES, offs=[offsets(slots, m) for m in moves])
    assert any(not np.array_equal(at_rest[f], moved[f]) for f in range(6))


# ---- the CLIs' flag name ---------------------------------------------------------------------------------------------
def test_flag_parsing():
    import rust_doom_b200 as b2d
    from rust_doom_b200 import cli
    assert cli.automap_flag_names("others") == ("", False)
    assert cli.automap_flag_options("rotate,others,seen") == ("rotate", True, True)
    assert cli.automap_flag_options("things") == ("things", False, False)
    for bad in ("other", "others,bogus"):
        with pytest.raises(ValueError):
            cli.automap_flag_options(bad)
    with pytest.raises(ValueError):
        b2d.automap_flags("others")                       # a CLI name: the library takes the arrows themselves
    assert cli.OTHER_COLOURS == (112, 96, 64, 176)


def test_compiled_cli_parses_others(tmp_path):
    """the compiled CLI takes `others` and refuses a misspelling as a usage error, before it opens any device"""
    from rust_doom_b200 import synthwad
    from tests.test_cli import _b2d_binary
    wad = tmp_path / "syn.wad"
    wad.write_bytes(synthwad.build_iwad(1, ("E1M1",)))
    bad = subprocess.run([_b2d_binary(), "-i", str(wad), "--dump", str(tmp_path / "d.ppm"), "--automap", "0.2",
                          "--automap-flags", "others,bogus"], capture_output=True, text=True)
    assert bad.returncode == 2 and "others" in bad.stderr
    assert not (tmp_path / "d.ppm").exists()
