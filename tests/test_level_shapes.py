"""Levels shaped like a node builder's output on real maps, without a GPU.  The generated levels have at most 12 segs in a
subsector, a BSP at most 18 levels deep and no seg longer than 256 units; real maps have round rooms and long walls cut
into many collinear segs.  The levels here are built by hand (synthwad's graphics, a small node builder below) so that:

- rotundas: convex N-gon rooms that stay one subsector each, N = 31, 32, 33, 64, 65 and 146 (the walk's 32-wide seg
  chunks: one short of a chunk, one, one over, two, two and one over, five), with two-sided windows into alcoves with
  higher floors and lower ceilings, masked middles in some windows, decoration things in a 65-seg subsector, and a
  zero-length seg and a 1-unit seg in the largest one;
- a long hall: 16384 units, one side a single one-sided seg, the other cut every 32 units into collinear segs that end up
  in subsectors of 128, with raised and lowered floor patches far down the hall;
- deep BSP: stair corridors whose tree is a comb (each node splits off one step) deep enough that the walk's BSP stack
  needs exactly its 128 entries, and one step more.

Every level is first shown to be a valid case here -- both scene compilers give the same blob, hostcheck (the CPU
execution of the kernels' maths) gives the oracle's frames, and the oracle agrees with the float64 ray caster -- so that
tests/test_gpu_level_shapes.py spends GPU time on cases known to be right."""
import functools
import math
import struct

import numpy as np
import pytest

from oracle import render
from oracle import scene as S
from oracle import wad as W
from tests.conftest import oracle_blob
from tests.refcheck import glcaster
from tests.test_refcheck import Tally
from tests.test_scale import DECOR_KINDS, STACK_DEPTH
from tests.test_view_range import projection_bound

LEAF = 0x80000000
LEVEL_LUMPS = ("THINGS", "LINEDEFS", "SIDEDEFS", "VERTEXES", "SEGS", "SSECTORS", "NODES", "SECTORS", "REJECT", "BLOCKMAP")
SIZES = ((320, 200), (333, 187), (1920, 1080))


def _iround(v: float) -> int:
    """round half away from zero (symmetric, so mirrored polygon vertices stay mirrored)"""
    return int(math.copysign(math.floor(abs(v) + 0.5), v))


# ---- level description ---------------------------------------------------------------------------------------------
class Map:
    """Vertices, sectors, sidedefs, linedefs and the segs a node builder starts from (one per linedef side, or a linedef cut
    into several collinear segs at given points), plus things."""

    def __init__(self):
        self.verts, self._vindex = [], {}
        self.sectors, self.sides, self.lines, self.segs, self.things = [], [], [], [], []

    def v(self, p) -> int:
        key = (int(p[0]), int(p[1]))
        assert -32768 <= key[0] < 32768 and -32768 <= key[1] < 32768
        if key not in self._vindex:
            self._vindex[key] = len(self.verts)
            self.verts.append(key)
        return self._vindex[key]

    def sector(self, floor, ceil, flat="FLOOR1", ceil_flat="CEIL1", light=176) -> int:
        from rust_doom_b200 import synthwad as G
        self.sectors.append(G.Sector(floor, ceil, flat, ceil_flat, light))
        return len(self.sectors) - 1

    def _side(self, sector, middle="-", upper="-", lower="-", xoff=0) -> int:
        from rust_doom_b200 import synthwad as G
        self.sides.append(G.Sidedef(xoff, 0, upper, lower, middle, sector))
        return len(self.sides) - 1

    def _cut(self, a, b, line, direction, cuts):
        pts = [a] + list(cuts) + [b]
        for p, q in zip(pts, pts[1:]):
            self.segs.append((self.v(p), self.v(q), line, direction, _iround(math.hypot(p[0] - a[0], p[1] - a[1]))))

    def wall(self, a, b, sector, tex="BRICK1", cuts=(), xoff=0) -> int:
        """one-sided linedef a -> b, `sector` on its right; `cuts`: points on it where its seg is cut"""
        from rust_doom_b200 import synthwad as G
        line = len(self.lines)
        self.lines.append(G.Linedef(self.v(a), self.v(b), 0x0001, 0, 0, self._side(sector, tex, xoff=xoff), -1))
        self._cut(a, b, line, 0, cuts)
        return line

    def window(self, a, b, front, back, front_tex=("BRICK2", "STEP2", "-"), back_tex=("BRICK1", "STEP1", "-"), cuts=()) -> int:
        """two-sided linedef a -> b: `front` on its right, `back` on its left; textures (upper, lower, middle)"""
        from rust_doom_b200 import synthwad as G
        line = len(self.lines)
        rs = self._side(front, upper=front_tex[0], lower=front_tex[1], middle=front_tex[2], xoff=3)
        ls = self._side(back, upper=back_tex[0], lower=back_tex[1], middle=back_tex[2], xoff=5)
        self.lines.append(G.Linedef(self.v(a), self.v(b), 0x0004, 0, 0, rs, ls))
        self._cut(a, b, line, 0, cuts)
        self._cut(b, a, line, 1, list(reversed(cuts)))
        return line

    def seg_sector(self, seg) -> int:
        line = self.lines[seg[2]]
        return self.sides[line.right if seg[3] == 0 else line.left].sector


# ---- node builder ----------------------------------------------------------------------------------------------------
def build_nodes(m: Map, hints=(), comb=False, max_leaf=None):
    """A small general node builder: partition with a seg's line (or one of `hints`, lines given as (x, y, dx, dy)), split
    the segs it crosses, stop at convex sets (of at most `max_leaf` segs).  Candidates are ranked by the number of
    splits, then by balance -- or, with `comb`, by the size of the smaller side, so that each node splits off as little
    as it can (a comb).  Writes m.out_segs, m.ssectors [(count, first)] and m.nodes [(x, y, dx, dy, rbox, lbox, rchild,
    lchild)], root last.  Boxes are the segs' bounding boxes (the scene compilers recompute them)."""
    out_segs, ssectors, nodes = [], [], []

    def ends(segs):
        a = np.array([m.verts[s[0]] for s in segs], np.int64)
        b = np.array([m.verts[s[1]] for s in segs], np.int64)
        return a, b

    def sides(part, a, b):
        px, py, dx, dy = part
        return ((a[:, 1] - py) * dx - (a[:, 0] - px) * dy, (b[:, 1] - py) * dx - (b[:, 0] - px) * dy)

    def classify(part, a, b):
        """-1 right, +1 left, 0 split"""
        sa, sb = sides(part, a, b)
        d = b - a
        along = d[:, 0] * part[2] + d[:, 1] * part[3]
        c = np.zeros(len(a), np.int64)
        c[((sa <= 0) & (sb <= 0)) & ((sa < 0) | (sb < 0))] = -1
        c[((sa >= 0) & (sb >= 0)) & ((sa > 0) | (sb > 0))] = 1
        on = (sa == 0) & (sb == 0)
        c[on] = np.where(along[on] < 0, 1, -1)       # collinear: same direction -> right (front), opposite -> left
        return c, sa, sb

    def convex(segs):
        a, b = ends(segs)
        d = b - a
        for i in range(len(segs)):
            if not d[i].any():
                continue
            part = (a[i, 0], a[i, 1], d[i, 0], d[i, 1])
            c, _, _ = classify(part, a, b)
            if (c != -1).any():
                return False
        return True

    def bbox(segs):
        a, b = ends(segs)
        p = np.concatenate([a, b])
        return (int(p[:, 1].max()), int(p[:, 1].min()), int(p[:, 0].min()), int(p[:, 0].max()))

    def choose(segs):
        a, b = ends(segs)
        d = b - a
        seen, cands = set(), []
        for i in range(len(segs)):
            if not d[i].any():
                continue
            g = math.gcd(int(d[i, 0]), int(d[i, 1]))
            ux, uy = int(d[i, 0]) // g, int(d[i, 1]) // g
            if ux < 0 or (ux == 0 and uy < 0):
                ux, uy = -ux, -uy
            key = (ux, uy, uy * int(a[i, 0]) - ux * int(a[i, 1]))
            if key not in seen:
                seen.add(key)
                cands.append((int(a[i, 0]), int(a[i, 1]), int(d[i, 0]), int(d[i, 1])))
        best = None
        for part in list(hints) + cands:
            c, _, _ = classify(part, a, b)
            nr, nl, ns = int((c == -1).sum()), int((c == 1).sum()), int((c == 0).sum())
            if nr + ns == 0 or nl + ns == 0:
                continue
            rank = (ns, min(nr, nl), part[0], part[1]) if comb else (ns, abs(nr - nl))
            if best is None or rank < best[0]:
                best = (rank, part)
        assert best is not None, "no partition divides a non-convex set of %d segs" % len(segs)
        return best[1]

    def divide(segs, part):
        a, b = ends(segs)
        c, sa, sb = classify(part, a, b)
        right, left = [], []
        for k, s in enumerate(segs):
            if c[k] < 0:
                right.append(s)
            elif c[k] > 0:
                left.append(s)
            else:
                t = sa[k] / float(sa[k] - sb[k])
                p = (_iround(a[k, 0] + t * (b[k, 0] - a[k, 0])), _iround(a[k, 1] + t * (b[k, 1] - a[k, 1])))
                mid = m.v(p)
                first = (s[0], mid, s[2], s[3], s[4])
                second = (mid, s[1], s[2], s[3], s[4] + _iround(math.hypot(p[0] - a[k, 0], p[1] - a[k, 1])))
                (left if sa[k] > 0 else right).append(first)
                (left if sb[k] > 0 else right).append(second)
        return right, left

    def rec(segs):
        if (max_leaf is None or len(segs) <= max_leaf) and convex(segs):
            secs = {m.seg_sector(s) for s in segs}
            assert len(secs) == 1, "a convex leaf faces sectors %s" % secs
            ssectors.append((len(segs), len(out_segs)))
            out_segs.extend(segs)
            return 0x8000 | (len(ssectors) - 1), bbox(segs)
        part = choose(segs)
        right, left = divide(segs, part)
        rc, rb = rec(right)
        lc, lb = rec(left)
        nodes.append(part + (rb, lb, rc, lc))
        assert len(nodes) < 0x8000
        return len(nodes) - 1, (max(rb[0], lb[0]), min(rb[1], lb[1]), min(rb[2], lb[2]), max(rb[3], lb[3]))

    rec(list(m.segs))
    m.out_segs, m.ssectors, m.nodes = out_segs, ssectors, nodes
    return m


def level_wad(m: Map) -> bytes:
    """The map as level 0 of a generated IWAD that has masked textures and the decoration sprites (its own level lumps
    replaced)."""
    from rust_doom_b200 import synthwad as G
    base = G.build_iwad(1, ("E1M1",), cfg=G.SynthConfig(mid_pct=30, thing_pct=30))
    lb = struct.pack
    nodes = b""
    for (x, y, dx, dy, rb, lbox, rc, lc) in m.nodes:
        nodes += lb("<hhhh4h4hHH", x, y, dx, dy, *rb, *lbox, rc, lc)
    mine = {
        "THINGS": b"".join(lb("<hhhHH", *t) for t in m.things),
        "LINEDEFS": b"".join(lb("<HHHHHhh", l.v1, l.v2, l.flags, l.special, l.tag, l.right, l.left) for l in m.lines),
        "SIDEDEFS": b"".join(lb("<hh8s8s8sH", s.xoff, s.yoff, G._name8(s.upper), G._name8(s.lower), G._name8(s.middle), s.sector)
                             for s in m.sides),
        "VERTEXES": b"".join(lb("<hh", *v) for v in m.verts),
        "SEGS": b"".join(lb("<HHHHHH", a, b, _seg_angle(m, a, b), line, d, off & 0xFFFF) for (a, b, line, d, off) in m.out_segs),
        "SSECTORS": b"".join(lb("<HH", n, f) for n, f in m.ssectors),
        "NODES": nodes,
        "SECTORS": b"".join(lb("<hh8s8shHH", s.floor, s.ceil, G._name8(s.floor_flat), G._name8(s.ceil_flat), s.light, 0, 0)
                            for s in m.sectors),
        "REJECT": bytes((len(m.sectors) ** 2 + 7) // 8),
        "BLOCKMAP": lb("<hhHH", 0, 0, 0, 0),
    }
    a = W.Archive(base)
    marker = a.levels[0]
    lumps = []
    for k, (name, pos, size) in enumerate(a.lumps):
        name = name.rstrip(b"\0").decode("ascii")
        if marker < k <= marker + len(LEVEL_LUMPS) and name in mine:
            lumps.append((name, mine[name]))
        else:
            lumps.append((name, base[pos:pos + size]))
    return G.assemble_wad(lumps)


def _seg_angle(m, a, b) -> int:
    (ax, ay), (bx, by) = m.verts[a], m.verts[b]
    return int(round(math.atan2(by - ay, bx - ax) * 32768.0 / math.pi)) & 0xFFFF if (ax, ay) != (bx, by) else 0


class Level:
    """A built level: wad bytes, the oracle's blob, its poses [(x, y, z, angle in BAM, what)] and facts the tests check."""

    def __init__(self, m: Map, poses, **facts):
        self.map = m
        self.wad = level_wad(m)
        self.blob = oracle_blob(self.wad)
        self.poses = poses
        self.facts = facts

    def pose_array(self, which=None) -> np.ndarray:
        sel = self.poses if which is None else [self.poses[i] for i in which]
        out = np.concatenate([render.make_pose(x, y, z, 0.0) for (x, y, z, _, _) in sel])
        out["angle"] = [a & 0xFFFFFFFF for (_, _, _, a, _) in sel]
        return out


def bam(deg: float) -> int:
    return int(round(deg / 360.0 * 4294967296.0)) & 0xFFFFFFFF


# ---- 1. rotundas -----------------------------------------------------------------------------------------------------
# (sides, radius, an alcove on every m-th edge, floor): alcove windows far enough apart that no alcove straddles another
# alcove's window line, so the node builder cuts the alcoves off without splitting the room
ROTUNDAS = ((31, 448, 5, 0), (32, 448, 5, 8), (33, 480, 5, -16), (64, 704, 10, 24), (65, 704, 10, 0), (144, 1120, 24, 16))
ALCOVE_DEPTH = 48
THINGS_IN = 65              # the rotunda whose subsector also holds decoration things
BIG = 144                   # the rotunda that also holds a zero-length seg and a 1-unit seg (146 segs)


@functools.lru_cache(maxsize=None)
def rotunda_level() -> Level:
    m = Map()
    ext = [r + ALCOVE_DEPTH + 16 for (_, r, _, _) in ROTUNDAS]
    x = -(sum(ext) * 2 + 128 * (len(ROTUNDAS) - 1)) // 2
    hints, poses, rooms = [], [], {}
    for k, (n, r, every, floor) in enumerate(ROTUNDAS):
        cx = x + ext[k]
        x = cx + ext[k] + 128
        if k + 1 < len(ROTUNDAS):
            hints.append((x - 64, 0, 0, 256))
        ceil = floor + 192
        rot = m.sector(floor, ceil, "FLOOR%d" % (1 + k % 6), "CEIL%d" % (1 + k % 4), 160 + 8 * k)
        th = [math.pi * (2 * i + 1) / n for i in range(n)]
        vs = [(cx + _iround(r * math.cos(t)), _iround(r * math.sin(t))) for t in th]
        for i in range(n):                                   # strictly convex after rounding
            (ax, ay), (bx, by), (qx, qy) = vs[i - 2], vs[i - 1], vs[i]
            assert (bx - ax) * (qy - by) - (by - ay) * (qx - bx) > 0, (n, i)
        s = 1.0 + ALCOVE_DEPTH / r
        alcoves = list(range(every // 2, n - every // 2, every))
        first_alcove = None
        for i in range(n):
            a, b = vs[i], vs[(i + 1) % n]                    # counter-clockwise edge; walls run b -> a (room on the right)
            if i in alcoves:
                j = alcoves.index(i)
                alc = m.sector(floor + 24, ceil - 64, "FLOOR%d" % (1 + (k + j) % 6), "CEIL%d" % (1 + j % 4), 144 + 16 * (j % 3))
                mid = ("GRATE1", "FENCE72", "-")[j % 3]
                m.window(b, a, rot, alc, front_tex=("BRICK2", "STEP2", mid), back_tex=("TECH1", "STEP1", "-"))
                oa = (cx + _iround(s * (a[0] - cx)), _iround(s * a[1]))
                ob = (cx + _iround(s * (b[0] - cx)), _iround(s * b[1]))
                m.wall(b, ob, alc, "PANEL72")
                m.wall(ob, oa, alc, "TECH2")
                m.wall(oa, a, alc, "PANEL72")
                if first_alcove is None:
                    first_alcove = ((oa[0] + ob[0] + 2 * a[0] + 2 * b[0]) / 6.0, (oa[1] + ob[1] + 2 * a[1] + 2 * b[1]) / 6.0, floor + 24)
            elif n == BIG and i == n - 1:
                # the vertical edge at the east side: one linedef cut into a 1-unit seg and the rest
                m.wall(b, a, rot, "WIDE1", cuts=[(b[0], b[1] - 1)])
            else:
                m.wall(b, a, rot, ("BRICK3", "WIDE1", "COMBO1", "PANEL2")[i % 4])
            if n == BIG and i == n // 2:
                # a zero-length seg at a vertex no partition line passes through, in the subsector's third chunk
                assert i not in alcoves and i - 1 not in alcoves
                m.segs.append((m.v(b), m.v(b), len(m.lines) - 1, 0, 0))
        rooms[n] = (rot, cx)
        z = floor + 41
        poses += [(cx, 0, z, bam(a), "rotunda %d centre" % n) for a in (0, 77, 161, 250)]
        poses.append((cx - 0.8 * r, 0.1 * r, z, bam(-5), "rotunda %d by the west wall" % n))      # sees most of the room
        poses.append((cx + 0.3 * r, -0.6 * r, z, bam(100), "rotunda %d off centre" % n))
        ax_, ay_, af = first_alcove
        poses.append((ax_, ay_, af + 41, bam(math.degrees(math.atan2(-ay_, cx - ax_))), "rotunda %d from an alcove" % n))
        if n == THINGS_IN:
            for t in range(8):
                a = 2 * math.pi * t / 8
                m.things.append((cx + _iround(0.45 * r * math.cos(a)), _iround(0.45 * r * math.sin(a)), 0, DECOR_KINDS[t % len(DECOR_KINDS)], 7))
    m.things.append((rooms[ROTUNDAS[0][0]][1], 0, 0, 1, 7))            # player start
    build_nodes(m, hints=hints)
    return Level(m, poses, rooms=rooms)


# ---- 2. long hall ----------------------------------------------------------------------------------------------------
HALL_X = 8192               # the hall runs from x = -8192 to 8192 (16384 units), y from -128 to 128
PATCHES = ((5120, 5632, 24), (6656, 7168, -24))      # (x0, x1, floor): 32 <= y <= 96, far from the west end


@functools.lru_cache(maxsize=None)
def hall_level() -> Level:
    m = Map()
    hall = m.sector(0, 160, "FLOOR2", "CEIL3", 192)
    X = HALL_X
    m.wall((X, -128), (-X, -128), hall, "WIDE1")                                             # one seg of 16384 units
    m.wall((-X, 128), (X, 128), hall, "BRICK3", cuts=[(x, 128) for x in range(-X + 32, X, 32)])  # 512 segs of 32
    m.wall((-X, -128), (-X, 0), hall, "PANEL1")
    m.wall((-X, 0), (-X, 128), hall, "PANEL1")
    m.wall((X, 128), (X, 0), hall, "PANEL2")
    m.wall((X, 0), (X, -128), hall, "PANEL2")
    for (x0, x1, f) in PATCHES:
        p = m.sector(f, 160, "FLOOR4", "CEIL3", 192)
        pts = [(x0, 32), (x1, 32), (x1, 96), (x0, 96)]                  # counter-clockwise: the patch on the left
        for a, b in zip(pts, pts[1:] + pts[:1]):
            m.window(a, b, hall, p, front_tex=("-", "STEP2", "-"), back_tex=("-", "STEP1", "-"))
    m.things.append((-X + 48, 0, 0, 1, 7))                             # player start
    # the hall's axis, then cuts across its north half (the patches' edges and the 32-unit cuts all meet these at vertices)
    build_nodes(m, hints=[(-X, 0, 2 * X, 0)] + [(x, 0, 0, 128) for x in (-4096, 0, 4096)], max_leaf=160)
    poses = []
    for x, a, what in ((-X + 48, 0, "west end"), (X - 48, 180, "east end")):
        for y in (0, 64, -100):
            for d in (0, 1, -1):
                poses.append((x, y, 41, (bam(a) + d) & 0xFFFFFFFF, "hall %s y=%d %+d BAM" % (what, y, d)))
    poses += [(-X + 2000, -40, 41, bam(3), "hall looking at the patches"), (0, 0, 41, bam(90), "hall middle across"),
              (5376, 64, 65, bam(180), "hall on the raised patch"), (6912, 64, 17, bam(0), "hall on the lowered patch")]
    return Level(m, poses)


# ---- 3. deep BSP: a stair corridor whose tree is a comb --------------------------------------------------------------
STEP_W = 32


@functools.lru_cache(maxsize=None)
def corridor_level(k: int) -> Level:
    """k steps of 32 units along x, each a sector 4 units higher than the one west of it; the comb splits off the west
    step first, so from the east end looking west every node pushes the step it splits off and its near child."""
    m = Map()
    x0 = -(k * STEP_W) // 2
    xs = [x0 + STEP_W * j for j in range(k + 1)]
    secs = [m.sector(4 * j, 4 * j + 128, "FLOOR%d" % (1 + j % 6), "CEIL%d" % (1 + j % 4), 144 + 8 * (j % 8)) for j in range(k)]
    m.wall((xs[0], -48), (xs[0], 48), secs[0], "PANEL1")
    m.wall((xs[k], 48), (xs[k], -48), secs[-1], "PANEL1")
    for j in range(k):
        m.wall((xs[j], 48), (xs[j + 1], 48), secs[j], "BRICK1")
        m.wall((xs[j + 1], -48), (xs[j], -48), secs[j], "BRICK2")
        if j:
            m.window((xs[j], -48), (xs[j], 48), secs[j], secs[j - 1], front_tex=("TECH1", "STEP1", "-"), back_tex=("TECH2", "STEP2", "-"))
    m.things.append((xs[k] - 16, 0, 180, 1, 7))                        # player start
    build_nodes(m, comb=True)
    z = [4 * j + 41 for j in range(k)]
    poses = [(xs[k] - 16, 0, z[-1], bam(180), "east end looking west"),
             (xs[k] - 16, 20, z[-1], bam(172), "east end looking west, off axis"),
             (xs[k] - 16, 0, z[-1], bam(0), "east end looking east"),
             (xs[0] + 16, 0, z[0], bam(180), "west end looking west"),
             (xs[0] + 16, 0, z[0], bam(0), "west end looking east"),
             (xs[k - 2] + 16, 0, z[k - 2], bam(180), "second step from the east looking west"),
             (xs[k // 2] + 16, -10, z[k // 2], bam(185), "middle looking west")]
    return Level(m, poses)


def stack_need(blob: bytes, view, pose) -> int:
    """The most entries the walk kernel's BSP stack holds for this pose: its push rule restated -- pop a child; at a node,
    the far child is pushed, then the near one, each only if its box's column range is on screen (box_range); the walk
    overflows when sp + need > 128.  The walk also leaves out a child whose columns are all closed by solid walls drawn so
    far; that only lowers the need, and is ignored here (the result is the need with nothing drawn yet, exact in the comb
    corridors, where every node is popped before any subsector)."""
    nodes = S.section(blob, "nodes").astype(np.int64)
    root = S.header(blob)[S.H_ROOT]
    cosq, sinq = render.sincos_q30(int(pose["angle"]))
    px, py = int(pose["x"]), int(pose["y"])
    px8, py8 = px >> 8, py >> 8
    W_, F = view.W, view.F

    def on_screen(box):                          # box_range of b2d_math.cuh: box = top, bottom, left, right
        all_behind, any_near, mn, mx = True, False, None, None
        for i in range(4):
            dx, dy = (int(box[2 + (i & 1)]) << 8) - px8, (int(box[i >> 1]) << 8) - py8
            tx, tz = (dx * sinq - dy * cosq) >> 30, (dx * cosq + dy * sinq) >> 30
            if tz >= -256:
                all_behind = False
            if tz < 32 * 256:
                any_near = True
                continue
            xc = ((tx * F) // tz - 1 + W_) // 2
            mn = xc if mn is None else min(mn, xc)
            mx = xc if mx is None else max(mx, xc)
        if all_behind:
            return False
        if any_near:
            return True
        return not (mx + 2 < 0 or mn - 2 > W_ - 1)

    stack, worst = [root & 0xFFFFFFFF], 1
    while stack:
        child = stack.pop()
        if child & LEAF or child >= len(nodes):
            continue
        n = nodes[child]
        sd = (py - (int(n[1]) << 16)) * int(n[2]) - (px - (int(n[0]) << 16)) * int(n[3])
        side = 1 if sd > 0 else 0
        boxes = (n[4:8], n[8:12])
        near_c, far_c = int(n[12 + side]) & 0xFFFFFFFF, int(n[12 + (side ^ 1)]) & 0xFFFFFFFF
        far_vis, near_vis = on_screen(boxes[side ^ 1]), on_screen(boxes[side])
        worst = max(worst, len(stack) + far_vis + near_vis)
        if far_vis:
            stack.append(far_c)
        if near_vis:
            stack.append(near_c)
    return worst


@functools.lru_cache(maxsize=None)
def deep_levels():
    """(at the limit, one step deeper): the corridors whose worst pose needs exactly STACK_DEPTH and STACK_DEPTH + 1
    stack entries at 320x200"""
    view = render.make_view(320, 200)
    found = {}
    for k in range(STACK_DEPTH - 2, STACK_DEPTH + 4):
        lv = corridor_level(k)
        need = max(stack_need(lv.blob, view, p) for p in lv.pose_array())
        found.setdefault(need, lv)
    return found[STACK_DEPTH], found[STACK_DEPTH + 1]


def levels():
    at, over = deep_levels()
    return {"rotundas": rotunda_level(), "hall": hall_level(), "deep128": at, "deep129": over}


LEVEL_NAMES = ("rotundas", "hall", "deep128", "deep129")


def subsector_sizes(blob: bytes) -> np.ndarray:
    return S.section(blob, "ssectors")[:, 1]


def seg_lengths(blob: bytes) -> np.ndarray:
    verts = S.section(blob, "verts").astype(np.float64)
    segs = S.section(blob, "segs")
    return np.hypot(*(verts[segs[:, 1]] - verts[segs[:, 0]]).T)


def level_eyes(blob: bytes):
    """the corners of the level's bounding box: the farthest an eye inside the level can be from any vertex"""
    verts = S.section(blob, "verts")
    (x0, y0), (x1, y1) = verts.min(0), verts.max(0)
    return [(x0, y0), (x0, y1), (x1, y0), (x1, y1)]


# ---- the levels reach their targets ----------------------------------------------------------------------------------
def test_rotundas_reach_the_seg_chunk_boundaries(hostcheck, b2d):
    lv = rotunda_level()
    sizes = subsector_sizes(lv.blob).tolist()
    for n in (31, 32, 33, 64, 65):
        assert sizes.count(n) == 1, "no subsector of exactly %d segs: %s" % (n, sorted(sizes)[-8:])
    assert max(sizes) == BIG + 2 > 4 * 32
    ss = S.section(lv.blob, "ssectors")
    big = int(np.argmax(sizes))
    first, num = int(ss[big, 0]), int(ss[big, 1])
    lengths = seg_lengths(lv.blob)[first:first + num]
    assert (lengths == 0).sum() == 1 and (lengths == 1).sum() == 1, "the zero-length and 1-unit segs"
    things = int(ss[sizes.index(THINGS_IN), 3]) >> 24
    assert things == 8, "the 65-seg subsector holds %d sprites" % things
    h = S.header(lv.blob)
    assert h[S.H_NMIDS] >= 6
    # some pose's worklist takes more than two chunks' worth of segs from one subsector
    _, counts, ids = hostcheck(lv.blob, b2d.make_view(320, 200), lv.pose_array())
    most = 0
    for i in range(len(lv.poses)):
        got = ids[i, :counts[i]]
        for k in range(len(ss)):
            most = max(most, int(((got >= ss[k, 0]) & (got < ss[k, 0] + ss[k, 1])).sum()))
    assert most > 64, most


def test_hall_reaches_its_targets():
    lv = hall_level()
    lengths = seg_lengths(lv.blob)
    assert lengths.max() >= 16384
    segs = S.section(lv.blob, "segs")
    ss = S.section(lv.blob, "ssectors")
    collinear = []
    for first, num, _, _ in ss:
        ys = S.section(lv.blob, "verts")[segs[first:first + num, 0], 1]
        collinear.append(int(((ys == 128) & (lengths[first:first + num] == 32)).sum()))
    assert sum(c >= 100 for c in collinear) >= 3, collinear


def test_deep_levels_need_exactly_the_stack_and_one_more():
    at, over = deep_levels()
    view = render.make_view(320, 200)
    for lv, want in ((at, STACK_DEPTH), (over, STACK_DEPTH + 1)):
        needs = [stack_need(lv.blob, view, p) for p in lv.pose_array()]
        assert max(needs) == want, needs
    # one step deeper, a pose near the east end still needs exactly the whole stack
    assert STACK_DEPTH in [stack_need(over.blob, view, p) for p in over.pose_array()]


@pytest.mark.parametrize("name", LEVEL_NAMES)
def test_projection_fits_at_every_eye(name):
    """seg_frame_setup's M = F * C bound (test_view_range.projection_bound) for an eye anywhere in the level"""
    blob = levels()[name].blob
    assert projection_bound(blob, level_eyes(blob)) < 2.0 ** 29


@pytest.mark.parametrize("name", LEVEL_NAMES)
def test_shape_level_blob_matches_oracle(b2d, name):
    lv = levels()[name]
    assert b2d.Scene(b2d.Archive.from_bytes(lv.wad), 0).blob == lv.blob


@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
@pytest.mark.parametrize("name", LEVEL_NAMES)
def test_shape_level_hostcheck_matches_oracle(b2d, hostcheck, name, size):
    """Bit for bit, except the poses over the stack limit, which hostcheck must report as an overflow (a negative count);
    the restated stack need agrees with hostcheck on which poses those are."""
    lv = levels()[name]
    w, h = size
    view, oview = b2d.make_view(w, h), render.make_view(w, h)
    poses = lv.pose_array()
    ofb = render.render(lv.blob, oview, poses, threads=8)
    hfb, counts, _ = hostcheck(lv.blob, view, poses)
    needs = [stack_need(lv.blob, oview, p) for p in poses]
    over = [i for i in range(len(poses)) if needs[i] > STACK_DEPTH]
    assert [i for i in range(len(poses)) if counts[i] < 0] == over, (needs, counts.tolist())
    assert all(counts[i] == -1 for i in over)                    # -kStatusStackOverflow
    assert bool(over) == (name == "deep129")
    bad = [(lv.poses[i][4], int((ofb[i] != hfb[i]).sum())) for i in range(len(poses)) if i not in over and not np.array_equal(ofb[i], hfb[i])]
    assert not bad, "%s %dx%d: frames differ (pose, pixels): %s" % (name, w, h, bad[:6])


# ---- the oracle against the float64 ray caster -----------------------------------------------------------------------
def _cast(lv, w, h, idx, cols=None):
    a = W.Archive(lv.wad)
    tex = W.TextureDirectory(a)
    view = render.make_view(w, h)
    t = Tally()
    for i in idx:
        x, y, z, ang, what = lv.poses[i]
        g, _, dbg = glcaster.render(a, tex, 0, w, h, x, y, z, ang * 360.0 / 4294967296.0, focal2=(view.F, view.FY2), cols=cols, debug=True)
        dbg["far_depth"] = FAR_STEP_DEPTH * view.FY2
        o = render.render(lv.blob, view, lv.pose_array([i]))[0]
        t.add(g, o if cols is None else o[:, cols], dbg, what)
    return t


# Walls farther than 4 FY2 units from the eye (1256 at 320x200) are textured at iscale's cap of 8 texels per row
# (DESIGN.md 4): far_step pixels, at most 8.6e-5 of these frames (measured on the 129-step corridor at 320x200)
FAR_STEP_DEPTH = 4
FAR_STEP_BOUND = 2e-4
RAYCAST_POSES = {"rotundas": None, "hall": None, "deep128": (0, 1, 2, 4, 6), "deep129": (0, 5)}


@pytest.mark.parametrize("name", LEVEL_NAMES)
def test_shape_level_oracle_agrees_with_raycaster(name):
    """320x200 at the level's poses, and every eighth column of two of them at 1920x1080: every differing pixel explained
    under the usual bounds.  This checks the long-seg and large-level arithmetic the oracle shares with the kernels."""
    lv = levels()[name]
    idx = RAYCAST_POSES[name] or range(len(lv.poses))
    t = _cast(lv, 320, 200, idx)
    t.check(far_step_bound=FAR_STEP_BOUND)
    t2 = _cast(lv, 1920, 1080, list(idx)[:2], cols=np.arange(0, 1920, 8))
    print("%s: 320x200 %d px %s; 1080p %d px %s" % (name, t.px, t.sum, t2.px, t2.sum))
    t2.check(far_step_bound=FAR_STEP_BOUND)
