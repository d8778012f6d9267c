"""State-automap oracle (DESIGN.md C21), test infrastructure: Doom's AM_drawWalls with the live heights of a line's sectors
and AM_drawPlayers' other arrows, restated in plain Python integers on top of oracle/automap.py's transform, shapes and
line pixels.  lines() is the C19 line table at per-sector floor and ceiling offsets; automap() draws C19's items with
each frame's list of other players' arrows after its own arrow and before the things.  Without offsets and arrows they
equal oracle/automap.py's lines() and automap().  Independent of libb2d."""
from typing import List, Sequence, Tuple

import numpy as np

from oracle import automap as A
from oracle import render
from oracle import wad as W


def _offset(off, sec: int) -> int:
    if off is None:
        return 0
    if isinstance(off, dict):
        return int(off.get(sec, 0))
    return int(off[sec])


def lines(level: W.Level, floor_off=None, ceil_off=None) -> List[Tuple[int, int, int, int, int, int, int]]:
    """(x0, y0, x1, y1, colour, colour_all, linedef) per linedef whose vertices exist, in LINEDEFS order, with Doom's
    AM_drawWalls colours at each sector's SECTORS heights plus floor_off / ceil_off ({sector: offset} or a sequence per
    sector, map units; None: 0)"""
    nv, ns, nsec = len(level.vertices), len(level.sidedefs), len(level.sectors)

    def sector(side):
        if not 0 <= side < ns:
            return None
        sec = int(level.sidedefs[side]["sector"])
        return sec if sec < nsec else None

    def floor(sec):
        return int(level.sectors[sec]["floor"]) + _offset(floor_off, sec)

    def ceil(sec):
        return int(level.sectors[sec]["ceil"]) + _offset(ceil_off, sec)

    out = []
    for i, l in enumerate(level.linedefs):
        v1, v2 = int(l["v1"]), int(l["v2"])
        if v1 >= nv or v2 >= nv:
            continue
        front, back = sector(int(l["right"])), sector(int(l["left"]))
        flags = int(l["flags"])
        if front is None or back is None:
            colour = A.WALL
        elif int(l["special"]) == 39:
            colour = A.TELEPORT
        elif flags & A.ML_SECRET:
            colour = A.WALL
        elif floor(front) != floor(back):
            colour = A.FLOOR_STEP
        elif ceil(front) != ceil(back):
            colour = A.CEIL_STEP
        else:
            colour = 0
        a, b = level.vertices[v1], level.vertices[v2]
        out.append((int(a["x"]), int(a["y"]), int(b["x"]), int(b["y"]), 0 if flags & A.ML_DONTDRAW else colour,
                    colour or A.PLAIN, i))
    return out


def automap(table: Sequence, thing_xy: Sequence, width: int, height: int, poses: np.ndarray, scale: int, flags: int,
            arrows=None) -> np.ndarray:
    """uint8 [n, height, width]: oracle/automap.py's automap of each pose, with arrows[f] (a list of (x, y, angle,
    colour): 16.16 map units, BAM, palette index; None: none) drawn after the pose's own arrow and before the things.  An
    arrow's centre goes through the frame's map transform; its shape is turned by its angle north-up, or by its angle +
    90 degrees - the pose's angle under ROTATE, then scaled like the map and added to the centre."""
    assert A.SCALE_MIN <= scale <= A.SCALE_MAX and not flags & ~7
    out = np.zeros((len(poses), height, width), np.uint8)
    for f, p in enumerate(poses):
        px, py, angle = int(p["x"]), int(p["y"]), int(p["angle"]) & 0xFFFFFFFF
        rot = bool(flags & A.ROTATE)
        c, s = render.sincos_q30((0x40000000 - angle) & 0xFFFFFFFF)
        ac, as_ = render.sincos_q30(0x40000000 if rot else angle)

        def mapped(mx, my):
            return A._screen(mx - px, my - py, rot, c, s, scale, width, height)

        items = []
        for (x0, y0, x1, y1, colour, colour_all, _) in table:
            col = colour_all if flags & A.ALL_LINES else colour
            if col:
                items.append((mapped(x0 << 16, y0 << 16), mapped(x1 << 16, y1 << 16), col))
        for (a, b) in A.ARROW_SEGS:
            items.append((A._screen(a[0], a[1], True, ac, as_, scale, width, height),
                          A._screen(b[0], b[1], True, ac, as_, scale, width, height), A.ARROW))
        for (ox, oy, oang, ocol) in ([] if arrows is None or arrows[f] is None else arrows[f]):
            Xc, Yc = mapped(int(ox), int(oy))
            phi = (int(oang) + 0x40000000 - angle) & 0xFFFFFFFF if rot else int(oang) & 0xFFFFFFFF
            oc, os_ = render.sincos_q30(phi)

            def shape(v):
                rx, ry = (v[0] * oc - v[1] * os_) >> 30, (v[0] * os_ + v[1] * oc) >> 30
                return Xc + ((rx * scale) >> 24), Yc - ((ry * scale) >> 24)
            for (a, b) in A.ARROW_SEGS:
                items.append((shape(a), shape(b), int(ocol)))
        if flags & A.THINGS:
            for (tx, ty) in thing_xy:
                for (a, b) in A.THING_SEGS:
                    items.append((mapped((tx << 16) + a[0], (ty << 16) + a[1]), mapped((tx << 16) + b[0], (ty << 16) + b[1]),
                                  A.THING))
        frame = out[f]
        for (P, Q, col) in items:
            for (x, y) in A._line_pixels(P[0], P[1], Q[0], Q[1], width, height):
                if 0 <= x < width and 0 <= y < height:
                    frame[y, x] = col
    return out
