"""Automap oracle (DESIGN.md C19), restated from the contract in plain Python integers: the line table of a level from
oracle/wad.py's Level, and W x H palette-index automap frames drawn pixel by pixel in draw order (later items overwrite
earlier ones).  Independent of libb2d: only the Q30 sine / cosine comes from the oracle's own C restatement
(render.sincos_q30)."""
from typing import List, Sequence, Tuple

import numpy as np

from oracle import render
from oracle import scene as S
from oracle import wad as W

ROTATE, ALL_LINES, THINGS = 1, 2, 4
SCALE_MIN, SCALE_MAX = 256, 64 << 16
WALL, TELEPORT, FLOOR_STEP, CEIL_STEP, PLAIN = 176, 184, 64, 231, 96
ARROW, THING = 209, 112
ML_SECRET, ML_DONTDRAW = 0x20, 0x80

_R = 8 * 16 * 65536 // 7
ARROW_SEGS = [((-_R + _R // 8, 0), (_R, 0)),
              ((_R, 0), (_R - _R // 2, _R // 4)),
              ((_R, 0), (_R - _R // 2, -(_R // 4))),
              ((-_R + _R // 8, 0), (-_R - _R // 8, _R // 4)),
              ((-_R + _R // 8, 0), (-_R - _R // 8, -(_R // 4))),
              ((-_R + 3 * _R // 8, 0), (-_R + _R // 8, _R // 4)),
              ((-_R + 3 * _R // 8, 0), (-_R + _R // 8, -(_R // 4)))]
THING_SEGS = [((-524288, -734000), (1048576, 0)),
              ((1048576, 0), (-524288, 734000)),
              ((-524288, 734000), (-524288, -734000))]


def lines(level: W.Level) -> List[Tuple[int, int, int, int, int, int, int]]:
    """(x0, y0, x1, y1, colour, colour_all, linedef) per linedef whose vertices exist, in LINEDEFS order."""
    nv, ns, nsec = len(level.vertices), len(level.sidedefs), len(level.sectors)

    def sector(side):
        if not 0 <= side < ns:
            return None
        sec = int(level.sidedefs[side]["sector"])
        return sec if sec < nsec else None

    out = []
    for i, l in enumerate(level.linedefs):
        v1, v2 = int(l["v1"]), int(l["v2"])
        if v1 >= nv or v2 >= nv:
            continue
        front, back = sector(int(l["right"])), sector(int(l["left"]))
        flags = int(l["flags"])
        if front is None or back is None:
            colour = WALL
        elif int(l["special"]) == 39:
            colour = TELEPORT
        elif flags & ML_SECRET:
            colour = WALL
        elif int(level.sectors[front]["floor"]) != int(level.sectors[back]["floor"]):
            colour = FLOOR_STEP
        elif int(level.sectors[front]["ceil"]) != int(level.sectors[back]["ceil"]):
            colour = CEIL_STEP
        else:
            colour = 0
        a, b = level.vertices[v1], level.vertices[v2]
        out.append((int(a["x"]), int(a["y"]), int(b["x"]), int(b["y"]), 0 if flags & ML_DONTDRAW else colour,
                    colour or PLAIN, i))
    return out


def things(blob: bytes) -> List[Tuple[int, int]]:
    """the (x, y) of the scene's decoration sprites, in blob order"""
    return [(int(r[0]), int(r[1])) for r in S.section(blob, "sprites")]


def _line_pixels(X0, Y0, X1, Y1, W_, H_):
    """the on-screen pixels of the Q8 line (X0, Y0) - (X1, Y1) by the C19 rule"""
    xmaj = abs(X1 - X0) >= abs(Y1 - Y0)
    M0, m0, M1, m1 = (X0, Y0, X1, Y1) if xmaj else (Y0, X0, Y1, X1)
    if M1 < M0:
        M0, m0, M1, m1 = M1, m1, M0, m0
    # pixel centres 256 i + 128 with M0 <= centre <= M1
    lo = -((128 - M0) // 256)                         # ceil((M0 - 128) / 256)
    hi = (M1 - 128) // 256
    if lo > hi:
        return [(X0 // 256, Y0 // 256)]
    lo, hi = max(lo, 0), min(hi, (W_ if xmaj else H_) - 1)
    out = []
    for i in range(lo, hi + 1):
        c = 256 * i + 128
        if M1 == M0:
            v = m0
        else:
            v = m0 * (M1 - M0) + (c - M0) * (m1 - m0)     # the minor coordinate times (M1 - M0)
            v = v // (M1 - M0)                              # floor
        j = v // 256
        out.append((i, j) if xmaj else (j, i))
    return out


def _screen(dx, dy, rot, c, s, scale, W_, H_):
    if rot:
        dx, dy = (dx * c - dy * s) >> 30, (dx * s + dy * c) >> 30
    return (W_ << 7) + ((dx * scale) >> 24), (H_ << 7) - ((dy * scale) >> 24)


def automap(table: Sequence, thing_xy: Sequence, width: int, height: int, poses: np.ndarray, scale: int, flags: int) -> np.ndarray:
    """uint8 [n, height, width]: the automap of each pose (b2d_pose records) over one level's line table and things"""
    assert SCALE_MIN <= scale <= SCALE_MAX and not flags & ~7
    out = np.zeros((len(poses), height, width), np.uint8)
    for f, p in enumerate(poses):
        px, py, angle = int(p["x"]), int(p["y"]), int(p["angle"]) & 0xFFFFFFFF
        rot = bool(flags & ROTATE)
        c, s = render.sincos_q30((0x40000000 - angle) & 0xFFFFFFFF)
        ac, as_ = render.sincos_q30(0x40000000 if rot else angle)

        def mapped(mx, my):
            return _screen(mx - px, my - py, rot, c, s, scale, width, height)

        items = []
        for (x0, y0, x1, y1, colour, colour_all, _) in table:
            col = colour_all if flags & ALL_LINES else colour
            if col:
                items.append((mapped(x0 << 16, y0 << 16), mapped(x1 << 16, y1 << 16), col))
        for (a, b) in ARROW_SEGS:
            items.append((_screen(a[0], a[1], True, ac, as_, scale, width, height),
                          _screen(b[0], b[1], True, ac, as_, scale, width, height), ARROW))
        if flags & THINGS:
            for (tx, ty) in thing_xy:
                for (a, b) in THING_SEGS:
                    items.append((mapped((tx << 16) + a[0], (ty << 16) + a[1]), mapped((tx << 16) + b[0], (ty << 16) + b[1]), THING))
        frame = out[f]
        for (A, B, col) in items:
            for (x, y) in _line_pixels(A[0], A[1], B[0], B[1], width, height):
                if 0 <= x < width and 0 <= y < height:
                    frame[y, x] = col
    return out
