"""Marks-automap oracle (DESIGN.md C22), test infrastructure: Doom's AM_drawGrid and AM_drawMarks restated in plain Python
integers on top of oracle/automap_states.py, and the loader side they need: a level's grid origin from its BLOCKMAP
header and the AMMNUM0 .. AMMNUM9 digit patches, from oracle/wad.py's archive and picture decoder.  automap() draws the
grid under C21's items and the marks over them; without the grid flag and marks it equals oracle/automap_states.py's
automap().  Independent of libb2d."""
from typing import List, Optional, Sequence, Tuple

import numpy as np

from oracle import automap as A
from oracle import automap_states as AST
from oracle import render
from oracle import wad as W

GRID = 16
GRID_COLOUR = 104                    # GRIDCOLORS = GRAYS + GRAYSRANGE / 2
GRID_STEP = 128                      # MAPBLOCKUNITS
GRID_MIN, GRID_MAX = -32768, 32767   # the map range every grid line lies in and spans
DIGITS = 10

Digit = Optional[Tuple[np.ndarray, int, int]]      # (u16 texels [h, w], leftoffset, topoffset); None: missing


# ---- loaders ---------------------------------------------------------------------------------------------------------
def grid_origin(wad: W.Archive, level_index: int) -> Tuple[int, int]:
    """the two int16 at the start of the lump at marker + 10 (ML_BLOCKMAP) when it is named BLOCKMAP and holds at least 8
    bytes inside the file; (0, 0) otherwise"""
    at = wad.levels[level_index] + 10
    if at < len(wad.lumps) and wad.lumps[at][0] == W.wad_name(b"BLOCKMAP") and wad.lumps[at][2] >= 8:
        try:
            raw = wad.read(at)
        except W.WadError:
            return 0, 0
        return int(np.frombuffer(raw[:2], "<i2")[0]), int(np.frombuffer(raw[2:4], "<i2")[0])
    return 0, 0


def digit_name(d: int) -> bytes:
    return b"AMMNUM%d" % d


def archive_digits(wad: W.Archive) -> List[Digit]:
    """AMMNUM0 .. AMMNUM9 by name (a later lump wins), decoded with their offsets; None when absent or not a picture"""
    out: List[Digit] = []
    for d in range(DIGITS):
        i = wad.named(digit_name(d))
        try:
            px, xo, yo = W.decode_picture(wad.read(i)) if i is not None else (None, 0, 0)
        except W.WadError:
            px = None
        out.append(None if px is None or px.size == 0 else (px, int(xo), int(yo)))
    return out


def image_digits(images) -> List[Digit]:
    """the digits of a scene from lumps: images {name: u16 texels [h, w]} (the b2d_textures entries; a later entry of a
    name wins) of the AMMNUM names, at offsets 0"""
    out: List[Digit] = []
    for d in range(DIGITS):
        px = images.get(digit_name(d))
        out.append(None if px is None or np.asarray(px).size == 0 else (np.asarray(px, np.uint16), 0, 0))
    return out


# ---- pixels ----------------------------------------------------------------------------------------------------------
def lattice(o: int) -> Tuple[int, int]:
    """[jlo, jhi]: every j whose line o + 128 j lies in [-32768, 32767]"""
    return -((o - GRID_MIN) // GRID_STEP), (GRID_MAX - o) // GRID_STEP


def mark_k(height: int) -> int:
    return max(1, height // 200)


def _frame_line_pixels(X0, Y0, X1, Y1, w, h):
    """the pixels of the C19 line rule (oracle/automap.py) that lie inside the frame: lines whose pixel box misses it are
    skipped, and the major range is narrowed, with a 2-pixel margin, to where the line's minor coordinate is on screen;
    each remaining pixel is computed and tested exactly"""
    if max(X0, X1) >> 8 < 0 or min(X0, X1) >> 8 >= w or max(Y0, Y1) >> 8 < 0 or min(Y0, Y1) >> 8 >= h:
        return []
    xmaj = abs(X1 - X0) >= abs(Y1 - Y0)
    M0, m0, M1, m1 = (X0, Y0, X1, Y1) if xmaj else (Y0, X0, Y1, X1)
    if M1 < M0:
        M0, m0, M1, m1 = M1, m1, M0, m0
    lo = -((128 - M0) // 256)
    hi = (M1 - 128) // 256
    if lo > hi:
        p = (X0 // 256, Y0 // 256)
        return [p] if 0 <= p[0] < w and 0 <= p[1] < h else []
    lo, hi = max(lo, 0), min(hi, (w if xmaj else h) - 1)
    if M1 != M0 and m1 != m0:                              # the major range whose minor lies within 2 pixels of the frame
        mlim = h if xmaj else w
        a = M0 + (-512 - m0) * (M1 - M0) / (m1 - m0)
        b = M0 + (mlim * 256 + 512 - m0) * (M1 - M0) / (m1 - m0)
        lo, hi = max(lo, int(min(a, b)) // 256 - 2), min(hi, int(max(a, b)) // 256 + 2)
    out = []
    for i in range(lo, hi + 1):
        c = 256 * i + 128
        v = m0 if M1 == M0 else (m0 * (M1 - M0) + (c - M0) * (m1 - m0)) // (M1 - M0)
        j = v // 256
        x, y = (i, j) if xmaj else (j, i)
        if 0 <= x < w and 0 <= y < h:
            out.append((x, y))
    return out


def automap(table: Sequence, thing_xy: Sequence, width: int, height: int, poses: np.ndarray, scale: int, flags: int,
            arrows=None, origin=(0, 0), digits: Optional[Sequence[Digit]] = None, marks=None) -> np.ndarray:
    """uint8 [n, height, width]: oracle/automap_states.py's automap of each pose (flags below GRID), with GRID the grid
    lines of `origin` (map units) in 104 under every item, and marks[f] (a list of (x, y, number): 16.16 map units, digit
    0..9; None: none) over everything in list order, each drawn with digits[number] magnified mark_k(height) times when
    its whole rectangle fits the frame."""
    assert A.SCALE_MIN <= scale <= A.SCALE_MAX and not flags & ~31
    items = AST.automap(table, thing_xy, width, height, poses, scale, flags & 7, arrows)
    out = np.zeros_like(items)
    k = mark_k(height)
    for f, p in enumerate(poses):
        px, py, angle = int(p["x"]), int(p["y"]), int(p["angle"]) & 0xFFFFFFFF
        rot = bool(flags & A.ROTATE)
        c, s = render.sincos_q30((0x40000000 - angle) & 0xFFFFFFFF)

        def mapped(mx, my):
            return A._screen(mx - px, my - py, rot, c, s, scale, width, height)

        frame = out[f]
        if flags & GRID:                                    # the grid, then C21's items over it (their colours are never 0)
            for vertical, o in ((True, int(origin[0])), (False, int(origin[1]))):
                jlo, jhi = lattice(o)
                for j in range(jlo, jhi + 1):
                    at = (o + GRID_STEP * j) << 16
                    P = mapped(at, GRID_MIN << 16) if vertical else mapped(GRID_MIN << 16, at)
                    Q = mapped(at, GRID_MAX << 16) if vertical else mapped(GRID_MAX << 16, at)
                    for (x, y) in _frame_line_pixels(P[0], P[1], Q[0], Q[1], width, height):
                        frame[y, x] = GRID_COLOUR
        drawn = items[f] != 0
        frame[drawn] = items[f][drawn]
        for (mx, my, number) in ([] if marks is None or marks[f] is None else marks[f]):
            d = None if digits is None else digits[int(number)]
            if d is None:
                continue
            px_, left_off, top_off = d
            X, Y = mapped(int(mx), int(my))
            left, top = (X >> 8) - k * left_off, (Y >> 8) - k * top_off
            dh, dw = px_.shape
            if left < 0 or top < 0 or left + k * dw > width or top + k * dh > height:
                continue
            for ty in range(dh):
                for tx in range(dw):
                    t = int(px_[ty, tx])
                    if t >> 8 == 0:
                        frame[top + k * ty:top + k * ty + k, left + k * tx:left + k * tx + k] = t
    return out
