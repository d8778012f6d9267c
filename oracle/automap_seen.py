"""Seen-automap oracle (DESIGN.md C20), test infrastructure: Doom's AM_drawWalls with mapped lines, restated on top of
oracle/automap.py.  Each line of a frame gets its colour from the frame's mapped row, then oracle/automap.py draws the
frame with that colour as the line's only one.  Independent of libb2d."""
import numpy as np

from oracle import automap as A
from oracle import wad as W

ALLMAP, ALLMAP_COLOUR = 8, 99


def dontdraw(level: W.Level):
    """{linedef: True} for the level's ML_DONTDRAW linedefs"""
    return {i: bool(int(l["flags"]) & A.ML_DONTDRAW) for i, l in enumerate(level.linedefs)}


def line_colour(line, hidden: bool, mapped: bool, flags: int) -> int:
    """AM_drawWalls: all lines (IDDT) -> colour_all; mapped -> colour; computer area map and not don't-draw -> 99; else 0"""
    colour, colour_all = line[4], line[5]
    if flags & A.ALL_LINES:
        return colour_all
    if mapped:
        return colour
    if flags & ALLMAP and not hidden:
        return ALLMAP_COLOUR
    return 0


def automap(table, hidden, thing_xy, width: int, height: int, poses: np.ndarray, scale: int, flags: int, mapped=None) -> np.ndarray:
    """uint8 [n, height, width]: frame f's automap with its lines coloured by row f of `mapped` (uint32 words, bit l & 31
    of word l >> 5 for linedef l; None: every line mapped); `hidden` from dontdraw()"""
    assert not flags & ~15
    out = np.zeros((len(poses), height, width), np.uint8)
    for f in range(len(poses)):
        row = None if mapped is None else np.asarray(mapped[f], np.uint32)

        def is_mapped(ld):
            return row is None or bool((int(row[ld >> 5]) >> (ld & 31)) & 1)

        t = []
        for line in table:
            c = line_colour(line, hidden[line[6]], is_mapped(line[6]), flags)
            t.append(line[:4] + (c, c, line[6]))
        out[f:f + 1] = A.automap(t, thing_xy, width, height, poses[f:f + 1], scale, flags & (A.ROTATE | A.THINGS))
    return out
