"""Seen-lines oracle (DESIGN.md C20), test infrastructure: the segs that own a column of each frame, from
oracle/b2d_seen.c (the oracle rasteriser's walk and clip loop without drawing), and the rows of linedef bits they make
through the level's SEGS lump as oracle/wad.py reads it.  Independent of libb2d.

`python -m oracle.seen` compiles oracle/b2d_seen.c into oracle/libb2d_seen.so with oracle/build.py's compiler flags."""
import ctypes
import os
import subprocess
import sys

import numpy as np

from oracle import build as _build
from oracle import render
from oracle import wad as W

SRC = os.path.join(_build.HERE, "b2d_seen.c")
OUT = os.path.join(_build.HERE, "libb2d_seen.so")
HOST = OUT + ".host"


def build(force: bool = False) -> str:
    """Compiled for the host that runs it, and rebuilt when it or the rasteriser it includes changed (as oracle/build.py)."""
    fresh = (os.path.exists(OUT) and os.path.getmtime(OUT) >= max(os.path.getmtime(SRC), os.path.getmtime(_build.SRC)))
    if not force and fresh:
        try:
            with open(HOST) as f:
                if f.read().strip() == _build.host_signature():
                    return OUT
        except OSError:
            pass
    subprocess.check_call(["gcc"] + _build.FLAGS + ["-o", OUT, SRC])
    with open(HOST, "w") as f:
        f.write(_build.host_signature() + "\n")
    return OUT


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(build())
        L.b2o_seen.argtypes = [ctypes.c_void_p, ctypes.POINTER(render.View), ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        L.b2o_seen.restype = ctypes.c_int
        _lib = L
    return _lib


def seg_owned(blob: bytes, view: render.View, poses: np.ndarray) -> np.ndarray:
    """bool [n, n_segs]: seg s owns at least one column of frame i in the solid pass of the compiled scene `blob` (a
    state's blob for a frame at that state)"""
    poses = np.ascontiguousarray(poses, dtype=render.POSE)
    n = len(poses)
    nsegs = int(np.frombuffer(blob, dtype="<u4", count=32)[6])
    owned = np.zeros((n, nsegs), dtype=np.uint8)
    buf = (ctypes.c_char * len(blob)).from_buffer_copy(blob)
    rc = lib().b2o_seen(ctypes.addressof(buf), ctypes.byref(view), poses.ctypes.data, n, owned.ctypes.data)
    if rc != 0:
        raise RuntimeError("b2o_seen failed: %d" % rc)
    return owned.astype(bool)


def seen_lines(level: W.Level, seg_owned_rows: np.ndarray, words: int) -> np.ndarray:
    """uint32 [n, words]: bit l & 31 of word l >> 5 of row i set for linedef l of every seg frame i owns; segs whose
    linedef is not in LINEDEFS set nothing"""
    owned = np.atleast_2d(np.asarray(seg_owned_rows, dtype=bool))
    out = np.zeros((len(owned), words), dtype=np.uint32)
    line = np.asarray(level.segs["linedef"], dtype=np.int64)
    nlines = len(level.linedefs)
    for i, row in enumerate(owned):
        for l in np.unique(line[:len(row)][row]):
            if l < nlines:
                out[i, l >> 5] |= np.uint32(1 << (int(l) & 31))
    return out


def words_for(levels) -> int:
    """the length of a row of seen lines for a set of oracle/wad.py levels: the largest ceil(n_linedefs / 32), at least 1"""
    return max([1] + [(len(lv.linedefs) + 31) // 32 for lv in levels])


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
