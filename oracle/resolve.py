"""ORACLE (test infrastructure): numpy restatement of C17, the resolve of index frames (DESIGN.md §4).

Output pixel (x, y), channel c, of frame f on level l = levels[f] at factor k:

    out_c = (sum_{i,j < k} T_l[idx[f][k*y + j][k*x + i]].c + k*k // 2) // (k*k)

with T_l level l's PLAYPAL[0] (R, G, B) for the colour formats and the luma Y = (77 R + 150 G + 29 B + 128) >> 8 of each
entry for grey.  Integer arithmetic throughout."""
from __future__ import annotations

import numpy as np

FORMATS = ("rgba", "rgb", "rgb_planar", "gray")


def palette_rgb(playpal) -> np.ndarray:
    """(256, 3) int32 R, G, B of a PLAYPAL (768 bytes, or anything shaped (256, 3))."""
    if isinstance(playpal, (bytes, bytearray)):
        playpal = np.frombuffer(bytes(playpal)[:768], np.uint8)
    return np.asarray(playpal, dtype=np.int32).reshape(256, 3)


def luma(playpal) -> np.ndarray:
    """(256,) int32 grey table: Y = (77 R + 150 G + 29 B + 128) >> 8 per palette entry."""
    p = palette_rgb(playpal)
    return (77 * p[:, 0] + 150 * p[:, 1] + 29 * p[:, 2] + 128) >> 8


def resolve(index: np.ndarray, playpals, factor: int, fmt: str, levels=None) -> np.ndarray:
    """The C17 resolve of (n, H, W) uint8 index frames; playpals[l] is level l's PLAYPAL, levels[f] the level of frame f
    (None: level 0).  Returns rgba: uint32 (n, H/k, W/k) packed R | G<<8 | B<<16 | 0xFF<<24; rgb: uint8 (n, H/k, W/k, 3);
    rgb_planar: uint8 (n, 3, H/k, W/k); gray: uint8 (n, H/k, W/k)."""
    index = np.asarray(index, dtype=np.uint8)
    n, h, w = index.shape
    k = int(factor)
    assert 1 <= k <= 8 and h % k == 0 and w % k == 0, "factor must be in 1..8 and divide the frame's sides"
    assert fmt in FORMATS, fmt
    lv = np.zeros(n, np.int64) if levels is None else np.asarray(levels, dtype=np.int64).reshape(n)
    tables = [luma(p)[:, None] if fmt == "gray" else palette_rgb(p) for p in playpals]
    chans = 1 if fmt == "gray" else 3
    sums = np.empty((n, h // k, w // k, chans), np.int32)          # at most 64 * 255 per channel
    for f in range(n):
        v = tables[int(lv[f])][index[f]]                                  # (H, W, chans)
        sums[f] = v.reshape(h // k, k, w // k, k, chans).sum(axis=(1, 3))
    out = ((sums + k * k // 2) // (k * k)).astype(np.uint8)
    if fmt == "gray":
        return out[..., 0]
    if fmt == "rgb":
        return out
    if fmt == "rgb_planar":
        return np.ascontiguousarray(out.transpose(0, 3, 1, 2))
    o = out.astype(np.uint32)
    return o[..., 0] | (o[..., 1] << 8) | (o[..., 2] << 16) | np.uint32(0xFF000000)
