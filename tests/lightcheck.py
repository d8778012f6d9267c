"""Test reference for the player's light effects (DESIGN.md C18), built on the oracle as it is: oracle/b2d_oracle.c,
oracle/render.py and oracle/scene.py know nothing of fixed colormaps or extra light, so both effects are restated here as
changes of the scene and of the oracle's per-sector light overrides.

* Extra light e: apply_extralight rewrites the static light bytes of the scene (sectors without a light effect, their
  segs and their sprites) as C12 gives them at `light >> 3` + 2e steps, and sector_lights_at gives the bytes of the
  sectors with a light effect, clamp(level_at(t) + f32(2e) / f32(31)) * 255; the oracle renders that scene with those
  overrides (its own b2o_render_t entry point).
* Fixed colormap r: off the sky, the frame of the scene whose COLORMAP rows 0..31 are all row r (the blob keeps 34 rows,
  so r = 32 is INVERSECOLORMAP); on the sky, the normal frame.  The sky pixels are found by rendering the scene with every
  texel of its sky texture set to 1, every other texture and flat texel to 2 (opacity masks kept) and identity rows.
"""
import ctypes

import numpy as np

from oracle import render as R
from oracle import scene as S

f32 = np.float32


def light_byte_steps(steps: int, contrast: int) -> int:
    """C12's static light byte with the level given in steps of 1/31 (a SECTORS light >> 3): light.rs:82-115 and
    lights.rs:26-29, float32 operation by operation"""
    level = f32(steps) / f32(31.0)
    if contrast:
        level = level + (f32(2.0) / f32(31.0) if contrast > 0 else f32(-2.0) / f32(31.0))
        level = f32(1.0) if level > f32(1.0) else (f32(0.0) if level < f32(0.0) else level)
    level = f32(1.0) if level > f32(1.0) else (f32(0.0) if level < f32(0.0) else level)
    v = float(level * f32(255.0))
    return int(v) & 0xFF if v >= 0 else 0


def light_byte_at(info, tics: int, extralight: int) -> int:
    """the byte of a sector with a light effect at `tics` with extra light: lights.rs:26-30 with f32(2e) / f32(31) added to
    the level before the clamp"""
    with np.errstate(all="ignore"):
        time = f32(f32(int(tics) & 0xFFFFFFFF) / f32(35.0))
        v = S.light_level_at(info, time)
        if extralight:
            v = f32(v + f32(f32(2 * extralight) / f32(31.0)))
        v = f32(0.0) if v < f32(0.0) else (f32(1.0) if v > f32(1.0) else v)
        r = float(f32(v * f32(255.0)))
    return int(r) & 0xFF if r >= 0 else 0


def _lights(blob: bytes) -> np.ndarray:
    h = S.header(blob)
    n = h[S.H_NSECTORS]
    return np.frombuffer(blob, dtype="<u4", count=8 * n, offset=h[S.H_OFF_LIGHTS]).reshape(n, 8)


def sector_lights_at(blob: bytes, tics: int, extralight: int = 0) -> np.ndarray:
    """int16 per sector: the byte at `tics` with `extralight` of a sector with a light effect, -1 for the others"""
    rec = _lights(blob)
    out = np.full(len(rec), -1, dtype=np.int16)
    for i in range(len(rec)):
        if rec[i, 0] != S.LIGHT_NONE:
            fl = rec[i, 1:6].copy().view("<f4")
            out[i] = light_byte_at((int(rec[i, 0]), fl[0], fl[1], fl[2], fl[3], fl[4]), tics, extralight)
    return out


def apply_extralight(blob: bytes, extralight: int) -> bytes:
    """The scene with its static light bytes raised by `extralight` (0..2) steps of Doom's 16-level scale: every sector
    without a light effect, its segs and its sprites lit as if its SECTORS light were light + 16 e.  A sector's
    `light >> 3` is its lights record's level * 31 (the record holds (light >> 3) / 31 for every sector); a seg's fake
    contrast follows from its vertices as the scene compiler derives it (visitor.rs:887-901)."""
    e = int(extralight)
    if e == 0:
        return blob
    h = S.header(blob)
    out = bytearray(blob)
    rec = _lights(blob)
    n = len(rec)
    effect = rec[:, 0] != S.LIGHT_NONE
    steps = [int(round(float(v) * 31.0)) for v in rec[:, 1].copy().view("<f4")]
    sectors = S.section(blob, "sectors").copy()
    for i in range(n):
        if not effect[i]:
            sectors[i, 4] = light_byte_steps(steps[i] + 2 * e, 0)
    verts = S.section(blob, "verts")
    segs = S.section(blob, "segs").copy()
    for seg in segs:
        f = int(seg[2])
        if seg[3] & S.SEG_INVALID or not 0 <= f < n or effect[f]:
            continue
        dx = int(verts[seg[1], 0]) - int(verts[seg[0], 0])
        dy = int(verts[seg[1], 1]) - int(verts[seg[0], 1])
        seg[12] = light_byte_steps(steps[f] + 2 * e, 1 if dy == 0 else (-1 if dx == 0 else 0))
    sprites = S.section(blob, "sprites").copy()
    for p in sprites:
        if 0 <= int(p[5]) < n and not effect[p[5]]:
            p[4] = light_byte_steps(steps[p[5]] + 2 * e, 0)
    for off, a in ((h[S.H_OFF_SECTORS], sectors), (h[S.H_OFF_SEGS], segs), (h[S.H_OFF_SPRITES], sprites)):
        data = a.astype("<i4").tobytes()
        out[off:off + len(data)] = data
    return bytes(out)


def tables_at(blob: bytes, tics: int, moves=(), extralight: int = 0) -> bytes:
    """oracle/scene.py tables_at with extra light: the tables of apply_extralight's scene, with the bytes of the sectors
    with a light effect (and of their segs and sprites) those of sector_lights_at with the same extra light"""
    t = bytearray(S.tables_at(apply_extralight(blob, extralight), tics, moves))
    if not extralight:
        return bytes(t)
    h = S.header(blob)
    ntex, n, nseg, nspr = h[S.H_NTEX], h[S.H_NSECTORS], h[S.H_NSEGS], h[S.H_NSPRITES]
    sectors = np.frombuffer(t, "<i4", 8 * n, 32 * ntex).reshape(n, 8).copy()
    segs = np.frombuffer(t, "<i4", 16 * nseg, 32 * ntex + 32 * n).reshape(nseg, 16).copy()
    sprites = np.frombuffer(t, "<i4", 8 * nspr, 32 * ntex + 32 * n + 64 * nseg).reshape(nspr, 8).copy()
    lights = sector_lights_at(blob, tics, extralight)
    effect = lights >= 0
    sectors[effect, 4] = lights[effect]
    for seg in segs:
        if not seg[3] & S.SEG_INVALID and 0 <= seg[2] < n and effect[seg[2]]:
            seg[12] = lights[seg[2]]
    for p in sprites:
        if 0 <= p[5] < n and effect[p[5]]:
            p[4] = lights[p[5]]
    at = 32 * ntex
    for a in (sectors, segs, sprites):
        data = a.astype("<i4").tobytes()
        t[at:at + len(data)] = data
        at += len(data)
    return bytes(t)


def with_colormap_rows(blob: bytes, row: int) -> bytes:
    """the scene with COLORMAP rows 0..31 all replaced by row `row` (of the 34 the blob keeps)"""
    off = S.header(blob)[S.H_OFF_COLORMAP]
    out = bytearray(blob)
    r = blob[off + 256 * row: off + 256 * row + 256]
    for k in range(32):
        out[off + 256 * k: off + 256 * k + 256] = r
    return bytes(out)


def sky_mask(blob: bytes, view, poses, tics: int = 0) -> np.ndarray:
    """the sky pixels of the frames, found without any light rule: every texel of the sky texture becomes 1 and every
    other texture and flat texel 2 (opacity masks kept), with COLORMAP rows 0..31 the identity.  (A wall that uses the sky
    texture would count as sky; the scenes this is used on have none.)"""
    h = S.header(blob)
    out = bytearray(blob)
    texels, flats, cm = h[S.H_OFF_TEXELS], h[S.H_OFF_FLATS], h[S.H_OFF_COLORMAP]
    sky = h[S.H_SKY_TEX]
    for i, t in enumerate(S.section(blob, "textures")):
        at, n = texels + int(t[0]), int(t[1]) * int(t[2])
        out[at:at + n] = bytes([1 if i == sky else 2]) * n
    out[flats:flats + 4096 * h[S.H_NFLATS]] = b"\x02" * (4096 * h[S.H_NFLATS])
    for k in range(32):
        out[cm + 256 * k: cm + 256 * k + 256] = bytes(range(256))
    return R.render(bytes(out), view, poses, tics=tics) == 1


def _render_lit(blob: bytes, view, poses, tics: int, extralight: int) -> np.ndarray:
    """the oracle's frames of apply_extralight's scene with sector_lights_at's overrides (b2o_render_t)"""
    poses = np.ascontiguousarray(poses, dtype=R.POSE)
    lit = apply_extralight(blob, extralight)
    buf = (ctypes.c_char * len(lit)).from_buffer_copy(lit)
    ov = np.ascontiguousarray(sector_lights_at(blob, tics, extralight), dtype=np.int16)
    fb = np.empty((len(poses), view.H, view.W), dtype=np.uint8)
    rc = R.lib().b2o_render_t(ctypes.addressof(buf), ctypes.byref(view), poses.ctypes.data, len(poses), int(tics) & 0xFFFFFFFF,
                              ov.ctypes.data if len(ov) else None, fb.ctypes.data, None, None, 1)
    if rc != 0:
        raise RuntimeError("b2o_render_t failed: %d" % rc)
    return fb


def render(blob: bytes, view, poses, tics: int = 0, fixed_colormap: int = -1, extralight: int = 0) -> np.ndarray:
    """(n, H, W) index frames of `poses` with the player's light effects of C18"""
    if not -1 <= fixed_colormap <= 32 or not 0 <= extralight <= 2:
        raise ValueError("fixed_colormap takes -1..32 and extralight 0..2")
    if fixed_colormap < 0:
        return _render_lit(blob, view, poses, tics, extralight) if extralight else R.render(blob, view, poses, tics=tics)
    flat = R.render(with_colormap_rows(blob, fixed_colormap), view, poses, tics=tics)
    normal = R.render(blob, view, poses, tics=tics)
    return np.where(sky_mask(blob, view, poses, tics), normal, flat)
