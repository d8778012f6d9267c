"""ORACLE (test infrastructure): level lumps + texture directory -> compiled scene blob.

Restates which surfaces a level contributes and how they are textured and lit, following the
reference's one-and-only geometry emitter `LevelWalker` and its visitor in `game/`:

* seg -> wall pieces, pegging, offsets        wad/src/visitor.rs:711-937
* fake contrast + static light byte           wad/src/visitor.rs:887-901, wad/src/light.rs:27-115,
                                              game/src/lights.rs:14-30
* flats / sky flats                           wad/src/visitor.rs:939-985, wad/src/util.rs:8-10
* player-1 start marker, sector_at            wad/src/visitor.rs:1010-1060, game/src/level.rs:757-762,
                                              game/src/player.rs:72-92 (camera_height)
* sky texture per level                       wad/src/meta.rs:156-172, assets/meta/doom.toml:29-68

The blob layout ("B2DS" v6) is the contract shared with the product's scene compiler
(rust-doom_b200/csrc/b2d_scene.cpp, written independently); tests compare the two byte-for-byte.
All fields are little-endian int32 unless noted.

header  : 64 x u32 (see H_* indices below)
verts   : {x, y}                                                   8 B
nodes   : {x, y, dx, dy, rbox[4], lbox[4], rchild, lchild, 0, 0}   64 B  (box = top,bottom,left,right;
          child bit31 = subsector)
ssectors: {first_seg, num_segs, sector, sprites}                   16 B  (sprites = first | count<<24)
sprites : {x, y, low, tex, light, sector, hanging, 0}                 32 B  decoration things grouped by subsector:
          billboard of the sprite image's size standing on the floor / hanging from the ceiling
          (visitor.rs:1062-1137), lit by the sector light without contrast
segs    : {v1, v2, front, flags, uoff, len_q12, texA, tA, hA, texB, tB, hB, light, otop, obot, mid}   64 B
          (mid = index into mids or -1)
mids    : {tex, t_high, low, high, 0, 0, 0, 0}                     32 B  masked two-sided middle texture:
          vertical extent [low, high) in map units and the texture row at `high` (visitor.rs:808-836,875-919)
sectors : {floor, ceil, floor_flat, ceil_flat, light, 0, 0, 0}     32 B  (flat: >=0 id, -1 sky, -2 missing)
textures: {texel_off, w, h, hmagic, hbias, mask_off, anim_first, anim_nk}  32 B  (mask_off = 0xFFFFFFFF: opaque;
          anim_nk = n | k<<16: this texture is frame k of an n-frame animation whose texture ids are
          anim[anim_first .. +n); n = 0: not animated)
anim    : i32 ids (texture ids, then flat ids) of animation frames, group by group
flatanim: {anim_first, anim_nk} per flat                           8 B
lights  : {kind, level, alt, speed, duration, sync, 0, 0} per sector  32 B  (kind u32: 0 none, 1 glow, 2 random,
          3 alternate; the rest float32: light.rs:27-80); the `light` fields above hold the value at tic 0
texels  : u8 row-major, textures back to back (transparent texels stored as 0); a texture with holes is
          followed by its opacity plane (1 = opaque), same layout, at mask_off
flats   : n x 4096 u8
colormap: 34 x 256 u8 (zero padded if the WAD has fewer)
palette : 256 x u32  R | G<<8 | B<<16 | 0xFF<<24  from PLAYPAL[0]
segdyn  : {back, bits} per seg                                     8 B   what apply_moves needs beyond the seg record:
          back sector (-1 one-sided), bits 1 = lower-unpegged line, 2 = the back ceiling is sky
dyn     : {sector, floor_min, floor_max, ceil_min, ceil_max, 0, 0, 0}  32 B  the sectors that may move and the height
          ranges the host's LevelAnalysis found for them (visitor.rs:146-245)

Moving sectors (doors, lifts; DESIGN.md C16).  The reference attaches every wall quad, flat and decoration to the floor or
ceiling *object* of a sector and translates it rigidly with that object's height offset (visitor.rs:733-836 object_id;
game/src/level.rs:201-245); quads next to a dynamic sector are pre-extended over the sector's height range so that
nothing opens up while it moves.  Here the same rule is applied to the per-seg pieces: `compile_scene(dynamic=...)`
resolves, for segs that touch a declared sector, the pieces that can come into existence while it moves, and
`apply_moves` re-derives the height-dependent records for one state (a floor and a ceiling offset per declared sector).
"""
from __future__ import annotations

import math
import re
import struct
from typing import Dict, List, Tuple

import numpy as np

from . import wad as W

MAGIC = 0x53443242
VERSION = 6
HEADER_WORDS = 64
(H_MAGIC, H_VERSION, H_TOTAL, H_NVERTS, H_NNODES, H_NSSECTORS, H_NSEGS, H_NSECTORS, H_NTEX, H_NFLATS,
 H_OFF_VERTS, H_OFF_NODES, H_OFF_SSECTORS, H_OFF_SEGS, H_OFF_SECTORS, H_OFF_TEX, H_OFF_TEXELS,
 H_TEXEL_BYTES, H_OFF_FLATS, H_OFF_COLORMAP, H_OFF_PALETTE, H_ROOT, H_SKY_TEX, H_START_X, H_START_Y,
 H_START_Z, H_START_ANGLE, H_HAS_START, H_MIN_H, H_MAX_H, H_NMIDS, H_OFF_MIDS, H_NSPRITES, H_OFF_SPRITES, H_NANIM, H_OFF_ANIM, H_OFF_FLAT_ANIM,
 H_OFF_LIGHTS, H_NDYN, H_OFF_DYN, H_OFF_SEGDYN) = range(41)

SEGDYN_UNPEG_LOWER = 1
SEGDYN_BACK_SKY = 2

SEG_TWO_SIDED = 1
SEG_SCROLL = 2            # linedef special 0x30: texture scrolls 35 units/s along s (visitor.rs:922)
SEG_INVALID = 0x80
LEAF = 0x80000000

LIGHT_NONE, LIGHT_GLOW, LIGHT_RANDOM, LIGHT_ALTERNATE = 0, 1, 2, 3

FLAT_SKY = -1
FLAT_MISSING = -2
TEX_NONE = -1

# assets/meta/doom.toml:29-68 (first regex match wins, fallback = entry 0)
SKY_TABLE = [
    (r"E1M.", b"SKY1"), (r"E2M.", b"SKY2"), (r"E3M.", b"SKY3"), (r"E4M.", b"SKY4"),
    (r"MAP(0[1-9]|10|11)", b"SKY1"), (r"MAP(1[2-9]|20)", b"SKY2"), (r"MAP(2[1-9]|32)", b"SKY3"),
]


def sky_for(level_name: bytes) -> bytes:
    s = level_name.rstrip(b"\0").decode("ascii")
    for pat, tex in SKY_TABLE:
        if re.search(pat, s):          # regex `is_match` = unanchored search
            return W.wad_name(tex)
    return W.wad_name(SKY_TABLE[0][1])


def _align16(n: int) -> int:
    return (n + 15) & ~15


def _floormod(a: int, b: int) -> int:
    return a - b * (a // b)


def sector_at(level: W.Level, x: float, y: float) -> int:
    return subsector_at(level, x, y)[1]


def subsector_at(level: W.Level, x: float, y: float):
    """LevelWalker::sector_at (visitor.rs:1028-1060).  Returns (subsector id, sector id) or (-1, -1).  Works
    in WAD coordinates; the reference's `signed_distance` sign is (py-oy)*dx - (px-ox)*dy > 0 => left."""
    r = _subsector_at(level, x, y)
    return r if r[1] >= 0 else (-1, -1)


def _subsector_at(level: W.Level, x: float, y: float):
    if len(level.nodes) == 0:
        return -1, -1
    child = len(level.nodes) - 1
    leaf = False
    for _ in range(4096):
        if leaf:
            break
        n = level.nodes[child]
        sd = (y - float(n["y"])) * float(n["dx"]) - (x - float(n["x"])) * float(n["dy"])
        nxt = int(n["left"]) if sd > 0.0 else int(n["right"])
        child, leaf = nxt & 0x7FFF, bool(nxt & 0x8000)
        if not leaf and child >= len(level.nodes):
            return -1, -1
    if not leaf or child >= len(level.subsectors):
        return -1, -1
    ss = level.subsectors[child]
    first, num = int(ss["first_seg"]), int(ss["num_segs"])
    if num == 0 or first + num > len(level.segs):
        return -1, -1
    segs = level.segs[first:first + num]
    side = level.seg_sidedef_index(segs[0])
    if side < 0:
        return -1, -1
    sector = int(level.sidedefs[side]["sector"])
    if sector >= len(level.sectors):
        return -1, -1
    for s in segs:
        if s["v1"] >= len(level.vertices) or s["v2"] >= len(level.vertices):
            continue
        a, b = level.vertices[s["v1"]], level.vertices[s["v2"]]
        dx, dy = float(b["x"]) - float(a["x"]), float(b["y"]) - float(a["y"])
        ln = math.hypot(dx, dy)
        if ln < 1e-14:
            continue
        sd = ((y - float(a["y"])) * dx - (x - float(a["x"])) * dy) / ln
        if sd > 10.0:                       # SEG_TOLERANCE = 0.1 world units = 10 map units
            return -1, -1
    return child, sector


_f = np.float32


def _f32bits(v) -> int:
    return int(np.array([v], dtype="<f4").view("<u4")[0])


def light_info(level: "W.Level", i: int) -> Tuple[int, np.float32, np.float32, np.float32, np.float32, np.float32]:
    """wad/src/light.rs:27-115 new_light: (kind, level, alt_level, speed, duration, sync), all float32."""
    s = level.sectors[i]
    base = _f(np.int16(s["light"]) >> 3) / _f(31.0)
    stype = int(s["type"])
    none = (LIGHT_NONE, base, _f(0), _f(0), _f(0), _f(0))
    if stype not in W.EFFECT_TYPES:
        return none
    alt = _f(np.int16(level.sector_min_light(i)) >> 3) / _f(31.0)
    if abs(alt - base) < _f(1.1920929e-07):                         # f32::EPSILON
        return none
    if stype in (12, 13, 8):                                         # SLOW_STROBE_SYNC, FAST_STROBE_SYNC, GLOW
        sync = _f(0.0)
    else:                                                            # id_to_sync, light.rs:109-111
        sync = _f(((i * 1664525 + 1013904223) & 0xFFFF)) / _f(15.0)
    kind, speed, duration = {
        1: (LIGHT_RANDOM, 20.0, 0.06), 17: (LIGHT_RANDOM, 8.0, 0.5),
        3: (LIGHT_ALTERNATE, 1.0, 0.85), 12: (LIGHT_ALTERNATE, 1.0, 0.85),
        2: (LIGHT_ALTERNATE, 2.0, 0.7), 4: (LIGHT_ALTERNATE, 2.0, 0.7), 13: (LIGHT_ALTERNATE, 2.0, 0.7),
        8: (LIGHT_GLOW, 0.5, 0.0)}[stype]
    return (kind, base, alt, _f(speed), _f(duration), sync)


def _fract(x: np.float32) -> np.float32:
    return _f(x - np.floor(x))


def _sin_f32(x: np.float32) -> np.float32:
    """The correctly rounded float32 sine (double-precision sine, rounded once): DESIGN.md C15."""
    return _f(math.sin(float(x)))


def light_level_at(info, time: np.float32) -> np.float32:
    """game/src/lights.rs:33-66, float32 operation by operation."""
    kind, level, alt, speed, duration, sync = info
    if kind == LIGHT_NONE:
        return level
    if kind == LIGHT_GLOW:
        scale = _f(level - alt)
        phase = _f(_f(time * speed) / scale)
        return _f(_f(_f(abs(_f(_f(0.5) - _fract(phase))) * _f(2.0)) * scale) + alt)
    if kind == LIGHT_RANDOM:
        t = np.floor(_f(time * speed))
        arg = _f(_f(_f(sync + _f(t / _f(1000.0))) * _f(12.9898)) + _f(sync * _f(78.233)))
        noise = _fract(_f(_f(1.0) + _f(_sin_f32(arg) * _f(43758.547))))
        return alt if noise < duration else level
    ph = _fract(_f(_f(time * speed) + _f(sync * _f(3.5435))))
    return alt if ph < duration else level


def light_byte_at(info, tics: int) -> int:
    """lights.rs:26-30: (clamp(level_at(time)) * 255.0) as u8 with time = tics / 35 seconds."""
    with np.errstate(all="ignore"):
        time = _f(_f(int(tics) & 0xFFFFFFFF) / _f(35.0))
        v = light_level_at(info, time)
        v = _f(0.0) if v < _f(0.0) else (_f(1.0) if v > _f(1.0) else v)
        r = float(_f(v * _f(255.0)))
    return int(r) & 0xFF if r >= 0 else 0


def sector_lights_at(blob: bytes, tics: int) -> np.ndarray:
    """int16 per sector: the light byte at `tics` for sectors with a light effect, -1 for the others."""
    h = header(blob)
    n = h[H_NSECTORS]
    rec = np.frombuffer(blob, dtype="<u4", count=8 * n, offset=h[H_OFF_LIGHTS]).reshape(n, 8)
    out = np.full(n, -1, dtype=np.int16)
    for i in range(n):
        if rec[i, 0] != LIGHT_NONE:
            fl = rec[i, 1:6].copy().view("<f4")
            out[i] = light_byte_at((int(rec[i, 0]), fl[0], fl[1], fl[2], fl[3], fl[4]), tics)
    return out


def compile_scene(archive: W.Archive, tex: W.TextureDirectory, level_index: int, dynamic=()) -> bytes:
    """`dynamic`: (sector, floor_min, floor_max, ceil_min, ceil_max) per sector that may move (the ranges are widened to
    contain the sector's own heights, like visitor.rs:232-245 merge_range)."""
    level = W.Level(archive, level_index)
    nverts, nsegs = len(level.vertices), len(level.segs)
    nsect, nss, nnodes = len(level.sectors), len(level.subsectors), len(level.nodes)
    dyn: Dict[int, Tuple[int, int, int, int]] = {}
    for d in dynamic:
        sec, fmin, fmax, cmin, cmax = (int(v) for v in d)
        if not 0 <= sec < nsect or sec in dyn:
            raise W.WadError("dynamic sector %d: out of range or listed twice" % sec)
        f0, c0 = int(level.sectors[sec]["floor"]), int(level.sectors[sec]["ceil"])
        dyn[sec] = (min(fmin, fmax, f0), max(fmin, fmax, f0), min(cmin, cmax, c0), max(cmin, cmax, c0))

    def floor_range(sec: int) -> Tuple[int, int]:
        f0 = int(level.sectors[sec]["floor"])
        return dyn[sec][0:2] if sec in dyn else (f0, f0)

    def ceil_range(sec: int) -> Tuple[int, int]:
        c0 = int(level.sectors[sec]["ceil"])
        return dyn[sec][2:4] if sec in dyn else (c0, c0)

    # --- texture / flat id assignment in first-use order -------------------------------------
    tex_ids: Dict[bytes, int] = {}
    tex_list: List[np.ndarray] = []

    from .anim_table import FLATS as ANIM_FLATS, WALLS as ANIM_WALLS
    anim_frames: List[int] = []                 # texture ids group by group, then (offset) flat ids
    tex_anim: Dict[int, Tuple[int, int, int]] = {}      # tex id -> (first, n, k)
    flat_anim: Dict[int, Tuple[int, int, int]] = {}

    def _group_of(name: bytes, groups):
        s = name.rstrip(b"\0").decode("ascii")
        for g in groups:
            if s in g:
                return g
        return None

    def tex_id(name: bytes, _follow=True) -> int:
        if W.is_untextured(name):
            return TEX_NONE
        if name in tex_ids:
            return tex_ids[name]
        img = tex.textures.get(name)
        if img is None or img.shape[0] == 0 or img.shape[1] == 0:
            return TEX_NONE                           # visitor.rs:857-860: skip + warn
        tex_ids[name] = len(tex_list)
        tex_list.append(img)
        tid = tex_ids[name]
        g = _group_of(name, ANIM_WALLS) if _follow else None
        if g is not None:
            # all existing frames of the animation, in group order (tex.rs:421-473, static.vert:23-39)
            ids = [tex_id(W.wad_name(n.encode()), False) for n in g]
            ids = [i for i in ids if i >= 0]
            if len(ids) > 1:
                first = len(anim_frames)
                anim_frames.extend(ids)
                for k, i in enumerate(ids):
                    tex_anim[i] = (first, len(ids), k)
        return tid

    sky_tex = tex_id(sky_for(level.name))

    flat_ids: Dict[bytes, int] = {}
    flat_list: List[bytes] = []

    flat_groups: List[List[int]] = []

    def flat_id(name: bytes, _follow=True) -> int:
        if W.is_sky_flat(name):
            return FLAT_SKY
        if name in flat_ids:
            return flat_ids[name]
        data = tex.flats.get(name)
        if data is None or len(data) < 4096:
            return FLAT_MISSING
        flat_ids[name] = len(flat_list)
        flat_list.append(data[:4096])
        fid = flat_ids[name]
        g = _group_of(name, ANIM_FLATS) if _follow else None
        if g is not None:
            ids = [flat_id(W.wad_name(n.encode()), False) for n in g]
            ids = [i for i in ids if i >= 0]
            if len(ids) > 1:
                flat_groups.append(ids)
        return fid

    def raw_name(arr, i, field) -> bytes:
        dt = arr.dtype
        off = dt.fields[field][1]
        b = arr.tobytes()[i * dt.itemsize + off:i * dt.itemsize + off + 8]
        return W.wad_name(b)

    # --- sectors --------------------------------------------------------------------------------
    sectors = np.zeros((nsect, 8), dtype=np.int32)
    sec_bytes = level.sectors.tobytes()
    has_effect = []
    lights = np.zeros((nsect, 8), dtype="<u4")     # {kind, level, alt, speed, duration, sync (f32 bits), 0, 0}
    sector_light0 = []                             # light byte at tic 0 (effects evaluated, lights.rs:26-30)
    for i in range(nsect):
        s = level.sectors[i]
        fname = W.wad_name(sec_bytes[i * 26 + 4:i * 26 + 12])
        cname = W.wad_name(sec_bytes[i * 26 + 12:i * 26 + 20])
        info = light_info(level, i)
        has_effect.append(info[0] != LIGHT_NONE)
        lights[i, 0] = info[0]
        lights[i, 1:6] = [_f32bits(v) for v in info[1:]]
        sector_light0.append(light_byte_at(info, 0) if has_effect[i] else W.light_byte(int(s["light"]), 0))
        sectors[i] = [int(s["floor"]), int(s["ceil"]), flat_id(fname), flat_id(cname),
                      sector_light0[i], 0, 0, 0]
    if nsect:
        min_h = int(level.sectors["floor"].min()) - 512      # visitor.rs:1173-1182
        max_h = int(level.sectors["ceil"].max()) + 512
    else:
        min_h, max_h = -512, 512

    # --- subsectors (sector = sector of the first seg's front sidedef, visitor.rs:636-643) -------
    ssectors = np.zeros((nss, 4), dtype=np.int32)
    seg_front = np.full(nsegs, -1, dtype=np.int64)
    for i in range(nss):
        first, num = int(level.subsectors[i]["first_seg"]), int(level.subsectors[i]["num_segs"])
        sector = -1
        if num > 0 and first + num <= nsegs:
            side = level.seg_sidedef_index(level.segs[first])
            if side >= 0 and int(level.sidedefs[side]["sector"]) < nsect:
                sector = int(level.sidedefs[side]["sector"])
            seg_front[first:first + num] = sector
        else:
            first, num = 0, 0
        ssectors[i] = [first, num, sector, 0]

    # --- segs ------------------------------------------------------------------------------------
    segs = np.zeros((nsegs, 16), dtype=np.int32)
    segdyn = np.zeros((nsegs, 2), dtype=np.int32)
    segdyn[:, 0] = -1
    mids: List[List[int]] = []
    side_bytes = level.sidedefs.tobytes()

    def side_name(idx: int, which: int) -> bytes:
        o = idx * 30 + 4 + 8 * which          # 0 upper, 1 lower, 2 middle
        return W.wad_name(side_bytes[o:o + 8])

    for i in range(nsegs):
        sg = level.segs[i]
        rec = [0] * 16
        rec[3] = SEG_INVALID
        rec[6] = rec[9] = TEX_NONE
        rec[15] = -1
        v1, v2 = int(sg["v1"]), int(sg["v2"])
        ok = v1 < nverts and v2 < nverts and int(sg["linedef"]) < len(level.linedefs)
        side = level.seg_sidedef_index(sg) if ok else -1
        front = int(seg_front[i])
        if front < 0 and side >= 0 and int(level.sidedefs[side]["sector"]) < nsect:
            front = int(level.sidedefs[side]["sector"])     # seg outside any subsector (never drawn)
        if not ok or side < 0 or front < 0:
            segs[i] = rec
            continue
        line = level.linedefs[sg["linedef"]]
        sd = level.sidedefs[side]
        fsec = level.sectors[front]
        ff, fc = int(fsec["floor"]), int(fsec["ceil"])
        a, b = level.vertices[v1], level.vertices[v2]
        dx, dy = int(b["x"]) - int(a["x"]), int(b["y"]) - int(a["y"])
        flags_line = int(line["flags"])
        unpeg_upper = bool(flags_line & 0x0008)
        unpeg_lower = bool(flags_line & 0x0010)
        xoff, yoff = int(sd["xoff"]), int(sd["yoff"])
        # light: sector light + fake contrast when the sector has no effect (visitor.rs:887-901).
        # world X = -wad_y, world Z = -wad_x: "v1[0]==v2[0]" <=> wad dy == 0 => Brighten.
        contrast = 0
        if not has_effect[front]:
            if dy == 0:
                contrast = 1
            elif dx == 0:
                contrast = -1
        light = sector_light0[front] if has_effect[front] else W.light_byte(int(fsec["light"]), contrast)

        back_side = level.seg_back_sidedef_index(sg)
        back = -1
        if back_side >= 0 and int(level.sidedefs[back_side]["sector"]) < nsect:
            back = int(level.sidedefs[back_side]["sector"])

        def piece(name: bytes, t_top_expr):
            """-> (tex id, t row at anchor reduced mod texture height)."""
            tid = tex_id(name)
            if tid < 0:
                return TEX_NONE, 0
            th = int(tex_list[tid].shape[0])
            return tid, _floormod(t_top_expr(th) + yoff, th)

        rec[0], rec[1], rec[2] = v1, v2, front
        scroll = SEG_SCROLL if int(line["special"]) == 0x30 else 0
        rec[4] = int(sg["offset"]) + xoff                     # s1 (visitor.rs:904)
        rec[5] = math.isqrt((dx * dx + dy * dy) << 24)        # |v2-v1| in Q12 (visitor.rs:905)
        rec[12] = light
        rec[15] = back
        if back < 0:
            # one-sided: full-height middle, Peg::Bottom if lower-unpegged else Peg::Top
            # (visitor.rs:733-749; t at `high`: Top -> 0, Bottom -> texh - (ceil - floor), :909-912)
            if unpeg_lower:
                tid, t = piece(side_name(side, 2), lambda th: th - (fc - ff))
            else:
                tid, t = piece(side_name(side, 2), lambda th: 0)
            rec[3] = scroll
            rec[6], rec[7], rec[8] = tid, t, fc
            rec[13], rec[14] = fc, ff
            segdyn[i] = [-1, SEGDYN_UNPEG_LOWER if unpeg_lower else 0]
        else:
            bsec = level.sectors[back]
            bf, bc = int(bsec["floor"]), int(bsec["ceil"])
            back_sky = W.is_sky_flat(raw_name(level.sectors, back, "ceil_tex"))
            rec[3] = SEG_TWO_SIDED | scroll
            # next to a sector that may move, the pieces that can come into existence are resolved too (the reference
            # pre-extends the lower quad over the floor ranges, visitor.rs:772-790; the upper one we extend likewise)
            segdyn[i] = [back, (SEGDYN_UNPEG_LOWER if unpeg_lower else 0) | (SEGDYN_BACK_SKY if back_sky else 0)]
            # upper: exists iff back_ceil < ceil and the back ceiling is not sky (visitor.rs:791-807);
            # Peg::Top if upper-unpegged else Peg::Bottom (t at `high`=ceil: 0 / texh - (ceil-back_ceil)).
            otop = fc
            if ceil_range(back)[0] < ceil_range(front)[1] and not back_sky:     # = bc < fc for sectors that never move
                if bc < fc:
                    otop = bc
                if unpeg_upper:
                    tid, t = piece(side_name(side, 0), lambda th: 0)
                else:
                    tid, t = piece(side_name(side, 0), lambda th: th - (fc - bc))
                rec[6], rec[7] = tid, t
            rec[8] = fc
            # lower: exists iff back_floor > floor (visitor.rs:772-790); Peg::BottomLower if
            # lower-unpegged (t at `high`=back_floor: texh - (back_floor-floor) + (ceil-floor)) else Top.
            obot = ff
            bf_hi, ff_lo = floor_range(back)[1], floor_range(front)[0]
            if bf_hi > ff_lo:                                 # = bf > ff for sectors that never move
                if bf > ff:
                    obot = bf
                if unpeg_lower:                               # quad height = back_range.1 - front_range.0 (:777-780, :913-917)
                    tid, t = piece(side_name(side, 1), lambda th: th - (bf_hi - ff_lo) + (fc - ff))
                else:
                    tid, t = piece(side_name(side, 1), lambda th: 0)
                rec[9], rec[10] = tid, t
            rec[11] = bf if bf_hi > ff_lo else obot           # anchor of tB: the back floor (moves with it)
            rec[13], rec[14] = otop, obot
            # masked middle (visitor.rs:808-836): between max(floors) and min(ceilings); float pegs clamp the
            # quad to the texture height (visitor.rs:875-885); t at `high`: Top/Floats 0, Bottom texh-height
            low0, high0 = (bf if bf_hi > ff_lo else ff), (bc if bc < fc else fc)
            mname = side_name(side, 2)
            mtid = tex_id(mname) if low0 < high0 else TEX_NONE
            rec[15] = -1
            if mtid >= 0:
                th = int(tex_list[mtid].shape[0])
                if unpeg_lower:
                    peg = "topfloat" if W.is_untextured(side_name(side, 0)) else "bottom"
                else:
                    peg = "bottomfloat" if W.is_untextured(side_name(side, 1)) else "top"
                low, high = low0, high0
                if peg == "topfloat":
                    low, high = low0 + yoff, low0 + th + yoff
                elif peg == "bottomfloat":
                    low, high = high0 + yoff - th, high0 + yoff
                t_high = (th - (high - low)) if peg == "bottom" else 0
                rec[15] = len(mids)
                mids.append([mtid, _floormod(t_high + yoff, th), low, high, 0, 0, 0, 0])
        segs[i] = rec

    # --- decoration things -> sprites (visitor.rs:1010-1026, 1062-1137; thing table from doom.toml) ------
    from .thing_table import THINGS
    sprite_rows = []            # (subsector, thing index, [x, y, low, tex, light, 0, 0, 0])
    for ti, t in enumerate(level.things):
        ttype = int(t["type"])
        if ttype in (1, 2, 3, 4, 11, 14):                     # markers (visitor.rs:1345-1364)
            continue
        ssid, sec = subsector_at(level, float(t["x"]), float(t["y"]))
        if sec < 0 or ttype not in THINGS or ssid >= nss or int(ssectors[ssid, 2]) != sec:
            continue
        prefix, frame, hanging = THINGS[ttype]
        tid = TEX_NONE
        for rot in (b"0", b"1"):                              # try <sprite><frame>0 then ...1
            try:
                nm = W.wad_name(prefix.encode() + frame.encode() + rot)
            except W.WadError:
                break
            if nm in tex.textures:
                tid = tex_id(nm)
                break
        if tid < 0:
            continue
        th = int(tex_list[tid].shape[0])
        sct = level.sectors[sec]
        low = int(sct["ceil"]) - th if hanging else int(sct["floor"])
        sprite_rows.append((ssid, ti, [int(t["x"]), int(t["y"]), low, tid, sector_light0[sec], sec, 1 if hanging else 0, 0]))
    sprite_rows.sort(key=lambda r: (r[0], r[1]))
    sprites = np.array([r[2] for r in sprite_rows], dtype=np.int64).reshape(-1, 8)
    k = 0
    while k < len(sprite_rows):
        ssid = sprite_rows[k][0]
        j = k
        while j < len(sprite_rows) and sprite_rows[j][0] == ssid:
            j += 1
        if j - k > 255:
            raise W.WadError("more than 255 decoration things in one subsector")
        cnt = j - k
        word = k | (cnt << 24)                            # a count of 128..255 sets the sign bit of the int32 record
        ssectors[ssid, 3] = word - (1 << 32) if word >= 1 << 31 else word
        k = j

    # --- nodes -----------------------------------------------------------------------------------
    nodes = np.zeros((nnodes, 16), dtype=np.int64)

    def child(c: int) -> int:
        idx = c & 0x7FFF
        return (idx | LEAF) if (c & 0x8000) else idx

    # Child bounding boxes are NOT taken from the file: they are recomputed from the segs each subtree
    # actually holds, so that bounding-box culling stays conservative for any (even inconsistent) map.
    # box = (top, bottom, left, right); an empty subtree gets (0,0,0,0); a cyclic reference gets the
    # whole coordinate range.  Iterative post-order, identical in the product's compiler.
    FULL = (32767, -32768, -32768, 32767)
    EMPTY = (0, 0, 0, 0)

    def leaf_box(ss_id: int):
        if ss_id >= nss:
            return None
        first, num = int(ssectors[ss_id, 0]), int(ssectors[ss_id, 1])
        box = None
        for k in range(first, first + num):
            if segs[k, 3] & SEG_INVALID:
                continue
            for v in (int(segs[k, 0]), int(segs[k, 1])):
                x, y = int(level.vertices[v]["x"]), int(level.vertices[v]["y"])
                box = (y, y, x, x) if box is None else (max(box[0], y), min(box[1], y), min(box[2], x), max(box[3], x))
        return box

    def union(a, b):
        if a is None:
            return b
        if b is None:
            return a
        return (max(a[0], b[0]), min(a[1], b[1]), min(a[2], b[2]), max(a[3], b[3]))

    state = [0] * nnodes            # 0 unvisited, 1 on the stack, 2 done
    node_box = [None] * nnodes      # union of both children once done
    child_box = [[None, None] for _ in range(nnodes)]

    def resolve(c: int):
        """box of child id c if already known, else the node index that must be visited first"""
        if c & LEAF:
            return leaf_box(c & 0x7FFFFFFF), -1
        if c >= nnodes:
            return None, -1
        if state[c] == 2:
            return node_box[c], -1
        if state[c] == 1:
            return FULL, -1
        return None, c

    if nnodes > 0:
        stack = [nnodes - 1]
        state[nnodes - 1] = 1
        while stack:
            i = stack[-1]
            n = level.nodes[i]
            pending = -1
            for side, raw in ((0, int(n["right"])), (1, int(n["left"]))):
                box, need = resolve(child(raw))
                if need >= 0:
                    pending = need
                    break
                child_box[i][side] = box
            if pending >= 0:
                state[pending] = 1
                stack.append(pending)
                continue
            node_box[i] = union(child_box[i][0], child_box[i][1])
            state[i] = 2
            stack.pop()

    for i in range(nnodes):
        n = level.nodes[i]
        if state[i] == 2:
            rb = list(child_box[i][0] or EMPTY)
            lb = list(child_box[i][1] or EMPTY)
        else:                       # unreachable from the root: never traversed
            rb, lb = list(EMPTY), list(EMPTY)
        nodes[i, :14] = [int(n["x"]), int(n["y"]), int(n["dx"]), int(n["dy"])] + rb + lb + \
                        [child(int(n["right"])), child(int(n["left"]))]

    verts = np.zeros((nverts, 2), dtype=np.int32)
    verts[:, 0] = level.vertices["x"]
    verts[:, 1] = level.vertices["y"]

    # --- textures ---------------------------------------------------------------------------------
    ntex = len(tex_list)
    texrec = np.zeros((ntex, 8), dtype=np.uint32)
    texels = bytearray()
    for i, img in enumerate(tex_list):
        h, w = img.shape
        holes = (img >> 8) != 0
        px = np.where(holes, 0, img & 0xFF).astype(np.uint8)
        hmagic = (1 << 32) // h + 1
        hbias = h * ((16384 + h - 1) // h)
        a_first, a_n, a_k = tex_anim.get(i, (0, 0, 0))
        texrec[i] = [len(texels), w, h, hmagic & 0xFFFFFFFF, hbias, 0xFFFFFFFF, a_first, a_n | (a_k << 16)]
        texels += px.tobytes()
        while len(texels) % 16:
            texels += b"\0"
        if holes.any():
            texrec[i][5] = len(texels)
            texels += (~holes).astype(np.uint8).tobytes()
            while len(texels) % 16:
                texels += b"\0"

    # flat animation groups are appended to the frame list after the texture groups
    flat_anim_rec = np.zeros((len(flat_list), 2), dtype=np.int64)
    for ids in flat_groups:
        first = len(anim_frames)
        anim_frames.extend(ids)
        for k, i in enumerate(ids):
            flat_anim_rec[i] = [first, len(ids) | (k << 16)]
    colormap = bytearray(34 * 256)
    for k in range(min(34, len(tex.colormaps))):
        colormap[k * 256:(k + 1) * 256] = tex.colormaps[k]
    pal = np.frombuffer(tex.palettes[0], dtype=np.uint8).reshape(256, 3).astype(np.uint32)
    palette = (pal[:, 0] | (pal[:, 1] << 8) | (pal[:, 2] << 16) | np.uint32(0xFF000000)).astype("<u4")

    # --- player start (visitor.rs:1010-1026, game/src/level.rs:757-762) -------------------------
    has_start, sx, sy, sz, sang = 0, 0, 0, 0, 0
    for t in level.things:
        if int(t["type"]) != 1:
            continue
        sec = sector_at(level, float(t["x"]), float(t["y"]))
        if sec < 0:
            continue
        ang = float(np.round(np.float32(t["angle"]) / np.float32(45.0)) * np.float32(45.0))
        has_start = 1
        sx, sy = int(t["x"]) - 32, int(t["y"])
        sz = int(level.sectors[sec]["floor"]) + 50 + 12
        sang = int(ang) % 360
        # no break: visit_marker overwrites start_pos on every player-1 start -- the LAST one wins (level.rs:757-762)

    # --- assemble ---------------------------------------------------------------------------------
    parts = [("verts", verts.astype("<i4").tobytes()), ("nodes", (nodes & 0xFFFFFFFF).astype("<u4").tobytes()),
             ("ssectors", ssectors.astype("<i4").tobytes()), ("segs", segs.astype("<i4").tobytes()),
             ("sectors", sectors.astype("<i4").tobytes()), ("tex", texrec.astype("<u4").tobytes()),
             ("mids", np.array(mids, dtype="<i4").reshape(-1, 8).tobytes()),
             ("sprites", (sprites & 0xFFFFFFFF).astype("<u4").tobytes()),
             ("anim", np.array(anim_frames, dtype="<i4").tobytes()),
             ("flatanim", flat_anim_rec.astype("<i4").tobytes()), ("lights", lights.tobytes()),
             ("texels", bytes(texels)), ("flats", b"".join(flat_list)), ("colormap", bytes(colormap)),
             ("palette", palette.tobytes()), ("segdyn", segdyn.astype("<i4").tobytes()),
             ("dyn", np.array([[sec] + list(dyn[sec]) + [0, 0, 0] for sec in sorted(dyn)], dtype="<i4").reshape(-1, 8).tobytes())]
    off = 4 * HEADER_WORDS
    offs = {}
    for name, data in parts:
        offs[name] = off
        off = _align16(off + len(data))
    total = off
    hdr = [0] * HEADER_WORDS
    hdr[H_MAGIC], hdr[H_VERSION], hdr[H_TOTAL] = MAGIC, VERSION, total
    hdr[H_NVERTS], hdr[H_NNODES], hdr[H_NSSECTORS], hdr[H_NSEGS] = nverts, nnodes, nss, nsegs
    hdr[H_NSECTORS], hdr[H_NTEX], hdr[H_NFLATS] = nsect, ntex, len(flat_list)
    hdr[H_OFF_VERTS], hdr[H_OFF_NODES], hdr[H_OFF_SSECTORS] = offs["verts"], offs["nodes"], offs["ssectors"]
    hdr[H_OFF_SEGS], hdr[H_OFF_SECTORS], hdr[H_OFF_TEX] = offs["segs"], offs["sectors"], offs["tex"]
    hdr[H_OFF_TEXELS], hdr[H_TEXEL_BYTES], hdr[H_OFF_FLATS] = offs["texels"], len(texels), offs["flats"]
    hdr[H_OFF_COLORMAP], hdr[H_OFF_PALETTE] = offs["colormap"], offs["palette"]
    if nnodes > 0:
        hdr[H_ROOT] = nnodes - 1
    else:
        hdr[H_ROOT] = LEAF | 0
    hdr[H_SKY_TEX] = sky_tex & 0xFFFFFFFF
    hdr[H_START_X], hdr[H_START_Y], hdr[H_START_Z] = sx & 0xFFFFFFFF, sy & 0xFFFFFFFF, sz & 0xFFFFFFFF
    hdr[H_START_ANGLE], hdr[H_HAS_START] = sang, has_start
    hdr[H_MIN_H], hdr[H_MAX_H] = min_h & 0xFFFFFFFF, max_h & 0xFFFFFFFF
    hdr[H_NMIDS], hdr[H_OFF_MIDS] = len(mids), offs["mids"]
    hdr[H_NSPRITES], hdr[H_OFF_SPRITES] = len(sprite_rows), offs["sprites"]
    hdr[H_NANIM], hdr[H_OFF_ANIM], hdr[H_OFF_FLAT_ANIM] = len(anim_frames), offs["anim"], offs["flatanim"]
    hdr[H_OFF_LIGHTS] = offs["lights"]
    hdr[H_NDYN], hdr[H_OFF_DYN], hdr[H_OFF_SEGDYN] = len(dyn), offs["dyn"], offs["segdyn"]
    blob = bytearray(total)
    blob[0:4 * HEADER_WORDS] = struct.pack("<%dI" % HEADER_WORDS, *hdr)
    for name, data in parts:
        blob[offs[name]:offs[name] + len(data)] = data
    return bytes(blob)


def apply_moves(blob: bytes, moves) -> bytes:
    """The scene with some of its declared sectors moved: `moves` = (sector, floor_offset, ceil_offset) in map units
    relative to the heights in the level lumps.  Every record that depends on a height is re-derived the way the
    reference moves its meshes -- rigidly with the floor / ceiling object they are attached to:

    * sector floor / ceiling (flats, sky)               own floor / ceiling object   visitor.rs:957-983
    * one-sided wall                                    own floor if the line is lower-unpegged, else own ceiling  :736-740
    * upper piece                                       back ceiling                 :797
    * lower piece                                       back floor                   :777
    * masked middle texture                             own floor if lower-unpegged, else own ceiling   :812-816
    * decoration                                        floor of its sector, ceiling if it hangs   :1106-1121
    and the opening of a two-sided seg follows the moved heights (what the depth test leaves visible of the
    pre-extended quads)."""
    h = header(blob)
    out = bytearray(blob)
    nsect = h[H_NSECTORS]
    dyn = section(blob, "dyn")
    ranges = {int(r[0]): [int(v) for v in r[1:5]] for r in dyn}
    df, dc = np.zeros(nsect, dtype=np.int64), np.zeros(nsect, dtype=np.int64)
    sectors = section(blob, "sectors").astype(np.int64)
    for sec, dfl, dcl in moves:
        sec = int(sec)
        if sec not in ranges:
            raise ValueError("sector %d was not declared dynamic" % sec)
        f1, c1 = int(sectors[sec, 0]) + int(dfl), int(sectors[sec, 1]) + int(dcl)
        r = ranges[sec]
        if not (r[0] <= f1 <= r[1] and r[2] <= c1 <= r[3] and f1 <= c1):
            raise ValueError("sector %d moved outside its declared range" % sec)
        df[sec], dc[sec] = int(dfl), int(dcl)
    sectors[:, 0] += df
    sectors[:, 1] += dc
    segs = section(blob, "segs").astype(np.int64)
    segdyn = section(blob, "segdyn")
    mids = section(blob, "mids").astype(np.int64)
    for i in range(len(segs)):
        S = segs[i]
        if S[3] & SEG_INVALID:
            continue
        f, b, bits = int(S[2]), int(segdyn[i, 0]), int(segdyn[i, 1])
        own = df[f] if bits & SEGDYN_UNPEG_LOWER else dc[f]
        if not (S[3] & SEG_TWO_SIDED):
            S[8] += own
            S[13], S[14] = sectors[f, 1], sectors[f, 0]
            continue
        S[8] += dc[b]
        S[11] += df[b]
        ff, fc, bf, bc = sectors[f, 0], sectors[f, 1], sectors[b, 0], sectors[b, 1]
        S[13] = bc if (bc < fc and not bits & SEGDYN_BACK_SKY) else fc
        S[14] = bf if bf > ff else ff
        if S[15] >= 0:
            mids[S[15], 2] += own
            mids[S[15], 3] += own
    sprites = section(blob, "sprites").astype(np.int64)
    for i in range(len(sprites)):
        sec = int(sprites[i, 5])
        sprites[i, 2] += dc[sec] if sprites[i, 6] else df[sec]

    def put(off, a):
        data = a.astype("<i4").tobytes()
        out[off:off + len(data)] = data
    put(h[H_OFF_SECTORS], sectors)
    put(h[H_OFF_SEGS], segs)
    put(h[H_OFF_MIDS], mids)
    put(h[H_OFF_SPRITES], sprites)
    return bytes(out)


def tables_at(blob: bytes, tics: int, moves=()) -> bytes:
    """The state-dependent tables at level time `tics` with `moves` applied, laid out [textures | sectors | segs | sprites |
    mids] as the product's b2d_scene_tables_at returns them.  Restated from DESIGN.md C14-C16 on top of apply_moves:
    an animated texture or flat shows group frame (tics >> 3) mod n, whichever frame name the map uses (the texture record
    is that frame's record); a scrolling seg adds tics & 0xFFFFFF to its column offset; a sector with a light effect, its
    segs and its sprites carry its light byte at `tics`."""
    tics = int(tics) & 0xFFFFFFFF
    b = apply_moves(blob, moves)
    h = header(b)
    anim = np.frombuffer(b, dtype="<i4", count=h[H_NANIM], offset=h[H_OFF_ANIM])

    def frame_now(first: int, nk: int, own: int) -> int:
        n = nk & 0xFFFF
        return own if n < 2 else int(anim[first + (tics >> 3) % n])

    tex0 = section(b, "textures")
    tex = np.array([tex0[frame_now(int(t[6]), int(t[7]), i)] for i, t in enumerate(tex0)], dtype="<u4").reshape(-1, 8)
    flatanim = np.frombuffer(b, dtype="<i4", count=2 * h[H_NFLATS], offset=h[H_OFF_FLAT_ANIM]).reshape(-1, 2)
    sectors = section(b, "sectors").astype(np.int64)
    for row in sectors:
        for c in (2, 3):
            if row[c] >= 0:
                row[c] = frame_now(int(flatanim[row[c], 0]), int(flatanim[row[c], 1]), int(row[c]))
    segs = section(b, "segs").astype(np.int64)
    sprites = section(b, "sprites").astype(np.int64)
    lights = sector_lights_at(b, tics)
    effect = lights >= 0
    sectors[effect, 4] = lights[effect]
    for S in segs:
        if S[3] & SEG_INVALID:
            continue
        if S[3] & SEG_SCROLL:
            S[4] = (S[4] + (tics & 0xFFFFFF) + (1 << 31)) % (1 << 32) - (1 << 31)
        if effect[S[2]]:
            S[12] = lights[S[2]]
    for P in sprites:
        if effect[P[5]]:
            P[4] = lights[P[5]]
    return b"".join([tex.tobytes(), sectors.astype("<i4").tobytes(), segs.astype("<i4").tobytes(),
                     sprites.astype("<i4").tobytes(), section(b, "mids").astype("<i4").tobytes()])


def header(blob: bytes) -> List[int]:
    return list(struct.unpack_from("<%dI" % HEADER_WORDS, blob, 0))


def section(blob: bytes, which: str) -> np.ndarray:
    """Convenience view of one section as an int32 (or u8) array."""
    h = header(blob)
    def arr(off, n, width, dt="<i4"):
        return np.frombuffer(blob, dtype=dt, count=n * width, offset=off).reshape(n, width)
    if which == "verts":
        return arr(h[H_OFF_VERTS], h[H_NVERTS], 2)
    if which == "nodes":
        return arr(h[H_OFF_NODES], h[H_NNODES], 16)
    if which == "ssectors":
        return arr(h[H_OFF_SSECTORS], h[H_NSSECTORS], 4)
    if which == "segs":
        return arr(h[H_OFF_SEGS], h[H_NSEGS], 16)
    if which == "sectors":
        return arr(h[H_OFF_SECTORS], h[H_NSECTORS], 8)
    if which == "textures":
        return arr(h[H_OFF_TEX], h[H_NTEX], 8, "<u4")
    if which == "mids":
        return arr(h[H_OFF_MIDS], h[H_NMIDS], 8)
    if which == "sprites":
        return arr(h[H_OFF_SPRITES], h[H_NSPRITES], 8)
    if which == "segdyn":
        return arr(h[H_OFF_SEGDYN], h[H_NSEGS], 2)
    if which == "dyn":
        return arr(h[H_OFF_DYN], h[H_NDYN], 8)
    raise KeyError(which)
