"""TEST-ONLY: a per-pixel ray caster that restates what the *reference's own pipeline* would put on screen.

rust-doom renders a level as a static triangle soup with a depth buffer (engine/src/renderer.rs:49-57):
wall quads per seg (wad/src/visitor.rs:711-937), one floor and one ceiling polygon per subsector at the
sector heights (visitor.rs:939-985), sky quads/polys at level min-512 / max+512 (visitor.rs:987-1008,
1173-1182), shaded per fragment by assets/shaders/static.{vert,frag} and sky.{vert,frag}.  With a depth test,
"what is on screen at pixel p" is simply "the nearest surface along the ray through p".  This module computes
exactly that with float64 ray casting -- no BSP ordering, no column clipping, no fixed point -- so it is an
algorithmically independent check of the oracle's *scene semantics* (which surface, which texel, which
colormap row).  Agreement cannot be bit-exact (float vs fixed point at texel/row boundaries, silhouette
pixels), so tests assert a high identical-pixel fraction instead.

Masked two-sided middle textures are modelled (transparent texels let the ray through, static.frag:21-22).
Decoration things are modelled as camera-facing billboards (visitor.rs:1062-1137, sprite.vert:40-42,
sprite.frag:15-27).  Not modelled: POLY_BIAS.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import scene as S
from oracle import wad as W


def _sector_at_vec(level: W.Level, px: np.ndarray, py: np.ndarray) -> np.ndarray:
    """Vectorised LevelWalker::sector_at (visitor.rs:1028-1060) without the seg tolerance test."""
    n = len(px)
    nodes = level.nodes
    cur = np.full(n, len(nodes) - 1, dtype=np.int64)
    leaf = np.zeros(n, dtype=bool)
    nx, ny = nodes["x"].astype(np.float64), nodes["y"].astype(np.float64)
    ndx, ndy = nodes["dx"].astype(np.float64), nodes["dy"].astype(np.float64)
    right, left = nodes["right"].astype(np.int64), nodes["left"].astype(np.int64)
    for _ in range(64):
        act = ~leaf
        if not act.any():
            break
        c = cur[act]
        sd = (py[act] - ny[c]) * ndx[c] - (px[act] - nx[c]) * ndy[c]
        nxt = np.where(sd > 0.0, left[c], right[c])
        cur[act] = nxt & 0x7FFF
        leaf[act] = (nxt & 0x8000) != 0
    ss = level.subsectors
    first = ss["first_seg"].astype(np.int64)[np.clip(cur, 0, len(ss) - 1)]
    seg0 = level.segs[np.clip(first, 0, len(level.segs) - 1)]
    line = level.linedefs[seg0["linedef"]]
    side = np.where(seg0["direction"] == 0, line["right"], line["left"]).astype(np.int64)
    sec = level.sidedefs["sector"].astype(np.int64)[np.clip(side, 0, len(level.sidedefs) - 1)]
    return np.where(leaf & (side >= 0), sec, -1)


def render(archive: W.Archive, tex: W.TextureDirectory, level_index: int, width: int, height: int,
           x: float, y: float, z: float, angle_deg: float, fov_deg: float = 65.0, focal2=None,
           tics: int = 0, cols=None, debug: bool = False, dynamic=(), moves=()):
    """`cols`: optional subset of screen columns to cast (the result then has shape (height, len(cols))); `debug`: also
    return, per pixel, which image / texel / colormap row / surface produced it (for classifying differences)."""
    level = W.Level(archive, level_index)
    from oracle.anim_table import FLATS as ANIM_FLATS, WALLS as ANIM_WALLS
    # moving sectors, literally as the reference builds and moves its meshes: quads pre-extended over the declared height
    # ranges (visitor.rs:146-155, 733-790), every quad / flat / decoration translated with the floor or ceiling object it
    # is attached to (game/src/level.rs:201-245), the depth test (= nearest hit) sorting out what is visible
    nsec_ = len(level.sectors)
    rng = [[int(level.sectors[i]["floor"])] * 2 + [int(level.sectors[i]["ceil"])] * 2 for i in range(nsec_)]
    for d in dynamic:
        sec_, f0_, c0_ = int(d[0]), rng[int(d[0])][0], rng[int(d[0])][2]
        rng[sec_] = [min(int(d[1]), int(d[2]), f0_), max(int(d[1]), int(d[2]), f0_), min(int(d[3]), int(d[4]), c0_), max(int(d[3]), int(d[4]), c0_)]
    dfl, dcl = [0.0] * nsec_, [0.0] * nsec_
    for m_ in moves:
        dfl[int(m_[0])], dcl[int(m_[0])] = float(m_[1]), float(m_[2])

    def anim_name(name, groups, table):
        """static.vert:23-39 with u_time = tics/35: frame_index = floor(mod(u_time / (8/35), n)), added to the atlas
        position of the group's FIRST frame (tex.rs:260, 302-306 bind every frame name to it): the image shown is group
        frame frame_index whichever frame name the map uses."""
        for g in groups:
            frames = [W.wad_name(f.encode()) for f in g]
            if name in frames:
                have = [f for f in frames if table.get(f) is not None]
                if len(have) < 2 or name not in have:
                    return name
                fi = int(math.floor(math.fmod((tics / 35.0) / (8.0 / 35.0) + 1e-9, len(have))))
                return have[fi % len(have)]
        return name

    W_, H_ = width, height
    tany = math.tan(math.radians(fov_deg) / 2.0)
    tanx = (W_ / H_) * 1.2 * tany                         # perspective(fovy, aspect*1.2), player.rs:84-89
    if focal2 is not None:                                # the renderer's integer focal lengths (2*focal px)
        tanx, tany = W_ / float(focal2[0]), H_ / float(focal2[1])
    a = math.radians(angle_deg)
    fx, fy = math.cos(a), math.sin(a)                     # forward (wad x east, y north)
    rx, ry = math.sin(a), -math.cos(a)                    # right
    xs = (np.arange(W_) + 0.5) / W_ * 2.0 - 1.0
    if cols is not None:
        xs = xs[np.asarray(cols, dtype=np.int64)]
    WC = len(xs)
    ys = 1.0 - (np.arange(H_) + 0.5) / H_ * 2.0
    ndx, ndy = np.meshgrid(xs, ys)
    # ray direction with unit forward component: depth along forward = t
    dx = fx + rx * ndx * tanx
    dy = fy + ry * ndx * tanx
    dz = ndy * tany
    npx = WC * H_
    dx, dy, dz = dx.reshape(-1), dy.reshape(-1), dz.reshape(-1)
    images, image_ids = [], {}
    d_img = np.full(npx, -1, dtype=np.int32)
    d_u = np.zeros(npx, dtype=np.int32)
    d_v = np.zeros(npx, dtype=np.int32)
    d_row = np.zeros(npx, dtype=np.int32)
    d_surf = np.full(npx, -1, dtype=np.int64)

    def image_id(key, arr):
        if key not in image_ids:
            image_ids[key] = len(images)
            images.append(np.asarray(arr))
        return image_ids[key]
    best_t = np.full(npx, np.inf)
    out = np.zeros(npx, dtype=np.uint8)                   # void = 0, as in the oracle
    kind = np.zeros(npx, dtype=np.int8)                   # 0 none, 1 wall, 2 flat, 3 sky

    cmaps = np.stack([np.frombuffer(tex.colormaps[k], np.uint8) for k in range(32)])
    secs = level.sectors
    sec_bytes = secs.tobytes()
    floor_name = [W.wad_name(sec_bytes[i * 26 + 4:i * 26 + 12]) for i in range(len(secs))]
    ceil_name = [W.wad_name(sec_bytes[i * 26 + 12:i * 26 + 20]) for i in range(len(secs))]
    min_h = int(secs["floor"].min()) - 512
    max_h = int(secs["ceil"].max()) + 512
    side_bytes = level.sidedefs.tobytes()

    def side_name(idx, which):
        o = idx * 30 + 4 + 8 * which
        return W.wad_name(side_bytes[o:o + 8])

    def palette_row(light_byte, depth):
        """static.vert:41-43 + static.frag:15-27; depth in map units (w = depth/100)."""
        v = light_byte / 255.0
        w = depth / 100.0
        dist = np.minimum(1.0, 1.0 - 0.9 / (w + 0.9))
        light = v * 2.0 - dist
        return np.clip(np.floor((1.0 - light) * 32.0), 0, 31).astype(np.int64)

    def sky_pixels(mask, record=True):
        """sky.vert:9-16, sky.frag:12-26 at pitch 0: uv = (ndc.x - 4*yaw/pi, 1 - ndc.y), mirrored below."""
        name = S.sky_for(level.name)
        img = tex.textures.get(name)
        if img is None:
            return np.zeros(mask.sum(), dtype=np.uint8)
        sh, sw = img.shape
        u = ndx.reshape(-1)[mask] - 4.0 * a / math.pi
        v = 1.0 - ndy.reshape(-1)[mask]
        v = np.where(v >= 1.0, 1.0 - v, v)
        ui = np.floor((u - np.floor(u)) * sw).astype(np.int64) % sw
        vi = np.floor((v - np.floor(v)) * sh).astype(np.int64) % sh
        if record:
            d_img[mask] = image_id(("tex", name), img)
            d_u[mask], d_v[mask], d_row[mask], d_surf[mask] = ui, vi, 0, 3000000
        return cmaps[0][(img[vi, ui] & 0xFF).astype(np.int64)]

    # ---- walls -----------------------------------------------------------------------------------------
    has_effect = []
    for i in range(len(secs)):
        eff = int(secs[i]["type"]) in W.EFFECT_TYPES and (level.sector_min_light(i) >> 3) != (int(secs[i]["light"]) >> 3)
        has_effect.append(eff)

    def effect_light_byte(i):
        """Light of an effect sector at u_time = tics/35 (wad/src/light.rs:27-80 parameters, game/src/lights.rs:26-66
        evaluation), in the reference's float32 arithmetic."""
        f = np.float32
        stype = int(secs[i]["type"])
        level_f = f(np.int16(secs[i]["light"]) >> 3) / f(31.0)
        alt = f(np.int16(level.sector_min_light(i)) >> 3) / f(31.0)
        sync = f(0.0) if stype in (12, 13, 8) else f((i * 1664525 + 1013904223) & 0xFFFF) / f(15.0)
        time = f(tics & 0xFFFFFFFF) / f(35.0)
        fract = lambda x: f(x - np.floor(x))                 # noqa: E731
        if stype == 8:                                       # glow
            scale = f(level_f - alt)
            phase = f(f(time * f(0.5)) / scale)
            val = f(f(f(abs(f(f(0.5) - fract(phase))) * f(2.0)) * scale) + alt)
        elif stype in (1, 17):                               # flash / flicker: hash noise per time slot
            speed, duration = (f(20.0), f(0.06)) if stype == 1 else (f(8.0), f(0.5))
            slot = np.floor(f(time * speed))
            arg = f(f(f(sync + f(slot / f(1000.0))) * f(12.9898)) + f(sync * f(78.233)))
            noise = fract(f(f(1.0) + f(f(math.sin(float(arg))) * f(43758.547))))
            val = alt if noise < duration else level_f
        else:                                                # strobes
            speed, duration = (f(1.0), f(0.85)) if stype in (3, 12) else (f(2.0), f(0.7))
            val = alt if fract(f(f(time * speed) + f(sync * f(3.5435)))) < duration else level_f
        val = min(max(float(val), 0.0), 1.0)
        return int(float(f(f(val) * f(255.0))))

    sector_byte = [effect_light_byte(i) if has_effect[i] else W.light_byte(int(secs[i]["light"]), 0)
                   for i in range(len(secs))]
    ss_sector = {}
    for ssi in range(len(level.subsectors)):
        first, num = int(level.subsectors[ssi]["first_seg"]), int(level.subsectors[ssi]["num_segs"])
        if num == 0:
            continue
        sd0 = level.seg_sidedef_index(level.segs[first])
        for k in range(first, first + num):
            ss_sector[k] = int(level.sidedefs[sd0]["sector"]) if sd0 >= 0 else -1

    for si in range(len(level.segs)):
        sg = level.segs[si]
        front = ss_sector.get(si, -1)
        side = level.seg_sidedef_index(sg)
        if front < 0 or side < 0:
            continue
        v1, v2 = level.vertices[sg["v1"]], level.vertices[sg["v2"]]
        ax, ay, bx, by = float(v1["x"]), float(v1["y"]), float(v2["x"]), float(v2["y"])
        ex, ey = bx - ax, by - ay
        length = math.hypot(ex, ey)
        if length == 0:
            continue
        if (y - ay) * ex - (x - ax) * ey >= 0:            # camera must be on the right (front) side
            continue
        # ray/segment intersection: (x,y) + t*(dx,dy) = A + s*(E)
        den = dx * ey - dy * ex
        with np.errstate(divide="ignore", invalid="ignore"):
            t = ((ax - x) * ey - (ay - y) * ex) / den
            s = ((ax - x) * dy - (ay - y) * dx) / den
        ok = (t > 0) & (s >= 0) & (s <= 1) & np.isfinite(t)
        if not ok.any():
            continue
        hz = z + t * dz                                     # height of the hit point
        fsec = secs[front]
        ff, fc = float(fsec["floor"]), float(fsec["ceil"])
        line = level.linedefs[sg["linedef"]]
        sd = level.sidedefs[side]
        xoff, yoff = float(sd["xoff"]), float(sd["yoff"])
        unpeg_upper, unpeg_lower = bool(line["flags"] & 8), bool(line["flags"] & 16)
        contrast = 0
        if not has_effect[front]:
            contrast = 1 if ey == 0 else (-1 if ex == 0 else 0)
        lb = sector_byte[front] if has_effect[front] else W.light_byte(int(fsec["light"]), contrast)
        back_side = level.seg_back_sidedef_index(sg)
        back = int(level.sidedefs[back_side]["sector"]) if back_side >= 0 else -1
        pieces = []                                         # (low, high, texture name or 'SKY', t at high[, object offset])
        maxh = float(rng[front][3] - rng[front][0])         # SectorInfo::max_height
        if back < 0:
            name = side_name(side, 2)
            img = tex.textures.get(name)
            th = img.shape[0] if img is not None else 0
            if unpeg_lower:
                pieces.append((ff, ff + maxh, name, th - maxh, dfl[front]))
            else:
                pieces.append((fc - maxh, fc, name, 0.0, dcl[front]))
            if W.is_sky_flat(ceil_name[front]):
                pieces.append((fc, float(max_h), "SKY", 0.0, dcl[front]))
            if W.is_sky_flat(floor_name[front]):
                pieces.append((float(min_h), ff, "SKY", 0.0, dfl[front]))
        else:
            bsec = secs[back]
            bf, bc = float(bsec["floor"]), float(bsec["ceil"])
            if W.is_sky_flat(ceil_name[front]) and not W.is_sky_flat(ceil_name[back]):
                pieces.append((fc, float(max_h), "SKY", 0.0, dcl[front]))
            if W.is_sky_flat(floor_name[front]) and not W.is_sky_flat(floor_name[back]):
                pieces.append((float(min_h), ff, "SKY", 0.0, dfl[front]))
            lower_exists = rng[back][1] > rng[front][0]
            if lower_exists:
                name = side_name(side, 1)
                img = tex.textures.get(name)
                th = img.shape[0] if img is not None else 0
                qh = float(rng[back][1] - rng[front][0])
                pieces.append((bf - qh, bf, name, (th - qh + (fc - ff)) if unpeg_lower else 0.0, dfl[back]))
            if bc < fc and not W.is_sky_flat(ceil_name[back]):
                name = side_name(side, 0)
                img = tex.textures.get(name)
                th = img.shape[0] if img is not None else 0
                pieces.append((bc, fc, name, 0.0 if unpeg_upper else (th - (fc - bc)), dcl[back]))
            # middle (visitor.rs:808-836,875-919): drawn last, so lower/upper win at equal depth (IfLess)
            low0, high0 = (bf if lower_exists else ff), (bc if bc < fc else fc)
            mname = side_name(side, 2)
            mimg = None if W.is_untextured(mname) else tex.textures.get(mname)
            if mimg is not None and low0 < high0:
                th = mimg.shape[0]
                if unpeg_lower:
                    peg = "topfloat" if W.is_untextured(side_name(side, 0)) else "bottom"
                else:
                    peg = "bottomfloat" if W.is_untextured(side_name(side, 1)) else "top"
                low, high = low0, high0
                if peg == "topfloat":
                    low, high = low0 + yoff, low0 + th + yoff
                elif peg == "bottomfloat":
                    low, high = high0 + yoff - th, high0 + yoff
                pieces.append((low, high, mname, (th - (high - low)) if peg == "bottom" else 0.0, dfl[front] if unpeg_lower else dcl[front]))
        for pi, (low, high, name, t_high, obj_off) in enumerate(pieces):
            if low >= high:
                continue
            low, high = low + obj_off, high + obj_off
            hit = ok & (hz >= low) & (hz < high) & (t < best_t)
            if not hit.any():
                continue
            if name == "SKY":
                best_t[hit] = t[hit]
                kind[hit] = 3
                continue
            if W.is_untextured(name):
                continue                                    # skipped by the mesh builder: ray passes through
            img = tex.textures.get(name)
            if img is None:
                continue
            img = tex.textures.get(anim_name(name, ANIM_WALLS, tex.textures))
            th, tw = img.shape
            scroll = 35.0 if int(line["special"]) == 0x30 else 0.0      # visitor.rs:922, static.vert:23
            su = float(sg["offset"]) + xoff + s[hit] * length + (tics / 35.0) * scroll
            tv = t_high + yoff + (high - hz[hit])
            ui = np.floor(su).astype(np.int64) % tw
            vi = np.floor(tv).astype(np.int64) % th
            texel = img[vi, ui]
            rows = palette_row(lb, t[hit])
            val = cmaps[rows, (texel & 0xFF).astype(np.int64)]
            opaque = (texel >> 8) == 0
            idx = np.nonzero(hit)[0][opaque]
            best_t[idx] = t[hit][opaque]
            out[idx] = val[opaque]
            kind[idx] = 1
            d_img[idx] = image_id(("tex", anim_name(name, ANIM_WALLS, tex.textures)), img)
            d_u[idx], d_v[idx], d_row[idx], d_surf[idx] = ui[opaque], vi[opaque], rows[opaque], si * 8 + pi

    # ---- decoration sprites: billboards at constant view depth ---------------------------------------------
    from oracle.thing_table import THINGS
    for th in level.things:
        ttype = int(th["type"])
        if ttype in (1, 2, 3, 4, 11, 14) or ttype not in THINGS:
            continue
        sec = S.sector_at(level, float(th["x"]), float(th["y"]))
        if sec < 0:
            continue
        prefix, frame, hanging = THINGS[ttype]
        img = None
        for rot in (b"0", b"1"):
            img = tex.textures.get(W.wad_name(prefix.encode() + frame.encode() + rot))
            if img is not None:
                break
        if img is None:
            continue
        sh, sw = img.shape
        low = float(secs[sec]["ceil"]) - sh + dcl[sec] if hanging else float(secs[sec]["floor"]) + dfl[sec]
        tx0, ty0 = float(th["x"]) - x, float(th["y"]) - y
        cz = tx0 * fx + ty0 * fy                              # view depth of the thing
        cx = tx0 * rx + ty0 * ry                              # offset to the right
        if cz <= 1.0:
            continue
        # my rays have unit forward component: the ray reaches depth cz at parameter t = cz
        hit_x = cz * (ndx.reshape(-1) * tanx)                 # rightward offset of the ray at that depth
        hz = z + cz * dz
        u = hit_x - (cx - sw / 2.0)
        v = (low + sh) - hz
        hit = (u >= 0) & (u < sw) & (v >= 0) & (v < sh) & (cz < best_t)
        if not hit.any():
            continue
        sui, svi = np.floor(u[hit]).astype(np.int64), np.floor(v[hit]).astype(np.int64)
        texel = img[svi, sui]
        vb = sector_byte[sec] / 255.0
        dist = min(1.0, 1.0 - 1.0 / (cz / 100.0 + 1.0))
        light = min(vb, vb * 2.0 - dist)                      # sprite.frag:24-26
        row = int(np.clip(np.floor((1.0 - light) * 32.0), 0, 31))
        opaque = (texel >> 8) == 0
        idx = np.nonzero(hit)[0][opaque]
        best_t[idx] = cz
        out[idx] = cmaps[row][(texel[opaque] & 0xFF).astype(np.int64)]
        kind[idx] = 4
        d_img[idx] = image_id(("sprite", id(img)), img)
        d_u[idx], d_v[idx], d_row[idx] = sui[opaque], svi[opaque], row
        d_surf[idx] = 1000000 + int(th["x"]) * 65536 + int(th["y"])

    # ---- flats: one horizontal plane per distinct height -------------------------------------------------
    floor_h = np.array([(min_h if W.is_sky_flat(floor_name[i]) else int(secs[i]["floor"])) + dfl[i] for i in range(len(secs))], dtype=np.float64)
    ceil_h = np.array([(max_h if W.is_sky_flat(ceil_name[i]) else int(secs[i]["ceil"])) + dcl[i] for i in range(len(secs))], dtype=np.float64)
    sec_light = np.array(sector_byte, dtype=np.float64)
    for is_ceiling, heights in ((False, floor_h), (True, ceil_h)):
        for h in np.unique(heights):
            with np.errstate(divide="ignore", invalid="ignore"):
                t = (h - z) / dz
            ok = np.isfinite(t) & (t > 0) & (t < best_t) & ((dz > 0) if is_ceiling else (dz < 0))
            if not ok.any():
                continue
            idx = np.nonzero(ok)[0]
            hx, hy = x + t[idx] * dx[idx], y + t[idx] * dy[idx]
            sec = _sector_at_vec(level, hx, hy)
            good = (sec >= 0) & (heights[np.clip(sec, 0, len(secs) - 1)] == h)
            if not good.any():
                continue
            idx, hx, hy, sec = idx[good], hx[good], hy[good], sec[good]
            tt = t[idx]
            names = ceil_name if is_ceiling else floor_name
            vals = np.zeros(len(idx), dtype=np.uint8)
            knd = np.full(len(idx), 2, dtype=np.int8)
            f_img = np.full(len(idx), -1, dtype=np.int32)
            f_u = np.zeros(len(idx), dtype=np.int32)
            f_v = np.zeros(len(idx), dtype=np.int32)
            f_row = np.zeros(len(idx), dtype=np.int32)
            f_surf = 2000000 + sec * 2 + (1 if is_ceiling else 0)
            for sid in np.unique(sec):
                m = sec == sid
                name = names[sid]
                if W.is_sky_flat(name):
                    knd[m] = 3
                    continue
                data = tex.flats.get(name)
                if data is None:
                    continue
                data = tex.flats.get(anim_name(name, ANIM_FLATS, tex.flats))
                fl = np.frombuffer(data, np.uint8)
                u = np.floor(hy[m]).astype(np.int64) % 64            # tile_uv = (wad_y, wad_x), level.rs:537-549
                v = np.floor(hx[m]).astype(np.int64) % 64
                rows = palette_row(sec_light[sid], tt[m])
                vals[m] = cmaps[rows, fl[u + 64 * v].astype(np.int64)]
                f_img[m] = image_id(("flat", anim_name(name, ANIM_FLATS, tex.flats)), fl.reshape(64, 64).astype(np.uint16))
                f_u[m], f_v[m], f_row[m] = u, v, rows
            best_t[idx] = tt
            out[idx] = vals
            kind[idx] = knd
            d_img[idx], d_u[idx], d_v[idx], d_row[idx], d_surf[idx] = f_img, f_u, f_v, f_row, f_surf
    sky = kind == 3
    if sky.any():
        out[sky] = sky_pixels(sky)
    if debug:
        sky_all = sky_pixels(np.ones(npx, dtype=bool), record=False).reshape(H_, WC)   # what the sky would show at each pixel
        dbg = {"images": images, "cmaps": cmaps, "sky_all": sky_all, "kind": kind.reshape(H_, WC), "img": d_img.reshape(H_, WC), "u": d_u.reshape(H_, WC), "v": d_v.reshape(H_, WC),
               "row": d_row.reshape(H_, WC), "surf": d_surf.reshape(H_, WC), "t": best_t.reshape(H_, WC)}     # t: view depth of the hit
        return out.reshape(H_, WC), kind.reshape(H_, WC), dbg
    return out.reshape(H_, WC), kind.reshape(H_, WC)
