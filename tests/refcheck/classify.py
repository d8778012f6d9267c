"""TEST-ONLY: explain every pixel on which the oracle and the reference-semantics ray caster (glcaster.py) differ.

A differing pixel is *explained* when the oracle's value is what the reference's own rules give for an adjacent sample:
  texel      the same surface, the texel next to the caster's (+-1 in u and/or v, wrapped), colormap row +-1
             (float vs fixed point at a texel or colormap-row boundary: static.frag:19-27)
  silhouette the pixel lies within one pixel of a boundary between two surfaces in the caster's image, or of a hole
             edge of a masked texture (rasterisation of an edge: which side a pixel centre falls on), and the oracle shows
             what the caster shows at one of the 8 neighbours (or a texel-adjacent variant of it)
  minified   the texture is minified at the pixel (the caster's texel jumps by more than one between this pixel and a
             neighbour on the same surface -- far floors near the horizon, distant walls): a sub-pixel shift of the sample
             point moves it by more than a texel, so the oracle may show any texel-adjacent value of the 8 neighbours
Three more categories are *deviations*, counted separately and bounded tightly by the tests (DESIGN.md 4):
  sky_hack      next to a sky surface the oracle shows the sky (at the pixel's own sky coordinates): a sky ceiling hides
                what pokes above it, as in Doom; the reference's sky polygon sits at level max + 512 and would not
  sprite_order  billboards are clipped by the column windows open when their subsector is entered instead of being
                depth-tested per pixel: a sprite that pokes into a wall, or overlaps a sprite of a neighbouring subsector
                (within a subsector they are depth-sorted)
  sliver        an edge pixel showing a third surface of which the caster has no pixel nearby, or a one-pixel-wide run
                (both neighbours across it agree): a surface seen edge-on that one renderer gives a column and the other none
  near_clamp    only when the caller sets dbg["near_depth"] (the renderer's wall depth clamp, max(1, FY2/16384) map units):
                the caster shows a wall nearer than that depth, which the renderer places at the clamp depth, so its top or
                bottom edge shows up to near_depth * H / FY2 map units nearer the eye height than it should (DESIGN.md 4)
Everything else -- a differing pixel away from any edge that no adjacent sample explains -- is *unexplained* and fails."""
import numpy as np


def _candidates(dbg, y, x):
    """Values the reference's rules give around the caster's sample at pixel (y, x): neighbouring texels x rows +-1."""
    i = int(dbg["img"][y, x])
    if i < 0:
        return {0}
    img = dbg["images"][i]
    h, w = img.shape
    u, v, r = int(dbg["u"][y, x]), int(dbg["v"][y, x]), int(dbg["row"][y, x])
    vals = set()
    for dv in (-1, 0, 1):
        for du in (-1, 0, 1):
            t = int(img[(v + dv) % h, (u + du) % w])
            if t >> 8:
                vals.add(-1)                                  # transparent texel next door: a hole edge
                continue
            for dr in (-1, 0, 1):
                rr = min(31, max(0, r + dr))
                vals.add(int(dbg["cmaps"][rr][t & 0xFF]))
    return vals


def _footprint(dbg, y, x, H, W):
    """Lit values of every texel inside the box the 3x3 neighbourhood (same surface) spans in texture space, +-1."""
    i = int(dbg["img"][y, x])
    img = dbg["images"][i]
    h, w = img.shape
    u, v, r = int(dbg["u"][y, x]), int(dbg["v"][y, x]), int(dbg["row"][y, x])
    dus, dvs, rows = [0], [0], [r]
    for yy in range(max(0, y - 1), min(H, y + 2)):
        for xx in range(max(0, x - 1), min(W, x + 2)):
            if dbg["surf"][yy, xx] != dbg["surf"][y, x]:
                continue
            du = (int(dbg["u"][yy, xx]) - u + w // 2) % w - w // 2
            dv = (int(dbg["v"][yy, xx]) - v + h // 2) % h - h // 2
            dus.append(du); dvs.append(dv); rows.append(int(dbg["row"][yy, xx]))
    vals = set()
    for dv in range(min(dvs) - 1, max(dvs) + 2):
        for du in range(min(dus) - 1, max(dus) + 2):
            t = int(img[(v + dv) % h, (u + du) % w])
            if t >> 8:
                continue
            for rr in range(max(0, min(rows) - 1), min(31, max(rows) + 1) + 1):
                vals.add(int(dbg["cmaps"][rr][t & 0xFF]))
    return vals


def classify(g, o, dbg):
    """Returns dict(differing, texel, silhouette, unexplained=[(y, x, caster value, oracle value), ...])."""
    H, W = g.shape
    ys, xs = np.nonzero(g != o)
    surf = dbg["surf"]
    img, uu, vv = dbg["img"], dbg["u"], dbg["v"]
    res = {"differing": int(len(ys)), "texel": 0, "silhouette": 0, "minified": 0, "sky_hack": 0, "sprite_order": 0, "sliver": 0, "near_clamp": 0, "unexplained": []}
    # every value a sprite image can produce (any texel, any colormap row): for the sprite-overlap category
    near = dbg.get("near_depth")
    sprite_values = None
    if (dbg["kind"] == 4).any():
        sprite_values = set()
        for i in set(np.unique(img[dbg["kind"] == 4]).tolist()):
            t = dbg["images"][i]
            texels = np.unique(t[(t >> 8) == 0] & 0xFF).astype(np.int64)
            sprite_values |= set(np.unique(dbg["cmaps"][:, texels]).tolist())

    for y, x in zip(ys.tolist(), xs.tolist()):
        ov = int(o[y, x])
        cand = _candidates(dbg, y, x)
        if ov in cand:
            res["texel"] += 1
            continue
        y0, y1, x0, x1 = max(0, y - 1), min(H, y + 2), max(0, x - 1), min(W, x + 2)
        edge = bool((surf[y0:y1, x0:x1] != surf[y, x]).any()) or (-1 in cand) or y in (0, H - 1)
        mini = False
        if not edge and img[y, x] >= 0:
            ih, iw = dbg["images"][int(img[y, x])].shape
            for (yy, xx) in ((y, x - 1), (y, x + 1), (y - 1, x), (y + 1, x)):
                if 0 <= yy < H and 0 <= xx < W and surf[yy, xx] == surf[y, x]:
                    du = abs(int(uu[yy, xx]) - int(uu[y, x])); du = min(du, iw - du)
                    dv = abs(int(vv[yy, xx]) - int(vv[y, x])); dv = min(dv, ih - dv)
                    if du > 1 or dv > 1:
                        mini = True
        ok = False
        if mini and ov in _footprint(dbg, y, x, H, W):
            ok = True
        if edge and not ok and (dbg["kind"][y0:y1, x0:x1] == 3).any():
            # next to a sky surface: the oracle may show the sky here -- at THIS pixel's sky coordinates
            sa = dbg["sky_all"]
            ok = any(int(sa[yy, xx]) == ov for yy in range(y0, y1) for xx in range(x0, x1))
        if (edge or mini) and not ok:
            for yy in range(y0, y1):
                for xx in range(x0, x1):
                    if int(g[yy, xx]) == ov or ov in _candidates(dbg, yy, xx) or (img[yy, xx] >= 0 and ov in _footprint(dbg, yy, xx, H, W)):
                        ok = True
                        break
                if ok:
                    break
        if ok:
            res["silhouette" if edge else "minified"] += 1
            continue
        # -- known semantic deviations of the column renderer (DESIGN.md 4, "deviations"), counted and bounded by the tests:
        ya, yb, xa, xb = max(0, y - 3), min(H, y + 4), max(0, x - 3), min(W, x + 4)
        sa = dbg["sky_all"]
        if near is not None and dbg["kind"][y, x] == 1 and dbg["t"][y, x] < near:
            res["near_clamp"] += 1     # a wall nearer than the depth clamp, drawn at the clamp depth: its edge rows move
        elif dbg["kind"][y, x] != 3 and any(int(sa[yy, xx]) == ov for yy in range(y0, y1) for xx in range(x0, x1)):
            res["sky_hack"] += 1       # a sky ceiling hides what pokes above it (Doom's sky hack; GL puts the sky poly at max+512)
        elif sprite_values is not None and ((dbg["kind"][y, x] == 4) or (ov in sprite_values and (dbg["kind"][ya:yb, xa:xb] == 4).any())):
            res["sprite_order"] += 1   # billboards are ordered / clipped per subsector and column window, not depth-tested per
                                       # pixel: two overlapping sprites of one subsector, a sprite poking into a wall
        elif edge or (0 < x < W - 1 and g[y, x - 1] == o[y, x - 1] and g[y, x + 1] == o[y, x + 1]) \
                or (0 < y < H - 1 and g[y - 1, x] == o[y - 1, x] and g[y + 1, x] == o[y + 1, x]):
            res["sliver"] += 1         # edge pixel showing a third surface the caster has no pixel of nearby (a 1-pixel sliver
                                       # of floor between two wall pieces, the top row of a masked texture): bounded by the tests
        else:
            res["unexplained"].append((y, x, int(g[y, x]), ov))
    return res
