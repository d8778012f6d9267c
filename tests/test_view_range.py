"""The whole accepted view range (b2d_view_init: width 1..4096, height 2..2160, 1 < fov < 170 degrees) at poses built for
the arithmetic's edges: walls nearer and farther than FY2 / 16384 map units (where the Q18 scale reaches 2^31), an eye a
fraction of a unit above a floor or below a ceiling looking down the longest line of sight, and a sprite and a masked
middle just beyond one unit.  hostcheck and the kernels must equal the oracle bit for bit at every case; at the head-on
poses the oracle must also agree with the float64 ray caster (tests/refcheck), which has no fixed point and so catches an
overflow that the oracle and the kernels share.  Views past the bounds (F < 2, W > 256 F) must be refused by both."""
import functools
import math

import numpy as np
import pytest

from oracle import render, scene, wad
from tests.refcheck import glcaster
from tests.test_refcheck import Tally

FOVS = (1.01, 2.0, 5.0, 10.0, 15.0, 20.0, 40.0, 65.0, 104.0, 110.0, 150.0, 169.9)     # 104: 4096x24 at W = 256 F
SIZES = ((1, 2), (31, 3), (64, 2160), (4096, 24), (1920, 1080), (4096, 2160))
HEAD_ON = (1.0, 2.0, 4.0, 8.0, 16.0, 20.0)          # distances straddling FY2 / 16384 (1 .. 15 units at 2160 rows)
ROW_SCALE_MAX = (1 << 31) - 1
# Every accepted case is ray-cast and every differing pixel must be explained (tests/refcheck/classify.py), with these
# allowances, measured on this grid and bounded:
# - rounding residue: the usual 1 % between 10 and 65 degrees.  Narrower views magnify a texel over many rows (at 1 degree
#   one texel of a wall 20 units away spans ~300 rows), so a float-vs-fixed texel boundary moves whole runs of pixels: up
#   to 5 % (4.6 % measured at 1.01 degrees).  Wider views sample walls at grazing angles near the screen edges: up to 8 %
#   (6.9 % measured at 169.9 degrees).  Every such pixel is still an adjacent texel, a silhouette or a counted deviation.
# - near_clamp: walls nearer than the renderer's depth clamp max(1, FY2 / 16384) are drawn at the clamp depth, which an eye
#   a fraction of a unit above a floor sees in oblique columns (DESIGN.md 4): at most 2.5 % (2.0 % measured at 169.9).
# - two cases the classifier does not explain yet, each bounded to what it shows: at 169.9 degrees the masked-middle pose's
#   bottom edge lies two rows lower than the ray caster's in every column (one row of each 2160-row frame), and a 31x3 view
#   at 10-15 degrees of a wall 317 units away, minified 18 texels per row, gives 1-2 pixels outside the texel footprint.
NEAR_CLAMP_BOUND = 0.025
KNOWN_UNEXPLAINED = {169.9: 62, 10.0: 2, 15.0: 1}


def _residue(fov):
    return 0.05 if fov < 10 else (0.08 if fov > 65 else 0.01)


def _accepted(w, view):
    return view.F >= 2 and view.FY2 >= 2 and w <= 256 * view.F


def _cols(w):
    """every column of a narrow view, about 64 spread over a wide one (always both edges)"""
    return np.unique(np.r_[np.arange(0, w, max(1, w // 64)), w - 1])


@functools.lru_cache(maxsize=None)
def _micro():
    from tests.test_scene import _micro_level
    data = _micro_level()
    a = wad.Archive(data)
    tex = wad.TextureDirectory(a)
    return data, a, tex, scene.compile_scene(a, tex, 0)


@functools.lru_cache(maxsize=None)
def _rich():
    """The content-rich generated level, with a pose 1.25 units in front of a sprite and one in front of a masked middle."""
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=30, thing_pct=70))
    a = wad.Archive(data)
    tex = wad.TextureDirectory(a)
    blob = scene.compile_scene(a, tex, 0)
    level = wad.Level(a, 0)
    texrec = scene.section(blob, "textures")
    poses = []

    def room(x, y, z):
        sec = scene.sector_at(level, x, y)
        return sec >= 0 and int(level.sectors[sec]["floor"]) + 1 < z < int(level.sectors[sec]["ceil"]) - 1

    for sp in scene.section(blob, "sprites"):         # facing north at it, eye at its middle
        x, y, z = int(sp[0]), int(sp[1]) - 1.25, int(sp[2]) + int(texrec[int(sp[3]), 2]) / 2
        if 0 <= sp[3] < len(texrec) and room(x, y, z):
            poses.append((x, y, z, 90.0))
            break
    verts, mids = scene.section(blob, "verts"), scene.section(blob, "mids")
    for s in scene.section(blob, "segs"):             # facing the middle of the seg from its front side
        if s[15] < 0 or s[15] >= len(mids):
            continue
        (ax, ay), (bx, by) = verts[s[0]], verts[s[1]]
        dx, dy = float(bx - ax), float(by - ay)
        ln = math.hypot(dx, dy)
        if ln < 16:
            continue
        x, y = (ax + bx) / 2 + 1.25 * dy / ln, (ay + by) / 2 - 1.25 * dx / ln
        z = (int(mids[s[15], 2]) + int(mids[s[15], 3])) / 2
        if room(x, y, z):
            poses.append((round(x * 256) / 256, round(y * 256) / 256, z, math.degrees(math.atan2(dx, -dy))))
            break
    assert len(poses) == 2, "no sprite / masked middle with room in front of it"
    return data, a, tex, blob, tuple(poses)


def _micro_poses():
    """Room A spans x -256..0, y 0..256, floor 0, ceiling 128; room B (x 0..256) has floor 24, ceiling 96."""
    head_on = [(-128.0, d, 60.0, 270.0) for d in HEAD_ON]                 # facing room A's south wall
    return head_on + [(-255.5, 0.5, 0.25, 45.0),                         # corner, eye 1/4 unit above the floor, across both rooms
                      (-255.5, 128.0, 127.75, 0.0),                      # eye 1/4 unit below the ceiling, looking east
                      (-255.5, 255.5, 24.125, 315.0)]                    # eye 1/8 unit above room B's floor height, diagonal


def _scale64(view, pose, a, b):
    """column_eval's 64-bit scale (Q18 px per unit, before any cap) of the one-sided seg a -> b at every column it covers."""
    c, s = render.sincos_q30(pose["angle"][0])
    px8, py8 = int(pose["x"][0]) >> 8, int(pose["y"][0]) >> 8

    def to_view(wx, wy):
        dx, dy = (wx << 8) - px8, (wy << 8) - py8
        return (dx * s - dy * c) >> 30, (dx * c + dy * s) >> 30
    (ax, az), (bx, bz) = to_view(*a), to_view(*b)
    W, F, FY2 = view.W, view.F, view.FY2
    dxs, dzs = bx - ax, bz - az
    C = az * dxs - ax * dzs
    if C <= 0:
        return []
    sh = max(0, (abs(dxs) * F + abs(dzs) * W).bit_length() - 31)
    M = F * C
    shm = M.bit_length() - 31
    Rm = min((1 << 62) // (M >> shm if shm >= 0 else M << -shm), 0xFFFFFFFF)
    e = 5 - sh + shm
    out = []
    for x in range(W):
        N, D = az * (2 * x + 1 - W) - ax * F, dxs * F - dzs * (2 * x + 1 - W)
        if D <= 0 or N < 0 or N > D or (D >> sh) < 1:
            continue
        P = ((min(D, M >> 8) >> sh) * Rm) >> 32
        scale = (FY2 * P) >> e if e >= 0 else (FY2 * P) << -e
        out.append(min(scale, FY2 << 17))
    return out


@pytest.mark.parametrize("fov", FOVS)
def test_oracle_agrees_with_raycaster_over_the_view_range(b2d, hostcheck, fov):
    """Every size at one field of view, in one tally (the 1 % rounding-residue rule means nothing for a 2-pixel frame)."""
    t, known_px = Tally(), 0
    for w, h in SIZES:
        view = render.make_view(w, h, fov)
        if not _accepted(w, view):
            with pytest.raises(b2d.B2dError) as e:
                b2d.make_view(w, h, fov)
            assert e.value.code == b2d.ERR_INVALID_ARG
            with pytest.raises(RuntimeError):
                render.render(_micro()[3], view, render.make_pose(-128, 1, 60, 270))
            continue
        pv = b2d.make_view(w, h, fov)
        assert (pv.width, pv.height, pv.F, pv.FY2) == (view.W, view.H, view.F, view.FY2)
        cols = _cols(w)
        for (data, a, tex, blob), poses in ((_micro(), _micro_poses()), (_rich()[:4], list(_rich()[4]))):
            pa = np.concatenate([render.make_pose(*p) for p in poses])
            ofb = render.render(blob, view, pa, threads=4)
            hfb, counts, _ = hostcheck(blob, pv, pa)
            bad = [(poses[i], int((ofb[i] != hfb[i]).sum())) for i in range(len(poses)) if not np.array_equal(ofb[i], hfb[i])]
            assert not bad, "%dx%d: hostcheck differs from the oracle (pose, pixels): %s" % (w, h, bad[:4])
            assert (counts >= 0).all()
            for i, pose in enumerate(poses):
                known = (fov == 169.9 and h == 2160 and pose == _rich()[4][1]) or (fov in (10.0, 15.0) and (w, h) == (31, 3)
                                                                                    and pose == _micro_poses()[-1])
                g, kind, dbg = glcaster.render(a, tex, 0, w, h, *pose, focal2=(view.F, view.FY2), cols=cols, debug=True)
                dbg["near_depth"] = max(1.0, view.FY2 / 16384.0)
                n0 = len(t.unexplained)
                t.add(g, ofb[i][:, cols], dbg, (w, h) + pose)
                if known:                       # counted against KNOWN_UNEXPLAINED instead
                    known_px += len(t.unexplained) - n0
                    t.sum["differing"] -= len(t.unexplained) - n0
                    del t.unexplained[n0:]
        if view.FY2 > 16384:
            # the nearest head-on pose must reach the 2^31 scale regime, or this test no longer tests it
            pose = render.make_pose(-128, HEAD_ON[0], 60, 270)
            assert max(_scale64(view, pose, (0, 0), (-256, 0))) > ROW_SCALE_MAX, (w, h)
    assert known_px <= KNOWN_UNEXPLAINED.get(fov, 0), known_px
    t.check(residue=_residue(fov), near_clamp_bound=NEAR_CLAMP_BOUND)


def test_wide_views_are_refused_at_the_width_bound(b2d):
    """W <= 256 F: the widest view b2d_view_init accepts at 24 rows, and the first it refuses."""
    ok = b2d.make_view(4096, 24, 104.0)
    assert ok.F == 16
    with pytest.raises(b2d.B2dError) as e:
        b2d.make_view(4096, 24, 105.0)
    assert e.value.code == b2d.ERR_INVALID_ARG
    assert render.make_view(4096, 24, 105.0).F == 15


def test_focal_lengths_fit_the_largest_generated_level(b2d):
    """seg_frame_setup's M = F * C in 63 bits: |C| <= (eye-to-vertex distance) * (seg length) in Q8 x Q8, for an eye anywhere a
    pose can put it (|x|, |y| < 32768 units: Q16 in int32), on the largest generated level, at the largest F a renderer accepts
    (and b2d_view_init's largest)."""
    from tests.test_scale import sweep_level
    blob = sweep_level(32)[1]
    verts = scene.section(blob, "verts").astype(np.int64)
    segs = scene.section(blob, "segs")
    diag = math.hypot(*(np.abs(verts).max(0) + 32768)) * 256
    seglen = max(math.hypot(*(verts[s[1]] - verts[s[0]])) for s in segs) * 256
    assert b2d.make_view(4096, 2160, 1.0001).FY2 < (1 << 18)
    assert (1 << 18) * diag * seglen < 2.0 ** 63


# ---- the same grid through the kernels ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_gpu_kernels_equal_oracle_over_the_view_range(b2d, size):
    """Index and RGBA frames, host path and b2d_render_device, at every field of view of the grid."""
    import torch
    w, h = size
    scenes = [b2d.Scene(b2d.Archive.from_bytes(d), 0) for d in (_micro()[0], _rich()[0])]
    for fov in FOVS:
        view = render.make_view(w, h, fov)
        if not _accepted(w, view):
            continue
        pv = b2d.make_view(w, h, fov)
        for sc, blob, poses in zip(scenes, (_micro()[3], _rich()[3]), (_micro_poses(), list(_rich()[4]))):
            pa = np.concatenate([render.make_pose(*p) for p in poses])
            ofb, orgba = render.render(blob, view, pa, rgba=True, threads=8)
            r = b2d.Renderer(sc, pv, max_batch=len(pa))
            idx, rgba = r.render(pa, rgba=True)
            assert r.status() == 0
            bad = [(poses[i], int((ofb[i] != idx[i]).sum())) for i in range(len(poses)) if not np.array_equal(ofb[i], idx[i])]
            assert not bad, "fov %s %dx%d: kernels differ from the oracle (pose, pixels): %s" % (fov, w, h, bad[:4])
            assert np.array_equal(orgba, rgba), "fov %s %dx%d: RGBA" % (fov, w, h)
            dp = torch.from_numpy(np.ascontiguousarray(pa).view(np.int32).reshape(-1, 4).copy()).cuda()
            di = torch.full((len(pa), h, w), 0xA5, dtype=torch.uint8, device="cuda")
            dr = torch.zeros((len(pa), h, w), dtype=torch.int32, device="cuda")
            r.render_device(dp.data_ptr(), len(pa), di.data_ptr(), dr.data_ptr())
            torch.cuda.synchronize()
            assert r.status() == 0
            assert np.array_equal(di.cpu().numpy(), ofb), "fov %s %dx%d: render_device index" % (fov, w, h)
            assert np.array_equal(dr.cpu().numpy().view(np.uint32), orgba), "fov %s %dx%d: render_device RGBA" % (fov, w, h)
