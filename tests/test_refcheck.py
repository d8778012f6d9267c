"""Scene-semantics pin for the oracle.  The reference has no CPU renderer to compare pixels with, but its
pipeline is well defined: a static triangle soup + depth test + the GLSL in assets/shaders/.  With a depth
test the visible surface at a pixel is the nearest one along the pixel's ray, so tests/refcheck/glcaster.py
ray-casts the level in float64 straight from the reference's geometry and shader rules (no BSP order, no column
clipping, no fixed point).  The oracle -- a completely different algorithm -- must agree with it pixel for pixel up
to rounding: tests/refcheck/classify.py explains EVERY differing pixel (adjacent texel / colormap row +-1, within one
pixel of a silhouette, sub-pixel shift on a minified texture), counts the three known deviations of a column renderer
separately under tight bounds, and the tests assert that nothing is left unexplained."""
import numpy as np
import pytest

from oracle import render, scene, wad
from tests.refcheck import classify, glcaster


def _poses_in(level, want_sky, n, seed):
    rng = np.random.default_rng(seed)
    sec_bytes = level.sectors.tobytes()
    out = []
    while len(out) < n:
        x, y = rng.uniform(-1280, 1280), rng.uniform(-1152, 1152)
        sec = scene.sector_at(level, x, y)
        if sec < 0:
            continue
        s = level.sectors[sec]
        is_sky = wad.is_sky_flat(wad.wad_name(sec_bytes[sec * 26 + 12:sec * 26 + 20]))
        if is_sky != want_sky or int(s["ceil"]) - int(s["floor"]) < 56:
            continue
        out.append((round(x * 4) / 4, round(y * 4) / 4, int(s["floor"]) + 41, float(rng.integers(0, 720)) / 2))
    return out


class Tally:
    """Sums the classification of several frames and applies the acceptance rule."""

    def __init__(self):
        self.px = 0
        self.sum = {}
        self.unexplained = []

    def add(self, g, o, dbg, what):
        r = classify.classify(g, o, dbg)
        self.px += g.size
        for k, v in r.items():
            if k != "unexplained":
                self.sum[k] = self.sum.get(k, 0) + v
        self.unexplained += [(what,) + u for u in r["unexplained"]]
        return r

    def check(self, allow=None, sky_hack_bound=2e-4, residue=0.01, near_clamp_bound=0.0):
        """`allow`: deviation counts of another tally (the same poses before a change) that are not held against this one;
        `sky_hack_bound`: share of the pixels the sky-hack deviation may take (it grows with the amount of tall geometry
        standing behind lower open-air sectors); `residue`: share of the pixels all differing ones may take; `near_clamp_bound`:
        share the near-clamp deviation may take (only counted when the frames' debug data carry the clamp depth)"""
        s = self.sum
        base = allow.sum if allow is not None else {}
        assert not self.unexplained, "unexplained pixels: %s" % self.unexplained[:10]
        assert s["texel"] + s["silhouette"] + s["minified"] + s["sky_hack"] + s["sprite_order"] + s["sliver"] + s["near_clamp"] \
            == s["differing"]
        assert s["differing"] < residue * self.px, s                    # rounding residue: well under 1 % of the pixels by default
        assert s["near_clamp"] <= near_clamp_bound * self.px, s
        for k in ("sky_hack", "sliver", "sprite_order"):
            assert s[k] - base.get(k, 0) <= (sky_hack_bound if k == "sky_hack" else 2e-4) * self.px, (k, s, base)


def _frame(a, tex, blob, W_, H_, pose, tics=0, cols=None):
    x, y, z, ang = pose
    view = render.make_view(W_, H_)
    g, kind, dbg = glcaster.render(a, tex, 0, W_, H_, x, y, z, ang, focal2=(view.F, view.FY2), tics=tics, cols=cols, debug=True)
    o = render.render(blob, view, render.make_pose(x, y, z, ang), tics=tics)[0]
    return g, (o if cols is None else o[:, cols]), kind, dbg


@pytest.mark.parametrize("want_sky", [False, True])
def test_oracle_agrees_with_reference_semantics_raycaster(synth_wad, oracle_scene, want_sky):
    a = wad.Archive(synth_wad)
    tex = wad.TextureDirectory(a)
    level = wad.Level(a, 0)
    t, sky_share = Tally(), []
    for pose in _poses_in(level, want_sky, 6, 7 + want_sky):
        g, o, kind, dbg = _frame(a, tex, oracle_scene, 320, 200, pose)
        t.add(g, o, dbg, pose)
        sky_share.append(float((kind == 3).mean()))
        if (kind == 3).any():
            assert (g == o)[kind == 3].mean() > 0.97, "sky mapping disagrees"
    t.check()
    if want_sky:
        assert max(sky_share) > 0.05, "no pose actually saw the sky"


def test_oracle_agrees_with_raycaster_at_1920x1080(synth_wad, oracle_scene):
    """The benchmark resolution: every fourth column of two 1080p frames (an indoor pose and one under the sky)."""
    a = wad.Archive(synth_wad)
    tex = wad.TextureDirectory(a)
    level = wad.Level(a, 0)
    cols = np.arange(0, 1920, 4)
    t = Tally()
    for pose in _poses_in(level, False, 1, 47) + _poses_in(level, True, 1, 48):
        g, o, kind, dbg = _frame(a, tex, oracle_scene, 1920, 1080, pose, cols=cols)
        t.add(g, o, dbg, pose)
    t.check()
    assert t.px == 2 * 480 * 1080


def test_oracle_agrees_with_raycaster_at_3840x2160(synth_wad, oracle_scene):
    """BASELINE.json's 4K configuration: every sixteenth column of one 3840x2160 frame."""
    a = wad.Archive(synth_wad)
    tex = wad.TextureDirectory(a)
    level = wad.Level(a, 0)
    cols = np.arange(0, 3840, 16)
    t = Tally()
    for pose in _poses_in(level, False, 1, 49):
        g, o, kind, dbg = _frame(a, tex, oracle_scene, 3840, 2160, pose, cols=cols)
        t.add(g, o, dbg, pose)
    t.check()
    assert t.px == 240 * 2160


def test_masked_middle_textures_agree_with_raycaster():
    """Two-sided middle textures with holes (visitor.rs:808-836; transparent texels discarded,
    static.frag:21-22): the oracle's deferred back-to-front pass vs rays that pass through the holes."""
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=45))
    a = wad.Archive(data)
    tex = wad.TextureDirectory(a)
    blob = scene.compile_scene(a, tex, 0)
    level = wad.Level(a, 0)
    assert scene.header(blob)[scene.H_NMIDS] > 50
    view = render.make_view(320, 200)
    t, twice = Tally(), 0
    for pose in _poses_in(level, False, 6, 17) + _poses_in(level, True, 4, 18):
        g, o, kind, dbg = _frame(a, tex, blob, 320, 200, pose)
        t.add(g, o, dbg, pose)
        _, hits = render.render(blob, view, render.make_pose(*pose), seg_hits=True)
        twice += int(hits.sum()) - 320 * 200          # pixels overdrawn by masked textures
    t.check()
    assert twice > 5000, "the poses never looked through a masked texture"
    g, o, kind, dbg = _frame(a, tex, blob, 1920, 1080, _poses_in(level, False, 1, 19)[0], cols=np.arange(0, 1920, 8))
    t2 = Tally()
    t2.add(g, o, dbg, "1080p")
    t2.check()


def test_decoration_sprites_agree_with_raycaster():
    """Thing sprites (visitor.rs:1062-1137, sprite.vert/frag): the oracle's per-subsector deferred billboards vs
    depth-tested billboards in the ray caster."""
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=30, thing_pct=70))
    a = wad.Archive(data)
    tex = wad.TextureDirectory(a)
    blob = scene.compile_scene(a, tex, 0)
    level = wad.Level(a, 0)
    assert scene.header(blob)[scene.H_NSPRITES] > 30
    t, sprite_px, sprite_same = Tally(), 0, 0
    for pose in _poses_in(level, False, 6, 27) + _poses_in(level, True, 4, 28):
        g, o, kind, dbg = _frame(a, tex, blob, 320, 200, pose)
        t.add(g, o, dbg, pose)
        sprite_px += int((kind == 4).sum())
        sprite_same += int(((g == o) & (kind == 4)).sum())
    t.check()
    assert sprite_px > 2000 and sprite_same / sprite_px > 0.97, (sprite_px, sprite_same)


def test_animation_and_scrolling_agree_with_raycaster():
    """u_time semantics (static.vert:23-39, visitor.rs:922): frame = floor(tics/8) mod n of the group (tex.rs:260,
    302-306: whichever frame name the map uses), scroll = 1 texel per tic."""
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(anim=True))
    a = wad.Archive(data)
    tex = wad.TextureDirectory(a)
    blob = scene.compile_scene(a, tex, 0)
    level = wad.Level(a, 0)
    view = render.make_view(320, 200)
    t, moved = Tally(), 0
    poses = _poses_in(level, False, 4, 37) + _poses_in(level, True, 2, 38)
    for tics in (0, 5, 8, 19, 1000):
        for pose in poses:
            g, o, kind, dbg = _frame(a, tex, blob, 320, 200, pose, tics=tics)
            t.add(g, o, dbg, (tics,) + pose)
            o0 = render.render(blob, view, render.make_pose(*pose))[0]
            moved += int((o != o0).sum())
    t.check()
    assert moved > 20000, "time never changed a pixel"


def test_moving_sectors_agree_with_raycaster():
    """Doors / lifts as a per-batch state (DESIGN.md C16).  The ray caster builds the reference's meshes literally --
    quads pre-extended over the declared height ranges, every quad, flat and decoration translated with the floor or
    ceiling object it is attached to (visitor.rs:733-836, 957-983, 1106-1121; game/src/level.rs:201-245), nearest hit
    wins -- and the oracle renders the re-derived per-seg pieces (oracle/scene.py apply_moves).  States in which the
    reference itself opens a hole (tests/refcheck/moves.py) are not drawn."""
    from rust_doom_b200 import synthwad
    from tests.refcheck import moves as MV
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=30, thing_pct=50))
    a = wad.Archive(data)
    tex = wad.TextureDirectory(a)
    level = wad.Level(a, 0)
    view = render.make_view(320, 200)
    t, rest, changed = Tally(), Tally(), 0
    for seed in (5, 6, 7):
        dyn, mv = MV.pick(level, seed, 14)
        blob = scene.compile_scene(a, tex, 0, dynamic=dyn)
        moved = scene.apply_moves(blob, mv)
        for pose in _poses_in(level, False, 4, 30 + seed) + _poses_in(level, True, 2, 40 + seed):
            x, y, z, ang = pose
            g, kind, dbg = glcaster.render(a, tex, 0, 320, 200, x, y, z, ang, focal2=(view.F, view.FY2), debug=True, dynamic=dyn, moves=mv)
            o = render.render(moved, view, render.make_pose(x, y, z, ang))[0]
            t.add(g, o, dbg, (seed,) + pose)
            g0, _, dbg0 = glcaster.render(a, tex, 0, 320, 200, x, y, z, ang, focal2=(view.F, view.FY2), debug=True)
            o0 = render.render(blob, view, render.make_pose(x, y, z, ang))[0]
            rest.add(g0, o0, dbg0, (seed,) + pose)
            changed += int((o != o0).sum())
    t.check(allow=rest)             # the known deviations (sky hack, slivers) of these poses at rest are not the moves' doing
    assert changed > 20000, "the moves never changed a pixel"


def test_light_effects_agree_with_raycaster(synth_wad, oracle_scene):
    """Sector light effects over time (wad/src/light.rs:27-115, game/src/lights.rs:26-66: glow, flash / flicker, strobes):
    the light byte of an effect sector at `tics`, as the ray caster evaluates it from the reference's float32 formulas,
    picks the same colormap row as the oracle's at every pixel of the sector's walls, flats and sprites."""
    a = wad.Archive(synth_wad)
    tex = wad.TextureDirectory(a)
    level = wad.Level(a, 0)
    lights = scene.section(oracle_scene, "sectors")[:, 4]
    n_fx = sum(1 for i in range(len(level.sectors)) if scene.light_info(level, i)[0] != scene.LIGHT_NONE)
    assert n_fx >= 5, "the generated level has too few light-effect sectors"
    view = render.make_view(320, 200)
    t, moved = Tally(), 0
    poses = _poses_in(level, False, 4, 57) + _poses_in(level, True, 2, 58)
    for tics in (3, 17, 35, 211, 100000):
        assert (scene.sector_lights_at(oracle_scene, tics) >= 0).sum() == n_fx
        for pose in poses:
            g, o, kind, dbg = _frame(a, tex, oracle_scene, 320, 200, pose, tics=tics)
            t.add(g, o, dbg, (tics,) + pose)
            moved += int((o != render.render(oracle_scene, view, render.make_pose(*pose))[0]).sum())
    t.check()
    assert moved > 20000, "the light effects never changed a pixel"
    del lights


@pytest.mark.parametrize("seed,name,cfg", [(7, "E2M3", {}), (21, "MAP12", dict(odd_tex=True, mid_pct=20)), (33, "MAP25", dict(odd_tex=True, thing_pct=40, anim=True))])
def test_other_levels_agree_with_raycaster(seed, name, cfg):
    """Other generated levels: another episode's sky (E2 / MAP12 / MAP25: wad/src/meta.rs:156-172), wall textures with odd
    heights and non-power-of-two widths (floor-mod sampling, static.frag:19-22), mixed content, another field of view."""
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(seed, (name,), cfg=synthwad.SynthConfig(**cfg))
    a = wad.Archive(data)
    tex = wad.TextureDirectory(a)
    blob = scene.compile_scene(a, tex, 0)
    level = wad.Level(a, 0)
    t = Tally()
    for fov, (w, h) in ((65.0, (320, 200)), (90.0, (400, 300))):
        view = render.make_view(w, h, fov)
        for pose in _poses_in(level, False, 3, seed + int(fov)) + _poses_in(level, True, 2, seed + 1 + int(fov)):
            x, y, z, ang = pose
            g, kind, dbg = glcaster.render(a, tex, 0, w, h, x, y, z, ang, fov_deg=fov, focal2=(view.F, view.FY2), tics=9, debug=True)
            o = render.render(blob, view, render.make_pose(x, y, z, ang), tics=9)[0]
            t.add(g, o, dbg, (fov,) + pose)
    # the MAP25-style level has open-air sectors of very different ceiling heights next to tall buildings: the Doom-style
    # sky (a sky ceiling hides what pokes above it) shows on up to 0.6 % of the pixels there; everything else as usual
    t.check(sky_hack_bound=6e-3 if name == "MAP25" else 2e-4)
