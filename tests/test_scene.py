"""Scene compiler: the product's C++ compiler must emit the same bytes as the oracle's restatement of
LevelWalker (wad/src/visitor.rs:711-937) for every map, plus spot checks of the pegging rules."""
import os

import numpy as np
import pytest

from oracle import scene as S
from oracle import wad as W


@pytest.mark.parametrize("seed,maps", [(1, ("E1M1", "E1M2")), (7, ("E2M3",)), (21, ("MAP01", "MAP12", "MAP25"))])
def test_blob_identical(b2d, seed, maps):
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(seed, maps)
    oa = W.Archive(data)
    ot = W.TextureDirectory(oa)
    pa = b2d.Archive.from_bytes(data)
    for i in range(len(maps)):
        ob = S.compile_scene(oa, ot, i)
        ps = b2d.Scene(pa, i)
        pb = ps.blob
        if ob != pb:
            A, B = np.frombuffer(ob, np.uint8), np.frombuffer(pb, np.uint8)
            n = min(len(A), len(B))
            first = int(np.nonzero(A[:n] != B[:n])[0][0]) if (A[:n] != B[:n]).any() else n
            pytest.fail("blob differs for %s at byte %d (sizes %d / %d)" % (maps[i], first, len(A), len(B)))


def test_sky_table():
    assert S.sky_for(W.wad_name(b"E1M1")) == W.wad_name(b"SKY1")
    assert S.sky_for(W.wad_name(b"E3M7")) == W.wad_name(b"SKY3")
    assert S.sky_for(W.wad_name(b"MAP11")) == W.wad_name(b"SKY1")
    assert S.sky_for(W.wad_name(b"MAP12")) == W.wad_name(b"SKY2")
    assert S.sky_for(W.wad_name(b"MAP32")) == W.wad_name(b"SKY3")
    assert S.sky_for(W.wad_name(b"MAP30")) == W.wad_name(b"SKY1")      # no match -> entry 0


def test_light_byte_matches_integer_rule():
    # (light>>3)/31 (+-2/31 clamped) * 255 truncated, in float32 (light.rs:82-115, lights.rs:26-29)
    for light in range(0, 256):
        for c in (-1, 0, 1):
            l5 = min(31, max(0, (light >> 3) + 2 * c))
            assert W.light_byte(light, c) == (l5 * 255) // 31, (light, c)


def test_sector_at_agrees(b2d, synth_wad, product_scene):
    oa = W.Archive(synth_wad)
    lv = W.Level(oa, 0)
    rng = np.random.default_rng(3)
    inside = 0
    for _ in range(400):
        x, y = rng.uniform(-1400, 1400), rng.uniform(-1300, 1300)
        so = S.sector_at(lv, float(x), float(y))
        sp, fl, ce = product_scene.sector_at(float(x), float(y))
        assert so == sp
        if so >= 0:
            inside += 1
            assert (fl, ce) == (int(lv.sectors[so]["floor"]), int(lv.sectors[so]["ceil"]))
    assert inside > 100


def test_view_constants(b2d):
    from oracle import render
    for (w, h, fov) in ((320, 200, 65.0), (1920, 1080, 65.0), (3840, 2160, 65.0), (1280, 720, 90.0)):
        pv, ov = b2d.make_view(w, h, fov), render.make_view(w, h, fov)
        assert (pv.width, pv.height, pv.F, pv.FY2) == (ov.W, ov.H, ov.F, ov.FY2)
    v = b2d.make_view(1920, 1080)
    assert (v.F, v.FY2) == (1413, 1695)     # 2*focal: fovy 65 deg, aspect correction 1.2


def _micro_level(two_sided_flags=0x0004, front=(0, 128), back=(24, 96), tex_h=128, yoff=0, mid="-", upper=None,
                 lower="STEP2"):
    """Two square rooms A (x<0) and B (x>0) sharing the edge x=0; returns seg records of the shared line."""
    from rust_doom_b200 import synthwad as G
    import struct
    rng = G.SplitMix64(9)
    playpal = G.make_playpal()
    patches, tex, flats = G.make_graphics(rng)
    pn, t1 = G.make_pnames_texture1(list(patches.keys()), tex)
    V = [(-256, 0), (0, 0), (0, 256), (-256, 256), (256, 0), (256, 256)]
    secs = [G.Sector(front[0], front[1], "FLOOR1", "CEIL1", 160), G.Sector(back[0], back[1], "FLOOR2", "F_SKY1" if back[1] == -1 else "CEIL2", 160)]
    sides = [G.Sidedef(0, 0, "-", "-", "BRICK1", 0) for _ in range(3)] + \
            [G.Sidedef(0, 0, "-", "-", "BRICK1", 1) for _ in range(3)] + \
            [G.Sidedef(8, yoff, upper if upper is not None else ("PANEL72" if tex_h == 72 else "BRICK2"), lower, mid, 0),
             G.Sidedef(8, yoff, "BRICK2", "STEP2", mid, 1)]
    # room A walls: clockwise so the room is on the right
    L = [G.Linedef(0, 3, 1, 0, 0, 0, -1), G.Linedef(3, 2, 1, 0, 0, 1, -1), G.Linedef(1, 0, 1, 0, 0, 2, -1),
         G.Linedef(2, 5, 1, 0, 0, 3, -1), G.Linedef(5, 4, 1, 0, 0, 4, -1), G.Linedef(4, 1, 1, 0, 0, 5, -1),
         G.Linedef(2, 1, two_sided_flags, 0, 0, 6, 7)]     # 2->1 points south: A (west) is on the right
    segsA = [(0, 3, 0, 0), (3, 2, 1, 0), (1, 0, 2, 0), (2, 1, 6, 0)]
    segsB = [(2, 5, 3, 0), (5, 4, 4, 0), (4, 1, 5, 0), (1, 2, 6, 1)]
    lb = struct.pack
    lumps = [("PLAYPAL", playpal), ("COLORMAP", G.make_colormap(playpal)), ("E1M1", b""),
             ("THINGS", lb("<hhhHH", -128, 128, 0, 1, 7)),
             ("LINEDEFS", b"".join(lb("<HHHHHhh", l.v1, l.v2, l.flags, 0, 0, l.right, l.left) for l in L)),
             ("SIDEDEFS", b"".join(lb("<hh8s8s8sH", s.xoff, s.yoff, G._name8(s.upper), G._name8(s.lower), G._name8(s.middle), s.sector) for s in sides)),
             ("VERTEXES", b"".join(lb("<hh", *v) for v in V)),
             ("SEGS", b"".join(lb("<HHHHHH", a, b, 0, l, d, 0) for (a, b, l, d) in segsA + segsB)),
             ("SSECTORS", lb("<HH", 4, 0) + lb("<HH", 4, 4)),
             # partition x=0 pointing north: right = east = B (subsector 1), left = A (subsector 0)
             ("NODES", lb("<hhhh4h4hHH", 0, 0, 0, 256, 256, 0, 0, 256, 256, 0, -256, 0, 0x8001, 0x8000)),
             ("SECTORS", b"".join(lb("<hh8s8shHH", s.floor, s.ceil, G._name8(s.floor_flat), G._name8(s.ceil_flat), s.light, 0, 0) for s in secs)),
             ("TEXTURE1", t1), ("PNAMES", pn)] + list(patches.items()) + \
            [("S_START", b""), ("S_END", b""), ("F_START", b"")] + list(flats.items()) + [("F_END", b"")]
    return G.assemble_wad(lumps)


def test_pegging_rules(b2d):
    # visitor.rs:772-807,909-913 with texture BRICK2/STEP2 heights 128 / 24
    data = _micro_level(two_sided_flags=0x0004, front=(0, 128), back=(24, 96))
    oa = W.Archive(data)
    blob = S.compile_scene(oa, W.TextureDirectory(oa), 0)
    assert blob == b2d.Scene(b2d.Archive.from_bytes(data), 0).blob
    segs = S.section(blob, "segs")
    tex = S.section(blob, "textures")
    s = segs[3]                      # A's side of the shared line
    assert s[3] == S.SEG_TWO_SIDED and s[2] == 0 and s[15] == -1     # two-sided, front sector 0, no masked middle
    assert (s[13], s[14]) == (96, 24)                      # opening: back ceil / back floor
    hA, hB = int(tex[s[6]][2]), int(tex[s[9]][2])
    assert (hA, hB) == (128, 24)
    assert s[7] == (hA - (128 - 96)) % hA and s[8] == 128  # upper, pegged: bottom of texture at back ceil
    assert s[10] == 0 and s[11] == 24                      # lower, pegged: top of texture at back floor
    assert s[4] == 8 and s[5] == 256 << 12                 # x offset, length Q12
    # unpegged variants
    data = _micro_level(two_sided_flags=0x0004 | 0x0008 | 0x0010, front=(0, 128), back=(24, 96), yoff=5)
    oa = W.Archive(data)
    blob = S.compile_scene(oa, W.TextureDirectory(oa), 0)
    assert blob == b2d.Scene(b2d.Archive.from_bytes(data), 0).blob
    s = S.section(blob, "segs")[3]
    assert s[7] == 5                                       # upper unpegged: top of texture at front ceil
    assert s[10] == (24 - 24 + 128 + 5) % 24               # lower unpegged: aligned to the front ceiling
    # the B side sees no upper/lower (its floor is higher, ceiling lower)
    sb = S.section(blob, "segs")[7]
    assert sb[6] == -1 and sb[9] == -1 and (sb[13], sb[14]) == (96, 24)


def test_contrast_rule(b2d):
    # visitor.rs:887-901: wad dy == 0 -> brighten (+2/31), dx == 0 -> darken (-2/31)
    data = _micro_level()
    oa = W.Archive(data)
    segs = S.section(S.compile_scene(oa, W.TextureDirectory(oa), 0), "segs")
    base = W.light_byte(160, 0)
    assert segs[0][12] == W.light_byte(160, -1)     # (-256,0)->(-256,256): dx == 0
    assert segs[1][12] == W.light_byte(160, +1)     # horizontal
    assert W.light_byte(160, -1) < base < W.light_byte(160, +1)


def test_wad_layout_quirks(b2d):
    """IWAD layout variations real files have: TEXTURE2, nested F1_START/F1_END markers (virtual lumps inside
    F_START..F_END), a duplicated lump name (the later one wins, archive.rs:85), lower-case texture names in
    sidedefs (upper-cased on read, name.rs:41-75) and a sprite that shadows a texture name (tex.rs:475-497)."""
    import struct
    from rust_doom_b200 import synthwad as G
    rng = G.SplitMix64(5)
    playpal = G.make_playpal()
    patches, tex, flats = G.make_graphics(rng)
    names = list(patches.keys())
    pn, t1 = G.make_pnames_texture1(names, tex[:9])
    _, t2 = G.make_pnames_texture1(names, tex[9:])
    lvl = G.LevelBuilder("E1M1", 42, G.SynthConfig(gx=4, gy=3, origin=(-512, -384))).generate()
    lumps = lvl.lumps()
    # lower-case the texture names of the first 20 sidedefs
    sd = bytearray(dict(lumps)["SIDEDEFS"])
    for i in range(20):
        for f in range(3):
            o = i * 30 + 4 + 8 * f
            sd[o:o + 8] = bytes(sd[o:o + 8]).lower()
    lumps = [(n, bytes(sd) if n == "SIDEDEFS" else d) for n, d in lumps]
    flat_items = list(flats.items())
    wadlumps = [("PLAYPAL", playpal), ("COLORMAP", G.make_colormap(playpal))] + lumps + \
               [("TEXTURE1", t1), ("TEXTURE2", t2), ("PNAMES", pn)] + list(patches.items()) + \
               [("S_START", b""), ("BRICK1", G.encode_picture(G._img_gradient(rng, 64, 128, 9))), ("S_END", b""),
                ("F_START", b""), ("F1_START", b"")] + flat_items[:6] + [("F1_END", b""), ("F2_START", b"")] + \
               flat_items[6:] + [("F2_END", b""), ("FLOOR1", flat_items[3][1]), ("F_END", b"")]
    data = G.assemble_wad(wadlumps)
    oa = W.Archive(data)
    ot = W.TextureDirectory(oa)
    assert len(ot.textures) >= len(tex)                       # TEXTURE1 + TEXTURE2 (+ the sprite)
    assert ot.flats[W.wad_name(b"FLOOR1")] == flat_items[3][1]       # later duplicate wins
    assert ot.textures[W.wad_name(b"BRICK1")].shape == (128, 64)      # sprite shadows the texture
    ob = S.compile_scene(oa, ot, 0)
    pb = b2d.Scene(b2d.Archive.from_bytes(data), 0).blob
    assert ob == pb
    segs = S.section(ob, "segs")
    assert (segs[:, 6] >= 0).sum() > 10                       # lower-case names resolved to textures


def test_middle_texture_pegging(b2d):
    """visitor.rs:808-836 (peg choice), 875-885 (float pegs clamp the quad to the texture height),
    909-919 (t at `high`); COMBO2 is 64x128."""
    def mid_of(**kw):
        data = _micro_level(mid="COMBO2", **kw)
        oa = W.Archive(data)
        blob = S.compile_scene(oa, W.TextureDirectory(oa), 0)
        assert blob == b2d.Scene(b2d.Archive.from_bytes(data), 0).blob
        s = S.section(blob, "segs")[3]
        assert s[15] >= 0
        return [int(v) for v in S.section(blob, "mids")[s[15]][:4]], S.section(blob, "textures")
    # opening between back floor 24 and back ceiling 96 (height 72)
    (tex, t_high, low, high), texs = mid_of(two_sided_flags=0x0004)                       # Peg::Top
    assert (int(texs[tex][1]), int(texs[tex][2])) == (64, 128) and (t_high, low, high) == (0, 24, 96)
    (_, t_high, low, high), _ = mid_of(two_sided_flags=0x0004 | 0x0010)                   # Peg::Bottom
    assert (t_high, low, high) == (128 - 72, 24, 96)
    (_, t_high, low, high), _ = mid_of(two_sided_flags=0x0004 | 0x0010, upper="-", yoff=6)    # Peg::TopFloat
    assert (t_high, low, high) == (6, 24 + 6, 24 + 128 + 6)
    (_, t_high, low, high), _ = mid_of(two_sided_flags=0x0004, lower="-", yoff=-5)        # Peg::BottomFloat
    assert (t_high, low, high) == ((-5) % 128, 96 - 5 - 128, 96 - 5)


def test_light_effect_parameters_and_hand_values():
    """new_light (light.rs:27-80) restated; hand-computed values of light_level_at (lights.rs:33-66)."""
    f = np.float32
    # glow: level 1.0, alt 0.5, speed 0.5: triangle wave of period scale/speed = 1 s between level and alt
    info = (S.LIGHT_GLOW, f(1.0), f(0.5), f(0.5), f(0.0), f(0.0))
    assert S.light_byte_at(info, 0) == 255                      # phase 0 -> level
    assert 126 <= S.light_byte_at(info, 17) <= 131              # ~half a period -> ~alt (0.5*255 = 127.5)
    assert S.light_byte_at(info, 35) == 255                     # one full period (time = 1.0 exactly)
    # strobe, sync 0: alt during the first `duration` of each 1/speed period
    info = (S.LIGHT_ALTERNATE, f(1.0), f(0.0), f(2.0), f(0.7), f(0.0))
    assert [S.light_byte_at(info, t) for t in (0, 5, 12, 13, 17, 18, 30)] == [0, 0, 0, 255, 255, 0, 255]
    # flash: alt with probability ~duration
    info = (S.LIGHT_RANDOM, f(1.0), f(0.0), f(20.0), f(0.06), f(123.4))
    vals = [S.light_byte_at(info, t) for t in range(0, 7000, 7)]
    assert set(vals) == {0, 255} and 0.02 < vals.count(0) / len(vals) < 0.12
    # static sector: clamped, truncated
    assert S.light_byte_at((S.LIGHT_NONE, f(144 >> 3) / f(31.0), f(0), f(0), f(0), f(0)), 99) == W.light_byte(144, 0)


def test_fixture_blob_identical(product_scene, oracle_scene):
    """The level every generic test runs on (generated, or B2D_IWAD): both scene compilers give the same bytes."""
    assert product_scene.blob == oracle_scene


def test_suite_runs_on_a_supplied_iwad(tmp_path):
    """B2D_IWAD hook (CPU tier): the generic fixtures take their level from the file the variable names.  A generated
    IWAD on disk stands in for doom1.wad: the scene-compiler and hostcheck tests must pass on it."""
    import subprocess
    import sys
    from rust_doom_b200 import synthwad
    path = tmp_path / "custom.wad"
    path.write_bytes(synthwad.build_iwad(9, ("E1M1", "E1M2"), cfg=synthwad.SynthConfig(mid_pct=10, thing_pct=10)))
    env = dict(os.environ, B2D_IWAD=str(path))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "not gpu", "tests/test_scene.py", "tests/test_hostcheck.py",
                          "-k", "fixture_blob_identical or sector_at_agrees or hostcheck_320x200 or hostcheck_odd_sizes"], cwd=root, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]


@pytest.mark.parametrize("seed,maps,level,cfg", [(1, ("E1M1", "E1M2"), 1, {}), (5, ("MAP03",), 0, dict(mid_pct=30, thing_pct=40, anim=True, odd_tex=True))])
def test_scene_from_lumps_equals_scene_from_wad(b2d, seed, maps, level, cfg):
    """b2d_scene_create_from_lumps (SURVEY 8b: 'caller-owned raw lump bytes + composed textures + COLORMAP + PLAYPAL[0]'):
    a host that has parsed the WAD itself -- here the oracle's loader stands in for rust-doom's wad crate -- hands over
    the level's eight lumps and its decoded images; the compiled scene is byte-identical to the one built from the
    WAD file, and so is sector_at."""
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(seed, maps, cfg=synthwad.SynthConfig(**cfg))
    a = W.Archive(data)
    td = W.TextureDirectory(a)
    marker = a.levels[level]
    lumps = {key: a.read(marker + 1 + k) for k, key in enumerate(b2d.Scene.LUMP_ORDER)}
    sc = b2d.Scene.from_lumps(a.lumps[marker][0], lumps, list(td.textures.items()), list(td.flats.items()), td.colormaps, td.palettes[0])
    ref = b2d.Scene(b2d.Archive.from_bytes(data), level)
    assert sc.blob == ref.blob
    assert sc.info.n_segs == ref.info.n_segs and sc.info.has_start == ref.info.has_start
    assert sc.start_pose.tobytes() == ref.start_pose.tobytes()
    assert sc.sector_at(100.0, 50.0) == ref.sector_at(100.0, 50.0)
    # errors follow wad::ErrorKind::CorruptWad: a lump whose size is not a multiple of the record size
    bad = dict(lumps, segs=lumps["segs"][:-1])
    with pytest.raises(b2d.B2dError) as e:
        b2d.Scene.from_lumps(a.lumps[marker][0], bad, [], [], td.colormaps, td.palettes[0])
    assert e.value.code == b2d.ERR_CORRUPT_WAD


def test_last_player_start_wins(b2d):
    """game/src/level.rs:757-762 overwrites start_pos on every player-1 start marker: with several (voodoo dolls) the
    LAST one in THINGS is the spawn.  Turn the last decoration thing of a generated level into a second type-1 thing."""
    import struct
    from rust_doom_b200 import synthwad
    data = bytearray(synthwad.build_iwad(4, ("E1M1",), cfg=synthwad.SynthConfig(thing_pct=40)))
    a = W.Archive(bytes(data))
    _, pos, size = a.lumps[a.levels[0] + 1]                   # THINGS: 10-byte records
    n = size // 10
    first = [i for i in range(n) if struct.unpack_from("<h", data, pos + 10 * i + 6)[0] == 1]
    assert len(first) == 1
    # the last thing that stands inside the level becomes a second player-1 start
    lv = W.Level(a, 0)
    cand = [i for i in range(n) if i != first[0] and S.sector_at(lv, float(lv.things[i]["x"]), float(lv.things[i]["y"])) >= 0]
    k = max(cand)
    assert k > first[0]
    struct.pack_into("<h", data, pos + 10 * k + 6, 1)
    x, y, ang = struct.unpack_from("<hhh", data, pos + 10 * k)
    a2 = W.Archive(bytes(data))
    ob = S.compile_scene(a2, W.TextureDirectory(a2), 0)
    sc = b2d.Scene(b2d.Archive.from_bytes(bytes(data)), 0)
    assert sc.blob == ob
    assert sc.info.has_start and sc.info.start.x == (x - 32) * 65536 and sc.info.start.y == y * 65536


def _moving_case(seed, cfg):
    from rust_doom_b200 import synthwad
    from tests.refcheck import moves as MV
    data = synthwad.build_iwad(seed, ("E1M1",), cfg=synthwad.SynthConfig(**cfg))
    a = W.Archive(data)
    tex = W.TextureDirectory(a)
    dyn, mv = MV.pick(W.Level(a, 0), seed + 100, 12)
    return data, a, tex, dyn, mv


@pytest.mark.parametrize("seed", [1, 9])
def test_dynamic_sectors_compile_and_move_like_the_oracle(b2d, seed):
    """Moving sectors (DESIGN.md C16): the product's scene compiler given the dynamic-sector list, and its re-derivation
    of the height-dependent tables for one state, are byte-identical to the oracle's numpy restatement."""
    data, a, tex, dyn, mv = _moving_case(seed, dict(mid_pct=30, thing_pct=50))
    ob = S.compile_scene(a, tex, 0, dynamic=dyn)
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0, dynamic=dyn)
    assert sc.blob == ob and sc.info.n_dynamic == len(dyn)
    assert S.header(ob)[S.H_NDYN] == len(dyn)
    # declaring sectors resolves more pieces (textures of walls that only appear while a sector moves), never fewer
    static = S.compile_scene(a, tex, 0)
    assert S.header(ob)[S.H_NTEX] >= S.header(static)[S.H_NTEX]
    assert (S.section(ob, "sectors") == S.section(static, "sectors")).all()
    moved = S.apply_moves(ob, mv)
    assert sc.tables_at(0, mv) == S.tables_at(ob, 0, mv)
    assert sc.tables_at(0, ()) == S.tables_at(ob, 0)
    assert moved != ob and S.apply_moves(ob, ()) == ob
    from tests.refcheck import moves as MV
    level = W.Level(a, 0)
    for k in range(25):                                  # more states of the same declaration, any height inside the ranges
        st = MV.state(level, dyn, 1000 * seed + k, hole_free=False)
        assert sc.tables_at(k, st) == sc.tables_at(k, list(reversed(st)))            # order of the list does not matter
        got = np.frombuffer(sc.tables_at(k, st), np.int32)
        want = np.frombuffer(S.tables_at(ob, k, st), np.int32)
        assert (got == want).all(), "state %d" % k
    # rest heights + offsets, openings follow
    s0, s1 = S.section(ob, "sectors"), S.section(moved, "sectors")
    for sec, dfl, dcl in mv:
        assert s1[sec, 0] == s0[sec, 0] + dfl and s1[sec, 1] == s0[sec, 1] + dcl
    segs, segdyn = S.section(moved, "segs"), S.section(ob, "segdyn")
    for i in range(len(segs)):
        if segs[i, 3] & S.SEG_INVALID:
            continue
        f, b = int(segs[i, 2]), int(segdyn[i, 0])
        if b < 0:
            assert (segs[i, 13], segs[i, 14]) == (s1[f, 1], s1[f, 0])
        else:
            assert segs[i, 14] == max(s1[f, 0], s1[b, 0]) and segs[i, 13] <= s1[f, 1]


def test_dynamic_sector_arguments_are_checked(b2d):
    data, a, tex, dyn, mv = _moving_case(3, {})
    arch = b2d.Archive.from_bytes(data)
    sc = b2d.Scene(arch, 0, dynamic=dyn)
    undeclared = next(i for i in range(sc.info.n_sectors) if i not in {d[0] for d in dyn})
    with pytest.raises(b2d.B2dError):
        sc.tables_at(0, [(undeclared, 1, 0)])                       # not declared dynamic
    with pytest.raises(b2d.B2dError):
        sc.tables_at(0, [(dyn[0][0], 4000, 0)])                     # outside the declared range
    with pytest.raises(ValueError):
        S.apply_moves(sc.blob, [(undeclared, 1, 0)])
    with pytest.raises(ValueError):
        S.apply_moves(sc.blob, [(dyn[0][0], 4000, 0)])
    with pytest.raises(b2d.B2dError):
        b2d.Scene(arch, 0, dynamic=[dyn[0], dyn[0]])                # listed twice
    with pytest.raises(b2d.B2dError):
        b2d.Scene(arch, 0, dynamic=[(100000, 0, 0, 0, 0)])
    with pytest.raises(W.WadError):
        S.compile_scene(a, tex, 0, dynamic=[dyn[0], dyn[0]])
    # the lumps entry point (b2d_scene_create_from_lumps_dynamic) takes the same list and compiles the same scene
    marker = a.levels[0]
    lumps = {key: a.read(marker + 1 + k) for k, key in enumerate(b2d.Scene.LUMP_ORDER)}
    from_lumps = b2d.Scene.from_lumps(a.lumps[marker][0], lumps, list(tex.textures.items()), list(tex.flats.items()),
                                      tex.colormaps, tex.palettes[0], dynamic=dyn)
    assert from_lumps.blob == S.compile_scene(a, tex, 0, dynamic=dyn) and from_lumps.info.n_dynamic == len(dyn)
    assert from_lumps.tables_at(7, mv) == sc.tables_at(7, mv)
    with pytest.raises(b2d.B2dError):
        b2d.Scene.from_lumps(a.lumps[marker][0], lumps, list(tex.textures.items()), list(tex.flats.items()),
                             tex.colormaps, tex.palettes[0], dynamic=[(100000, 0, 0, 0, 0)])


def test_time_and_moves_compose(b2d):
    """Level time and sector state are one table set: animation / light effects at `tics` plus the moved heights."""
    data, a, tex, dyn, mv = _moving_case(5, dict(mid_pct=20, thing_pct=30, anim=True))
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0, dynamic=dyn)
    ob = S.compile_scene(a, tex, 0, dynamic=dyn)
    h = S.header(ob)
    for tics in (0, 9, 1000):
        t0, t1 = sc.tables_at(tics, ()), sc.tables_at(tics, mv)
        # texture records do not depend on heights
        ntex = h[S.H_NTEX] * 32
        assert t0[:ntex] == t1[:ntex]
        assert t0 == S.tables_at(ob, tics) and t1 == S.tables_at(ob, tics, mv)


# ---- the state rule over level kinds and edge tics ----------------------------------------------------------------------
# Five generated levels whose tables depend on different parts of a state, so that each reduction of the compact state
# (DESIGN.md §3: the tic kept as tics & ~7 when a level only animates, tics & 0xFFFFFF when it only scrolls, 0 when it does
# neither) is taken by one of them.
STATE_KINDS = ("lights", "anim", "scroll", "moves", "all")
EDGE_TICS = (0, 7, 8, 15, (1 << 24) - 1, 1 << 24, (1 << 24) + 7, (1 << 32) - 8, (1 << 32) - 1)


def declare_doors(level, seed=5, n_sectors=16):
    """tests/refcheck/moves.py's declaration, with the ceilings of the first few non-sky sectors allowed down to their floor;
    -> (dynamic, doors = [(sector, floor, ceiling)])"""
    from tests.refcheck import moves as MV
    dyn = MV.declare(level, seed, n_sectors)
    doors = []
    for k, (s, fmin, fmax, cmin, cmax) in enumerate(dyn):
        f0, c0 = int(level.sectors[s]["floor"]), int(level.sectors[s]["ceil"])
        if cmin != cmax and len(doors) < 4:
            dyn[k] = (s, fmin, fmax, min(cmin, f0), cmax)
            doors.append((s, f0, c0))
    return dyn, doors


def _patch_level(data: bytes, lump: str, record: int, fields, fn) -> bytes:
    """`data` with fn(8-byte name) -> 8-byte name applied to the name fields at byte offsets `fields` of every `record`-byte
    record of the first level's lump `lump` (one of Scene.LUMP_ORDER)"""
    from rust_doom_b200 import Scene
    a = W.Archive(data)
    _, pos, size = a.lumps[a.levels[0] + 1 + Scene.LUMP_ORDER.index(lump)]
    out = bytearray(data)
    for r in range(pos, pos + size, record):
        for f in fields:
            out[r + f:r + f + 8] = fn(bytes(out[r + f:r + f + 8]))
    return bytes(out)


def _static_names(groups, replacement: bytes):
    frames = {W.wad_name(n.encode()) for g in groups for n in g}
    return lambda name: replacement if W.wad_name(name) in frames else name


def state_level(kind: str):
    """-> (wad bytes, dynamic sectors, doors, level) of one level kind:
    lights  the c2 level (bench.py): light effects only
    anim    animated textures and flats only (the scrolling special 0x30 cleared in LINEDEFS)
    scroll  scrolling walls only (animated names in SIDEDEFS and SECTORS replaced by static ones)
    moves   dynamic sectors only (doors)
    all     animation, scrolling, light effects, doors, masked middles and sprites"""
    import struct
    from oracle.anim_table import FLATS, WALLS
    from rust_doom_b200 import synthwad
    cfg = {"lights": {}, "anim": dict(anim=True, light_fx=False), "scroll": dict(anim=True, light_fx=False),
           "moves": dict(light_fx=False), "all": dict(anim=True, mid_pct=20, thing_pct=30)}[kind]
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(**cfg))
    if kind == "anim":                          # special (u16 at byte 6 of a linedef) 0x30 -> 0
        data = _patch_level(data, "linedefs", 14, [6], lambda b: struct.pack("<H", 0) + b[2:] if b[:2] == b"\x30\0" else b)
    if kind == "scroll":
        data = _patch_level(data, "sidedefs", 30, [4, 12, 20], _static_names(WALLS, W.wad_name(b"BRICK1")))
        data = _patch_level(data, "sectors", 26, [4, 12], _static_names(FLATS, W.wad_name(b"FLOOR1")))
    level = W.Level(W.Archive(data), 0)
    dyn, doors = declare_doors(level) if kind in ("moves", "all") else ([], [])
    return data, dyn, doors, level


def state_moves(level, dyn, doors, seed):
    """move lists for a level kind: at rest, all offsets zero (at rest too), doors shut, one random state"""
    from tests.refcheck import moves as MV
    if not dyn:
        return [[]]
    return [[], [(dyn[0][0], 0, 0), (dyn[-1][0], 0, 0)], [(s, 0, f0 - c0) for (s, f0, c0) in doors],
            MV.state(level, dyn, seed, hole_free=False)]


def assert_kind(blob: bytes, kind: str):
    """what the blob holds is what the kind says"""
    h = S.header(blob)
    n = h[S.H_NSECTORS]
    lights = set(np.frombuffer(blob, "<u4", 8 * n, h[S.H_OFF_LIGHTS]).reshape(n, 8)[:, 0].tolist()) - {S.LIGHT_NONE}
    scrolls = bool((S.section(blob, "segs")[:, 3] & S.SEG_SCROLL).any())
    want = {"lights": (False, False, True, False), "anim": (True, False, False, False), "scroll": (False, True, False, False),
            "moves": (False, False, False, True), "all": (True, True, True, True)}[kind]
    assert (h[S.H_NANIM] > 0, scrolls, bool(lights), h[S.H_NDYN] > 0) == want, kind
    assert lights <= {S.LIGHT_GLOW, S.LIGHT_RANDOM, S.LIGHT_ALTERNATE}
    if kind == "all":
        assert lights == {S.LIGHT_GLOW, S.LIGHT_RANDOM, S.LIGHT_ALTERNATE}


@pytest.mark.parametrize("kind", STATE_KINDS)
def test_tables_at_equals_oracle_restatement(b2d, kind):
    """b2d_scene_tables_at (the product's state rule, scene_at_time) equals oracle/scene.py tables_at byte for byte on every
    level kind, at the edge tics of the animation step, the 24-bit scroll wrap and the 32-bit tic range, and at random tics,
    with no moves, an all-zero move list, shut doors and random states."""
    data, dyn, doors, level = state_level(kind)
    a = W.Archive(data)
    ob = S.compile_scene(a, W.TextureDirectory(a), 0, dynamic=dyn)
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0, dynamic=dyn)
    assert sc.blob == ob
    assert_kind(ob, kind)
    rng = np.random.default_rng(STATE_KINDS.index(kind))
    tics = list(EDGE_TICS) + rng.integers(0, 1 << 32, 6, dtype=np.uint64).tolist()
    for i, t in enumerate(tics):
        for mv in state_moves(level, dyn, doors, 100 + i):
            got, want = sc.tables_at(t, mv), S.tables_at(ob, t, mv)
            if got != want:
                g, w = np.frombuffer(got, np.int32), np.frombuffer(want, np.int32)
                pytest.fail("%s: tics %d, moves %s: tables differ at word %s" % (kind, t, mv, np.nonzero(g != w)[0][:8]))
