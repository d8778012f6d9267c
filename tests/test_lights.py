"""The player's light effects without a GPU (DESIGN.md C18): the test reference of tests/lightcheck.py checked against
independent renders -- extra light against a level whose SECTORS lights are raised by 16 e, the sky mask of the fixed
colormap against a second way of finding the sky -- and against hand-computed bytes; the C ABI, exports and ctypes
prototypes of the _lights calls; and the CLIs' refusals of bad --fixed-colormap / --extralight values, which happen
before any device is touched."""
import ctypes
import os
import re
import struct
import subprocess

import numpy as np
import pytest

from oracle import render
from oracle import scene as S
from oracle import wad as W
from tests import lightcheck as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def raise_sector_lights(data: bytes, level: int, amount: int) -> bytes:
    """the IWAD with every SECTORS light of `level` raised by `amount` (the light is the int16 at byte 20 of a 26-byte
    sector record)"""
    a = W.Archive(data)
    name, off, size = a.lumps[a.levels[level] + 8]
    assert name.rstrip(b"\0") == b"SECTORS" and size % 26 == 0
    out = bytearray(data)
    for k in range(size // 26):
        at = off + 26 * k + 20
        (light,) = struct.unpack_from("<h", out, at)
        struct.pack_into("<h", out, at, light + amount)
    return bytes(out)


def static_wad(seed=3):
    from rust_doom_b200 import synthwad
    return synthwad.build_iwad(seed, ("E1M1",), cfg=synthwad.SynthConfig(light_fx=False, mid_pct=30, thing_pct=40))


def rich_wad():
    from rust_doom_b200 import synthwad
    return synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=30, thing_pct=40, anim=True))


def blob_of(data: bytes, level: int = 0) -> bytes:
    a = W.Archive(data)
    return S.compile_scene(a, W.TextureDirectory(a), level)


def poses_of(data: bytes, n: int, seed: int):
    """seeded poses inside the level (random points and a fly-through)"""
    import rust_doom_b200 as b2d
    from tests.conftest import sample_poses
    return sample_poses(b2d, b2d.Scene(b2d.Archive.from_bytes(data), 0), n, seed)


# ---- extra light -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("e", (1, 2))
def test_extralight_renders_like_sector_lights_raised_by_16e(e):
    """On a level with static lights only (masked middles and sprites included), extra light e gives the frames and the
    tables of the same level with every SECTORS light raised by 16 e, compiled from its own lumps."""
    data = static_wad()
    blob, raised = blob_of(data), blob_of(raise_sector_lights(data, 0, 16 * e))
    assert S.section(blob, "sprites").shape[0] > 0 and S.section(blob, "mids").shape[0] > 0
    assert (S.sector_lights_at(blob, 0) == -1).all()
    assert L.tables_at(blob, 17, extralight=e) == S.tables_at(raised, 17)
    assert L.tables_at(blob, 17, extralight=e) != S.tables_at(blob, 17)
    view = render.make_view(160, 100)
    poses = poses_of(data, 6, 5)
    got = L.render(blob, view, poses, extralight=e)
    want = render.render(raised, view, poses)
    assert np.array_equal(got, want)
    assert not np.array_equal(got, render.render(blob, view, poses))


def test_extralight_bytes_by_hand():
    """tables_at with extra light against bytes computed here: static sectors (clamped at 255), their segs with fake
    contrast, their sprites, and a sector with a light effect, whose byte is clamp(level_at(t) + 2e/31) * 255."""
    f = np.float32
    blob = blob_of(raise_sector_lights(rich_wad(), 0, 80))       # bright enough that extra light clamps somewhere
    n = S.header(blob)[S.H_NSECTORS]
    rec = np.frombuffer(blob, dtype="<u4", count=8 * n, offset=S.header(blob)[S.H_OFF_LIGHTS]).reshape(n, 8)
    effect = np.nonzero(rec[:, 0] != S.LIGHT_NONE)[0]
    static = np.nonzero(rec[:, 0] == S.LIGHT_NONE)[0]
    assert len(effect) and len(static)
    steps = np.rint(rec[:, 1].copy().view("<f4").astype(np.float64) * 31).astype(int)
    top = [int(sec) for sec in static if 29 <= steps[sec] <= 31]
    assert top, "no static sector that extra light takes past full brightness"
    tics = 123
    for e in (1, 2):
        t = L.tables_at(blob, tics, extralight=e)
        h = S.header(blob)
        ntex, nseg, nspr = h[S.H_NTEX], h[S.H_NSEGS], h[S.H_NSPRITES]
        sectors = np.frombuffer(t, "<i4", 8 * n, 32 * ntex).reshape(n, 8)
        segs = np.frombuffer(t, "<i4", 16 * nseg, 32 * ntex + 32 * n).reshape(nseg, 16)
        sprites = np.frombuffer(t, "<i4", 8 * nspr, 32 * ntex + 32 * n + 64 * nseg).reshape(nspr, 8)
        level = rec[:, 1].copy().view("<f4")

        def static_byte(sec, contrast):
            v = f(int(round(float(level[sec]) * 31)) + 2 * e) / f(31)
            if contrast:
                v = min(max(v + (f(2) / f(31) if contrast > 0 else f(-2) / f(31)), f(0)), f(1))
            return int(float(min(max(v, f(0)), f(1)) * f(255)))

        for sec in static:
            assert sectors[sec, 4] == static_byte(sec, 0), (e, sec)
        assert all(sectors[sec, 4] == 255 for sec in top if steps[sec] + 2 * e >= 31)
        for sec in effect:
            fl = rec[sec, 1:6].copy().view("<f4")
            v = S.light_level_at((int(rec[sec, 0]), *fl), f(f(tics) / f(35)))
            v = min(max(f(v + f(2 * e) / f(31)), f(0)), f(1))
            assert sectors[sec, 4] == int(float(f(v * f(255)))), (e, sec)
        verts = S.section(blob, "verts")
        for S_ in segs:
            if S_[3] & S.SEG_INVALID:
                continue
            fr = int(S_[2])
            if fr in set(effect.tolist()):
                assert S_[12] == sectors[fr, 4]
                continue
            dx, dy = int(verts[S_[1], 0] - verts[S_[0], 0]), int(verts[S_[1], 1] - verts[S_[0], 1])
            assert S_[12] == static_byte(fr, 1 if dy == 0 else (-1 if dx == 0 else 0))
        for P in sprites:
            assert P[4] == sectors[P[5], 4]


def rich_wad_blob():
    return blob_of(rich_wad())


# ---- fixed colormap --------------------------------------------------------------------------------------------------
def test_sky_mask_is_where_the_sky_texture_shows():
    """the sky mask of the fixed-colormap reference equals the pixels that change when only the sky texture's texels do
    (identity COLORMAP rows, every sky texel 7, then 9)"""
    data = rich_wad()
    blob = blob_of(data)
    view = render.make_view(160, 100)
    poses = poses_of(data, 6, 11)
    h = S.header(blob)
    T = S.section(blob, "textures")[h[S.H_SKY_TEX]]
    at, n = h[S.H_OFF_TEXELS] + int(T[0]), int(T[1]) * int(T[2])
    frames = []
    for v in (7, 9):
        b = bytearray(blob)
        b[at:at + n] = bytes([v]) * n
        for k in range(32):
            b[h[S.H_OFF_COLORMAP] + 256 * k: h[S.H_OFF_COLORMAP] + 256 * k + 256] = bytes(range(256))
        frames.append(render.render(bytes(b), view, poses, tics=40))
    sky = L.sky_mask(blob, view, poses, 40)
    assert sky.any() and (~sky).any()
    assert np.array_equal(sky, frames[0] != frames[1])


@pytest.mark.parametrize("row", (0, 1, 31, 32))
def test_fixed_colormap_reference(row):
    """off the sky, a fixed-colormap frame is the frame of the scene whose rows 0..31 are row r, and differs from the
    normal frame; on the sky it is the normal frame; extra light changes nothing under it"""
    data = rich_wad()
    blob = blob_of(data)
    view = render.make_view(160, 100)
    poses = poses_of(data, 6, 11)
    got = L.render(blob, view, poses, tics=40, fixed_colormap=row)
    normal = render.render(blob, view, poses, tics=40)
    sky = L.sky_mask(blob, view, poses, 40)
    assert np.array_equal(got[sky], normal[sky])
    assert np.array_equal(got[~sky], render.render(L.with_colormap_rows(blob, row), view, poses, tics=40)[~sky])
    assert not np.array_equal(got[~sky], normal[~sky])
    assert np.array_equal(L.render(blob, view, poses, tics=40, fixed_colormap=row, extralight=2), got)


# ---- ABI -------------------------------------------------------------------------------------------------------------
CALLS = ("b2d_render_levels_states_lights", "b2d_render_device_levels_states_lights", "b2d_walk_device_levels_states_lights")


def test_header_declares_the_struct_and_calls():
    with open(os.path.join(ROOT, "include", "b2d.h")) as f:
        h = f.read()
    assert re.search(r"typedef struct b2d_frame_light \{\s*int32_t fixed_colormap;[^}]*uint32_t extralight;[^}]*\} b2d_frame_light;", h)
    for name in CALLS:
        m = re.search(r"int %s\(([^;]*)\);" % name, h)
        assert m, name
        args = [a.strip() for a in m.group(1).split(",")]
        assert args[3] == "const b2d_frame_state *states" and args[4] == "const b2d_frame_light *lights", args


def test_library_exports_and_prototypes(b2d):
    from rust_doom_b200 import _lib
    L = _lib.load()
    assert ctypes.sizeof(_lib.FrameLight) == 8
    for name in CALLS:
        assert name in _lib.EXPORTS
        fn = getattr(L, name)
        assert fn.argtypes[3] is ctypes.POINTER(_lib.FrameState) and fn.argtypes[4] is ctypes.POINTER(_lib.FrameLight)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH],
                         capture_output=True, text=True, check=True).stdout
    for name in CALLS:
        assert re.search(r" T %s$" % name, out, re.M), name


# ---- CLIs ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra,needle", [
    (["--levels", "0", "--fixed-colormap", "33"], "--fixed-colormap"),
    (["--levels", "0", "--fixed-colormap", "-2"], "--fixed-colormap"),
    (["--levels", "0", "--extralight", "3"], "--extralight"),
    (["--fixed-colormap", "32"], "--levels"),
    (["--extralight", "1"], "--levels"),
    (["--levels", "0", "--world", "2", "--id-file", "x", "--fixed-colormap", "32"], "--world"),
])
def test_clis_refuse_bad_lights_before_any_device(tmp_path, b2d, capsys, extra, needle):
    from rust_doom_b200 import cli, synthwad
    from tests.test_cli import _b2d_binary
    wad = tmp_path / "syn.wad"
    wad.write_bytes(synthwad.build_iwad(1, ("E1M1",)))
    assert cli.main(["--iwad", str(wad), "-r", "64x40"] + extra) == 2
    assert needle in capsys.readouterr().err
    out = subprocess.run([_b2d_binary(), "-i", str(wad), "-r", "64x40"] + extra, capture_output=True, text=True)
    assert out.returncode == 2 and needle in out.stderr, (out.returncode, out.stderr)
