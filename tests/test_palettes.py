"""Per-frame palettes without a GPU: the palettes a scene keeps (b2d_scene_num_palettes, b2d_scene_set_palettes and their
refusals), C17 with a palette per frame restated through oracle/resolve.py and checked by hand, the C ABI and ctypes
prototypes of the new calls, and the CLIs' --palette refusals, which happen before any device is touched."""
import ctypes
import inspect
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import resolve as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def resolve_palettes(index, playpals, factor, fmt, levels=None, palettes=None):
    """C17 with per-frame palettes: frame f through palette palettes[f] of level levels[f] (None: 0), where playpals[l] is
    level l's PLAYPAL, n_l x 768 bytes.  The renderer's colour table -- every level's palettes in order, level l's palette
    p at table base[l] + p -- is handed to the oracle as its list of palettes, and each frame's table index as its level."""
    tables, base = [], []
    for pp in playpals:
        raw = bytes(pp)
        assert raw and len(raw) % 768 == 0
        base.append(len(tables))
        tables += [raw[i:i + 768] for i in range(0, len(raw), 768)]
    n = len(index)
    lv = np.zeros(n, np.int64) if levels is None else np.asarray(levels, np.int64).reshape(n)
    pv = np.zeros(n, np.int64) if palettes is None else np.asarray(palettes, np.int64).reshape(n)
    counts = [len(bytes(pp)) // 768 for pp in playpals]
    assert all(0 <= pv[f] < counts[lv[f]] for f in range(n)), "palette out of range of its level"
    return R.resolve(index, tables, factor, fmt, [base[lv[f]] + pv[f] for f in range(n)])


def lump_scene(b2d, data: bytes, level: int = 0, palette=None):
    """the scene of `level` built from lumps (b2d_scene_create_from_lumps) with PLAYPAL[0], or `palette`"""
    from oracle import wad as W
    a = W.Archive(data)
    td = W.TextureDirectory(a)
    marker = a.levels[level]
    lumps = {key: a.read(marker + 1 + k) for k, key in enumerate(b2d.Scene.LUMP_ORDER)}
    return b2d.Scene.from_lumps(a.lumps[marker][0], lumps, list(td.textures.items()), list(td.flats.items()), td.colormaps,
                                td.palettes[0] if palette is None else palette)


@pytest.fixture(scope="module")
def playpal():
    from rust_doom_b200 import synthwad
    return synthwad.make_playpal()


# ---- scenes ----------------------------------------------------------------------------------------------------------
def test_archive_scene_keeps_every_playpal_entry(b2d, synth_wad):
    sc = b2d.Scene(b2d.Archive.from_bytes(synth_wad), 0)
    assert sc.num_palettes == 14
    assert sc.num_palettes == b2d.Scene(b2d.Archive.from_bytes(synth_wad), 1).num_palettes


def test_lump_scene_keeps_its_palette_and_takes_the_playpal(b2d, synth_wad, playpal):
    sc = lump_scene(b2d, synth_wad)
    blob = sc.blob
    assert sc.num_palettes == 1
    sc.set_palettes(playpal)
    assert sc.num_palettes == 14 and sc.blob == blob                  # the blob and its version do not change
    sc.set_palettes(playpal[:3 * 768])
    assert sc.num_palettes == 3
    sc.set_palettes(playpal[:768])
    assert sc.num_palettes == 1


def test_lump_scene_without_a_palette_holds_zero_bytes(b2d, synth_wad):
    sc = lump_scene(b2d, synth_wad, palette=bytes(768))
    assert sc.num_palettes == 1
    sc.set_palettes(bytes(768) + bytes(range(256)) * 3)
    assert sc.num_palettes == 2


def test_set_palettes_refusals_leave_the_scene_as_it_was(b2d, synth_wad, playpal):
    from rust_doom_b200 import _lib
    L = _lib.load()
    sc = lump_scene(b2d, synth_wad)
    sc.set_palettes(playpal[:2 * 768])
    buf = ctypes.create_string_buffer(playpal, len(playpal))
    assert L.b2d_scene_set_palettes(sc._h, None, 14) == b2d.ERR_INVALID_ARG
    assert L.b2d_scene_set_palettes(sc._h, buf, 0) == b2d.ERR_INVALID_ARG
    assert L.b2d_scene_set_palettes(None, buf, 14) == b2d.ERR_INVALID_ARG
    assert sc.num_palettes == 2
    for wrong in (playpal[768:], bytes(255 - v for v in playpal[:768]) + playpal[768:]):
        with pytest.raises(b2d.B2dError) as e:
            sc.set_palettes(wrong)
        assert e.value.code == b2d.ERR_INVALID_ARG and "palette 0" in e.value.message
        assert sc.num_palettes == 2
    one = bytearray(playpal)
    one[767] ^= 1                                                     # one byte of palette 0 differs
    with pytest.raises(b2d.B2dError):
        sc.set_palettes(bytes(one))
    for bad in (b"", playpal[:700]):
        with pytest.raises(ValueError):
            sc.set_palettes(bad)
    assert sc.num_palettes == 2
    assert L.b2d_scene_num_palettes(None) == b2d.ERR_INVALID_ARG
    # an archive scene's palette 0 is its PLAYPAL[0] as well
    arch = b2d.Scene(b2d.Archive.from_bytes(synth_wad), 0)
    with pytest.raises(b2d.B2dError):
        arch.set_palettes(bytes(768))
    arch.set_palettes(playpal[:768])
    assert arch.num_palettes == 1


# ---- the rule --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", R.FORMATS)
@pytest.mark.parametrize("k", (1, 2, 3))
def test_palette_zero_everywhere_is_the_resolve_without_palettes(playpal, fmt, k):
    rng = np.random.default_rng(k)
    idx = rng.integers(0, 256, (5, 6 * k, 4 * k), dtype=np.uint8)
    other = bytes(255 - v for v in playpal)                           # a second level with different palettes
    lv = [0, 1, 1, 0, 1]
    want = R.resolve(idx, [playpal[:768], other[:768]], k, fmt, lv)
    assert np.array_equal(resolve_palettes(idx, [playpal, other], k, fmt, lv, [0] * 5), want)
    assert np.array_equal(resolve_palettes(idx, [playpal, other], k, fmt, lv), want)


def test_red_and_green_palettes_by_hand():
    """level 0 holds a normal and a red palette, level 1 only a green one; 2 x 2 blocks resolved by hand"""
    normal = np.zeros((256, 3), np.uint8)
    normal[:, 0] = normal[:, 1] = normal[:, 2] = np.arange(256)
    red = np.zeros((256, 3), np.uint8)
    red[:, 0] = 255 - np.arange(256)
    green = np.zeros((256, 3), np.uint8)
    green[:, 1] = np.arange(256) // 2
    pals = [normal.tobytes() + red.tobytes(), green.tobytes()]
    idx = np.array([[[10, 20], [30, 41]]] * 3, np.uint8)              # three frames of one 2 x 2 block: sum 101
    out = resolve_palettes(idx, pals, 2, "rgb", levels=[0, 0, 1], palettes=[0, 1, 0])
    assert out[0, 0, 0].tolist() == [25, 25, 25]                      # (101 + 2) // 4
    assert out[1, 0, 0].tolist() == [(4 * 255 - 101 + 2) // 4, 0, 0]   # 229.75 -> 230
    assert out[2, 0, 0].tolist() == [0, (5 + 10 + 15 + 20 + 2) // 4, 0]   # 50 / 4 = 12.5 -> 13
    grey = resolve_palettes(idx, pals, 2, "gray", levels=[0, 0, 1], palettes=[0, 1, 0])
    y = lambda r, g, b: (77 * r + 150 * g + 29 * b + 128) >> 8          # noqa: E731
    assert grey[1, 0, 0] == (sum(y(255 - v, 0, 0) for v in (10, 20, 30, 41)) + 2) // 4
    assert grey[2, 0, 0] == (sum(y(0, v // 2, 0) for v in (10, 20, 30, 41)) + 2) // 4
    with pytest.raises(AssertionError):
        resolve_palettes(idx, pals, 2, "rgb", levels=[0, 0, 1], palettes=[0, 1, 1])     # level 1 has one palette


# ---- the C ABI -------------------------------------------------------------------------------------------------------
CALLS = {"b2d_scene_num_palettes": 1, "b2d_scene_set_palettes": 3, "b2d_resolve_palettes_device": 9,
         "b2d_render_sharded_levels_states_resolved_palettes": 16}


def _declaration(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2d.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+%s\s*\(([^;]*)\)\s*;" % name, text, flags=re.S)
    assert m, "b2d.h does not declare %s" % name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def test_header_declares_the_palette_forms_next_to_their_bases():
    for name, arity in CALLS.items():
        assert len(_declaration(name)) == arity, name
    base = _declaration("b2d_resolve_device")
    assert _declaration("b2d_resolve_palettes_device") == base[:3] + ["const uint32_t *palettes"] + base[3:]
    base = _declaration("b2d_render_sharded_levels_states_resolved")
    assert _declaration("b2d_render_sharded_levels_states_resolved_palettes") == base[:4] + ["const uint32_t *palettes"] + base[4:]


def test_library_exports_the_calls_with_argtypes_matching_the_header(b2d):
    from rust_doom_b200 import _lib
    lib = _lib.load()
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for name, arity in CALLS.items():
        assert name in _lib.EXPORTS and re.search(r"\bT %s$" % name, out, flags=re.M), name
        types = getattr(lib, name).argtypes
        assert types and len(types) == arity, name
        for decl, t in zip(_declaration(name), types):
            if decl.startswith("b2d_chunk_fn"):
                assert t is _lib.CHUNK_FN, (name, decl, t)
            elif "*" in decl:
                assert t is ctypes.c_void_p or hasattr(t, "_type_"), (name, decl, t)
            elif decl.startswith("size_t"):
                assert t is ctypes.c_size_t, (name, decl, t)
            else:
                assert decl.startswith("int ") and t is ctypes.c_int, (name, decl, t)
    r, p = lib.b2d_resolve_device.argtypes, lib.b2d_resolve_palettes_device.argtypes
    assert list(p) == list(r[:3]) + [ctypes.c_void_p] + list(r[3:])
    r = lib.b2d_render_sharded_levels_states_resolved.argtypes
    p = lib.b2d_render_sharded_levels_states_resolved_palettes.argtypes
    assert list(p) == list(r[:4]) + [ctypes.c_void_p] + list(r[4:])


def test_python_methods_take_palettes(b2d):
    for name in ("resolve_device", "resolve", "render_sharded_levels_states"):
        p = inspect.signature(getattr(b2d.Renderer, name)).parameters
        assert "palettes" in p and p["palettes"].default is None, name
    assert "palettes" not in inspect.signature(b2d.Renderer.render_sharded).parameters


def test_sharded_palettes_without_resolve_is_refused_before_the_library(b2d):
    r = object.__new__(b2d.Renderer)                                   # the check comes before any use of the renderer
    with pytest.raises(ValueError):
        b2d.Renderer.render_sharded_levels_states(r, None, np.zeros(1, b2d.POSE_DTYPE), [0], [0], palettes=[1])


# ---- the CLIs' refusals ----------------------------------------------------------------------------------------------
def _wad(tmp_path):
    from rust_doom_b200 import synthwad
    wad = tmp_path / "syn.wad"
    wad.write_bytes(synthwad.build_iwad(1, ("E1M1", "E1M2")))
    return wad


@pytest.mark.parametrize("extra", [[], ["--levels", "0,1"], ["--supersample", "2"]])
def test_python_cli_refuses_a_palette_outside_the_playpal(tmp_path, b2d, extra, capsys):
    from rust_doom_b200 import cli
    wad = _wad(tmp_path)
    for p in ("14", "-1"):
        assert cli.main(["--iwad", str(wad), "-r", "160x100", "--palette", p] + extra) == 2
        assert "--palette" in capsys.readouterr().err
    assert cli.main(["--iwad", str(wad), "--levels", "0", "--palette", "3", "--world", "2", "--id-file", "x"]) == 2
    assert "--palette" in capsys.readouterr().err


def test_compiled_cli_refuses_a_palette_outside_the_playpal(tmp_path, b2d):
    from tests.test_cli import _b2d_binary
    exe, wad = _b2d_binary(), _wad(tmp_path)
    for extra in ([], ["--levels", "0,1"], ["--supersample", "2"]):
        for p in ("14", "-1", "x", ""):
            out = subprocess.run([exe, "-i", str(wad), "-r", "160x100", "--palette", p] + extra, capture_output=True, text=True)
            assert out.returncode == 2 and "--palette" in out.stderr, (extra, p, out.stderr)
    out = subprocess.run([exe, "-i", str(wad), "--levels", "0", "--palette", "3", "--world", "2", "--id-file", "x"],
                         capture_output=True, text=True)
    assert out.returncode == 2 and "--palette" in out.stderr
