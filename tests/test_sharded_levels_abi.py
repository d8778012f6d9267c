"""Level sets on the sharded path and the per-frame-level palette kernel on the C ABI (no GPU needed): include/b2d.h
declares both calls, libb2d.so exports them, the ctypes binding matches the header, the restated partition of a level-set
job covers every pose once and pads with the last entry's level and state, and the compiled CLI parses --levels."""
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = {"b2d_render_sharded_levels_states": 13, "b2d_palette_lut_levels_device": 6}


def _declaration(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2d.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+%s\s*\(([^;]*)\)\s*;" % name, text, flags=re.S)
    assert m, "b2d.h does not declare %s" % name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def test_header_declares_the_calls():
    for name, arity in CALLS.items():
        assert len(_declaration(name)) == arity, name
    assert "Not covered: levels in b2d_render_sharded" not in open(os.path.join(ROOT, "include", "b2d.h")).read()


def test_library_exports_the_calls_with_argtypes_matching_the_header(b2d):
    import ctypes
    from rust_doom_b200 import _lib
    lib = _lib.load()
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    ptr_like = (ctypes.c_void_p,)
    for name, arity in CALLS.items():
        assert name in _lib.EXPORTS and re.search(r"\bT %s$" % name, out, flags=re.M), name
        types = getattr(lib, name).argtypes
        assert types and len(types) == arity, name
        for decl, t in zip(_declaration(name), types):
            if "*" in decl:
                assert t in ptr_like or hasattr(t, "_type_") or t is _lib.CHUNK_FN, (name, decl, t)
            elif decl.startswith("size_t"):
                assert t is ctypes.c_size_t, (name, decl, t)
            elif decl.startswith("int "):
                assert t is ctypes.c_int, (name, decl, t)
            elif decl.startswith("b2d_chunk_fn"):
                assert t is _lib.CHUNK_FN, (name, decl, t)
    for name in ("render_sharded_levels_states", "palette_lut_levels_device"):
        assert callable(getattr(b2d.Renderer, name))


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("n_total", [1, 5, 7, 24, 100, 257])
@pytest.mark.parametrize("chunk", [0, 1, 3, 64])
def test_partition_covers_every_pose_once(world, n_total, chunk):
    from rust_doom_b200 import parallel
    poses = np.arange(n_total)
    levels = np.arange(n_total) % 5
    tics = 1000 + np.arange(n_total)
    moves = [[(i, 8, 0)] for i in range(n_total)]
    per, plan = parallel.sharded_schedule(n_total, world, chunk, 7)
    seen = []
    for q in range(world):
        p, lv, t, m = parallel.padded_block_levels_states(poses, levels, tics, q, world, moves)
        assert len(p) == len(lv) == len(t) == len(m) == per
        assert sum(c for _, c in plan) == per and all(c <= min(chunk or 256, 7) for _, c in plan)
        for first, cnt in plan:
            for j in range(cnt):
                g = q * per + first + j                                   # frame j of rank q's slice of the chunk
                i = first + j
                if g < n_total:
                    seen.append(g)
                    assert (p[i], lv[i], t[i], m[i]) == (g, levels[g], tics[g], moves[g])
                else:                                                     # the padded tail: the last entry, whole
                    assert (p[i], lv[i], t[i], m[i]) == (n_total - 1, levels[-1], tics[-1], moves[-1])
    assert sorted(seen) == list(range(n_total))


def test_padded_block_is_the_levels_states_block_poses():
    from rust_doom_b200 import parallel
    poses = np.arange(10) * 3
    for q in range(4):
        assert np.array_equal(parallel.padded_block(poses, q, 4), parallel.padded_block_levels_states(poses, poses, poses, q, 4)[0])


def test_compiled_cli_parses_levels(tmp_path):
    """--levels takes `all` or comma-separated indices below the archive's level count: anything else is an argument error
    (exit 2) before any device work; an accepted list goes on to build the renderer (on a box without a GPU that is the
    library's fatal error, exit 1)."""
    from rust_doom_b200 import build, synthwad
    wad = tmp_path / "t.wad"
    wad.write_bytes(synthwad.build_iwad(1, ("E1M1", "E1M2")))
    exe = build.build_cli()
    base = [exe, "--iwad", str(wad), "-r", "64x40"]
    for bad in ("2", "-1", "0,", ",1", "0,x", "", "al"):
        res = subprocess.run(base + ["--levels", bad], capture_output=True, text=True, timeout=60)
        assert res.returncode == 2 and "--levels" in res.stderr, (bad, res.stderr)
    res = subprocess.run(base + ["--levels"], capture_output=True, text=True, timeout=60)
    assert res.returncode == 2
    import torch
    if not torch.cuda.is_available():
        for ok in ("all", "1,0", "1"):
            res = subprocess.run(base + ["--levels", ok], capture_output=True, text=True, timeout=60)
            assert res.returncode == 1 and "Fatal error: renderer" in res.stderr, (ok, res.stderr)


def test_python_cli_parses_levels(capsys):
    from rust_doom_b200 import cli
    assert cli.parse_levels("all", 3) == [0, 1, 2] and cli.parse_levels("2,0", 3) == [2, 0]
    for bad in ("3", "-1", "0,,1", "x"):
        with pytest.raises(ValueError):
            cli.parse_levels(bad, 3)
    assert cli.main(["--levels", "9"]) == 2
    assert cli.main(["--levels", "0", "--world", "1"]) == 2 and "--id-file" in capsys.readouterr().err
    assert cli.main(["--world", "2"]) == 2
