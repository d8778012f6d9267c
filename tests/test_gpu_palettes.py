"""-m gpu: per-frame palettes (b2d_resolve_palettes_device, b2d_render_sharded_levels_states_resolved_palettes, C17 with
T_{l,p}) bit for bit against oracle/resolve.py through tests/test_palettes.resolve_palettes.  The level set mixes an
archive scene with the generated IWAD's 14 palettes, a scene from lumps that keeps its one palette and a scene from lumps
of another WAD that was given its whole PLAYPAL, so the colour-table base of each level differs.  Also: palette 0
everywhere against b2d_resolve_device and the raster's RGBA, 1000 1080p frames, guard bytes and unaligned pointers,
refusals that enqueue nothing, the staging's stream order, the world-1 sharded call and both CLIs with --palette."""
import subprocess

import numpy as np
import pytest

from oracle import render
from tests.conftest import oracle_blob, sample_poses
from tests.test_gpu_resolve import FORMATS, _got, _random_index, clock, pending  # noqa: F401
from tests.test_palettes import lump_scene, resolve_palettes

pytestmark = pytest.mark.gpu


def _invert_playpal(data: bytes) -> bytes:
    """the WAD with every byte of its PLAYPAL lump (all 14 palettes) inverted"""
    buf = bytearray(data)
    n, diro = np.frombuffer(bytes(buf[4:12]), "<i4")
    for k in range(int(n)):
        pos, size = np.frombuffer(bytes(buf[diro + 16 * k:diro + 16 * k + 8]), "<i4")
        if bytes(buf[diro + 16 * k + 8:diro + 16 * k + 16]).rstrip(b"\0") == b"PLAYPAL":
            buf[pos:pos + size] = bytes(255 - v for v in buf[pos:pos + size])
            return bytes(buf)
    raise AssertionError("no PLAYPAL lump")


@pytest.fixture(scope="module")
def mix(b2d):
    """[{data, level, scene, playpal}]: an archive scene (14 palettes), a scene from lumps with its one palette, and a scene
    from lumps of a WAD with an inverted PLAYPAL given all 14 (table bases 0, 14, 15)"""
    from oracle import wad as W
    from rust_doom_b200 import synthwad
    a = synthwad.build_iwad(1, ("E1M1", "E1M2"))
    b = _invert_playpal(synthwad.build_iwad(7, ("E1M1",), cfg=synthwad.SynthConfig(gx=3, gy=3, origin=(-384, -384), light_fx=False)))
    pa, pb = (b"".join(W.TextureDirectory(W.Archive(d)).palettes) for d in (a, b))
    c = lump_scene(b2d, b)
    c.set_palettes(pb)
    out = [dict(data=a, level=0, scene=b2d.Scene(b2d.Archive.from_bytes(a), 0), playpal=pa),
           dict(data=a, level=1, scene=lump_scene(b2d, a, 1), playpal=pa[:768]),
           dict(data=b, level=0, scene=c, playpal=pb)]
    assert [L["scene"].num_palettes for L in out] == [14, 1, 14]
    return out


def _pals(mix):
    return [L["playpal"] for L in mix]


def _renderer(b2d, mix, w, h, max_batch=4):
    return b2d.Renderer.from_levels([L["scene"] for L in mix], b2d.make_view(w, h), max_batch=max_batch)


def _random_job(n, seed):
    """seeded random (level, palette) per frame, each palette below its level's count"""
    rng = np.random.default_rng(seed)
    lv = rng.integers(0, 3, n)
    pv = np.where(lv == 1, 0, rng.integers(0, 14, n))
    return lv, pv


@pytest.mark.parametrize("view", [(168, 120), (1920, 1080)], ids=["168x120", "1080p"])
def test_random_levels_and_palettes_every_format(b2d, mix, view):
    w, h = view
    n = 3 if w > 1000 else 12
    r = _renderer(b2d, mix, w, h, max_batch=1)
    idx = _random_index(n, h, w, w + 3)
    host = idx.cpu().numpy()
    lv, pv = _random_job(n, w)
    for k in (1, 2, 3, 8):
        for fmt in FORMATS:
            got = _got(r.resolve(idx, k, fmt, lv, pv))
            want = resolve_palettes(host, _pals(mix), k, fmt, lv, pv)
            assert got.shape == want.shape and np.array_equal(got, want), (view, k, fmt)
    # NULL levels: every frame on level 0, through its own palette
    assert np.array_equal(_got(r.resolve(idx, 2, "rgb", None, pv % 14)), resolve_palettes(host, _pals(mix), 2, "rgb", None, pv % 14))


def test_palette_zero_is_the_resolve_without_palettes_and_the_raster_rgba(b2d, mix):
    import torch
    w, h, n = 320, 200, 9
    r = _renderer(b2d, mix, w, h, max_batch=n)
    poses = np.concatenate([sample_poses(b2d, mix[k]["scene"], 3, 40 + k) for k in range(3)])
    lv = np.repeat([0, 1, 2], 3)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    idx = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
    rgba = torch.empty((n, h, w), dtype=torch.int32, device="cuda")
    r.render_device_levels(dp.data_ptr(), lv, n, idx.data_ptr(), rgba.data_ptr())
    zero = np.zeros(n, np.int64)
    for k in (1, 2, 4):
        for fmt in FORMATS:
            assert torch.equal(r.resolve(idx, k, fmt, lv, zero), r.resolve(idx, k, fmt, lv)), (k, fmt)
    assert torch.equal(r.resolve(idx, 1, "rgba", lv, zero), rgba)
    torch.cuda.synchronize()
    assert r.status() == 0
    # the tints differ from palette 0 wherever the frame shows anything
    tinted = _got(r.resolve(idx, 1, "rgba", lv, np.where(lv == 1, 0, 13)))
    assert (tinted[lv != 1] != _got(rgba)[lv != 1]).any()
    assert np.array_equal(tinted[lv == 1], _got(rgba)[lv == 1])


def test_thousand_1080p_frames_with_random_palettes(b2d, mix):
    import torch
    n, w, h, guard = 1000, 1920, 1080, 4096
    r = _renderer(b2d, mix, w, h, max_batch=1)
    idx = _random_index(n, h, w, 2000)
    lv, pv = _random_job(n, 2001)
    code = b2d.RESOLVE_GRAY8
    fb = r.resolve_frame_bytes(2, code)
    obuf = torch.full((2 * guard + n * fb,), 0x5A, dtype=torch.uint8, device="cuda")
    l0 = r.launch_count
    r.resolve_device(idx.data_ptr(), n, 2, code, obuf.data_ptr() + guard, lv, palettes=pv)
    torch.cuda.synchronize()
    assert r.launch_count == l0 + 1
    assert bool((obuf[:guard] == 0x5A).all()) and bool((obuf[guard + n * fb:] == 0x5A).all())
    out = obuf[guard:guard + n * fb].reshape(n, 540, 960)
    for f in (0, 1, 333, 500, 998, 999):
        want = resolve_palettes(idx[f:f + 1].cpu().numpy(), _pals(mix), 2, "gray", lv[f:f + 1], pv[f:f + 1])
        assert np.array_equal(out[f:f + 1].cpu().numpy(), want), f


def test_guard_bytes_and_unaligned_pointers(b2d, mix):
    import torch
    w, h, n, guard = 96, 48, 4, 4096
    r = _renderer(b2d, mix, w, h)
    src = _random_index(n, h, w, 78)
    host = src.cpu().numpy()
    lv, pv = [2, 0, 1, 0], [13, 5, 0, 9]
    ibuf = torch.empty(n * w * h + 16, dtype=torch.uint8, device="cuda")
    for off_i in range(16):
        ibuf[off_i:off_i + n * w * h].copy_(src.reshape(-1))
        off_o = (5 * off_i + 7) % 16
        for k in (1, 2, 3, 8):
            for fmt in FORMATS:
                code = b2d.RESOLVE_FORMATS[fmt]
                nbytes = n * r.resolve_frame_bytes(k, code)
                obuf = torch.full((2 * guard + nbytes + 16,), 0xA5, dtype=torch.uint8, device="cuda")
                r.resolve_device(ibuf.data_ptr() + off_i, n, k, code, obuf.data_ptr() + guard + off_o, lv, palettes=pv)
                got = obuf.cpu().numpy()
                lo, hi = guard + off_o, guard + off_o + nbytes
                assert (got[:lo] == 0xA5).all() and (got[hi:] == 0xA5).all(), (off_i, off_o, k, fmt)
                want = resolve_palettes(host, _pals(mix), k, fmt, lv, pv)
                assert np.array_equal(got[lo:hi], want.view(np.uint8).reshape(-1)), (off_i, off_o, k, fmt)


def test_invalid_arguments_enqueue_nothing(b2d, mix):
    import torch
    from rust_doom_b200 import _lib
    L = _lib.load()
    r = _renderer(b2d, mix, 320, 200)
    idx = torch.zeros((2, 200, 320), dtype=torch.uint8, device="cuda")
    out = torch.zeros(2 * 320 * 200 * 4, dtype=torch.uint8, device="cuda")
    a = lambda *v: np.array(v, np.uint32)              # noqa: E731
    lv, good, lv01, pv01, pv14, pv014, lv03 = a(0, 2), a(13, 13), a(0, 1), a(0, 1), a(14, 0), a(0, 14), a(0, 3)
    l0 = r.launch_count
    calls = [(idx.data_ptr(), lv01.ctypes.data, pv01.ctypes.data, 2, 2, 0, out.data_ptr()),     # palette 1 on 1 palette
             (idx.data_ptr(), lv.ctypes.data, pv14.ctypes.data, 2, 2, 0, out.data_ptr()),       # 14 on 14 palettes
             (idx.data_ptr(), None, pv014.ctypes.data, 2, 2, 0, out.data_ptr()),                # NULL levels: level 0
             (idx.data_ptr(), lv03.ctypes.data, good.ctypes.data, 2, 2, 0, out.data_ptr()),     # level out of range
             (None, lv.ctypes.data, good.ctypes.data, 2, 2, 0, out.data_ptr()),
             (idx.data_ptr(), lv.ctypes.data, good.ctypes.data, 2, 2, 0, None),
             (idx.data_ptr(), lv.ctypes.data, good.ctypes.data, 2, 3, 0, out.data_ptr()),       # 3 does not divide 320
             (idx.data_ptr(), lv.ctypes.data, good.ctypes.data, 2, 2, 4, out.data_ptr())]
    for ip, lp, pp, n, k, f, op in calls:
        assert L.b2d_resolve_palettes_device(r._h, ip, lp, pp, n, k, f, op, None) == b2d.ERR_INVALID_ARG, (n, k, f)
    assert L.b2d_resolve_palettes_device(None, idx.data_ptr(), None, None, 2, 2, 0, out.data_ptr(), None) == b2d.ERR_INVALID_ARG
    with pytest.raises(b2d.B2dError) as e:
        r.resolve(idx, 2, "rgb", [0, 1], [0, 1])
    assert e.value.code == b2d.ERR_INVALID_ARG and "palette" in e.value.message
    assert L.b2d_resolve_palettes_device(r._h, idx.data_ptr(), None, None, 0, 2, 0, out.data_ptr(), None) == 0     # n = 0
    torch.cuda.synchronize()
    assert r.launch_count == l0
    assert r.status() == 0


def test_second_call_waits_for_the_first_calls_staging_copy(b2d, mix, clock):
    """the table-index staging of b2d_resolve_device is rewritten only after the copy of the previous call that staged
    (with levels or palettes) has read it; a call with neither stages nothing and does not wait"""
    import torch
    r = _renderer(b2d, mix, 320, 200)
    idx = _random_index(6, 200, 320, 92)
    a, b, c = (torch.empty((6, 100, 160), dtype=torch.uint8, device="cuda") for _ in range(3))
    lva, pva = [0, 2, 1, 0, 2, 0], [1, 13, 0, 9, 4, 13]
    lvc = [2, 2, 0, 1, 0, 2]
    r.resolve_device(idx.data_ptr(), 6, 2, b2d.RESOLVE_GRAY8, a.data_ptr(), lva, palettes=pva)     # staging grown outside the hold
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    hold = clock.hold(s)
    r.resolve_device(idx.data_ptr(), 6, 2, b2d.RESOLVE_GRAY8, a.data_ptr(), lva, s.cuda_stream, pva)
    pending(hold, "first call")
    r.resolve_device(idx.data_ptr(), 6, 2, b2d.RESOLVE_GRAY8, b.data_ptr(), None, s.cuda_stream)
    pending(hold, "a call without levels or palettes")
    r.resolve_device(idx.data_ptr(), 6, 2, b2d.RESOLVE_GRAY8, c.data_ptr(), lvc, s.cuda_stream)
    assert hold.query(), "the second call rewrote the staging the first call's held copy reads"
    torch.cuda.synchronize()
    host = idx.cpu().numpy()
    assert np.array_equal(a.cpu().numpy(), resolve_palettes(host, _pals(mix), 2, "gray", lva, pva))
    assert np.array_equal(b.cpu().numpy(), resolve_palettes(host, _pals(mix), 2, "gray"))
    assert np.array_equal(c.cpu().numpy(), resolve_palettes(host, _pals(mix), 2, "gray", lvc))


# ---- world-1 sharded -------------------------------------------------------------------------------------------------
def _sharded_job(b2d, mix, n, seed):
    """3n poses, each sampled on its own random level, with a random palette and a level time per pose"""
    lv, pv = _random_job(3 * n, seed)
    samples = np.concatenate([sample_poses(b2d, mix[k]["scene"], 3 * n, seed + k) for k in range(3)])
    poses = samples[lv * 3 * n + np.arange(3 * n)]
    tics = (np.arange(3 * n) * 7) & 0xFFFF
    return poses, lv, pv, tics


@pytest.mark.parametrize("n,chunk", [(4, 5), (7, 4)])
def test_sharded_resolved_palettes_equal_the_resolve_of_the_rendered_frames(b2d, mix, n, chunk):
    import torch
    from rust_doom_b200 import _lib, jobs, parallel
    from tests.test_gpu_sharded_resolve import _run
    w, h, total = 320, 200, 3 * n
    comm = jobs.single_comm(0)
    r = _renderer(b2d, mix, w, h, max_batch=7)
    poses, lv, pv, tics = _sharded_job(b2d, mix, n, 300 + n)
    per, plan = parallel.sharded_schedule(total, 1, chunk, 7)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    idx = torch.empty((total, h, w), dtype=torch.uint8, device="cuda")
    r.render_device_levels_states(dp.data_ptr(), lv, tics, total, idx.data_ptr())
    for k, fmt in ((1, "rgba"), (2, "rgb_planar"), (2, "gray"), (4, "rgb")):
        code = b2d.RESOLVE_FORMATS[fmt]
        fb = r.resolve_frame_bytes(k, code)
        want = torch.empty(total * fb, dtype=torch.uint8, device="cuda")
        r.resolve_device(idx.data_ptr(), total, k, code, want.data_ptr(), lv, palettes=pv)
        torch.cuda.synchronize()
        got, seen, st = _run(lambda **kw: r.render_sharded_levels_states(comm, poses, lv, tics, None, chunk, **kw), total, per,
                             fb, mode=_lib.SHARD_RENDER_GATHER, resolve=(k, fmt), palettes=pv)
        assert seen == [(f, c, 1) for f, c in plan], (k, fmt)
        assert np.array_equal(got, want.cpu().numpy().reshape(total, fb)), (k, fmt)
        assert np.array_equal(got, resolve_palettes(idx.cpu().numpy(), _pals(mix), k, fmt, lv, pv).view(np.uint8).reshape(total, fb))
    assert r.status() == 0


def test_sharded_bad_palette_is_refused_before_any_launch(b2d, mix):
    from rust_doom_b200 import _lib, jobs
    comm = jobs.single_comm(0)
    r = _renderer(b2d, mix, 320, 200, max_batch=7)
    poses, lv, pv, tics = _sharded_job(b2d, mix, 5, 77)
    l0 = r.launch_count
    for bad in (np.flatnonzero(lv == 1)[-1], np.flatnonzero(lv != 1)[0]):
        pb = pv.copy()
        pb[bad] = 14 if lv[bad] != 1 else 1
        with pytest.raises(b2d.B2dError) as e:
            r.render_sharded_levels_states(comm, poses, lv, tics, None, 4, _lib.SHARD_RENDER_GATHER, None, resolve=(2, "rgb"),
                                           palettes=pb)
        assert e.value.code == b2d.ERR_INVALID_ARG and "palette" in e.value.message
    assert r.launch_count == l0


# ---- CLIs ------------------------------------------------------------------------------------------------------------
def _oracle_rgb_palette(data, level_of, poses, tics, w, h, k, palette):
    from oracle import wad as W
    playpal = b"".join(W.TextureDirectory(W.Archive(data)).palettes)
    blobs = {lv: oracle_blob(data, lv) for lv in set(level_of)}
    view = render.make_view(k * w, k * h)
    idx = np.empty((len(poses), k * h, k * w), np.uint8)
    for i in range(len(poses)):
        render.render(blobs[level_of[i]], view, poses[i:i + 1], tics=int(tics[i]), out=idx[i:i + 1])
    return resolve_palettes(idx, [playpal], k, "rgb", None, [palette] * len(poses))


@pytest.mark.parametrize("k", (1, 2))
def test_clis_palette(tmp_path, b2d, capsys, k):
    from rust_doom_b200 import cli
    from rust_doom_b200 import poses as P
    from tests.test_cli import _b2d_binary
    from tests.test_gpu_resolve import _cli_wad
    data, wad = _cli_wad(tmp_path)
    w, h = 160, 100
    arch = b2d.Archive.from_bytes(data)
    scenes = [b2d.Scene(arch, i) for i in (0, 1)]
    poses, levels, tics = cli.level_set_job(b2d, scenes, 3, 40)
    want_ls = _oracle_rgb_palette(data, [int(v) for v in levels], poses, tics, w, h, k, 3)
    look = np.repeat(scenes[0].start_pose, 4)
    look["angle"] = (look["angle"].astype(np.uint64) + (np.arange(4, dtype=np.uint64) << np.uint64(32)) // np.uint64(4)).astype(np.uint32)
    want_look = _oracle_rgb_palette(data, [0] * 4, look, [40] * 4, w, h, k, 3)
    want_fly = _oracle_rgb_palette(data, [0] * 4, P.flythrough_poses(scenes[0], 4, 2), [0] * 4, w, h, k, 3)
    stream, dump = tmp_path / "s.ppm", tmp_path / "d.ppm"
    base = ["-r", "%dx%d" % (w, h), "--palette", "3", "--supersample", str(k), "--stream", str(stream), "--dump", str(dump)]
    # the Python CLI: a level set, then one level's fly-through
    assert cli.main(["--iwad", str(wad), "--levels", "0,1", "--poses", "3", "--tics", "40"] + base) == 0
    assert "palette 3" in capsys.readouterr().out
    assert stream.read_bytes() == b"".join(cli.encode_ppm(f) for f in want_ls)
    for lvl in (0, 1):
        assert (tmp_path / ("d.%d.ppm" % lvl)).read_bytes() == cli.encode_ppm(want_ls[3 * lvl])
    assert cli.main(["--iwad", str(wad), "--poses", "4"] + base) == 0
    assert stream.read_bytes() == b"".join(cli.encode_ppm(f) for f in want_fly)
    assert dump.read_bytes() == cli.encode_ppm(want_fly[0])
    # the compiled CLI: a level set, then one level's look-around at tic 40
    exe = _b2d_binary()
    out = subprocess.run([exe, "-i", str(wad), "--levels", "0,1", "--poses", "3", "--tics", "40"] + base, capture_output=True, text=True)
    assert out.returncode == 0 and "palette 3" in out.stdout, out.stderr
    assert stream.read_bytes() == b"".join(cli.encode_ppm(f) for f in want_ls)
    for lvl in (0, 1):
        assert (tmp_path / ("d.%d.ppm" % lvl)).read_bytes() == cli.encode_ppm(want_ls[3 * lvl])
    out = subprocess.run([exe, "-i", str(wad), "--poses", "4", "--tics", "40"] + base, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert stream.read_bytes() == b"".join(cli.encode_ppm(f) for f in want_look)
    assert dump.read_bytes() == cli.encode_ppm(want_look[0])
    # a palette past the PLAYPAL: a usage error before any device work
    out = subprocess.run([exe, "-i", str(wad), "-r", "%dx%d" % (w, h), "--palette", "14"], capture_output=True, text=True)
    assert out.returncode == 2 and "--palette" in out.stderr
    assert cli.main(["--iwad", str(wad), "-r", "%dx%d" % (w, h), "--palette", "14"]) == 2
