"""-m gpu: the resolve kernel K4 (b2d_resolve_device, C17) bit for bit against its numpy restatement (oracle/resolve.py):
seeded random index frames in every format at every factor, views whose width is not a multiple of 16 as well as 1080p
and 4K, a level set from two WADs with different PLAYPALs, supersampled renders end to end, byte identity with K3 and the
raster's RGBA at factor 1, guard bytes and unaligned pointers, 1000 frames in one call, argument refusals that enqueue
nothing, stream order, and both CLIs with --supersample."""
import ctypes
import subprocess
import time

import numpy as np
import pytest

from oracle import render
from oracle import resolve as R
from tests.conftest import oracle_blob, sample_poses

pytestmark = pytest.mark.gpu

FORMATS = ("rgba", "rgb", "rgb_planar", "gray")
HOLD_MS = 200


def _other_palette(data: bytes) -> bytes:
    """the WAD with every byte of its PLAYPAL lump inverted (255 - v): a level set whose levels come from different WADs"""
    buf = bytearray(data)
    n, diro = np.frombuffer(bytes(buf[4:12]), "<i4")
    for k in range(int(n)):
        pos, size = np.frombuffer(bytes(buf[diro + 16 * k:diro + 16 * k + 8]), "<i4")
        if bytes(buf[diro + 16 * k + 8:diro + 16 * k + 16]).rstrip(b"\0") == b"PLAYPAL":
            buf[pos:pos + size] = bytes(255 - v for v in buf[pos:pos + size])
            return bytes(buf)
    raise AssertionError("no PLAYPAL lump")


@pytest.fixture(scope="module")
def lset(b2d):
    """two levels from WADs with different PLAYPALs: [{data, blob (oracle), scene, playpal}]"""
    from oracle import wad as W
    from rust_doom_b200 import synthwad
    out = []
    for data in (synthwad.build_iwad(1, ("E1M1",)),
                 _other_palette(synthwad.build_iwad(7, ("E1M1",), cfg=synthwad.SynthConfig(gx=3, gy=3, origin=(-384, -384),
                                                                                           light_fx=False)))):
        pal = W.TextureDirectory(W.Archive(data)).palettes[0]
        out.append(dict(data=data, blob=oracle_blob(data), scene=b2d.Scene(b2d.Archive.from_bytes(data), 0), playpal=pal))
    assert (np.frombuffer(out[0]["playpal"], np.uint8) != np.frombuffer(out[1]["playpal"], np.uint8)).all()
    return out


def _pals(lset):
    return [L["playpal"] for L in lset]


def _renderer(b2d, lset, w, h, max_batch=4):
    return b2d.Renderer.from_levels([L["scene"] for L in lset], b2d.make_view(w, h), max_batch=max_batch)


def _random_index(n, h, w, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (n, h, w), dtype=torch.uint8, device="cuda", generator=g)


def _got(t):
    a = t.cpu().numpy()
    return a.view(np.uint32) if a.dtype == np.int32 else a


# views and the factors each is tested at: 168 and 120 columns are not multiples of 16 (the byte path), 1920 x 1080 and
# 3840 x 2160 take every factor but 7, which 1792 x 1008 takes (1792 = 16 * 112: the vector path at factor 7)
VIEWS = [((168, 120), (1, 2, 3, 4, 6, 8)), ((21 * 5, 13 * 5), (1, 5)), ((21 * 7, 13 * 7), (1, 7)),
         ((1920, 1080), (1, 2, 3, 4, 5, 6, 8)), ((1792, 1008), (7,)), ((3840, 2160), (1, 2, 3, 4, 5, 6, 8))]


@pytest.mark.parametrize("view,factors", VIEWS, ids=["%dx%d" % v for v, _ in VIEWS])
def test_random_frames_every_format_and_factor(b2d, lset, view, factors):
    w, h = view
    n = 2 if w * h > 4_000_000 else 3
    r = _renderer(b2d, lset, w, h, max_batch=1)
    idx = _random_index(n, h, w, w + h)
    host = idx.cpu().numpy()
    lv = [1, 0, 1][:n]
    for k in factors:
        for fmt in FORMATS:
            for levels in ((lv, None) if n == 3 else (lv,)):
                got = _got(r.resolve(idx, k, fmt, levels))
                want = R.resolve(host, _pals(lset), k, fmt, levels)
                assert got.shape == want.shape and np.array_equal(got, want), (view, k, fmt, levels)
        assert r.resolve_frame_bytes(k, b2d.RESOLVE_RGB8) == (w // k) * (h // k) * 3


def test_random_per_frame_levels(b2d, lset):
    """seeded random levels over 24 frames; NULL levels is level 0 on every frame"""
    r = _renderer(b2d, lset, 320, 200)
    idx = _random_index(24, 200, 320, 11)
    host = idx.cpu().numpy()
    lv = np.random.default_rng(12).integers(0, 2, 24)
    for k, fmt in ((2, "rgb_planar"), (4, "gray"), (5, "rgba"), (8, "rgb")):
        assert np.array_equal(_got(r.resolve(idx, k, fmt, lv)), R.resolve(host, _pals(lset), k, fmt, lv)), (k, fmt)
        assert np.array_equal(_got(r.resolve(idx, k, fmt)), _got(r.resolve(idx, k, fmt, np.zeros(24, np.int64)))), (k, fmt)


def test_factor_one_rgba_is_k3_and_the_raster_rgba(b2d, lset):
    import torch
    w, h, n = 320, 200, 8
    r = _renderer(b2d, lset, w, h, max_batch=n)
    poses = np.concatenate([sample_poses(b2d, lset[k]["scene"], n // 2, 30 + k) for k in range(2)])
    lv = np.repeat([0, 1], n // 2)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    idx = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
    rgba = torch.empty((n, h, w), dtype=torch.int32, device="cuda")
    r.render_device_levels(dp.data_ptr(), lv, n, idx.data_ptr(), rgba.data_ptr())
    k3 = torch.empty_like(rgba)
    r.palette_lut_levels_device(idx.data_ptr(), lv, n, k3.data_ptr())
    k4 = r.resolve(idx, 1, "rgba", lv)
    torch.cuda.synchronize()
    assert r.status() == 0
    assert torch.equal(k4, rgba) and torch.equal(k4, k3)
    assert np.array_equal(_got(k4), R.resolve(idx.cpu().numpy(), _pals(lset), 1, "rgba", lv))


@pytest.mark.parametrize("k", [2, 3])
def test_supersampled_levels_states_end_to_end(b2d, lset, k):
    """render_device_levels_states at k x a 160 x 100 view, then the resolve: equal to the numpy resolve of the oracle's
    frames at the same poses, levels and tics"""
    import torch
    w, h, n = 160 * k, 100 * k, 10
    r = _renderer(b2d, lset, w, h, max_batch=4)
    rng = np.random.default_rng(40 + k)
    lv = rng.integers(0, 2, n)
    pools = [sample_poses(b2d, lset[q]["scene"], n, 50 + q) for q in range(2)]
    poses = np.array([pools[lv[i]][i] for i in range(n)], dtype=pools[0].dtype)
    tics = rng.integers(0, 5000, n)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    idx = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
    r.render_device_levels_states(dp.data_ptr(), lv, tics, n, idx.data_ptr())
    outs = {fmt: _got(r.resolve(idx, k, fmt, lv)) for fmt in FORMATS}
    assert r.status() == 0
    view = render.make_view(w, h)
    want = np.empty((n, h, w), np.uint8)
    for i in range(n):
        render.render(lset[lv[i]]["blob"], view, poses[i:i + 1], tics=int(tics[i]), out=want[i:i + 1])
    assert np.array_equal(idx.cpu().numpy(), want)
    for fmt in FORMATS:
        assert np.array_equal(outs[fmt], R.resolve(want, _pals(lset), k, fmt, lv)), fmt


def test_guard_bytes_and_unaligned_pointers(b2d, lset):
    """4 KB of poisoned guard bytes on either side of the output stay untouched; index and output pointers offset by 0..15
    bytes give exact results (vector and byte paths, every format)"""
    import torch
    w, h, n, guard = 96, 48, 3, 4096
    r = _renderer(b2d, lset, w, h)
    src = _random_index(n, h, w, 77)
    host = src.cpu().numpy()
    lv = [1, 0, 1]
    ibuf = torch.empty(n * w * h + 16, dtype=torch.uint8, device="cuda")
    for off_i in range(16):
        ibuf[off_i:off_i + n * w * h].copy_(src.reshape(-1))
        off_o = (7 * off_i + 3) % 16
        for k in (1, 2, 3, 8):
            for fmt in FORMATS:
                code = b2d.RESOLVE_FORMATS[fmt]
                nbytes = n * r.resolve_frame_bytes(k, code)
                obuf = torch.full((2 * guard + nbytes + 16,), 0xA5, dtype=torch.uint8, device="cuda")
                r.resolve_device(ibuf.data_ptr() + off_i, n, k, code, obuf.data_ptr() + guard + off_o, lv)
                got = obuf.cpu().numpy()
                lo, hi = guard + off_o, guard + off_o + nbytes
                assert (got[:lo] == 0xA5).all() and (got[hi:] == 0xA5).all(), (off_i, off_o, k, fmt)
                want = R.resolve(host, _pals(lset), k, fmt, lv)
                assert np.array_equal(got[lo:hi], want.view(np.uint8).reshape(-1)), (off_i, off_o, k, fmt)


def test_thousand_1080p_frames_in_one_call(b2d, lset):
    """1000 frames of 1920 x 1080 -> 960 x 540 planar RGB in one call; sampled frames against numpy, guards intact"""
    import torch
    n, w, h, guard = 1000, 1920, 1080, 4096
    r = _renderer(b2d, lset, w, h, max_batch=1)
    idx = _random_index(n, h, w, 1000)
    lv = np.random.default_rng(1001).integers(0, 2, n)
    code = b2d.RESOLVE_RGB8_PLANAR
    fb = r.resolve_frame_bytes(2, code)
    assert fb == 3 * 960 * 540
    obuf = torch.full((2 * guard + n * fb,), 0x5A, dtype=torch.uint8, device="cuda")
    l0 = r.launch_count
    r.resolve_device(idx.data_ptr(), n, 2, code, obuf.data_ptr() + guard, lv)
    torch.cuda.synchronize()
    assert r.launch_count == l0 + 1
    assert bool((obuf[:guard] == 0x5A).all()) and bool((obuf[guard + n * fb:] == 0x5A).all())
    out = obuf[guard:guard + n * fb].reshape(n, 3, 540, 960)
    for f in (0, 1, 499, 500, 998, 999):
        want = R.resolve(idx[f:f + 1].cpu().numpy(), _pals(lset), 2, "rgb_planar", lv[f:f + 1])
        assert np.array_equal(out[f:f + 1].cpu().numpy(), want), f


def test_invalid_arguments_enqueue_nothing(b2d, lset):
    import torch
    from rust_doom_b200 import _lib
    L = _lib.load()
    r = _renderer(b2d, lset, 320, 200)
    idx = torch.zeros((2, 200, 320), dtype=torch.uint8, device="cuda")
    out = torch.zeros(2 * 320 * 200 * 4, dtype=torch.uint8, device="cuda")
    good = (np.zeros(2, np.uint32), np.ones(2, np.uint32))
    bad_levels = np.array([0, 2], np.uint32)
    l0 = r.launch_count
    calls = [(None, good[0].ctypes.data, 2, 2, 0, out.data_ptr()), (idx.data_ptr(), good[0].ctypes.data, 2, 2, 0, None)]
    calls += [(idx.data_ptr(), None, 2, k, 0, out.data_ptr()) for k in (0, -1, 9, 3, 7, 6)]      # 320 x 200: 3, 6, 7 do not divide
    calls += [(idx.data_ptr(), None, 2, 2, f, out.data_ptr()) for f in (-1, 4, 99)]
    calls += [(idx.data_ptr(), bad_levels.ctypes.data, 2, 2, 0, out.data_ptr())]
    calls += [(idx.data_ptr(), bad_levels.ctypes.data, 0, 9, 0, out.data_ptr())]                  # checked before n = 0
    for ip, lp, n, k, f, op in calls:
        assert L.b2d_resolve_device(r._h, ip, lp, n, k, f, op, None) == b2d.ERR_INVALID_ARG, (ip, n, k, f)
    size = ctypes.c_size_t(12345)
    for k, f in ((0, 0), (3, 0), (9, 1), (2, 4), (2, -1)):
        assert L.b2d_resolve_frame_bytes(r._h, k, f, ctypes.byref(size)) == b2d.ERR_INVALID_ARG
    assert size.value == 12345
    assert L.b2d_resolve_frame_bytes(r._h, 2, 0, None) == b2d.ERR_INVALID_ARG
    with pytest.raises(b2d.B2dError) as e:
        r.resolve(idx, 2, "rgb", [0, 2])
    assert e.value.code == b2d.ERR_INVALID_ARG and "level" in e.value.message
    assert L.b2d_resolve_device(r._h, idx.data_ptr(), None, 0, 2, 0, out.data_ptr(), None) == 0           # n = 0: nothing
    assert L.b2d_resolve_device(r._h, idx.data_ptr(), bad_levels.ctypes.data, 1, 2, 0, out.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert r.launch_count == l0 + 1                      # only the last call, whose one frame is on level 0
    assert r.status() == 0


# ---- stream order: a bounded sleep kernel holds a stream (helpers as in tests/test_gpu_stream_order.py) -----------------
class Clock:
    """Holds: a sleep kernel of `ms` milliseconds on a stream, and an event recorded after it."""

    def __init__(self, cycles_per_ms):
        self.cycles_per_ms = cycles_per_ms

    def sleep(self, stream, ms):
        import torch
        assert 0 < ms <= 500, "holds stay bounded"
        with torch.cuda.stream(stream):
            torch.cuda._sleep(int(self.cycles_per_ms * ms))

    def hold(self, stream, ms=HOLD_MS):
        self.sleep(stream, ms)
        return mark(stream)


@pytest.fixture(scope="module")
def clock(b2d):
    """cycles per millisecond of the sleep kernel, from CUDA events around one sleep"""
    import torch
    s = torch.cuda.Stream()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    cycles = 1 << 24
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 16)                  # loads the kernel
        a.record(s)
        torch.cuda._sleep(cycles)
        b.record(s)
    b.synchronize()
    return Clock(cycles / a.elapsed_time(b))


def mark(stream):
    import torch
    ev = torch.cuda.Event()
    ev.record(stream)
    return ev


def pending(hold, what):
    assert not hold.query(), "%s: the call blocked until the hold ended" % what


def must_wait(down, hold, what):
    """`down` must not complete before `hold`."""
    assert not hold.query(), "%s: the hold ended before the probe started" % what
    while True:
        d = down.query()
        if hold.query():
            break
        assert not d, "%s: finished while the hold it must wait for was pending" % what
        time.sleep(0.0005)
    down.synchronize()


def test_resolve_is_enqueued_on_its_stream(b2d, lset, clock):
    """the call returns while its stream is held, and its output is not written before the hold ends"""
    import torch
    r = _renderer(b2d, lset, 320, 200)
    idx = _random_index(6, 200, 320, 90)
    out = torch.full((6, 3, 100, 160), 0xA5, dtype=torch.uint8, device="cuda")
    lv = [0, 1, 0, 1, 1, 0]
    r.resolve_device(idx.data_ptr(), 6, 2, b2d.RESOLVE_RGB8_PLANAR, out.data_ptr(), lv)      # staging grown outside the hold
    out.fill_(0xA5)
    s, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    hold = clock.hold(s)
    r.resolve_device(idx.data_ptr(), 6, 2, b2d.RESOLVE_RGB8_PLANAR, out.data_ptr(), lv, s.cuda_stream)
    pending(hold, "resolve")
    with torch.cuda.stream(s2):
        early = out.cpu().numpy()
    pending(hold, "the read-back on another stream")
    assert (early == 0xA5).all(), "the resolve wrote its output while its stream was held"
    must_wait(mark(s), hold, "resolve behind the hold")
    assert np.array_equal(out.cpu().numpy(), R.resolve(idx.cpu().numpy(), _pals(lset), 2, "rgb_planar", lv))


def test_second_call_waits_for_the_first_calls_staging_copy(b2d, lset, clock):
    """the levels staging is rewritten only after the copy of the previous call with levels has read it; a call without
    levels stages nothing and does not wait"""
    import torch
    r = _renderer(b2d, lset, 320, 200)
    idx = _random_index(6, 200, 320, 91)
    a, b = (torch.empty((6, 100, 160), dtype=torch.uint8, device="cuda") for _ in range(2))
    lva, lvb = [0, 1, 1, 0, 0, 1], [1, 1, 0, 0, 1, 0]
    r.resolve_device(idx.data_ptr(), 6, 2, b2d.RESOLVE_GRAY8, a.data_ptr(), lva)             # staging grown outside the hold
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    hold = clock.hold(s)
    r.resolve_device(idx.data_ptr(), 6, 2, b2d.RESOLVE_GRAY8, a.data_ptr(), lva, s.cuda_stream)
    pending(hold, "first call")
    r.resolve_device(idx.data_ptr(), 6, 4, b2d.RESOLVE_GRAY8, b.data_ptr(), None, s.cuda_stream)
    pending(hold, "a call without levels")
    r.resolve_device(idx.data_ptr(), 6, 2, b2d.RESOLVE_GRAY8, b.data_ptr(), lvb, s.cuda_stream)
    assert hold.query(), "the second call rewrote the staging the first call's held copy reads"
    torch.cuda.synchronize()
    host = idx.cpu().numpy()
    assert np.array_equal(a.cpu().numpy(), R.resolve(host, _pals(lset), 2, "gray", lva))
    assert np.array_equal(b.cpu().numpy(), R.resolve(host, _pals(lset), 2, "gray", lvb))


# ---- CLIs ------------------------------------------------------------------------------------------------------------
def _cli_wad(tmp_path):
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1", "E1M2"))
    wad = tmp_path / "syn.wad"
    wad.write_bytes(data)
    return data, wad


def _oracle_rgb(data, level_of, poses, tics, w, h, k):
    """the numpy resolve to w x h RGB of the oracle's (k w) x (k h) frames; level_of[i], tics[i] per pose"""
    from oracle import wad as W
    pal = W.TextureDirectory(W.Archive(data)).palettes[0]
    blobs = {lv: oracle_blob(data, lv) for lv in set(level_of)}
    view = render.make_view(k * w, k * h)
    idx = np.empty((len(poses), k * h, k * w), np.uint8)
    for i in range(len(poses)):
        render.render(blobs[level_of[i]], view, poses[i:i + 1], tics=int(tics[i]), out=idx[i:i + 1])
    return R.resolve(idx, [pal], k, "rgb")


def test_python_cli_supersample(tmp_path, b2d, capsys):
    from rust_doom_b200 import cli
    from rust_doom_b200 import poses as P
    data, wad = _cli_wad(tmp_path)
    w, h, k = 160, 100, 2
    stream, dump = tmp_path / "s.ppm", tmp_path / "d.ppm"
    assert cli.main(["--iwad", str(wad), "-r", "%dx%d" % (w, h), "--levels", "0,1", "--poses", "3", "--tics", "40",
                     "--supersample", str(k), "--dump", str(dump), "--stream", str(stream)]) == 0
    assert "supersampled 2x" in capsys.readouterr().out
    arch = b2d.Archive.from_bytes(data)
    scenes = [b2d.Scene(arch, i) for i in (0, 1)]
    poses, levels, tics = cli.level_set_job(b2d, scenes, 3, 40)
    want = _oracle_rgb(data, [int(v) for v in levels], poses, tics, w, h, k)
    assert stream.read_bytes() == b"".join(cli.encode_ppm(f) for f in want)
    for lvl in (0, 1):
        assert (tmp_path / ("d.%d.ppm" % lvl)).read_bytes() == cli.encode_ppm(want[3 * lvl])
    # one level, a fly-through
    assert cli.main(["--iwad", str(wad), "-r", "%dx%d" % (w, h), "--poses", "4", "--supersample", str(k),
                     "--stream", str(stream), "--dump", str(dump)]) == 0
    poses = P.flythrough_poses(scenes[0], 4, 2)
    want = _oracle_rgb(data, [0] * 4, poses, [0] * 4, w, h, k)
    assert stream.read_bytes() == b"".join(cli.encode_ppm(f) for f in want)
    assert dump.read_bytes() == cli.encode_ppm(want[0])


def test_compiled_cli_supersample(tmp_path, b2d):
    from rust_doom_b200 import cli
    from tests.test_cli import _b2d_binary
    data, wad = _cli_wad(tmp_path)
    w, h, k = 160, 100, 2
    exe = _b2d_binary()
    stream, dump = tmp_path / "s.ppm", tmp_path / "d.ppm"
    out = subprocess.run([exe, "-i", str(wad), "-r", "%dx%d" % (w, h), "--levels", "0,1", "--poses", "3", "--tics", "40",
                          "--supersample", str(k), "--dump", str(dump), "--stream", str(stream)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    arch = b2d.Archive.from_bytes(data)
    scenes = [b2d.Scene(arch, i) for i in (0, 1)]
    poses, levels, tics = cli.level_set_job(b2d, scenes, 3, 40)
    want = _oracle_rgb(data, [int(v) for v in levels], poses, tics, w, h, k)
    assert stream.read_bytes() == b"".join(cli.encode_ppm(f) for f in want)
    for lvl in (0, 1):
        assert (tmp_path / ("d.%d.ppm" % lvl)).read_bytes() == cli.encode_ppm(want[3 * lvl])
    # one level: the look-around from the start at tic 40 (the renderer's own time)
    out = subprocess.run([exe, "-i", str(wad), "-r", "%dx%d" % (w, h), "--poses", "4", "--tics", "40", "--supersample", str(k),
                          "--stream", str(stream), "--dump", str(dump)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    poses = np.repeat(scenes[0].start_pose, 4)
    poses["angle"] = (poses["angle"].astype(np.uint64) + (np.arange(4, dtype=np.uint64) << np.uint64(32)) // np.uint64(4)).astype(np.uint32)
    want = _oracle_rgb(data, [0] * 4, poses, [40] * 4, w, h, k)
    assert stream.read_bytes() == b"".join(cli.encode_ppm(f) for f in want)
    assert dump.read_bytes() == cli.encode_ppm(want[0])
