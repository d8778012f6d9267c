"""-m gpu: the automap kernel (b2d_automap_device, DESIGN.md C19) bit for bit against oracle/automap.py on the c2 level, the
content-rich level and a three-level set with per-frame levels, at 320x200 and 1920x1080, with random poses and every
flag combination; map and pose coordinates at +-32767 units; automap frames through b2d_resolve_palettes_device against
oracle/resolve.py; the call's stream order (it overlaps a held raster on another stream, and its level staging waits as
the resolve's does); refusals that enqueue nothing; and both CLIs' --automap files."""
import subprocess

import numpy as np
import pytest

from oracle import automap as A
from oracle import render
from oracle import resolve as R
from oracle import wad as W
from tests.test_automap import _find_lump, random_poses
from tests.test_gpu_resolve import clock, mark, must_wait, pending  # noqa: F401
from tests.test_palettes import resolve_palettes

pytestmark = pytest.mark.gpu

SCALES = (A.SCALE_MIN, 13107, A.SCALE_MAX)


@pytest.fixture(scope="module")
def lset(b2d):
    """[(data, level, scene)]: the c2 level, the c2 WAD's second map and the content-rich level"""
    from rust_doom_b200 import synthwad
    from tests.test_lights import rich_wad
    c2, rich = synthwad.build_iwad(1, ("E1M1", "E1M2")), rich_wad()
    return [(d, lv, b2d.Scene(b2d.Archive.from_bytes(d), lv)) for d, lv in ((c2, 0), (c2, 1), (rich, 0))]


def _oracle_items(entry):
    data, lv, scene = entry
    return A.lines(W.Level(W.Archive(data), lv)), A.things(scene.blob)


def _device_poses(poses):
    import torch
    return torch.from_numpy(np.ascontiguousarray(poses).view(np.uint8).reshape(-1)).cuda()


def _automap(r, poses, scale, flags, levels=None, stream=0):
    import torch
    dp = _device_poses(poses)
    out = torch.full((len(poses), r.height, r.width), 0xEE, dtype=torch.uint8, device="cuda")
    r.automap_device(dp.data_ptr(), len(poses), out.data_ptr(), scale, flags, levels, stream)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _oracle(items_of, poses, levels, w, h, scale, flags):
    out = np.empty((len(poses), h, w), np.uint8)
    for i in range(len(poses)):
        table, things = items_of[levels[i] if levels is not None else 0]
        out[i:i + 1] = A.automap(table, things, w, h, poses[i:i + 1], scale, flags)
    return out


@pytest.mark.parametrize("w,h", [(320, 200), (1920, 1080)])
@pytest.mark.parametrize("which", [0, 2], ids=["c2", "rich"])
def test_one_level_every_flag(b2d, lset, w, h, which):
    r = b2d.Renderer(lset[which][2], b2d.make_view(w, h), max_batch=4)
    items = [_oracle_items(lset[which])]
    n = 3 if w == 320 else 1
    for flags in range(8):
        scale = SCALES[flags % 3] if w == 320 else 13107
        poses = random_poses(items[0][0], n, 10 * flags + which)
        got = _automap(r, poses, scale, flags)
        want = _oracle(items, poses, None, w, h, scale, flags)
        assert np.array_equal(got, want), (flags, scale, np.argwhere(got != want)[:5])
        assert (want != 0).any()


@pytest.mark.parametrize("w,h", [(320, 200), (1920, 1080)])
def test_level_set_per_frame_levels(b2d, lset, w, h):
    r = b2d.Renderer.from_levels([e[2] for e in lset], b2d.make_view(w, h), max_batch=4)
    items = [_oracle_items(e) for e in lset]
    rng = np.random.default_rng(7)
    n = 6 if w == 320 else 3
    for flags in range(8):
        levels = [int(v) for v in rng.integers(0, 3, n)]
        poses = np.concatenate([random_poses(items[lv][0], 1, 100 * flags + i) for i, lv in enumerate(levels)])
        got = _automap(r, poses, 13107, flags, levels)
        assert np.array_equal(got, _oracle(items, poses, levels, w, h, 13107, flags)), flags
    # no level array: every frame on level 0
    got = _automap(r, poses, 13107, 7)
    assert np.array_equal(got, _oracle(items, poses, [0] * n, w, h, 13107, 7))


def _extreme_wad(data: bytes) -> bytes:
    """the c2 level with its first vertices moved to the corners and edges of the map's range"""
    buf = bytearray(data)
    pos, size = _find_lump(data, b"VERTEXES")
    v = np.frombuffer(buf, W.VERTEX, count=size // 4, offset=pos)
    corners = [(32767, 32767), (-32768, -32768), (32767, -32768), (-32768, 32767), (0, 32767), (-32768, 0)]
    for k, (x, y) in enumerate(corners):
        v[k] = (x, y)
    return bytes(buf)


def test_extreme_coordinates(b2d, lset):
    data = _extreme_wad(lset[0][0])
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    items = [(A.lines(W.Level(W.Archive(data), 0)), A.things(sc.blob))]
    assert any(abs(t[0]) >= 32767 for t in items[0][0])
    poses = np.zeros(6, render.POSE)
    poses["x"] = [2 ** 31 - 1, -2 ** 31, 2 ** 31 - 1, -2 ** 31, 0, 2 ** 31 - 1]
    poses["y"] = [2 ** 31 - 1, -2 ** 31, -2 ** 31, 2 ** 31 - 1, 0, 0]
    poses["angle"] = [0x20000000, 0xA0000000, 0x60000000, 0xE0000000, 0x12345678, 0xFFFFFFFF]
    for w, h in ((320, 200), (333, 187)):
        r = b2d.Renderer(sc, b2d.make_view(w, h), max_batch=4)
        for flags in range(8):
            for scale in SCALES:
                got = _automap(r, poses, scale, flags)
                assert np.array_equal(got, _oracle(items, poses, None, w, h, scale, flags)), (w, h, flags, scale)


def test_resolved_automaps_match_the_oracle(b2d, lset):
    import torch
    r = b2d.Renderer.from_levels([e[2] for e in lset], b2d.make_view(320, 200), max_batch=4)
    items = [_oracle_items(e) for e in lset]
    levels = [0, 2, 1, 2]
    poses = np.concatenate([random_poses(items[lv][0], 1, 40 + i) for i, lv in enumerate(levels)])
    am = r.automap(poses, levels, 0.2, "rotate,things")
    want_idx = _oracle(items, poses, levels, 320, 200, 13107, A.ROTATE | A.THINGS)
    assert np.array_equal(am.cpu().numpy(), want_idx)
    pals = [b"".join(W.TextureDirectory(W.Archive(e[0])).palettes) for e in lset]
    palettes = [0, 3, 13, 9]
    for k, fmt in ((1, "rgb"), (2, "gray"), (2, "rgb_planar")):
        got = r.resolve(am, k, fmt, levels, palettes).cpu().numpy()
        assert np.array_equal(got, resolve_palettes(want_idx, pals, k, fmt, levels, palettes)), (k, fmt)
    got = r.resolve(am, 2, "rgb", levels).cpu().numpy()
    assert np.array_equal(got, R.resolve(want_idx, [p[:768] for p in pals], 2, "rgb", levels))
    torch.cuda.synchronize()


def test_unaligned_and_odd_outputs(b2d, lset):
    """a view whose width is not a multiple of 16 and an output 3 bytes past an aligned address: the byte path"""
    import torch
    items = [_oracle_items(lset[2])]
    poses = random_poses(items[0][0], 3, 77)
    for w, h in ((333, 187), (320, 200), (1, 2)):
        r = b2d.Renderer(lset[2][2], b2d.make_view(w, h), max_batch=4)
        dp = _device_poses(poses)
        buf = torch.full((3 * w * h + 16,), 0xEE, dtype=torch.uint8, device="cuda")
        r.automap_device(dp.data_ptr(), 3, buf.data_ptr() + 3, 13107, 7)
        host = buf.cpu().numpy()
        assert (host[:3] == 0xEE).all() and (host[3 + 3 * w * h:] == 0xEE).all(), (w, h)
        assert np.array_equal(host[3:3 + 3 * w * h].reshape(3, h, w), _oracle(items, poses, None, w, h, 13107, 7)), (w, h)


def test_invalid_arguments_enqueue_nothing(b2d, lset):
    import torch
    from rust_doom_b200 import _lib
    L = _lib.load()
    r = b2d.Renderer.from_levels([e[2] for e in lset], b2d.make_view(320, 200), max_batch=4)
    dp = _device_poses(random_poses(_oracle_items(lset[0])[0], 2, 1))
    out = torch.full((2, 200, 320), 0xEE, dtype=torch.uint8, device="cuda")
    good, bad = np.array([0, 2], np.uint32), np.array([0, 3], np.uint32)
    l0 = r.launch_count
    calls = [(None, dp.data_ptr(), None, 2, 13107, 0, out.data_ptr()), (r._h, None, None, 2, 13107, 0, out.data_ptr()),
             (r._h, dp.data_ptr(), None, 2, 13107, 0, None)]
    calls += [(r._h, dp.data_ptr(), None, 2, 13107, f, out.data_ptr()) for f in (8, 16, -1)]
    calls += [(r._h, dp.data_ptr(), None, 2, s, 0, out.data_ptr()) for s in (0, 255, (64 << 16) + 1, -13107)]
    calls += [(r._h, dp.data_ptr(), bad.ctypes.data, 2, 13107, 0, out.data_ptr())]
    calls += [(r._h, dp.data_ptr(), None, 0, 0, 0, out.data_ptr())]                          # checked before n = 0
    # more CTAs than one grid holds (21 tiles per 320 x 200 frame): refused before the first call uploads anything
    calls += [(r._h, dp.data_ptr(), None, 0x7FFFFFFF // 21 + 1, 13107, 0, out.data_ptr())]
    for h_, p, lv, n, s, f, o in calls:
        assert L.b2d_automap_device(h_, p, lv, n, s, f, o, None) == b2d.ERR_INVALID_ARG, (n, s, f)
    with pytest.raises(ValueError):
        r.automap(np.zeros(1, b2d.POSE_DTYPE), flags="rotate,iddqd")
    assert L.b2d_automap_device(r._h, dp.data_ptr(), bad.ctypes.data, 0, 13107, 0, out.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert r.launch_count == l0 and (out.cpu().numpy() == 0xEE).all()
    assert L.b2d_automap_device(r._h, dp.data_ptr(), good.ctypes.data, 2, 13107, 0, out.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert r.launch_count == l0 + 1 and r.status() == 0


def test_first_call_on_a_held_stream_orders_later_calls(b2d, lset, clock):
    """the first call uploads every level's tables on its own stream: it returns while that stream is held, and a call on
    another stream right after it waits for the upload, whose frames are then the oracle's"""
    import torch
    items = [_oracle_items(e) for e in lset]
    warm = b2d.Renderer(lset[1][2], b2d.make_view(320, 200), max_batch=4)
    levels = [2, 0, 1, 2]
    poses = np.concatenate([random_poses(items[lv][0], 1, 80 + i) for i, lv in enumerate(levels)])
    dp = _device_poses(poses)
    a, b = (torch.full((4, 200, 320), 0xEE, dtype=torch.uint8, device="cuda") for _ in range(2))
    warm.automap_device(dp.data_ptr(), 4, a.data_ptr(), 13107, 7)           # the kernel's module loaded outside the hold
    r = b2d.Renderer.from_levels([e[2] for e in lset], b2d.make_view(320, 200), max_batch=4)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    hold = clock.hold(s1)
    r.automap_device(dp.data_ptr(), 4, a.data_ptr(), 13107, 7, levels, s1.cuda_stream)
    pending(hold, "the first call")
    r.automap_device(dp.data_ptr(), 4, b.data_ptr(), 13107, 5, None, s2.cuda_stream)
    pending(hold, "a call on another stream")
    must_wait(mark(s2), hold, "the second call behind the first call's held upload")
    torch.cuda.synchronize()
    assert np.array_equal(a.cpu().numpy(), _oracle(items, poses, levels, 320, 200, 13107, 7))
    assert np.array_equal(b.cpu().numpy(), _oracle(items, poses, [0] * 4, 320, 200, 13107, 5))


def test_overlaps_a_held_raster_on_another_stream(b2d, lset, clock):
    """the automap has no edge with walks or rasters: it finishes while a raster is held back on another stream"""
    import torch
    r = b2d.Renderer(lset[0][2], b2d.make_view(320, 200), max_batch=4)
    poses = random_poses(_oracle_items(lset[0])[0], 4, 3)
    dp = _device_poses(poses)
    idx = torch.empty((4, 200, 320), dtype=torch.uint8, device="cuda")
    am = torch.empty((4, 200, 320), dtype=torch.uint8, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    # first-use work outside the hold: the automap tables, the worklist slots, and each kernel's module, which CUDA loads
    # lazily at its first launch in the process (a load made behind a held stream holds launches on other streams too)
    for st in (s1, s2, s1, s2):
        r.render_device(dp.data_ptr(), 4, idx.data_ptr(), 0, st.cuda_stream)
        r.automap_device(dp.data_ptr(), 4, am.data_ptr(), 13107, 7, None, st.cuda_stream)
    torch.cuda.synchronize()
    hold = clock.hold(s1)
    r.render_device(dp.data_ptr(), 4, idx.data_ptr(), 0, s1.cuda_stream)
    pending(hold, "the held render")
    r.automap_device(dp.data_ptr(), 4, am.data_ptr(), 13107, 7, None, s2.cuda_stream)
    done = mark(s2)
    done.synchronize()
    pending(hold, "the automap on another stream")
    must_wait(mark(s1), hold, "the raster behind the hold")
    items = [_oracle_items(lset[0])]
    assert np.array_equal(am.cpu().numpy(), _oracle(items, poses, None, 320, 200, 13107, 7))


def test_second_call_waits_for_the_first_calls_staging_copy(b2d, lset, clock):
    """the level staging is rewritten only after the copy of the previous call with levels has read it; a call without
    levels stages nothing and does not wait"""
    import torch
    r = b2d.Renderer.from_levels([e[2] for e in lset], b2d.make_view(320, 200), max_batch=4)
    items = [_oracle_items(e) for e in lset]
    lva, lvb = [0, 1, 2, 2, 1, 0], [2, 2, 0, 1, 0, 1]
    poses = np.concatenate([random_poses(items[lv][0], 1, 60 + i) for i, lv in enumerate(lva)])
    dp = _device_poses(poses)
    a, b = (torch.empty((6, 200, 320), dtype=torch.uint8, device="cuda") for _ in range(2))
    r.automap_device(dp.data_ptr(), 6, a.data_ptr(), 13107, 0, lva)          # staging grown outside the hold
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    hold = clock.hold(s)
    r.automap_device(dp.data_ptr(), 6, a.data_ptr(), 13107, 0, lva, s.cuda_stream)
    pending(hold, "first call")
    r.automap_device(dp.data_ptr(), 6, b.data_ptr(), 13107, 0, None, s.cuda_stream)
    pending(hold, "a call without levels")
    r.automap_device(dp.data_ptr(), 6, b.data_ptr(), 13107, 0, lvb, s.cuda_stream)
    assert hold.query(), "the second call rewrote the staging the first call's held copy reads"
    torch.cuda.synchronize()
    assert np.array_equal(a.cpu().numpy(), _oracle(items, poses, lva, 320, 200, 13107, 0))
    assert np.array_equal(b.cpu().numpy(), _oracle(items, poses, lvb, 320, 200, 13107, 0))


# ---- CLIs ------------------------------------------------------------------------------------------------------------
def _cli_expected(b2d, data, set_, poses, w, h, scale, flags):
    """the oracle's automap of each pose on its level, through palette 0 of the WAD"""
    pal = W.TextureDirectory(W.Archive(data)).palettes[0]
    out = []
    for lv, p in zip(set_, poses):
        sc = b2d.Scene(b2d.Archive.from_bytes(data), lv)
        idx = A.automap(A.lines(W.Level(W.Archive(data), lv)), A.things(sc.blob), w, h, p.reshape(1), scale, flags)
        out.append(R.resolve(idx, [pal], 1, "rgb")[0])
    return out


def test_python_cli_writes_automaps(tmp_path, b2d):
    from rust_doom_b200 import cli
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1", "E1M2"))
    wad = tmp_path / "syn.wad"
    wad.write_bytes(data)
    dump = tmp_path / "d.ppm"
    assert cli.main(["--iwad", str(wad), "-r", "160x100", "--levels", "0,1", "--poses", "2", "--dump", str(dump),
                     "--automap", "0.25", "--automap-flags", "rotate,things"]) == 0
    arch = b2d.Archive.from_bytes(data)
    poses, _, _ = cli.level_set_job(b2d, [b2d.Scene(arch, i) for i in (0, 1)], 2, 0)
    want = _cli_expected(b2d, data, [0, 1], poses[[0, 2]], 160, 100, 16384, A.ROTATE | A.THINGS)
    for lvl in (0, 1):
        assert (tmp_path / ("d.automap.%d.ppm" % lvl)).read_bytes() == cli.encode_ppm(want[lvl])
    assert cli.main(["--iwad", str(wad), "-r", "160x100", "--dump", str(dump), "--automap", "0.2"]) == 0
    sc = b2d.Scene(arch, 0)
    want = _cli_expected(b2d, data, [0], sc.start_pose, 160, 100, 13107, 0)
    assert (tmp_path / "d.automap.ppm").read_bytes() == cli.encode_ppm(want[0])
    assert cli.main(["--iwad", str(wad), "--dump", str(dump), "--automap", "0.2", "--automap-flags", "iddt"]) == 2


def test_compiled_cli_writes_automaps(tmp_path, b2d):
    from rust_doom_b200 import cli
    from rust_doom_b200 import synthwad
    from tests.test_cli import _b2d_binary
    data = synthwad.build_iwad(1, ("E1M1", "E1M2"))
    wad = tmp_path / "syn.wad"
    wad.write_bytes(data)
    exe = _b2d_binary()
    dump = tmp_path / "d.ppm"
    out = subprocess.run([exe, "-i", str(wad), "-r", "160x100", "--levels", "0,1", "--poses", "2", "--dump", str(dump),
                          "--automap", "0.25", "--automap-flags", "all,things"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    arch = b2d.Archive.from_bytes(data)
    scenes = [b2d.Scene(arch, i) for i in (0, 1)]
    first = [sc.start_pose[0].copy() for sc in scenes]      # the look-around's pose 0 is the start
    want = _cli_expected(b2d, data, [0, 1], first, 160, 100, 16384, A.ALL_LINES | A.THINGS)
    for lvl in (0, 1):
        assert (tmp_path / ("d.automap.%d.ppm" % lvl)).read_bytes() == cli.encode_ppm(want[lvl])
    out = subprocess.run([exe, "-i", str(wad), "-r", "160x100", "--dump", str(dump), "--automap", "0.2"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    want = _cli_expected(b2d, data, [0], scenes[0].start_pose, 160, 100, 13107, 0)
    assert (tmp_path / "d.automap.ppm").read_bytes() == cli.encode_ppm(want[0])
    out = subprocess.run([exe, "-i", str(wad), "--automap", "0.2"], capture_output=True, text=True)
    assert out.returncode == 2
