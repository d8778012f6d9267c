"""-m gpu: the player's light effects per frame (DESIGN.md C18) through b2d_render_levels_states_lights,
b2d_render_device_levels_states_lights and b2d_walk_device_levels_states_lights, on the four levels of
tests/test_gpu_levels.py (masked middles, sprites, sky, light effects, dynamic sectors, and a level without
time-dependent content).  Every frame is compared bit for bit, index and RGBA, with the oracle's frame of its pose, level,
state, fixed colormap and extra light (tests/lightcheck.py on the oracle); every table set with lightcheck.tables_at."""
import subprocess

import numpy as np
import pytest

from oracle import render
from tests import lightcheck as LC
from tests.conftest import oracle_blob
from tests.test_gpu_levels import RICH, SMALL, _assert_same, _dev, _mix, _palette, levels  # noqa: F401
from tests.test_gpu_levels_states import _per_frame, _timed
from tests.test_gpu_resolve import clock, pending  # noqa: F401

pytestmark = pytest.mark.gpu


def _lights(n, seed, p_fixed=0.4, p_extra=0.4):
    """a seeded (fixed_colormap, extralight) per frame: rows 32, 1 and random ones, extra light 0..2"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        fixed = -1
        if rng.random() < p_fixed:
            fixed = int(rng.choice([32, 1, 0, 31, int(rng.integers(0, 33))]))
        out.append((fixed, int(rng.integers(1, 3)) if rng.random() < p_extra else 0))
    return out


def _oracle_lights(levels, w, h, poses, lv, tics, moves, lights):
    from concurrent.futures import ThreadPoolExecutor
    import os
    from oracle import scene as S
    view = render.make_view(w, h)
    out = np.empty((len(poses), h, w), np.uint8)

    def one(i):
        L = levels[int(lv[i])]
        blob = S.apply_moves(L["blob"], moves[i]) if moves[i] else L["blob"]
        out[i:i + 1] = LC.render(blob, view, poses[i:i + 1], tics=int(tics[i]), fixed_colormap=lights[i][0],
                                 extralight=lights[i][1])

    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        list(ex.map(one, range(len(poses))))
    return out


def _renderer(b2d, levels, w, h, max_batch):
    return b2d.Renderer.from_levels([L["scene"] for L in levels], b2d.make_view(w, h), max_batch=max_batch)


@pytest.mark.parametrize("w,h,per_level", [(320, 200, 24), (1920, 1080, 5)])
def test_lights_match_oracle(b2d, levels, w, h, per_level):
    """Seeded per-frame levels, tics, moves, fixed colormaps and extra light: host path (n > max_batch) and device path,
    index and RGBA through each frame's level palette, equal to the oracle."""
    import torch
    poses, lv = _mix(b2d, levels, per_level, 71 + w)
    n = len(poses)
    tics, moves = _per_frame(levels, lv, 5 + w)
    lights = _lights(n, 9 + w)
    assert any(f == 32 for f, _ in lights) and any(e for _, e in lights)
    want = _oracle_lights(levels, w, h, poses, lv, tics, moves, lights)
    r = _renderer(b2d, levels, w, h, max_batch=max(n // 3, 1))
    idx, rgba = r.render_levels_states(poses, lv, tics, moves, rgba=True, lights=lights)
    _assert_same(want, idx, "host index")
    pal = [_palette(L["scene"]) for L in levels]
    want_rgba = np.stack([pal[int(lv[i])][want[i]] for i in range(n)])
    assert np.array_equal(rgba, want_rgba), "host RGBA"
    d_idx = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
    d_rgba = torch.empty((n, h, w), dtype=torch.int32, device="cuda")
    dp = _dev(poses)
    r.render_device_levels_states(dp.data_ptr(), lv, tics, n, d_idx.data_ptr(), d_rgba.data_ptr(), moves, lights=lights)
    torch.cuda.synchronize()
    _assert_same(want, d_idx.cpu().numpy(), "device index")
    assert np.array_equal(d_rgba.cpu().numpy().view(np.uint32), want_rgba), "device RGBA"


def test_no_lights_is_the_call_without_lights(b2d, levels):
    """lights = None and every frame {-1, 0}: the frames and the launch counts of render_levels_states"""
    import torch
    w, h = 640, 400
    poses, lv = _mix(b2d, levels, 6, 3)
    n = len(poses)
    tics, moves = _per_frame(levels, lv, 4)
    outs, counts = [], []
    dp = _dev(poses)
    for lights in ("plain", None, [(-1, 0)] * n):
        r = _renderer(b2d, levels, w, h, max_batch=n)
        d = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
        c0 = r.launch_count
        if lights == "plain":
            r.render_device_levels_states(dp.data_ptr(), lv, tics, n, d.data_ptr(), 0, moves)
        else:
            r.render_device_levels_states(dp.data_ptr(), lv, tics, n, d.data_ptr(), 0, moves, lights=lights)
        torch.cuda.synchronize()
        outs.append(d.cpu().numpy())
        counts.append(r.launch_count - c0)
    assert counts[0] == counts[1] == counts[2]
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2])


def test_table_sets_follow_level_state_and_extralight(b2d, levels):
    """Frames share a table set exactly as their (level, state, extra light) do; a frame with extra light on a level
    without time-dependent content has a set, one without none; every set equals lightcheck.tables_at."""
    timed = _timed(b2d, levels)
    assert not timed[SMALL]
    poses, lv = _mix(b2d, levels, 8, 12)
    n = len(poses)
    tics, moves = _per_frame(levels, lv, 13)
    tics[::3] = 77                                       # repeated states, so that sets are shared
    lights = _lights(n, 14, p_fixed=0.2, p_extra=0.6)
    r = _renderer(b2d, levels, 320, 200, max_batch=n)
    dp = _dev(poses)
    t = r.walk_device_levels_states(dp.data_ptr(), lv, tics, n, moves, lights=lights)
    slots = r.state_slots(n)
    keys = {}
    for i in range(n):
        e = lights[i][1]
        has = timed[int(lv[i])] or e > 0
        assert (slots[i] != 0xFFFFFFFF) == has, (i, int(lv[i]), e)
        if not has:
            continue
        key = (int(lv[i]), e, int(tics[i]) if timed[int(lv[i])] else 0, tuple(map(tuple, moves[i])))
        want = LC.tables_at(levels[key[0]]["blob"], key[2], moves[i], extralight=e)
        got = r.state_tables(int(slots[i]))
        assert got == want, "frame %d (level %d, extra light %d): set differs from tables_at" % (i, key[0], e)
        keys.setdefault(int(slots[i]), set()).add((key[0], e))
    assert all(len(v) == 1 for v in keys.values()), "a set shared across levels or extra lights"
    import torch
    out = torch.empty((n, 200, 320), dtype=torch.uint8, device="cuda")
    r.raster_device(t, out.data_ptr())
    torch.cuda.synchronize()
    _assert_same(_oracle_lights(levels, 320, 200, poses, lv, tics, moves, lights), out.cpu().numpy(), "walked ticket")


def test_bad_lights_enqueue_nothing(b2d, levels):
    import torch
    from rust_doom_b200 import B2dError
    poses, lv = _mix(b2d, levels, 2, 5)
    n = len(poses)
    r = _renderer(b2d, levels, 160, 100, max_batch=n)
    d = torch.empty((n, 100, 160), dtype=torch.uint8, device="cuda")
    dp = _dev(poses)
    c0 = r.launch_count
    for bad in ((33, 0), (-2, 0), (32, 3), (0, 7)):
        lights = [(-1, 0)] * n
        lights[n // 2] = bad
        with pytest.raises(B2dError):
            r.render_levels_states(poses, lv, 0, lights=lights)
        with pytest.raises(B2dError):
            r.render_device_levels_states(dp.data_ptr(), lv, 0, n, d.data_ptr(), lights=lights)
        with pytest.raises(B2dError):
            r.walk_device_levels_states(dp.data_ptr(), lv, 0, n, lights=lights)
    assert r.launch_count == c0
    # still usable, and the first row-32 request builds the level's planes once (two launches)
    r.render_device_levels_states(dp.data_ptr(), lv, 0, n, d.data_ptr(), lights=[(32, 0)] * n)
    c1 = r.launch_count
    r.render_device_levels_states(dp.data_ptr(), lv, 0, n, d.data_ptr(), lights=[(32, 0)] * n)
    assert r.launch_count - c1 == 3
    torch.cuda.synchronize()


def test_staging_waits_for_the_copy_two_batches_earlier(b2d, levels, clock):
    """The fixed colormaps are staged with the levels: the walk into a slot rewrites its staging only after the copy of
    the batch two walks earlier has read it, on held-back streams; frames are the oracle's."""
    import torch
    poses, lv = _mix(b2d, levels, 3, 8)
    n = len(poses)
    tics, moves = _per_frame(levels, lv, 9)
    L = [_lights(n, 20 + k, p_fixed=0.8) for k in range(3)]
    r = _renderer(b2d, levels, 320, 200, max_batch=n)
    outs = [torch.empty((n, 200, 320), dtype=torch.uint8, device="cuda") for _ in range(3)]
    dp = _dev(poses)
    for k in range(3):     # row-32 planes built and staging touched outside the hold
        r.render_device_levels_states(dp.data_ptr(), lv, tics, n, outs[k].data_ptr(), 0, moves, lights=L[k])
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    hold = clock.hold(s)
    t0 = r.walk_device_levels_states(dp.data_ptr(), lv, tics, n, moves, s.cuda_stream, lights=L[0])
    pending(hold, "first walk")
    t1 = r.walk_device_levels_states(dp.data_ptr(), lv, tics, n, moves, s.cuda_stream, lights=L[1])
    pending(hold, "second walk")
    r.raster_device(t0, outs[0].data_ptr(), 0, s.cuda_stream)
    pending(hold, "raster")
    t2 = r.walk_device_levels_states(dp.data_ptr(), lv, tics, n, moves, s.cuda_stream, lights=L[2])
    assert hold.query(), "the third walk rewrote the staging the first walk's held copy reads"
    r.raster_device(t1, outs[1].data_ptr(), 0, s.cuda_stream)
    r.raster_device(t2, outs[2].data_ptr(), 0, s.cuda_stream)
    torch.cuda.synchronize()
    for k in range(3):
        _assert_same(_oracle_lights(levels, 320, 200, poses, lv, tics, moves, L[k]), outs[k].cpu().numpy(), "batch %d" % k)


def test_clis_fixed_colormap_32(tmp_path, b2d, capsys):
    """Both CLIs render a --levels job with --fixed-colormap 32 (and --extralight 2, ignored under it) as the library does"""
    from rust_doom_b200 import cli
    from tests.test_cli import _b2d_binary
    from tests.test_gpu_resolve import _cli_wad
    data, wad = _cli_wad(tmp_path)
    w, h = 160, 100
    arch = b2d.Archive.from_bytes(data)
    scenes = [b2d.Scene(arch, i) for i in (0, 1)]
    poses, lv, tics = cli.level_set_job(b2d, scenes, 3, 40)
    r = b2d.Renderer.from_levels(scenes, b2d.make_view(w, h), max_batch=8)
    rgba = r.render_levels_states(poses, lv, tics, rgba=True, lights=[(32, 2)] * len(poses))[1]
    blobs = [oracle_blob(data, k) for k in (0, 1)]
    view = render.make_view(w, h)
    for i in range(len(poses)):
        want = LC.render(blobs[int(lv[i])], view, poses[i:i + 1], tics=int(tics[i]), fixed_colormap=32)
        assert np.array_equal(rgba[i], _palette(scenes[int(lv[i])])[want[0]])
    want = b"".join(cli.encode_ppm(cli.rgba_to_rgb(f)) for f in rgba)
    stream = tmp_path / "s.ppm"
    args = ["--levels", "0,1", "--poses", "3", "--tics", "40", "-r", "%dx%d" % (w, h), "--fixed-colormap", "32",
            "--extralight", "2", "--stream", str(stream)]
    assert cli.main(["--iwad", str(wad)] + args) == 0
    assert stream.read_bytes() == want
    out = subprocess.run([_b2d_binary(), "-i", str(wad)] + args, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert stream.read_bytes() == want
