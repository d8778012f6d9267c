"""-m gpu: level sets with per-frame states on the sharded path (b2d_render_sharded_levels_states) and the per-frame-level
palette kernel (b2d_palette_lut_levels_device), with a one-rank NCCL communicator; the two-rank variant is skipped on a box
with fewer than two GPUs.  The set: a plain level from a WAD with another PLAYPAL, a timed level (light effects,
animation, scrolling) and a level with declared dynamic sectors; every frame carries its own level and state."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.conftest import sample_poses
from tests.test_gpu_levels import C2, RICH, SMALL, _assert_same, _dev, _palette, levels  # noqa: F401
from tests.test_gpu_levels_states import _oracle_states, _per_frame

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARG = -4                                                        # B2D_ERR_INVALID_ARG


class _DevBytes:
    """n device bytes at ptr, for torch.as_tensor"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 2}


def _job(b2d, levels, n, seed):
    """(scenes, poses, frame levels, tics, moves) of n poses over the three levels C2, RICH, SMALL in a seeded order"""
    rng = np.random.default_rng(seed)
    lv = rng.integers(0, 3, n).astype(np.uint32)
    lv[:3] = [C2, RICH, SMALL]
    pools = [sample_poses(b2d, levels[k]["scene"], n, seed + 10 * k) for k in range(3)]
    poses = np.empty(n, dtype=pools[0].dtype)
    for i, k in enumerate(lv):
        poses[i] = pools[k][i]
    tics, moves = _per_frame(levels, lv, seed + 1, tic0=200)
    return [levels[k]["scene"] for k in range(3)], poses, lv, tics, moves


def _gathered(r, comm, poses, lv, tics, moves, chunk, mode, npix):
    """every frame the callback sees, copied out in gathered order, its checksum table and the calls' (first, cnt, ranks)"""
    import torch
    from rust_doom_b200 import jobs
    n = len(poses)
    frames = torch.zeros((n, npix), dtype=torch.uint8, device="cuda")
    table = jobs.ChecksumTable(1, n, npix, torch.device("cuda", 0))
    seen = []

    def on_chunk(k, first, cnt, ptr, ranks, stream):
        seen.append((first, cnt, ranks))
        table.on_chunk(k, first, cnt, ptr, ranks, stream)
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            src = torch.as_tensor(_DevBytes(ptr, ranks * cnt * npix), device="cuda").view(ranks * cnt, npix)
            frames[first:first + cnt].copy_(src[:cnt])
    st = r.render_sharded_levels_states(comm, poses, lv, tics, moves, chunk, mode, on_chunk)
    torch.cuda.synchronize()
    return frames.cpu().numpy(), table.host()[0], seen, st


@pytest.mark.parametrize("n,chunk", [(5, 5), (5, 2), (21, 7), (23, 0), (23, 4)])
def test_sharded_levels_states_world1(b2d, levels, n, chunk):
    """Chunks that divide the block and chunks that do not, jobs below and above max_batch (7): every gathered frame equals
    b2d_render_device_levels_states over the whole list, its device checksum the host restatement, and sampled frames the
    oracle at their own level and state; RENDER_ONLY hands the callback the same frames; the status word stays clear."""
    import torch
    from rust_doom_b200 import _lib, jobs, parallel
    w, h = 320, 200
    npix = w * h
    scenes, poses, lv, tics, moves = _job(b2d, levels, n, 1300 + n + chunk)
    r = b2d.Renderer.from_levels(scenes, b2d.make_view(w, h), max_batch=7)
    out = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
    r.render_device_levels_states(_dev(poses).data_ptr(), lv, tics, n, out.data_ptr(), moves_per_pose=moves)
    torch.cuda.synchronize()
    want = out.cpu().numpy().reshape(n, npix)
    comm = jobs.single_comm(0)
    per, plan = parallel.sharded_schedule(n, 1, chunk, 7)
    for mode in (_lib.SHARD_RENDER_GATHER, _lib.SHARD_RENDER_ONLY):
        got, sums, seen, st = _gathered(r, comm, poses, lv, tics, moves, chunk, mode, npix)
        assert seen == [(f, c, 1) for f, c in plan] and st["chunks"] == len(plan) and st["frames_local"] == n
        assert st["frames_gathered"] == (n if mode == _lib.SHARD_RENDER_GATHER else 0)
        _assert_same(want, got, "mode %d vs the device path" % mode)
        assert sums.tolist() == [b2d.frame_checksum(want[i]) for i in range(n)]
        assert r.status() == 0
    pick = [0, 1, 2, n - 1]
    oracle = _oracle_states(levels, w, h, poses[pick], lv[pick], tics[pick], [moves[i] for i in pick])
    _assert_same(oracle.reshape(len(pick), npix), want[pick], "oracle")
    comm.close()


def test_sharded_levels_on_level0_equals_render_sharded(b2d, levels):
    """Every pose on level 0 at the renderer's own time: the frames of b2d_render_sharded; the renderer's time is untouched
    by the level-set call, and b2d_render_sharded's launch count for a fixed job is 2 per chunk, as before."""
    import torch
    from rust_doom_b200 import _lib, jobs
    w, h = 320, 200
    npix = w * h
    poses = sample_poses(b2d, levels[C2]["scene"], 11, 1401)
    r = b2d.Renderer.from_levels([levels[k]["scene"] for k in range(3)], b2d.make_view(w, h), max_batch=4)
    r.set_time(77)
    comm = jobs.single_comm(0)
    l0 = r.launch_count
    a, sa, _, _ = _gathered(r, comm, poses, np.zeros(11, np.uint32), np.full(11, 77, np.uint32), None, 4,
                            _lib.SHARD_RENDER_GATHER, npix)
    l1 = r.launch_count
    plain = b2d.Renderer(levels[C2]["scene"], b2d.make_view(w, h), max_batch=4)
    plain.set_time(77)
    plain.render_sharded(comm, poses, 4, _lib.SHARD_RENDER_ONLY)        # the restate of the level's tables at time 77
    p0 = plain.launch_count
    st = plain.render_sharded(comm, poses, 4, _lib.SHARD_RENDER_GATHER)
    assert plain.launch_count - p0 == 2 * st["chunks"] == 6
    b, sb, _, _ = _gathered(r, comm, poses, np.zeros(11, np.uint32), np.full(11, 77, np.uint32), None, 4,
                            _lib.SHARD_RENDER_GATHER, npix)
    assert l1 - l0 == 3 * 3                                              # walk, raster, one state-set expansion per chunk
    table = jobs.ChecksumTable(1, 11, npix, torch.device("cuda", 0))
    plain.render_sharded(comm, poses, 4, _lib.SHARD_RENDER_GATHER, table.on_chunk)
    assert table.host()[0].tolist() == sa.tolist() == sb.tolist()
    _assert_same(a, b, "repeat")
    assert r.status() == 0 and plain.status() == 0
    comm.close()


def test_sharded_levels_invalid_inputs_launch_nothing(b2d, levels):
    """Each invalid input -- also placed where only the padded tail or another rank's block would meet it -- is
    B2D_ERR_INVALID_ARG with no launch, and the renderer renders correctly afterwards."""
    import ctypes
    from rust_doom_b200 import B2dError, _lib, jobs
    from rust_doom_b200 import _frame_states
    w, h = 160, 100
    scenes, poses, lv, tics, moves = _job(b2d, levels, 9, 1500)
    r = b2d.Renderer.from_levels(scenes, b2d.make_view(w, h), max_batch=4)
    comm = jobs.single_comm(0)
    L = _lib.load()
    ok = r.render_sharded_levels_states(comm, poses, lv, tics, moves, 4, _lib.SHARD_RENDER_ONLY)
    assert ok["chunks"] == 3
    l0 = r.launch_count
    bad_level = lv.copy()
    bad_level[-1] = 3                                                    # the last entry: what the padded tail repeats
    rich_moves = levels[RICH]["moves"]
    undeclared = [list(m) for m in moves]
    undeclared[-1] = rich_moves if lv[-1] != RICH else []
    if lv[-1] == RICH:
        undeclared[-1] = [(rich_moves[0][0], 1 << 20, 0)]               # out of its declared range
    for l, m in ((bad_level, moves), (lv, undeclared)):
        with pytest.raises(B2dError) as e:
            r.render_sharded_levels_states(comm, poses, l, tics, m, 4, _lib.SHARD_RENDER_GATHER)
        assert e.value.code == INVALID_ARG
    pc, lvc = np.ascontiguousarray(poses), np.ascontiguousarray(lv)
    st = _lib.ShardedStats()
    cb = _lib.CHUNK_FN(lambda *a: None)

    def raw(levels_ptr, states, arr, nm, mode=_lib.SHARD_RENDER_GATHER):
        return L.b2d_render_sharded_levels_states(r._h, comm._h, pc.ctypes.data, levels_ptr, states, 9, arr, nm, 4, mode, cb, None,
                                                  ctypes.byref(st))
    states, arr, nm = _frame_states(tics, moves, 9)
    assert raw(None, states, arr, nm) == INVALID_ARG
    assert raw(lvc.ctypes.data, None, arr, nm) == INVALID_ARG
    assert raw(lvc.ctypes.data, states, arr, nm, mode=7) == INVALID_ARG
    states[8] = _lib.FrameState(0, nm, 1)                                # a move range past n_moves
    assert raw(lvc.ctypes.data, states, arr, nm) == INVALID_ARG
    assert r.launch_count == l0
    again = _gathered(r, comm, poses, lv, tics, moves, 4, _lib.SHARD_RENDER_GATHER, w * h)
    first = r.render_levels_states(poses, lv, tics, moves).reshape(9, w * h)
    _assert_same(first, again[0], "after the refused calls")
    assert r.status() == 0
    comm.close()


def test_palette_levels_kernel(b2d, levels):
    """Each frame through its own level's palette (levels from WADs with different PLAYPALs): equal to the palette applied
    on the host and to the RGBA output of b2d_render_levels; on a set of one it equals b2d_palette_lut_device; a level out
    of range or a NULL argument is refused without a launch."""
    import torch
    from rust_doom_b200 import B2dError
    w, h = 1920, 1080
    npix = w * h
    scenes = [levels[k]["scene"] for k in (C2, SMALL)]
    pals = [_palette(s) for s in scenes]
    assert (pals[0] != pals[1]).any()
    r = b2d.Renderer.from_levels(scenes, b2d.make_view(w, h), max_batch=6)
    poses = np.concatenate([sample_poses(b2d, s, 3, 1600 + k) for k, s in enumerate(scenes)])
    lv = np.array([0, 1, 1, 0, 1, 0], np.uint32)
    poses = poses[[0, 3, 4, 1, 5, 2]]
    idx, rgba = r.render_levels(poses, lv, rgba=True)
    d_idx = torch.from_numpy(idx.reshape(-1).copy()).cuda()
    out = torch.zeros((6, h, w), dtype=torch.int32, device="cuda")
    r.palette_lut_levels_device(d_idx.data_ptr(), lv, 6, out.data_ptr())
    torch.cuda.synchronize()
    got = out.cpu().numpy().view(np.uint32)
    for i in range(6):
        assert np.array_equal(got[i], pals[lv[i]][idx[i]]), "frame %d: not its level's palette" % i
    _assert_same(rgba, got, "b2d_render_levels RGBA")
    # random index bytes, many frames, an odd frame size (no 128-bit path) on a set of one against K3
    one = b2d.Renderer.from_levels(scenes[1:], b2d.make_view(333, 101), max_batch=1)
    rnd = torch.randint(0, 256, (37 * 333 * 101,), dtype=torch.uint8, device="cuda")
    a = torch.zeros(37 * 333 * 101, dtype=torch.int32, device="cuda")
    b = torch.ones_like(a)
    one.palette_lut_levels_device(rnd.data_ptr(), [0] * 37, 37, a.data_ptr())
    one.palette_lut_device(rnd.data_ptr(), b.data_ptr(), 37 * 333 * 101)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    l0 = r.launch_count
    with pytest.raises(B2dError):
        r.palette_lut_levels_device(d_idx.data_ptr(), [0, 1, 2, 0, 0, 0], 6, out.data_ptr())
    with pytest.raises(B2dError):
        r.palette_lut_levels_device(0, lv, 6, out.data_ptr())
    assert r.launch_count == l0


def _wad3(tmp_path):
    """an IWAD of three levels: plain, timed (light effects, animation, scrolling walls), and a third map"""
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1", "E1M2", "E1M3"), cfg=synthwad.SynthConfig(mid_pct=20, thing_pct=30, anim=True))
    wad = tmp_path / "three.wad"
    wad.write_bytes(data)
    return data, wad


def _mirror_stream(b2d, data, set_, per_level, tics, w, h):
    from rust_doom_b200 import cli
    arch = b2d.Archive.from_bytes(data)
    scenes = [b2d.Scene(arch, i) for i in set_]
    poses, lv, t = cli.level_set_job(b2d, scenes, per_level, tics)
    r = b2d.Renderer.from_levels(scenes, b2d.make_view(w, h), max_batch=8)
    idx, rgba = r.render_levels_states(poses, lv, t, rgba=True)
    return idx, rgba, b"".join(cli.encode_ppm(cli.rgba_to_rgb(f)) for f in rgba)


def test_cli_levels_one_process_and_world1(b2d, tmp_path):
    """Compiled and Python --levels, in one process and (Python: gathered frames coloured on the device; compiled: the
    checksum sink) with --world 1: the streams equal the Python mirror's frames, the compiled checksum its restatement."""
    from rust_doom_b200 import build
    data, wad = _wad3(tmp_path)
    idx, rgba, want = _mirror_stream(b2d, data, [2, 0], 3, 40, 320, 200)
    exe = build.build_cli()
    args = ["--iwad", str(wad), "-r", "320x200", "--levels", "2,0", "--poses", "3", "--tics", "40"]
    res = subprocess.run([exe] + args + ["--stream", str(tmp_path / "c.ppm"), "--dump", str(tmp_path / "c.ppm")],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    assert (tmp_path / "c.ppm").read_bytes() == want
    from rust_doom_b200 import cli
    assert (tmp_path / "c.2.ppm").read_bytes() == cli.encode_ppm(cli.rgba_to_rgb(rgba[0]))
    assert (tmp_path / "c.0.ppm").read_bytes() == cli.encode_ppm(cli.rgba_to_rgb(rgba[3]))
    env = dict(os.environ, PYTHONPATH=ROOT)
    for extra in ([], ["--world", "1", "--rank", "0", "--id-file", str(tmp_path / "pid"), "--chunk", "4"]):
        out = tmp_path / ("p%d.ppm" % len(extra))
        res = subprocess.run([sys.executable, "-m", "rust_doom_b200.cli"] + args + ["--stream", str(out)] + extra,
                             capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
        assert res.returncode == 0, res.stdout + res.stderr
        assert out.read_bytes() == want, extra
    res = subprocess.run([exe] + args + ["--world", "1", "--rank", "0", "--id-file", str(tmp_path / "cid"), "--chunk", "4"],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    total = 0
    for f in idx:
        total = (total * 31 + b2d.frame_checksum(f)) & 0xFFFFFFFF
    assert "rank 0/1: 6 frames gathered in 2 chunk(s)" in res.stdout and ("checksum %08x" % total) in res.stdout, res.stdout


def test_cli_levels_two_ranks(b2d, tmp_path):
    """Two processes, two GPUs (skipped on a one-GPU box): the compiled CLI's ranks agree with the one-rank checksum, and
    the Python CLI's rank 0 writes the mirror's stream."""
    import re
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from rust_doom_b200 import build
    data, wad = _wad3(tmp_path)
    _, _, want = _mirror_stream(b2d, data, [0, 1, 2], 5, 7, 320, 200)
    exe = build.build_cli()
    args = ["--iwad", str(wad), "-r", "320x200", "--levels", "all", "--poses", "5", "--tics", "7", "--chunk", "3"]
    one = subprocess.run([exe] + args + ["--world", "1", "--rank", "0", "--id-file", str(tmp_path / "i1")], capture_output=True,
                         text=True, timeout=300)
    assert one.returncode == 0, one.stderr
    sums = re.search(r"checksum ([0-9a-f]{8})", one.stdout).group(1)
    for tag, cmd in (("c", [exe] + args), ("p", [sys.executable, "-m", "rust_doom_b200.cli"] + args + ["--stream", str(tmp_path / "p2.ppm")])):
        procs = [subprocess.Popen(cmd + ["--world", "2", "--rank", str(q), "--id-file", str(tmp_path / (tag + "2"))], cwd=ROOT,
                                  env=dict(os.environ, PYTHONPATH=ROOT), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
                 for q in range(2)]
        outs = [p.communicate(timeout=600)[0] for p in procs]
        assert all(p.returncode == 0 for p in procs), outs
        if tag == "c":
            assert [re.search(r"checksum ([0-9a-f]{8})", o).group(1) for o in outs] == [sums, sums]
    assert (tmp_path / "p2.ppm").read_bytes() == want
