"""-m gpu: the resolved sharded calls (b2d_render_sharded_resolved, b2d_render_sharded_levels_states_resolved) with a
one-rank NCCL communicator; the two-rank variant is skipped on a box with fewer than two GPUs.  Every resolved frame the
callback sees is compared with the numpy resolve (oracle/resolve.py) of the oracle's index frame for its pose, level and
state, and with Renderer.resolve of the frame the unresolved call gathers at the same position.  The level set is that
of tests/test_gpu_sharded_levels.py: a plain level, a timed level with declared dynamic sectors and a level from a WAD
with another PLAYPAL."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import resolve as R
from tests.conftest import sample_poses
from tests.test_gpu_levels import C2, RICH, SMALL, _oracle, levels  # noqa: F401
from tests.test_gpu_levels_states import _oracle_states
from tests.test_gpu_sharded_levels import _DevBytes, _job

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARG = -4                                                        # B2D_ERR_INVALID_ARG
FORMATS = ("rgba", "rgb", "rgb_planar", "gray")
# views and the factors each is tested at (3 and 5 divide 480 x 270, 1, 2 and 4 divide 320 x 200)
VIEWS = [((320, 200), (1, 2, 4)), ((480, 270), (3, 5))]
_ORACLE = {}


def _pal_rgb(blob):
    """(256, 3) R, G, B of the palette stored in an oracle-compiled scene blob (header word 20 = its offset)"""
    p = np.frombuffer(blob, "<u4", 256, int(np.frombuffer(blob, "<u4", 21)[20]))
    return np.stack([p & 0xFF, (p >> 8) & 0xFF, (p >> 16) & 0xFF], axis=1)


def _oracle_cached(key, fn):
    if key not in _ORACLE:
        _ORACLE[key] = fn()
    return _ORACLE[key]


def _bytes(a, n):
    """frames as (n, bytes per frame) uint8: numpy arrays of any dtype, or CUDA tensors"""
    if not isinstance(a, np.ndarray):
        a = a.cpu().numpy()
    return np.ascontiguousarray(a).view(np.uint8).reshape(n, -1)


def _run(call, n, per, frame_bytes, **kw):
    """(every frame the callback sees, copied out by pose and without the padded tail, as (n, frame_bytes) uint8; the
    calls' (first, cnt, ranks); the stats) of call(on_chunk=..., **kw)"""
    import torch
    frames = torch.zeros((n, frame_bytes), dtype=torch.uint8, device="cuda")
    seen = []

    def on_chunk(k, first, cnt, ptr, ranks, stream):
        seen.append((first, cnt, ranks))
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            src = torch.as_tensor(_DevBytes(ptr, ranks * cnt * frame_bytes), device="cuda").view(ranks * cnt, frame_bytes)
            for q in range(ranks):
                g = q * per + first
                m = min(cnt, n - g)
                if m > 0:
                    frames[g:g + m].copy_(src[q * cnt:q * cnt + m])
    st = call(on_chunk=on_chunk, **kw)
    torch.cuda.synchronize()
    return frames.cpu().numpy(), seen, st


def _calls(b2d, levels, comm, n, chunk, w, h, seed, max_batch=7):
    """the two calls on one job of n poses at a w x h view: {name: (renderer, call(**kw), frame levels or None, the
    oracle's index frames, palettes)}; the plain call renders C2 at the renderer's time, the level-set call the three
    levels with a state per pose"""
    scenes, poses, lv, tics, moves = _job(b2d, levels, n, seed)
    plain_poses = sample_poses(b2d, levels[C2]["scene"], n, seed + 50)
    ls = b2d.Renderer.from_levels(scenes, b2d.make_view(w, h), max_batch=max_batch)
    plain = b2d.Renderer(levels[C2]["scene"], b2d.make_view(w, h), max_batch=max_batch)
    want_ls = _oracle_cached(("ls", n, seed, w, h), lambda: _oracle_states(levels, w, h, poses, lv, tics, moves))
    want_pl = _oracle_cached(("pl", n, seed, w, h), lambda: _oracle(levels, w, h, plain_poses, np.zeros(n, np.uint32)))
    pals = [_pal_rgb(levels[k]["blob"]) for k in (C2, RICH, SMALL)]
    return {
        "levels_states": (ls, lambda **kw: ls.render_sharded_levels_states(comm, poses, lv, tics, moves, chunk, **kw), lv,
                          want_ls, pals),
        "plain": (plain, lambda **kw: plain.render_sharded(comm, plain_poses, chunk, **kw), None, want_pl, pals[:1]),
    }


@pytest.mark.parametrize("n,chunk", [(5, 5), (5, 2), (21, 7), (23, 0), (23, 4)])
def test_resolved_frames_equal_the_resolve_of_the_gathered_frames(b2d, levels, n, chunk):
    """Chunks that divide the block and chunks that do not, jobs below and above max_batch (7), every format at factors 1,
    2, 4 (320 x 200) and 3, 5 (480 x 270), both calls, RENDER_GATHER: every resolved frame equals the numpy resolve of the
    oracle's index frame and Renderer.resolve of the unresolved call's frame; RENDER_ONLY hands the callback this rank's
    resolved frames with ranks = 1; the stats count resolved bytes; the status word stays clear."""
    import torch
    from rust_doom_b200 import _lib, jobs, parallel
    comm = jobs.single_comm(0)
    per, plan = parallel.sharded_schedule(n, 1, chunk, 7)
    for (w, h), factors in VIEWS:
        for name, (r, call, lv, want_idx, pals) in _calls(b2d, levels, comm, n, chunk, w, h, 1700 + n).items():
            idx, seen, st = _run(call, n, per, w * h, mode=_lib.SHARD_RENDER_GATHER)
            assert np.array_equal(idx, _bytes(want_idx, n)), (name, w, h)
            d_idx = torch.from_numpy(idx.reshape(n, h, w)).cuda()
            for k in factors:
                for fmt in FORMATS:
                    fb = r.resolve_frame_bytes(k, b2d.RESOLVE_FORMATS[fmt])
                    got, seen, st = _run(call, n, per, fb, mode=_lib.SHARD_RENDER_GATHER, resolve=(k, fmt))
                    what = (name, w, h, k, fmt)
                    assert seen == [(f, c, 1) for f, c in plan], what
                    assert (st["chunks"], st["frames_local"], st["frames_gathered"], st["bytes_received"]) == (len(plan), n, n, 0)
                    assert np.array_equal(got, _bytes(R.resolve(want_idx, pals, k, fmt, lv), n)), what
                    assert np.array_equal(got, _bytes(r.resolve(d_idx, k, fmt, lv), n)), what
            k, fmt = factors[-1], "rgb"
            got, seen, st = _run(call, n, per, r.resolve_frame_bytes(k, b2d.RESOLVE_RGB8), mode=_lib.SHARD_RENDER_ONLY,
                                 resolve=(k, fmt))
            assert seen == [(f, c, 1) for f, c in plan] and st["frames_gathered"] == 0 and st["bytes_received"] == 0
            assert np.array_equal(got, _bytes(R.resolve(want_idx, pals, k, fmt, lv), n)), (name, "RENDER_ONLY")
            assert r.status() == 0
    comm.close()


def test_each_frame_through_its_own_levels_palette(b2d, levels):
    """A set of two levels whose WADs have different PLAYPALs, levels interleaved: every resolved frame is its oracle frame
    through its own level's palette, and differs from the same frame through the other level's palette."""
    from rust_doom_b200 import _lib, jobs
    w, h, n = 320, 200, 12
    pals = [_pal_rgb(levels[k]["blob"]) for k in (C2, SMALL)]
    assert (pals[0] != pals[1]).all()
    lv = np.array([0, 1, 1, 0, 1, 0, 0, 1, 0, 1, 1, 0], np.uint32)
    pools = [sample_poses(b2d, levels[k]["scene"], n, 1800 + k) for k in (C2, SMALL)]
    poses = np.array([pools[lv[i]][i] for i in range(n)], dtype=pools[0].dtype)
    tics = np.zeros(n, np.uint32)
    r = b2d.Renderer.from_levels([levels[C2]["scene"], levels[SMALL]["scene"]], b2d.make_view(w, h), max_batch=4)
    comm = jobs.single_comm(0)
    idx = _oracle(levels, w, h, poses, np.where(lv == 0, C2, SMALL))
    for fmt in ("rgb", "gray"):
        fb = r.resolve_frame_bytes(2, b2d.RESOLVE_FORMATS[fmt])
        got, _, _ = _run(lambda **kw: r.render_sharded_levels_states(comm, poses, lv, tics, None, 4, **kw), n, n, fb,
                         mode=_lib.SHARD_RENDER_GATHER, resolve=(2, fmt))
        assert np.array_equal(got, _bytes(R.resolve(idx, pals, 2, fmt, lv), n)), fmt
        swapped = _bytes(R.resolve(idx, pals, 2, fmt, 1 - lv), n)
        assert all(not np.array_equal(got[i], swapped[i]) for i in range(n)), fmt
    assert r.status() == 0
    comm.close()


def test_gather_only_carries_resolved_chunks(b2d, levels):
    """GATHER_ONLY renders nothing and hands the callback the exchange buffers at resolved size: right after a resolved
    RENDER_GATHER of the same two-chunk job they hold that job's resolved frames at the offsets the callback reads; the
    stats fields are as documented"""
    from rust_doom_b200 import _lib, jobs
    w, h, n, chunk = 320, 200, 8, 4
    comm = jobs.single_comm(0)
    for name, (r, call, lv, want_idx, pals) in _calls(b2d, levels, comm, n, chunk, w, h, 1900, max_batch=4).items():
        for k, fmt in ((1, "rgba"), (2, "rgb_planar"), (4, "gray")):
            fb = r.resolve_frame_bytes(k, b2d.RESOLVE_FORMATS[fmt])
            got, _, _ = _run(call, n, n, fb, mode=_lib.SHARD_RENDER_GATHER, resolve=(k, fmt))
            assert np.array_equal(got, _bytes(R.resolve(want_idx, pals, k, fmt, lv), n)), (name, k, fmt)
            l0 = r.launch_count
            again, seen, st = _run(call, n, n, fb, mode=_lib.SHARD_GATHER_ONLY, resolve=(k, fmt))
            assert r.launch_count == l0, (name, k, fmt)
            assert seen == [(0, 4, 1), (4, 4, 1)]
            assert (st["frames_local"], st["frames_gathered"], st["chunks"], st["chunk_frames"], st["bytes_received"]) == (8, 8, 2, 4, 0)
            assert np.array_equal(again, got), (name, k, fmt)
    comm.close()


def test_launches_are_the_unresolved_calls_plus_one_per_chunk(b2d, levels):
    from rust_doom_b200 import _lib, jobs
    comm = jobs.single_comm(0)
    for name, (r, call, _, _, _) in _calls(b2d, levels, comm, 23, 4, 320, 200, 2000).items():
        call(mode=_lib.SHARD_RENDER_GATHER)                                  # first-call set-up out of the count
        l0 = r.launch_count
        st = call(mode=_lib.SHARD_RENDER_GATHER)
        l1 = r.launch_count
        st2 = call(mode=_lib.SHARD_RENDER_GATHER, resolve=(2, "gray"))
        l2 = r.launch_count
        assert st["chunks"] == st2["chunks"] == 6
        assert l2 - l1 == (l1 - l0) + st2["chunks"], (name, l1 - l0, l2 - l1)
        assert r.status() == 0
    comm.close()


def test_resolved_call_between_unresolved_calls(b2d, levels):
    """On one communicator: an unresolved call, a resolved RGBA factor-1 call (its exchange buffers are 4x the index
    frames', so they grow), the unresolved call again: the first and last give the same frames and device checksums, and
    the RGBA frames are Renderer.resolve of the index frames"""
    import torch
    from rust_doom_b200 import _lib, jobs
    w, h, n, chunk = 320, 200, 20, 8
    comm = jobs.single_comm(0)
    r = b2d.Renderer(levels[C2]["scene"], b2d.make_view(w, h), max_batch=chunk)
    poses = sample_poses(b2d, levels[C2]["scene"], n, 2100)

    def unresolved():
        """the gathered frames and their device checksums"""
        table = jobs.ChecksumTable(1, n, w * h, torch.device("cuda", 0))

        def call(on_chunk, **kw):
            def both(*a):
                table.on_chunk(*a)
                on_chunk(*a)
            return r.render_sharded(comm, poses, chunk, on_chunk=both, **kw)
        frames, _, _ = _run(call, n, n, w * h, mode=_lib.SHARD_RENDER_GATHER)
        return frames, table.host()[0]
    a, sa = unresolved()
    fb = r.resolve_frame_bytes(1, b2d.RESOLVE_RGBA8)
    assert fb == 4 * w * h
    rgba, _, _ = _run(lambda **kw: r.render_sharded(comm, poses, chunk, **kw), n, n, fb, mode=_lib.SHARD_RENDER_GATHER,
                      resolve=(1, "rgba"))
    b, sb = unresolved()
    assert np.array_equal(a, b) and sa.tolist() == sb.tolist()
    assert sa.tolist() == [b2d.frame_checksum(f) for f in a]
    assert np.array_equal(rgba, _bytes(r.resolve(torch.from_numpy(a.reshape(n, h, w)).cuda(), 1, "rgba"), n))
    assert r.status() == 0
    comm.close()


@pytest.mark.parametrize("w,h,n,fmt", [(1920, 1080, 512, "gray"), (3840, 2160, 256, "rgb")], ids=["1080p_gray", "4k_rgb"])
def test_scale_checksums_against_the_oracle(b2d, levels, w, h, n, fmt):
    """The c5 poses (random_poses, seed 5) on the c5 level, chunks of 128, resolved by 2: device checksums of every
    gathered frame (ChecksumTable at the resolved frame size) equal, on sampled entries, the host checksum of the numpy
    resolve of the oracle's frame; three launches per chunk; the status word stays clear"""
    import torch
    from rust_doom_b200 import _lib, jobs
    from rust_doom_b200 import poses as P
    scene = levels[C2]["scene"]
    poses = P.random_poses(scene, n, 5)
    r = b2d.Renderer(scene, b2d.make_view(w, h), max_batch=128)
    comm = jobs.single_comm(0)
    fb = r.resolve_frame_bytes(2, b2d.RESOLVE_FORMATS[fmt])
    assert fb == (w // 2) * (h // 2) * (1 if fmt == "gray" else 3)
    table = jobs.ChecksumTable(1, n, fb, torch.device("cuda", 0))
    l0 = r.launch_count
    st = r.render_sharded(comm, poses, 128, _lib.SHARD_RENDER_GATHER, table.on_chunk, resolve=(2, fmt))
    sums = table.host()[0]
    assert r.status() == 0
    assert st["chunks"] == n // 128 and r.launch_count - l0 == 3 * st["chunks"]
    rng = np.random.default_rng(n)
    pick = sorted({0, 1, 127, 128, n - 1} | set(rng.choice(n, 3, replace=False).tolist()))
    idx = _oracle(levels, w, h, poses[pick], np.full(len(pick), C2))
    want = R.resolve(idx, [_pal_rgb(levels[C2]["blob"])], 2, fmt)
    assert [int(sums[i]) for i in pick] == [b2d.frame_checksum(f) for f in want]
    comm.close()


def test_refusals_launch_nothing(b2d, levels):
    """A factor of 0 or 9 or one that does not divide the view, a format of -1 or 4, and on the level-set call the level and
    move refusals of the unresolved call: B2D_ERR_INVALID_ARG with no launch (also with no poses at all); a valid call
    afterwards gives the right frames"""
    import ctypes
    from rust_doom_b200 import _frame_states, _lib, jobs
    w, h, n = 320, 200, 9
    scenes, poses, lv, tics, moves = _job(b2d, levels, n, 1500)
    ls = b2d.Renderer.from_levels(scenes, b2d.make_view(w, h), max_batch=4)
    plain = b2d.Renderer(levels[C2]["scene"], b2d.make_view(w, h), max_batch=4)
    comm = jobs.single_comm(0)
    L = _lib.load()
    st = _lib.ShardedStats()
    cb = _lib.CHUNK_FN(lambda *a: None)
    pc, lvc = np.ascontiguousarray(poses), np.ascontiguousarray(lv)
    pp = np.ascontiguousarray(sample_poses(b2d, levels[C2]["scene"], n, 1550))
    states, arr, nm = _frame_states(tics, moves, n)

    def raw_plain(k, f, count=n, mode=_lib.SHARD_RENDER_GATHER):
        return L.b2d_render_sharded_resolved(plain._h, comm._h, pp.ctypes.data, count, 4, k, f, mode, cb, None, ctypes.byref(st))

    def raw_ls(k, f, levels_ptr=lvc.ctypes.data, states=states, count=n, mode=_lib.SHARD_RENDER_GATHER):
        return L.b2d_render_sharded_levels_states_resolved(ls._h, comm._h, pc.ctypes.data, levels_ptr, states, count, arr, nm, 4,
                                                           k, f, mode, cb, None, ctypes.byref(st))
    # first-call set-up before the counts
    ls.render_sharded_levels_states(comm, poses, lv, tics, moves, 4, _lib.SHARD_RENDER_ONLY)
    plain.render_sharded(comm, pp, 4, _lib.SHARD_RENDER_ONLY)
    l0 = (ls.launch_count, plain.launch_count)
    for k, f in ((0, 0), (9, 0), (3, 0), (7, 1), (2, -1), (2, 4)):       # 3 and 7 divide neither 320 nor 200
        assert raw_plain(k, f) == INVALID_ARG, (k, f)
        assert raw_ls(k, f) == INVALID_ARG, (k, f)
        assert raw_plain(k, f, count=0) == INVALID_ARG and raw_ls(k, f, count=0) == INVALID_ARG, (k, f)
    assert raw_plain(2, 3, mode=7) == INVALID_ARG and raw_ls(2, 3, mode=7) == INVALID_ARG
    assert raw_plain(2, 3, count=0) == 0 and raw_ls(2, 3, count=0) == 0                # a valid empty job: nothing
    # the level-set call's own refusals, with a valid resolve
    bad_level = lvc.copy()
    bad_level[-1] = 3                                                    # the last entry: what the padded tail repeats
    assert raw_ls(2, 3, levels_ptr=bad_level.ctypes.data) == INVALID_ARG
    assert raw_ls(2, 3, levels_ptr=None) == INVALID_ARG
    assert raw_ls(2, 3, states=None) == INVALID_ARG
    past = (_lib.FrameState * n)(*states[:n])
    past[n - 1] = _lib.FrameState(0, nm, 1)                              # a move range past n_moves
    assert raw_ls(2, 3, states=past) == INVALID_ARG
    rich_moves = levels[RICH]["moves"]
    undeclared = [list(m) for m in moves]
    undeclared[-1] = rich_moves if lv[-1] != RICH else [(rich_moves[0][0], 1 << 20, 0)]
    with pytest.raises(b2d.B2dError) as e:
        ls.render_sharded_levels_states(comm, poses, lv, tics, undeclared, 4, _lib.SHARD_RENDER_GATHER, resolve=(2, "gray"))
    assert e.value.code == INVALID_ARG
    assert (ls.launch_count, plain.launch_count) == l0
    pals = [_pal_rgb(levels[k]["blob"]) for k in (C2, RICH, SMALL)]
    got, _, _ = _run(lambda **kw: ls.render_sharded_levels_states(comm, poses, lv, tics, moves, 4, **kw), n, n, w * h // 4,
                     mode=_lib.SHARD_RENDER_GATHER, resolve=(2, "gray"))
    want = ls.render_levels_states(poses, lv, tics, moves)
    assert np.array_equal(got, _bytes(R.resolve(want, pals, 2, "gray", lv), n))
    assert ls.status() == 0 and plain.status() == 0
    comm.close()


_WORKER = r"""
import json, sys
import numpy as np, torch
import rust_doom_b200 as b2d
from rust_doom_b200 import _lib, jobs
from tests.test_gpu_sharded_resolve import _two_rank_job
uid, rank, world, out = bytes.fromhex(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), sys.argv[4]
torch.cuda.set_device(rank)
comm = b2d.Comm(uid, rank, world, rank)
res = {}
for name, (r, call, n, fb) in _two_rank_job(b2d, rank).items():
    per = (n + world - 1) // world
    table = jobs.ChecksumTable(world, per, fb, torch.device("cuda", rank))
    st = call(comm, table.on_chunk)
    assert r.status() == 0
    res[name] = dict(sums=[int(v) for v in table.host().reshape(-1)], bytes_received=st["bytes_received"], fb=fb, per=per)
comm.close()
json.dump(res, open(out, "w"))
"""


def _two_rank_job(b2d, device):
    """the jobs of the two-rank test on `device`: {name: (renderer, call(comm, on_chunk), n, frame bytes)} -- the plain call
    resolved by 2 to RGB and a level set of two WADs with different PLAYPALs resolved by 2 to planar RGB"""
    from rust_doom_b200 import _lib, poses as P, synthwad
    from tests.test_gpu_levels import _other_palette
    view = b2d.make_view(320, 200)
    a = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",))), 0)
    bwad = _other_palette(synthwad.build_iwad(7, ("E1M1",), cfg=synthwad.SynthConfig(gx=3, gy=3, origin=(-384, -384), light_fx=False)))
    b = b2d.Scene(b2d.Archive.from_bytes(bwad), 0)
    n = 37
    poses = P.random_poses(a, n, 5)
    plain = b2d.Renderer(a, view, device=device, max_batch=8)
    lv = (np.arange(n) % 3 == 1).astype(np.uint32)
    pools = [P.random_poses(s, n, 6) for s in (a, b)]
    ls_poses = np.array([pools[lv[i]][i] for i in range(n)], dtype=pools[0].dtype)
    tics = (np.arange(n) * 11).astype(np.uint32)
    ls = b2d.Renderer.from_levels([a, b], view, device=device, max_batch=8)
    return {
        "plain": (plain, lambda comm, fn: plain.render_sharded(comm, poses, 8, _lib.SHARD_RENDER_GATHER, fn, resolve=(2, "rgb")),
                  n, plain.resolve_frame_bytes(2, b2d.RESOLVE_RGB8)),
        "levels_states": (ls, lambda comm, fn: ls.render_sharded_levels_states(comm, ls_poses, lv, tics, None, 8,
                                                                               _lib.SHARD_RENDER_GATHER, fn, resolve=(2, "rgb_planar")),
                          n, ls.resolve_frame_bytes(2, b2d.RESOLVE_RGB8_PLANAR)),
    }


def test_two_ranks_resolve_to_the_world1_frames(b2d, tmp_path):
    """Two processes, two GPUs (skipped on a one-GPU box): every rank's checksum table of the gathered resolved frames equals
    the world-1 table of the same job, and each rank receives per x frame bytes"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from rust_doom_b200 import jobs
    comm = jobs.single_comm(0)
    want = {}
    for name, (r, call, n, fb) in _two_rank_job(b2d, 0).items():
        table = jobs.ChecksumTable(1, n, fb, torch.device("cuda", 0))
        call(comm, table.on_chunk)
        want[name] = table.host()[0].tolist()
    comm.close()
    uid = b2d.Comm.unique_id().hex()
    outs = [tmp_path / ("rank%d.json" % q) for q in range(2)]
    procs = [subprocess.Popen([sys.executable, "-c", _WORKER, uid, str(q), "2", str(outs[q])], cwd=ROOT,
                              env=dict(os.environ, PYTHONPATH=ROOT), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for q in range(2)]
    logs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), logs
    for q in range(2):
        got = json.loads(outs[q].read_text())
        for name, w1 in want.items():
            g = got[name]
            assert g["sums"][:len(w1)] == w1, (q, name)
            assert g["bytes_received"] == g["per"] * g["fb"], (q, name)
