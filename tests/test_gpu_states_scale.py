"""-m gpu: per-frame states at the benchmark's batch sizes.  1000-frame 1080p batches pipelined the way bench.py and
tools/timeline_bench.py run them, with enough distinct states that b2d_state_sets_kernel's grid-stride loop takes more
than one pass; and worklist slots that hold plain and per-frame batches in turn.  Every frame is compared with the oracle
at its own state, and every expanded table set, read back, with oracle/scene.py tables_at."""
import numpy as np
import pytest

from tests.test_gpu_states import _assert_same, _level, _oracle, _states, check_state_sets
from tests.test_scene import EDGE_TICS, declare_doors

pytestmark = pytest.mark.gpu

N, WIDTH, HEIGHT = 1000, 1920, 1080


def _sms() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dev_poses(poses):
    import torch
    return torch.from_numpy(np.ascontiguousarray(poses).view(np.int32).reshape(-1, 4).copy()).cuda()


def _assert_oracle_chunked(oblob, poses, tics, moves, out, what, chunk=125):
    """frames of an (N, HEIGHT, WIDTH) device tensor against the oracle, `chunk` frames at a time (a 1080p batch is 2 GB)"""
    for c in range(0, len(poses), chunk):
        s = slice(c, c + chunk)
        _assert_same(_oracle(oblob, WIDTH, HEIGHT, poses[s], tics[s], moves[s]), out[s].cpu().numpy(), "%s, frames %d.." % (what, c))


def _records(blob) -> int:
    """records of one table set: textures + sectors + segs + sprites + mids"""
    from oracle import scene as S
    h = S.header(blob)
    return h[S.H_NTEX] + h[S.H_NSECTORS] + h[S.H_NSEGS] + h[S.H_NSPRITES] + h[S.H_NMIDS]


def test_states_pipelined_1000_frame_batches_rich_level(b2d):
    """The rich level with doors at 1920x1080, max_batch 1000: three batches, walk_device_states on a priority stream under
    raster_device on two alternating streams, a timeline of one tic per pose that continues across batches with the edge
    tics mixed in, moves drawn from a pool of six states; the third batch reuses slot 0's arena with new states.  After each
    walk the per-frame set indices and every table set are read back and compared with the oracle's tables; the batch's
    records outnumber the expansion grid's threads, so its grid-stride loop runs more than once."""
    import torch
    from oracle import scene as S, wad as W
    from rust_doom_b200 import poses as P, synthwad
    from tests.refcheck import moves as MV
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=30, thing_pct=40, anim=True))
    a = W.Archive(data)
    level = W.Level(a, 0)
    dyn, doors = declare_doors(level)
    oblob = S.compile_scene(a, W.TextureDirectory(a), 0, dynamic=dyn)
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0, dynamic=dyn)
    assert sc.blob == oblob and doors
    pool = [[], [(dyn[0][0], 0, 0)], [(s, 0, f0 - c0) for (s, f0, c0) in doors]] + \
           [MV.state(level, dyn, 500 + k, hole_free=False) for k in range(3)]
    rng = np.random.default_rng(17)
    base = P.flythrough_poses(sc, N, 2)
    batches = []
    for k in range(3):
        tics = np.arange(N, dtype=np.uint64) + N * k
        tics[50 + 97 * np.arange(len(EDGE_TICS))] = EDGE_TICS
        batches.append((np.roll(base, 333 * k), tics.astype(np.uint32), [pool[j] for j in rng.integers(0, len(pool), N)]))
    r = b2d.Renderer(sc, b2d.make_view(WIDTH, HEIGHT), max_batch=N)
    dps = [_dev_poses(p) for p, _, _ in batches]
    outs = [torch.empty((N, HEIGHT, WIDTH), dtype=torch.uint8, device="cuda") for _ in batches]
    s_walk, s_r = torch.cuda.Stream(priority=-1), (torch.cuda.Stream(), torch.cuda.Stream())
    threads = _sms() * 16 * 256                                     # launch_state_sets' grid cap
    torch.cuda.synchronize()

    def walk(k):
        _, tics, moves = batches[k]
        ticket = r.walk_device_states(dps[k].data_ptr(), tics, N, moves, s_walk.cuda_stream)
        slots, _ = check_state_sets(r, oblob, tics, moves, N)
        assert _records(oblob) * (int(slots.max()) + 1) > threads, "batch %d: one pass of the expansion grid" % k
        return ticket

    ticket = walk(0)
    for k in range(3):
        r.raster_device(ticket, outs[k].data_ptr(), 0, s_r[k % 2].cuda_stream)
        if k + 1 < 3:
            ticket = walk(k + 1)
    torch.cuda.synchronize()
    assert r.status() == 0
    for k, (poses, tics, moves) in enumerate(batches):
        _assert_oracle_chunked(oblob, poses, tics, moves, outs[k], "batch %d" % k)


def test_states_c2_1000_consecutive_tics(b2d):
    """The c2 level (light effects only: the compact state is the effect sectors' light bytes) at 1080p, one batch of 1000
    consecutive tics: one table set per distinct tables, each equal to the oracle's, and every frame equal to the
    oracle's."""
    import torch
    from oracle import scene as S, wad as W
    from rust_doom_b200 import poses as P, synthwad
    data = synthwad.build_iwad(1, ("E1M1",))
    a = W.Archive(data)
    oblob = S.compile_scene(a, W.TextureDirectory(a), 0)
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    assert sc.blob == oblob
    poses = P.flythrough_poses(sc, N, 2)
    tics = np.arange(N, dtype=np.uint32) + 5000
    moves = [[]] * N
    r = b2d.Renderer(sc, b2d.make_view(WIDTH, HEIGHT), max_batch=N)
    dp = _dev_poses(poses)
    out = torch.empty((N, HEIGHT, WIDTH), dtype=torch.uint8, device="cuda")
    r.render_device_states(dp.data_ptr(), tics, N, out.data_ptr())
    torch.cuda.synchronize()
    assert r.status() == 0
    slots, want = check_state_sets(r, oblob, tics, moves, N)
    assert int(slots.max()) + 1 == len(set(want)), "same set if and only if same tables"
    _assert_oracle_chunked(oblob, poses, tics, moves, out, "c2")


def test_slots_shared_by_plain_and_per_frame_batches(b2d):
    """Worklist slots that hold a plain batch and a per-frame batch in turn, at 320x200: a plain ticket walked at state A,
    the renderer moved to state B, a per-frame ticket walked, the per-frame ticket rastered before the plain one, then
    plain batches at B into both slots -- the second into the slot whose arena just held the per-frame sets, while its own
    table set still holds tic 0 at rest.  Each batch equals the oracle at its own state, each plain batch's table set equals
    the oracle's tables at A or B, and each batch launches what DESIGN.md §3 says: walk + raster, one expansion more when
    its slot's set holds another state, and one expansion for a per-frame batch."""
    import torch
    from oracle import scene as S
    from rust_doom_b200 import synthwad
    from tests.conftest import sample_poses
    sc, oblob, level, dyn, doors = _level(b2d, mid_pct=20, thing_pct=30)
    n = 8
    poses = sample_poses(b2d, sc, n, 91)
    tA, mA = 300, _states(level, dyn, doors, 3, 60)[2]
    tB, mB = (1 << 32) - 3, [(s, 0, f0 - c0) for (s, f0, c0) in doors]
    tics = np.arange(n, dtype=np.uint32) * 5 + 7
    moves = _states(level, dyn, doors, n, 70)
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=n)
    dp = _dev_poses(poses)
    outs = [torch.empty((n, 200, 320), dtype=torch.uint8, device="cuda") for _ in range(4)]
    s_walk, s_r = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    launches = []

    def counted(fn, *args):
        l0 = r.launch_count
        res = fn(*args)
        launches.append(r.launch_count - l0)
        return res

    r.set_time(tA)
    r.set_sector_moves(mA)
    t0 = counted(r.walk_device, dp.data_ptr(), n, s_walk.cuda_stream)               # slot 0, expanded from tic 0 to A
    assert r.state_tables(0) == S.tables_at(oblob, tA, mA)
    with pytest.raises(b2d.B2dError):
        r.state_tables(1)                                                           # a plain batch has one set
    r.set_time(tB)
    r.set_sector_moves(mB)
    t1 = counted(r.walk_device_states, dp.data_ptr(), tics, n, moves, s_walk.cuda_stream)     # slot 1's arena
    check_state_sets(r, oblob, tics, moves, n)
    counted(r.raster_device, t1, outs[1].data_ptr(), 0, s_r.cuda_stream)
    counted(r.raster_device, t0, outs[0].data_ptr(), 0, s_r.cuda_stream)
    t2 = counted(r.walk_device, dp.data_ptr(), n, s_walk.cuda_stream)               # slot 0: A -> B
    assert r.state_tables(0) == S.tables_at(oblob, tB, mB)
    counted(r.raster_device, t2, outs[2].data_ptr(), 0, s_r.cuda_stream)
    t3 = counted(r.walk_device, dp.data_ptr(), n, s_walk.cuda_stream)               # slot 1: its own set, tic 0 -> B
    assert r.state_tables(0) == S.tables_at(oblob, tB, mB)
    counted(r.raster_device, t3, outs[3].data_ptr(), 0, s_r.cuda_stream)
    t4 = counted(r.walk_device, dp.data_ptr(), n, s_walk.cuda_stream)               # slot 0 already holds B
    counted(r.raster_device, t4, outs[2].data_ptr(), 0, s_r.cuda_stream)
    torch.cuda.synchronize()
    assert r.status() == 0
    assert launches == [2, 2, 1, 1, 2, 1, 2, 1, 1, 1], launches
    at_a = _oracle(oblob, 320, 200, poses, [tA] * n, [mA] * n)
    at_b = _oracle(oblob, 320, 200, poses, [tB] * n, [mB] * n)
    _assert_same(at_a, outs[0].cpu().numpy(), "plain ticket walked at A, rastered after the per-frame one")
    _assert_same(_oracle(oblob, 320, 200, poses, tics, moves), outs[1].cpu().numpy(), "per-frame ticket")
    _assert_same(at_b, outs[2].cpu().numpy(), "plain batch at B in slot 0")
    _assert_same(at_b, outs[3].cpu().numpy(), "plain batch at B in the slot that held per-frame sets")
    assert not np.array_equal(at_a, at_b)
    plain = b2d.Scene(b2d.Archive.from_bytes(synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(light_fx=False))), 0)
    rp = b2d.Renderer(plain, b2d.make_view(320, 200), max_batch=n)
    rp.render(sample_poses(b2d, plain, n, 92))
    with pytest.raises(b2d.B2dError):
        rp.state_tables(0)                                          # no table sets on a scene without state
