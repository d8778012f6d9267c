"""-m gpu: the cross-stream ordering of the device-resident API, observed directly.  A test holds one of its own streams
with a bounded sleep kernel (about 200 ms, orders of magnitude longer than the 320x200 batches of six frames here), enqueues
library calls behind and beside it, and watches events:

  must_wait(down, hold)     the work behind `down` may not finish before the hold: an edge the library must have;
  must_overlap(down, hold)  the work behind `down` finishes while the hold is pending: an edge the library must not have;
  pending(hold)             the call returned while the hold was pending: it did not block the host.

The calls that do block the host are the ones include/b2d.h names: the rewrite of a worklist slot's pinned staging waits
for the copy that read it two batches earlier, and the palette staging of b2d_palette_lut_levels_device waits for the
previous call (its growth for the previous call's kernel).  Every scenario ends with every batch's frames equal to the
oracle's at that batch's own poses, levels and states, a clear status word and the launch counts of DESIGN.md section 3.
Holds run on non-default streams only (the legacy default stream would serialise everything)."""
import time

import numpy as np
import pytest

from tests.conftest import sample_poses
from tests.test_gpu_levels import C2, RICH, SMALL, _assert_same, _mix, _palette, levels  # noqa: F401
from tests.test_gpu_levels_states import _oracle_states, _per_frame, _rich_states

pytestmark = pytest.mark.gpu

W, H = 320, 200
N = 6                       # frames per batch
MAX_BATCH = 8
HOLD_MS = 200
SET = (RICH, C2, SMALL)     # level 0 has masked middles, sprites, time-dependent content and dynamic sectors
PLAIN_SET = (C2, SMALL)     # no masked content: rasters do not share a masked-entry arena
# the split walks; "restate" is walk_device after set_time / set_sector_moves (the slot's table set is re-expanded)
WALKS = ("plain", "restate", "states", "levels", "levels_states")
CALLS = ("plain", "states", "levels", "levels_states")
# launches per walked and rastered batch once both worklist slots hold the renderer's state (DESIGN.md section 3)
LAUNCHES = {"plain": 2, "restate": 3, "states": 3, "levels": 2, "levels_states": 3}


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
    per_ms = cycles / a.elapsed_time(b)
    print("\nhold calibration: %.0f cycles per ms (%s)" % (per_ms, torch.cuda.get_device_name()))
    return Clock(per_ms)


def mark(stream):
    import torch
    ev = torch.cuda.Event()
    ev.record(stream)
    return ev


def pending(hold, what):
    assert not hold.query(), "%s: the call blocked until the hold ended" % what


def must_wait(down, hold, what):
    """`down` must not complete before `hold`.  The downstream event is queried before the hold in each round, so a
    downstream that completes right after the hold is never taken for one that completed first."""
    assert not hold.query(), "%s: the hold ended before the probe started" % what
    while True:
        d = down.query()
        if hold.query():
            break
        assert not d, "%s: finished while the hold it must wait for was pending" % what
        time.sleep(0.0005)
    down.synchronize()


def must_overlap(down, hold, what):
    """`down` must complete while `hold` is still pending"""
    down.synchronize()
    assert not hold.query(), "%s: waited for a hold it does not depend on" % what


class Batch:
    """N frames: poses on the device, per-frame levels (indices into the renderer's set, and into `levels` for the
    oracle), tics and move lists, and the oracle's frames"""

    def __init__(self, b2d, levels, lset, kind, seed, own=(0, ()), oracle=True):
        """`own`: the renderer's (time, level-0 moves) that the plain and levels kinds render at"""
        import torch
        sub = [levels[k] for k in lset]
        if kind.startswith("levels"):
            self.poses, self.lv_set = _mix(b2d, sub, N // len(lset), seed)
        else:
            self.poses, self.lv_set = sample_poses(b2d, sub[0]["scene"], N, seed), np.zeros(N, np.uint32)
        self.lv = np.asarray(lset, np.uint32)[self.lv_set]
        if kind in ("states", "levels_states"):
            self.tics, self.moves = _per_frame(levels, self.lv, seed)
        else:
            self.tics = np.full(N, own[0], np.uint32)
            self.moves = [list(own[1]) if k == lset[0] else [] for k in self.lv]
        self.own = own
        self.dp = torch.from_numpy(np.ascontiguousarray(self.poses).view(np.int32).reshape(-1, 4).copy()).cuda()
        self.out = torch.full((N, H, W), 0x5A, dtype=torch.uint8, device="cuda")
        self.rgba = torch.zeros((N, H, W), dtype=torch.int32, device="cuda")
        self.want = _oracle_states(levels, W, H, self.poses, self.lv, self.tics, self.moves) if oracle else None
        torch.cuda.synchronize()                        # the inputs are on the device before any call reads them


def _batches(b2d, levels, lset, kind, count, seed):
    """`count` batches of one kind, each with its own poses and, for "restate", its own renderer state; consecutive batches'
    oracle frames differ, so a batch rendered from another batch's worklist, tables or staging changes pixels"""
    owns = [(0, ())] * count
    if kind == "restate":
        rich = _rich_states(levels, count + 1, seed)
        owns = [(1000 + 37 * k, tuple(rich[k + 1])) for k in range(count)]
    out = [Batch(b2d, levels, lset, kind, seed + 17 * k, owns[k]) for k in range(count)]
    for a, b in zip(out, out[1:]):
        assert not np.array_equal(a.want, b.want)
    return out


def _walk(r, kind, b, stream):
    s, dp = stream.cuda_stream, b.dp.data_ptr()
    if kind in ("plain", "restate"):
        if kind == "restate":
            r.set_time(b.own[0])
            r.set_sector_moves(b.own[1])
        return r.walk_device(dp, N, s)
    if kind == "states":
        return r.walk_device_states(dp, b.tics, N, b.moves, s)
    if kind == "levels":
        return r.walk_device_levels(dp, b.lv_set, N, s)
    return r.walk_device_levels_states(dp, b.lv_set, b.tics, N, b.moves, s)


def _raster(r, t, b, stream):
    r.raster_device(t, b.out.data_ptr(), b.rgba.data_ptr(), stream.cuda_stream)


def _render(r, kind, b, stream):
    """the one-call device entry point of `kind`, one batch"""
    s, dp, o, c = stream.cuda_stream, b.dp.data_ptr(), b.out.data_ptr(), b.rgba.data_ptr()
    if kind == "plain":
        r.render_device(dp, N, o, c, s)
    elif kind == "states":
        r.render_device_states(dp, b.tics, N, o, c, b.moves, s)
    elif kind == "levels":
        r.render_device_levels(dp, b.lv_set, N, o, c, s)
    else:
        r.render_device_levels_states(dp, b.lv_set, b.tics, N, o, c, b.moves, s)


def _rig(b2d, levels, lset):
    """A renderer over the levels `lset`, four streams, and one batch of every call kind walked and rastered through both
    worklist slots: first-use allocations and the growth of a slot's sections (which may free buffers, and cudaFree
    synchronises the device) happen here, not under a probe; both slots' table sets then hold the renderer's state."""
    import torch
    r = b2d.Renderer.from_levels([levels[k]["scene"] for k in lset], b2d.make_view(W, H), max_batch=MAX_BATCH)
    streams = [torch.cuda.Stream() for _ in range(4)]
    for kind in CALLS:
        b = Batch(b2d, levels, lset, kind, 7000, oracle=False)
        for i in range(2):
            _raster(r, _walk(r, kind, b, streams[0]), b, streams[1 + i])
            _render(r, kind, b, streams[i])
    d = torch.zeros(N * W * H, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    r.palette_lut_levels_device(d.data_ptr(), [0] * N, N, b.rgba.data_ptr(), streams[0].cuda_stream)
    torch.cuda.synchronize()
    assert r.status() == 0
    return r, streams


def _finish(r, lset, levels, batches, launches):
    """every batch's index and RGBA frames equal the oracle's, a clear status word, the expected launch count"""
    import torch
    torch.cuda.synchronize()
    assert r.status() == 0
    pals = [_palette(levels[k]["scene"]) for k in lset]
    for i, b in enumerate(batches):
        idx = b.out.cpu().numpy()
        _assert_same(b.want, idx, "batch %d" % i)
        rgba = b.rgba.cpu().numpy().view(np.uint32)
        for f in range(N):
            assert np.array_equal(rgba[f], pals[b.lv_set[f]][idx[f]]), "batch %d frame %d: RGBA is not its level's palette" % (i, f)
    assert r.launch_count == launches


# ---- a: the raster of a ticket waits for its walk ----------------------------------------------------------------------
@pytest.mark.parametrize("kind", WALKS)
def test_raster_waits_for_its_walk(b2d, levels, clock, kind):
    r, (w, s, _, _) = _rig(b2d, levels, SET)
    (b,) = _batches(b2d, levels, SET, kind, 1, 7100)
    l0 = r.launch_count
    hold = clock.hold(w)
    t = _walk(r, kind, b, w)
    pending(hold, "walk")
    _raster(r, t, b, s)
    pending(hold, "raster")
    must_wait(mark(s), hold, "raster_device on another stream than its walk")
    _finish(r, SET, levels, [b], l0 + LAUNCHES[kind])


# ---- b: a walk into a worklist slot waits for the slot's previous raster, and only for that ---------------------------
@pytest.mark.parametrize("kind", WALKS)
def test_slot_reuse_waits_for_the_slots_raster(b2d, levels, clock, kind):
    r, (w, s, s2, _) = _rig(b2d, levels, SET)
    bs = _batches(b2d, levels, SET, kind, 3, 7200)
    l0 = r.launch_count
    t0 = _walk(r, kind, bs[0], w)
    w.synchronize()                                     # the hold keeps raster k only
    hold = clock.hold(s)
    _raster(r, t0, bs[0], s)
    pending(hold, "raster k")
    t1 = _walk(r, kind, bs[1], w)
    pending(hold, "walk k+1")
    walk1 = mark(w)
    _raster(r, t1, bs[1], s2)
    pending(hold, "raster k+1")
    t2 = _walk(r, kind, bs[2], w)
    pending(hold, "walk k+2")
    walk2 = mark(w)
    _raster(r, t2, bs[2], s)
    must_overlap(walk1, hold, "walk k+1 into the other slot (the background walk runs under raster k)")
    must_wait(walk2, hold, "walk k+2 into the slot raster k reads")
    _finish(r, SET, levels, bs, l0 + 3 * LAUNCHES[kind])


# ---- c: a slot's pinned staging is rewritten after the copy that read it two batches earlier --------------------------
@pytest.mark.parametrize("kind", WALKS)
def test_staging_waits_for_the_copy_two_batches_back(b2d, levels, clock, kind):
    r, (w, s, s2, _) = _rig(b2d, levels, SET)
    bs = _batches(b2d, levels, SET, kind, 3, 7300)
    l0 = r.launch_count
    hold = clock.hold(w)
    t0 = _walk(r, kind, bs[0], w)
    pending(hold, "walk k")
    _raster(r, t0, bs[0], s)
    t1 = _walk(r, kind, bs[1], w)
    pending(hold, "walk k+1")
    _raster(r, t1, bs[1], s2)
    pending(hold, "raster k+1")
    t2 = _walk(r, kind, bs[2], w)
    if kind == "plain":
        pending(hold, "walk k+2 at an unchanged state (stages nothing)")
    else:
        assert hold.query(), "walk k+2 rewrote the staging walk k's held copy reads"
    _raster(r, t2, bs[2], s)
    _finish(r, SET, levels, bs, l0 + 3 * LAUNCHES[kind])


# ---- d: rasters with masked content share one arena; rasters without do not wait for each other -----------------------
@pytest.mark.parametrize("lset", [SET, PLAIN_SET], ids=["masked", "unmasked"])
def test_masked_rasters_run_one_after_the_other(b2d, levels, clock, lset):
    r, (w, a, b, _) = _rig(b2d, levels, lset)
    bs = _batches(b2d, levels, lset, "levels", 2, 7400)
    l0 = r.launch_count
    t = [_walk(r, "levels", x, w) for x in bs]
    w.synchronize()
    hold = clock.hold(a)
    _raster(r, t[0], bs[0], a)
    pending(hold, "raster k")
    _raster(r, t[1], bs[1], b)
    pending(hold, "raster k+1")
    if lset == SET:
        must_wait(mark(b), hold, "raster k+1 behind raster k (one masked-entry arena)")
    else:
        must_overlap(mark(b), hold, "rasters without masked content on two streams")
    _finish(r, lset, levels, bs, l0 + 2 * LAUNCHES["levels"])


# ---- e: the setters record host state and enqueue nothing --------------------------------------------------------------
def test_setters_enqueue_nothing(b2d, levels, clock):
    r, (w, s, s2, _) = _rig(b2d, levels, SET)
    rich = _rich_states(levels, 4, 7500)
    new = (4321, tuple(rich[3]))
    b0 = Batch(b2d, levels, SET, "plain", 7501)
    b1 = Batch(b2d, levels, SET, "levels", 7502, own=new)
    l0 = r.launch_count
    t0 = _walk(r, "plain", b0, w)
    w.synchronize()
    hold = clock.hold(s)
    r.set_time_async(new[0], s.cuda_stream)
    pending(hold, "set_time_async")
    r.set_sector_moves(rich[1], stream=s.cuda_stream)
    pending(hold, "set_sector_moves(stream=)")
    r.set_level_sector_moves(0, new[1])
    pending(hold, "set_level_sector_moves")
    assert r.launch_count == l0 + 1, "a setter launched work"
    _raster(r, t0, b0, s)                               # the held ticket: at the state it was walked at
    _raster(r, _walk(r, "levels", b1, w), b1, s2)       # the next batch: at the new state (every level re-expanded)
    pending(hold, "the next batch")
    _finish(r, SET, levels, [b0, b1], l0 + 2 + 2 + 2)   # RICH and C2 are timed: one expansion each for b1's slot


# ---- f: the one-call device entry points on two streams -------------------------------------------------------------
@pytest.mark.parametrize("kind", CALLS)
def test_one_call_renders_on_two_streams(b2d, levels, clock, kind):
    """On levels without masked content, call 2 (the other slot, another stream) overlaps the held call 1; call 3 lands in
    call 1's slot and waits for its raster.  A call that writes pinned staging waits on the host for the held copy of call
    1 two batches earlier instead, so for those call 3 returns after the hold."""
    r, (s1, s2, _, _) = _rig(b2d, levels, PLAIN_SET)
    bs = _batches(b2d, levels, PLAIN_SET, kind, 3, 7600)
    l0 = r.launch_count
    hold = clock.hold(s1)
    _render(r, kind, bs[0], s1)
    pending(hold, "call 1")
    _render(r, kind, bs[1], s2)
    pending(hold, "call 2")
    must_overlap(mark(s2), hold, "call 2 into the other slot on another stream")
    _render(r, kind, bs[2], s2)
    if kind == "plain":
        pending(hold, "call 3")
        must_wait(mark(s2), hold, "call 3 into the slot of call 1")
    else:
        assert hold.query(), "call 3 rewrote the staging call 1's held copy reads"
    _finish(r, PLAIN_SET, levels, bs, l0 + 3 * LAUNCHES[kind])


# ---- g: the per-level palette staging -----------------------------------------------------------------------------------
def test_palette_staging_waits_and_grows(b2d, levels, clock):
    """Call 2 rewrites the one-deep staging only after call 1's held copy; call 3 with more frames than the staging holds
    (1024 frames at first) replaces it only after call 2's held kernel; every frame goes through its own level's palette.
    K3 on two streams has no edge between them."""
    import torch
    scenes = [levels[k]["scene"] for k in PLAIN_SET]
    pals = [_palette(s) for s in scenes]
    w, h = 64, 40
    npix = w * h
    r = b2d.Renderer.from_levels(scenes, b2d.make_view(w, h), max_batch=1)
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    idx = torch.randint(0, 256, (1025 * npix,), dtype=torch.uint8, device="cuda")
    outs = [torch.zeros(1025 * npix, dtype=torch.int32, device="cuda") for _ in range(3)]
    rng = np.random.default_rng(7700)
    lv1 = rng.integers(0, 2, 8).astype(np.uint32)
    lvs = [lv1, 1 - lv1, rng.integers(0, 2, 1025).astype(np.uint32)]
    torch.cuda.synchronize()
    r.palette_lut_levels_device(idx.data_ptr(), lv1, 8, outs[0].data_ptr(), a.cuda_stream)     # the first staging
    torch.cuda.synchronize()
    l0 = r.launch_count
    hold_a = clock.hold(a)
    r.palette_lut_levels_device(idx.data_ptr(), lvs[0], 8, outs[0].data_ptr(), a.cuda_stream)
    pending(hold_a, "call 1")
    hold_b = clock.hold(b)
    r.palette_lut_levels_device(idx.data_ptr(), lvs[1], 8, outs[1].data_ptr(), b.cuda_stream)
    assert hold_a.query(), "call 2 rewrote the staging call 1's held copy reads"
    r.palette_lut_levels_device(idx.data_ptr(), lvs[2], 1025, outs[2].data_ptr(), b.cuda_stream)
    assert hold_b.query(), "call 3 replaced the staging before call 2's held kernel ran"
    torch.cuda.synchronize()
    assert r.launch_count == l0 + 3
    px = idx.cpu().numpy().reshape(1025, npix)
    for k, lv in enumerate(lvs):
        got = outs[k].cpu().numpy().view(np.uint32).reshape(1025, npix)
        for f in range(len(lv)):
            assert np.array_equal(got[f], pals[lv[f]][px[f]]), "call %d frame %d: not its level's palette" % (k + 1, f)
    k3 = [torch.zeros(8 * npix, dtype=torch.int32, device="cuda") for _ in range(2)]
    # K3's first launch in the process loads its module (CUDA lazy loading): made on a held stream, it held the K3 launch
    # on the other stream too.  So K3 runs once on each stream before the probe, like every call of the other scenarios.
    for st in (a, b):
        r.palette_lut_device(idx.data_ptr(), k3[0].data_ptr(), 8 * npix, st.cuda_stream)
    torch.cuda.synchronize()
    l0 = r.launch_count
    hold = clock.hold(a)
    r.palette_lut_device(idx.data_ptr(), k3[0].data_ptr(), 8 * npix, a.cuda_stream)
    pending(hold, "K3 on the held stream")
    r.palette_lut_device(idx.data_ptr(), k3[1].data_ptr(), 8 * npix, b.cuda_stream)
    pending(hold, "K3 on the other stream")
    must_overlap(mark(b), hold, "K3 on another stream")
    torch.cuda.synchronize()
    assert r.launch_count == l0 + 2
    want = pals[0][px[:8].reshape(-1)]
    assert np.array_equal(k3[0].cpu().numpy().view(np.uint32), want)
    assert np.array_equal(k3[1].cpu().numpy().view(np.uint32), want)


# ---- h: the sharded loop reuses a chunk buffer only after the consumer has read it ------------------------------------
@pytest.mark.parametrize("call", ["render_sharded", "render_sharded_levels_states"])
def test_sharded_chunk_buffers_wait_for_the_consumer(b2d, levels, clock, call):
    """World 1, five chunks of four frames; the callback holds the consumer stream it is handed before the checksum of
    each chunk, so the render of chunk k+2 into chunk k's buffer would change the checksums if it did not wait."""
    import torch
    from rust_doom_b200 import _lib, jobs
    r, _ = _rig(b2d, levels, SET)
    n, chunk = 20, 4
    kind = "plain" if call == "render_sharded" else "levels_states"
    sub = [Batch(b2d, levels, SET, kind, 7800 + 17 * k) for k in range(4)]          # 24 frames, the first 20 used
    poses = np.concatenate([x.poses for x in sub])[:n]
    want = np.concatenate([x.want for x in sub])[:n]
    comm = jobs.single_comm(0)
    table = jobs.ChecksumTable(1, n, W * H, torch.device("cuda", 0))
    seen = []

    def on_chunk(k, first, cnt, ptr, ranks, stream):
        seen.append(k)
        clock.sleep(torch.cuda.ExternalStream(stream), 50)
        table.on_chunk(k, first, cnt, ptr, ranks, stream)
    torch.cuda.synchronize()
    l0 = r.launch_count
    if call == "render_sharded":
        st = r.render_sharded(comm, poses, chunk, _lib.SHARD_RENDER_GATHER, on_chunk)
    else:
        lv = np.concatenate([x.lv_set for x in sub])[:n]
        tics = np.concatenate([x.tics for x in sub])[:n]
        moves = sum((x.moves for x in sub), [])[:n]
        st = r.render_sharded_levels_states(comm, poses, lv, tics, moves, chunk, _lib.SHARD_RENDER_GATHER, on_chunk)
    torch.cuda.synchronize()
    assert st["chunks"] == 5 and seen == list(range(5))
    assert table.host()[0].tolist() == [b2d.frame_checksum(want[i]) for i in range(n)]
    assert r.status() == 0
    assert r.launch_count == l0 + 5 * LAUNCHES[kind]
    comm.close()


# ---- the one-call renders refuse a walked, unrastered ticket up front ---------------------------------------------------
def test_one_call_renders_refuse_a_pending_ticket(b2d, levels):
    """With a ticket walked and not rastered, every one-call render that needs its slot -- host and device, two batches,
    and the sharded calls at world 1 with several chunks -- is B2D_ERR_INVALID_ARG with no launch and its output untouched;
    a single batch into the free slot renders exactly; the pending ticket then rasters to the oracle's frames, and the
    renderer's time is what it was (render_timed refused before setting it)."""
    import torch
    from rust_doom_b200 import B2dError, _frame_states, _lib, _levels_array, jobs
    L = _lib.load()
    r, (w, s, _, _) = _rig(b2d, levels, SET)
    comm = jobs.single_comm(0)
    held, one = _batches(b2d, levels, SET, "levels_states", 2, 7900)
    big = [Batch(b2d, levels, SET, "levels_states", 7910 + k) for k in range(2)]       # 12 frames: two batches
    n = 2 * N
    poses = np.ascontiguousarray(np.concatenate([x.poses for x in big]))
    lv = _levels_array(np.concatenate([x.lv_set for x in big]), n)
    tics = np.ascontiguousarray(np.concatenate([x.tics for x in big]), np.uint32)
    moves = sum((x.moves for x in big), [])
    states, arr, nm = _frame_states(tics, moves, n)
    plain_states, plain_arr, plain_nm = _frame_states(tics, None, n)
    dp = torch.cat([x.dp for x in big])
    d_out = torch.full((n, H, W), 0x5A, dtype=torch.uint8, device="cuda")
    h_out = np.full((n, H, W), 0x5A, np.uint8)
    h_rgba = np.full((n, H, W), 0x5A5A5A5A, np.uint32)
    chunks = []
    torch.cuda.synchronize()

    t = _walk(r, "levels_states", held, w)
    l0 = r.launch_count
    host = {
        "render": lambda: L.b2d_render(r._h, poses.ctypes.data, n, h_out.ctypes.data, h_rgba.ctypes.data),
        "render_timed": lambda: L.b2d_render_timed(r._h, poses.ctypes.data, tics.ctypes.data, n, h_out.ctypes.data, None),
        "render_states": lambda: L.b2d_render_states(r._h, poses.ctypes.data, plain_states, n, plain_arr, plain_nm,
                                                     h_out.ctypes.data, None),
        "render_levels": lambda: L.b2d_render_levels(r._h, poses.ctypes.data, lv.ctypes.data, n, h_out.ctypes.data, None),
        "render_levels_states": lambda: L.b2d_render_levels_states(r._h, poses.ctypes.data, lv.ctypes.data, states, n, arr, nm,
                                                                   h_out.ctypes.data, h_rgba.ctypes.data),
    }
    for name, call in host.items():
        assert call() == b2d.ERR_INVALID_ARG, name
        assert r.launch_count == l0, name
    o = d_out.data_ptr()
    device = {
        "render_device_timed": lambda: r.render_device_timed(dp.data_ptr(), tics, n, o, 0, s.cuda_stream),
        "render_device_states": lambda: r.render_device_states(dp.data_ptr(), tics, n, o, 0, None, s.cuda_stream),
        "render_device_levels": lambda: r.render_device_levels(dp.data_ptr(), lv, n, o, 0, s.cuda_stream),
        "render_device_levels_states": lambda: r.render_device_levels_states(dp.data_ptr(), lv, tics, n, o, 0, moves,
                                                                             s.cuda_stream),
        "render_sharded": lambda: r.render_sharded(comm, poses, N, _lib.SHARD_RENDER_GATHER, lambda *a: chunks.append(a)),
        "render_sharded_levels_states": lambda: r.render_sharded_levels_states(comm, poses, lv, tics, moves, N,
                                                                               _lib.SHARD_RENDER_GATHER,
                                                                               lambda *a: chunks.append(a)),
    }
    for name, call in device.items():
        with pytest.raises(B2dError) as e:
            call()
        assert e.value.code == b2d.ERR_INVALID_ARG and r.launch_count == l0, name
    torch.cuda.synchronize()
    assert not chunks, "a refused sharded call handed out a chunk"
    assert (d_out == 0x5A).all().item() and (h_out == 0x5A).all() and (h_rgba == 0x5A5A5A5A).all(), "a refused call wrote frames"

    idx, rgba = r.render_levels_states(one.poses, one.lv_set, one.tics, one.moves, rgba=True)    # one batch: the free slot
    _assert_same(one.want, idx, "a single batch into the free slot")
    pals = [_palette(levels[k]["scene"]) for k in SET]
    assert all(np.array_equal(rgba[f], pals[one.lv_set[f]][idx[f]]) for f in range(N))
    l1 = r.launch_count
    with pytest.raises(B2dError) as e:                  # the next slot is the pending ticket's: one batch is refused too
        r.render_device(one.dp.data_ptr(), N, o, 0, s.cuda_stream)
    assert e.value.code == b2d.ERR_INVALID_ARG and r.launch_count == l1
    _raster(r, t, held, s)
    _finish(r, SET, levels, [held], l1 + 1)
    assert r.status() == 0
    from tests.test_gpu_levels import _oracle
    own = sample_poses(b2d, levels[SET[0]]["scene"], n, 7920)
    _assert_same(_oracle(levels, W, H, own, np.full(n, SET[0])), r.render(own), "after the refusals, at the renderer's own time")
    comm.close()
