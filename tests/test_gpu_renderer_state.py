"""-m gpu: the renderer's own state (b2d_renderer_set_time[_async], b2d_renderer_set_sector_moves[_async]).  The setters
only record a compact state on the host; the next plain batch of each worklist slot expands it into the slot's table set,
so a ticket is rastered at exactly the state it was walked at.  Frames are compared with the oracle's frame at that state:
its own scene with the moves applied (oracle/scene.py apply_moves), rendered at the tics."""
import numpy as np
import pytest

from tests.conftest import sample_poses
from tests.test_gpu_states import _assert_same, _level, _oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("raster_on_walk_stream", [True, False])
def test_walked_ticket_keeps_its_state(b2d, raster_on_walk_stream):
    """walk_device at rest and tic t0, then set_sector_moves_async (doors shut: the openings, and so the walk's solid
    columns, change) and set_time_async(t1), then raster_device of that ticket: its frames are the (rest, t0) frames; the
    next walked batch shows (doors shut, t1)."""
    import torch
    sc, oblob, level, dyn, doors = _level(b2d, mid_pct=20, thing_pct=30)
    assert doors
    shut = [(s, 0, f0 - c0) for (s, f0, c0) in doors]
    n, t0, t1 = 8, 40, 1234
    poses = sample_poses(b2d, sc, n, 81)
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=n)
    r.set_time(t0)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    outs = [torch.empty((n, 200, 320), dtype=torch.uint8, device="cuda") for _ in range(2)]
    s_walk = torch.cuda.Stream()
    s_raster = s_walk if raster_on_walk_stream else torch.cuda.Stream()
    torch.cuda.synchronize()
    ticket = r.walk_device(dp.data_ptr(), n, s_walk.cuda_stream)
    r.set_sector_moves(shut, stream=s_walk.cuda_stream)
    r.set_time_async(t1, s_walk.cuda_stream)
    r.raster_device(ticket, outs[0].data_ptr(), 0, s_raster.cuda_stream)
    ticket = r.walk_device(dp.data_ptr(), n, s_walk.cuda_stream)
    r.raster_device(ticket, outs[1].data_ptr(), 0, s_raster.cuda_stream)
    torch.cuda.synchronize()
    assert r.status() == 0
    before, after = outs[0].cpu().numpy(), outs[1].cpu().numpy()
    _assert_same(_oracle(oblob, 320, 200, poses, [t0] * n, [[]] * n), before, "ticket walked at rest, tic %d" % t0)
    _assert_same(_oracle(oblob, 320, 200, poses, [t1] * n, [shut] * n), after, "next batch, doors shut, tic %d" % t1)
    assert not np.array_equal(before, after), "the state change never changed a pixel"


def test_setters_enqueue_nothing_and_each_slot_expands_once(b2d):
    """The setters launch nothing; after a state change the next batch of each worklist slot costs walk + expansion +
    raster and later batches at the same state walk + raster; going back to a state a slot already holds costs no
    expansion."""
    import torch
    sc, oblob, level, dyn, doors = _level(b2d, mid_pct=10, thing_pct=10)
    shut = [(s, 0, f0 - c0) for (s, f0, c0) in doors]
    n = 4
    poses = sample_poses(b2d, sc, n, 82)
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=n)
    dp = torch.from_numpy(poses.view(np.int32).reshape(-1, 4).copy()).cuda()
    out = torch.empty((n, 200, 320), dtype=torch.uint8, device="cuda")

    def batch():
        l0 = r.launch_count
        r.render_device(dp.data_ptr(), n, out.data_ptr())
        return r.launch_count - l0

    assert [batch(), batch()] == [2, 2]                 # both slots hold tic 0 at rest from creation
    l0 = r.launch_count
    r.set_time(1000)
    r.set_sector_moves(shut)
    r.set_time_async(1000, 0)
    r.set_sector_moves(shut, stream=0)
    assert r.launch_count == l0
    assert [batch(), batch(), batch(), batch()] == [3, 3, 2, 2]
    r.set_time(2000)
    assert batch() == 3                                 # slot 0 -> (shut, 2000); slot 1 still holds (shut, 1000)
    r.set_time(1000)
    assert [batch(), batch()] == [2, 3]
    torch.cuda.synchronize()
    assert r.status() == 0
    _assert_same(_oracle(oblob, 320, 200, poses, [1000] * n, [shut] * n), out.cpu().numpy(), "(shut, 1000)")
