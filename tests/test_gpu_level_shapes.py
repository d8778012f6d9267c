"""-m gpu: the node-builder-shaped levels of tests/test_level_shapes.py through the kernels, bit for bit against the
oracle -- subsectors of 31 to 146 segs (the walk's seg loop over several 32-wide chunks, with sprites in one of them), a
16384-unit seg and subsectors of 128 collinear segs, and BSP trees whose walk needs exactly the 128 stack entries the
kernel has, or one more (which must be reported, never drawn wrong).  tests/test_level_shapes.py shows on the CPU that
every case here is valid."""
import numpy as np
import pytest

from oracle import render
from tests.conftest import oracle_blob, sample_poses
from tests.test_gpu_scale import _assert_same, _assert_worklists, _background_walk, _dev_poses, _sms
from tests.test_level_shapes import STACK_DEPTH, THINGS_IN, deep_levels, levels, rotunda_level, stack_need

pytestmark = pytest.mark.gpu

RENDER_SIZES = ((320, 200), (333, 187), (1920, 1080), (3840, 2160))
AT_LIMIT = ("rotundas", "hall", "deep128")


def _scene(b2d, lv, dynamic=()):
    return b2d.Scene(b2d.Archive.from_bytes(lv.wad), 0, dynamic=dynamic)


@pytest.mark.parametrize("size", RENDER_SIZES, ids=["%dx%d" % s for s in RENDER_SIZES])
@pytest.mark.parametrize("name", AT_LIMIT)
def test_gpu_shape_level_render_matches_oracle(b2d, name, size):
    """Renderer.render, index and RGBA: 333 columns take the generic-width raster, 1920 and 3840 the specialised ones."""
    lv = levels()[name]
    w, h = size
    poses = lv.pose_array()
    if w == 3840:
        poses = poses[::3]
    ofb, orgba = render.render(lv.blob, render.make_view(w, h), poses, rgba=True, threads=8)
    r = b2d.Renderer(_scene(b2d, lv), b2d.make_view(w, h), max_batch=len(poses))
    idx, rgba = r.render(poses, rgba=True)
    assert r.status() == 0
    _assert_same(ofb, idx, "%s %dx%d" % (name, w, h))
    assert np.array_equal(orgba, rgba), "%s %dx%d: RGBA" % (name, w, h)


@pytest.mark.parametrize("name", AT_LIMIT)
def test_gpu_shape_level_device_paths_match_oracle(b2d, hostcheck, name):
    """render_device into a poisoned buffer (the frame past the batch stays poisoned), worklists vs hostcheck (counts and
    ids in order), and the persistent walk grid (walk_device + raster_device, n > SMs: CTAs walk several frames)."""
    import torch
    lv = levels()[name]
    sc = _scene(b2d, lv)
    view, oview = b2d.make_view(320, 200), render.make_view(320, 200)
    poses = lv.pose_array()
    n = len(poses)
    ofb = render.render(lv.blob, oview, poses, threads=8)
    r = b2d.Renderer(sc, view, max_batch=n)
    dp = _dev_poses(poses)
    out = torch.full((n + 1, 200, 320), 0xA5, dtype=torch.uint8, device="cuda")
    r.render_device(dp.data_ptr(), n, out.data_ptr())
    torch.cuda.synchronize()
    assert r.status() == 0
    _assert_same(ofb, out[:n].cpu().numpy(), "%s render_device" % name)
    assert bool((out[n] == 0xA5).all()), "render_device wrote past the batch"
    _assert_worklists(r, hostcheck, lv.blob, view, poses, "%s foreground" % name)
    big = 2 * _sms() + 5
    more = np.resize(poses, big)
    rb = b2d.Renderer(sc, view, max_batch=big)
    _, bout = _background_walk(rb, more, 320, 200)
    assert rb.status() == 0
    _assert_worklists(rb, hostcheck, lv.blob, view, more, "%s background" % name)
    _assert_same(np.resize(ofb, (big, 200, 320)), bout.cpu().numpy(), "%s background walk n=%d" % (name, big))


def test_gpu_rotunda_floor_states_match_oracle(b2d):
    """render_states with the 65-seg rotunda's floor declared dynamic (its sprites ride on it): the floor at both ends of
    its range and at rest, with level times, for the poses in and around that rotunda."""
    from oracle import scene as S, wad as W
    from tests.test_gpu_states import _oracle
    lv = rotunda_level()
    sec, _ = lv.facts["rooms"][THINGS_IN]
    f0, c0 = int(lv.map.sectors[sec].floor), int(lv.map.sectors[sec].ceil)
    dyn = [(sec, f0 - 24, f0 + 24, c0, c0)]
    a = W.Archive(lv.wad)
    blob = S.compile_scene(a, W.TextureDirectory(a), 0, dynamic=dyn)
    sc = _scene(b2d, lv, dyn)
    assert sc.blob == blob
    which = [i for i, p in enumerate(lv.poses) if "rotunda %d " % THINGS_IN in p[4]]
    poses = np.concatenate([lv.pose_array(which)] * 3)
    n = len(poses)
    pool = [[(sec, -24, 0)], [(sec, 24, 0)], []]
    moves = [pool[i % 3] for i in range(n)]
    tics = np.array([(37 * i + 11) % 2000 for i in range(n)], np.uint32)
    r = b2d.Renderer(sc, b2d.make_view(320, 200), max_batch=n)
    got = r.render_states(poses, tics, moves)
    assert r.status() == 0
    _assert_same(_oracle(blob, 320, 200, poses, tics, moves), got, "rotunda floor states")


def test_gpu_shape_levels_in_one_level_set(b2d):
    """Renderer.from_levels over the shape levels and the generated c2 level, frames alternating levels: the level-set
    walk reloads scenes of very different sizes from one frame to the next."""
    from rust_doom_b200 import synthwad
    names = ("rotundas", "hall", "deep128")
    c2 = synthwad.build_iwad(1, ("E1M1",))
    scenes = [_scene(b2d, levels()[k]) for k in names] + [b2d.Scene(b2d.Archive.from_bytes(c2), 0)]
    blobs = [levels()[k].blob for k in names] + [oracle_blob(c2)]
    pose_lists = [levels()[k].pose_array() for k in names] + [sample_poses(b2d, scenes[3], 12, 900)]
    n = 48
    lv = np.array([i % 4 for i in range(n)], np.int32)
    poses = np.concatenate([pose_lists[lv[i]][(i // 4) % len(pose_lists[lv[i]]):][:1] for i in range(n)])
    r = b2d.Renderer.from_levels(scenes, b2d.make_view(320, 200), max_batch=n)
    got = r.render_levels(poses, lv)
    assert r.status() == 0
    oview = render.make_view(320, 200)
    want = np.concatenate([render.render(blobs[lv[i]], oview, poses[i:i + 1]) for i in range(n)])
    _assert_same(want, got, "level set")


# ---- the BSP stack at its limit and one past it --------------------------------------------------------------------
@pytest.mark.parametrize("size", ((320, 200), (1920, 1080)), ids=["320x200", "1920x1080"])
def test_gpu_bsp_stack_limit(b2d, size):
    """The corridor whose worst pose needs exactly 128 entries renders every pose exactly with status 0.  One step deeper:
    the poses that still need at most 128 render exactly with status 0; a pose that needs 129 makes render raise the
    stack-overflow error, and the device paths (per-frame and persistent walk grids) set status bit 1 -- never bit 4 (a
    valid deep tree must not exhaust the termination budget), and never status 0."""
    import torch
    w, h = size
    view, oview = b2d.make_view(w, h), render.make_view(w, h)
    at, over = deep_levels()
    poses = at.pose_array()
    assert max(stack_need(at.blob, oview, p) for p in poses) == STACK_DEPTH
    r = b2d.Renderer(_scene(b2d, at), view, max_batch=len(poses))
    _assert_same(render.render(at.blob, oview, poses, threads=8), r.render(poses), "at the limit %dx%d" % size)
    assert r.status() == 0

    poses = over.pose_array()
    needs = [stack_need(over.blob, oview, p) for p in poses]
    fits = [i for i in range(len(poses)) if needs[i] <= STACK_DEPTH]
    past = [i for i in range(len(poses)) if needs[i] > STACK_DEPTH]
    assert past and STACK_DEPTH in [needs[i] for i in fits]
    r = b2d.Renderer(_scene(b2d, over), view, max_batch=len(poses) + _sms())
    _assert_same(render.render(over.blob, oview, poses[fits], threads=8), r.render(poses[fits]), "one deeper, fitting poses")
    assert r.status() == 0
    for i in past:
        with pytest.raises(b2d.B2dError, match="stack overflow"):
            r.render(poses[i:i + 1])
        r.status()
        dp = _dev_poses(poses[i:i + 1])
        out = torch.empty((1, h, w), dtype=torch.uint8, device="cuda")
        r.render_device(dp.data_ptr(), 1, out.data_ptr())
        st = r.status()
        assert st & 1 and not st & 4, "pose %s: status %d" % (over.poses[i][4], st)
    dp = _dev_poses(poses)
    out = torch.empty((len(poses), h, w), dtype=torch.uint8, device="cuda")
    r.render_device(dp.data_ptr(), len(poses), out.data_ptr())
    st = r.status()
    assert st & 1 and not st & 4, st
    more = np.resize(poses, len(poses) + _sms())
    _background_walk(r, more, w, h)
    st = r.status()
    assert st & 1 and not st & 4, st
