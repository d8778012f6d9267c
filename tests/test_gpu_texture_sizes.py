"""-m gpu: the texture-size gallery of tests/test_texture_sizes.py through the kernels, bit for bit against the oracle --
walls 1 to 4096 rows tall and 1 to 4096 columns wide head-on in every step class of the raster's wall paths, masked
middles with holes at odd heights and at one and two row quads, sprites of 1x1, 1xN, Nx1 and 300 rows, an animation
group whose frames differ in size, and skies of 1024x128, 256x200, 64x240 and 256x1.  tests/test_texture_sizes.py shows
on the CPU that every case here is valid and reads nothing outside its texture."""
import numpy as np
import pytest

from oracle import render
from tests.test_gpu_scale import _assert_same, _dev_poses
from tests.test_texture_sizes import ANIM_TICS, ONE, SIZES, SKIES, anim_bay, gallery, pose_array

pytestmark = pytest.mark.gpu


def _scene(b2d, g):
    return b2d.Scene(b2d.Archive.from_bytes(g.wad), 0)


@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_gpu_gallery_render_matches_oracle(b2d, size):
    """Renderer.render, index and RGBA, every bay at every step class: 333 columns take the generic-width raster, 1920
    and 3840 the specialised ones."""
    g = gallery()
    w, h = size
    poses = pose_array(g.poses(size))
    if w == 3840:
        poses = poses[::2]
    chunk = 16 if w == 3840 else 64                       # host memory: oracle index + RGBA frames of one chunk
    oview = render.make_view(w, h)
    r = b2d.Renderer(_scene(b2d, g), b2d.make_view(w, h), max_batch=chunk)
    for i in range(0, len(poses), chunk):
        ofb, orgba = render.render(g.blob, oview, poses[i:i + chunk], rgba=True, threads=8)
        idx, rgba = r.render(poses[i:i + chunk], rgba=True)
        assert r.status() == 0
        _assert_same(ofb, idx, "gallery %dx%d from pose %d" % (w, h, i))
        assert np.array_equal(orgba, rgba), "gallery %dx%d from pose %d: RGBA" % (w, h, i)


def test_gpu_gallery_render_device_matches_oracle(b2d):
    """render_device into a poisoned buffer: every pixel written, nothing past the batch."""
    import torch
    g = gallery()
    view, oview = b2d.make_view(320, 200), render.make_view(320, 200)
    poses = pose_array(g.poses((320, 200)))
    n = len(poses)
    ofb = render.render(g.blob, oview, poses, threads=8)
    r = b2d.Renderer(_scene(b2d, g), view, max_batch=n)
    dp = _dev_poses(poses)
    out = torch.full((n + 1, 200, 320), 0xA5, dtype=torch.uint8, device="cuda")
    r.render_device(dp.data_ptr(), n, out.data_ptr())
    torch.cuda.synchronize()
    assert r.status() == 0
    _assert_same(ofb, out[:n].cpu().numpy(), "gallery render_device")
    assert bool((out[n] == 0xA5).all()), "render_device wrote past the batch"


@pytest.mark.parametrize("size", ((320, 200), (1920, 1080)), ids=["320x200", "1920x1080"])
def test_gpu_gallery_animation_states_match_oracle(b2d, size):
    """render_states at tics showing each frame of the mixed-size animation group, mixed in one batch."""
    g = gallery()
    w, h = size
    base = pose_array(g.poses(size, bays={anim_bay()}))
    poses = np.concatenate([base] * len(ANIM_TICS))
    tics = np.repeat(np.array(ANIM_TICS, np.uint32), len(base))
    order = np.arange(len(poses)).reshape(len(ANIM_TICS), -1).T.ravel()       # neighbouring frames at different tics
    poses, tics = poses[order], tics[order]
    oview = render.make_view(w, h)
    want = np.concatenate([render.render(g.blob, oview, poses[i:i + 1], tics=int(tics[i])) for i in range(len(poses))])
    r = b2d.Renderer(_scene(b2d, g), b2d.make_view(w, h), max_batch=len(poses))
    got = r.render_states(poses, tics)
    assert r.status() == 0
    _assert_same(want, got, "animation states %dx%d" % size)


def test_gpu_gallery_sky_variants_in_one_level_set(b2d):
    """Renderer.from_levels over the gallery with every sky size, frames alternating levels, index and RGBA: each frame
    uses its own level's skyrow table and sky texture."""
    gs = [gallery(s) for s in SKIES]
    sky_bays = {k for k, b in enumerate(ONE) if b[4]}
    per = [pose_array(g.poses((320, 200), bays=sky_bays, classes=(0, 2, 5))) for g in gs]
    n = 60
    lv = np.array([i % len(gs) for i in range(n)], np.int32)
    poses = np.concatenate([per[lv[i]][(i // len(gs)) % len(per[lv[i]]):][:1] for i in range(n)])
    r = b2d.Renderer.from_levels([_scene(b2d, g) for g in gs], b2d.make_view(320, 200), max_batch=n)
    idx, rgba = r.render_levels(poses, lv, rgba=True)
    assert r.status() == 0
    oview = render.make_view(320, 200)
    want = [render.render(gs[lv[i]].blob, oview, poses[i:i + 1], rgba=True) for i in range(n)]
    _assert_same(np.concatenate([w[0] for w in want]), idx, "sky level set")
    assert np.array_equal(np.concatenate([w[1] for w in want]), rgba), "sky level set: RGBA"


@pytest.mark.parametrize("sky", SKIES[1:], ids=["sky%dx%d" % s for s in SKIES[1:]])
def test_gpu_gallery_sky_variant_render_matches_oracle(b2d, sky):
    g = gallery(sky)
    sky_bays = {k for k, b in enumerate(ONE) if b[4]}
    for size in ((333, 187), (1920, 1080)):
        poses = pose_array(g.poses(size, bays=sky_bays, classes=(0, 3, 5)))
        r = b2d.Renderer(_scene(b2d, g), b2d.make_view(*size), max_batch=len(poses))
        got = r.render(poses)
        assert r.status() == 0
        _assert_same(render.render(g.blob, render.make_view(*size), poses, threads=8), got, "sky %dx%d at %dx%d" % (sky + size))
