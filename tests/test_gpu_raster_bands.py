"""-m gpu: the raster's band-major draw phase (b2d_kernels.cu kBandRows, kItemCap) on the long-seg hall of
tests/test_level_shapes.py, whose CTAs draw hundreds of items with records crossing every band, and on a ring of 255
sprites in one subsector, whose CTAs defer masked entries and so draw their records whole, in record order: at 1080p, 4K
and a generic width, plain, with RGBA, with per-frame states, and in a level set with per-frame states (a CTA's warps
then hold frames of both kinds).  The CPU mirror of the same schedule (tests/hostcheck/raster_bands.cpp) shows which
CTAs take which order; the list-capacity fallback is checked there, at capacities below the shipped one."""
import numpy as np
import pytest

from oracle import render
from tests.test_gpu_raster_queue import _hall, _ring
from tests.test_gpu_scale import _assert_same
from tests.test_gpu_states import _oracle
from tests.test_hostcheck_bands import SHIPPED_BAND, SHIPPED_CAP, banded

pytestmark = pytest.mark.gpu

SIZES = ((1920, 1080), (3840, 2160), (1000, 750))


def _schedule(b2d, blob, poses, w, h):
    """The mirror's counts for these frames at the shipped band height and list capacity."""
    _, st = banded(blob, b2d.make_view(w, h), poses, SHIPPED_BAND, SHIPPED_CAP, frames=False)
    _, whole = banded(blob, b2d.make_view(w, h), poses, 0, frames=False)
    assert st["ctas_fallback"] == 0 and st["items"] > whole["items"], (st, whole)
    return st


@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
@pytest.mark.parametrize("shape", ["hall", "ring255"])
def test_gpu_bands_match_oracle(b2d, shape, size):
    w, h = size
    sc, blob, poses = (_hall if shape == "hall" else _ring)(b2d)
    st = _schedule(b2d, blob, poses, w, h)
    assert st["ctas_masked"] == (0 if shape == "hall" else st["ctas"]), st
    n = len(poses)
    r = b2d.Renderer(sc, b2d.make_view(w, h), max_batch=n)
    idx, rgba = r.render(poses, rgba=True)
    assert r.status() == 0
    ofb, orgba = render.render(blob, render.make_view(w, h), poses, rgba=True, threads=8)
    _assert_same(ofb, idx, "%s %dx%d" % (shape, w, h))
    assert np.array_equal(orgba, rgba), "%s %dx%d RGBA" % (shape, w, h)
    tics = np.array([(53 * i + 5) % 700 for i in range(n)], np.uint32)
    moves = [[] for _ in range(n)]
    got = r.render_states(poses, tics, moves)
    assert r.status() == 0
    _assert_same(_oracle(blob, w, h, poses, tics, moves), got, "%s %dx%d per-frame states" % (shape, w, h))


@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_gpu_bands_level_set_states(b2d, size):
    """Both shapes in one level set, frames alternating levels, each at its own level time, index and RGBA frames: a
    CTA's items come from frames of different levels, some CTAs banded and some in record order."""
    w, h = size
    hs, hblob, hposes = _hall(b2d)
    rs, rblob, rposes = _ring(b2d)
    n = 8
    lv = np.array([i % 2 for i in range(n)], np.int32)
    poses = np.concatenate([(hposes if lv[i] == 0 else rposes)[(i // 2) % 6:][:1] for i in range(n)])
    tics = np.array([(31 * i + 7) % 500 for i in range(n)], np.uint32)
    r = b2d.Renderer.from_levels([hs, rs], b2d.make_view(w, h), max_batch=n)
    idx, rgba = r.render_levels_states(poses, lv, tics, rgba=True)
    assert r.status() == 0
    blobs = (hblob, rblob)
    for i in range(n):
        ofb, orgba = render.render(blobs[lv[i]], render.make_view(w, h), poses[i:i + 1], rgba=True, tics=int(tics[i]))
        _assert_same(ofb, idx[i:i + 1], "level set frame %d %dx%d" % (i, w, h))
        assert np.array_equal(orgba[0], rgba[i]), "level set frame %d %dx%d RGBA" % (i, w, h)
