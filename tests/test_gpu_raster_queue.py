"""-m gpu: scenes whose raster CTAs fill their draw queue (b2d_kernels.cu DrawQueue), so that strips draw part of their
records themselves during the clip pass and hand the rest to the CTA's draw phase: the long-seg hall of
tests/test_level_shapes.py and a ring of 255 sprites in one subsector (masked kernels), at 1080p and 4K, plain, with
per-frame states, with RGBA, and in a level set with per-frame states.  The CPU mirror of the same schedule
(tests/hostcheck/raster_queue.cpp) shows that these frames do overflow the queue."""
import numpy as np
import pytest

from oracle import render
from tests.test_gpu_scale import _assert_same
from tests.test_gpu_states import _oracle
from tests.test_hostcheck_queue import SHIPPED_WORDS, _queued
from tests.test_level_shapes import levels
from tests.test_scale import cluster_level, cluster_poses

pytestmark = pytest.mark.gpu

SIZES = ((1920, 1080), (3840, 2160))


def _hall(b2d):
    lv = levels()["hall"]
    return b2d.Scene(b2d.Archive.from_bytes(lv.wad), 0), lv.blob, lv.pose_array()[:6]


def _ring(b2d):
    data, blob, _, _ = cluster_level(255, "ring")
    return b2d.Scene(b2d.Archive.from_bytes(data), 0), blob, cluster_poses(b2d, 255, "ring")[:6]


def _assert_overflows(b2d, blob, poses, w, h):
    _, st = _queued(blob, b2d.make_view(w, h), poses, 8, SHIPPED_WORDS)
    assert st["overflow"] > 0, st


@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
@pytest.mark.parametrize("shape", ["hall", "ring255"])
def test_gpu_queue_overflow_matches_oracle(b2d, shape, size):
    w, h = size
    sc, blob, poses = (_hall if shape == "hall" else _ring)(b2d)
    _assert_overflows(b2d, blob, poses, w, h)
    n = len(poses)
    r = b2d.Renderer(sc, b2d.make_view(w, h), max_batch=n)
    idx, rgba = r.render(poses, rgba=True)
    ofb, orgba = render.render(blob, render.make_view(w, h), poses, rgba=True, threads=8)
    _assert_same(ofb, idx, "%s %dx%d" % (shape, w, h))
    assert np.array_equal(orgba, rgba), "%s %dx%d RGBA" % (shape, w, h)
    tics = np.array([(53 * i + 5) % 700 for i in range(n)], np.uint32)
    moves = [[] for _ in range(n)]
    got = r.render_states(poses, tics, moves)
    assert r.status() == 0
    _assert_same(_oracle(blob, w, h, poses, tics, moves), got, "%s %dx%d per-frame states" % (shape, w, h))


@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_gpu_queue_overflow_level_set_states(b2d, size):
    """Both shapes in one level set, frames alternating levels, each at its own level time, index and RGBA frames: the
    records of a CTA's warps come from frames of different levels (each drawn with its owner's scene and palette)."""
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
