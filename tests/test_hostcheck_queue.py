"""The raster kernel's CTA draw queue, executed on the CPU by tests/hostcheck/raster_queue.cpp: each warp's clip pass appends
its strip's draws to a queue of bounded size shared by the CTA's warps, a draw that does not fit is drawn by its owner at
once, the queue is drawn after all clip passes, and the masked passes come last.  Whatever the queue size, the frames
must be the oracle's bit for bit."""
import ctypes
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import render
from tests.conftest import sample_poses

# per-lane words of the kernel's queue (b2d_kernels.cu kQueueWords): a flat span or void fill takes 32, a wall piece 96
SHIPPED_WORDS = 6144

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostcheck", "raster_queue.cpp")


@functools.lru_cache(maxsize=None)
def queue_mirror():
    """The queue mirror, compiled into a temporary directory (the source tree may be read-only)."""
    out = os.path.join(tempfile.mkdtemp(prefix="b2d_raster_queue_"), "libb2d_raster_queue.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out, SRC])
    return ctypes.CDLL(out)


def _queued(blob, view, poses, warps, words, tics=0):
    n = len(poses)
    fb = np.empty((n, view.height, view.width), np.uint8)
    q = np.zeros(4, np.int64)
    buf = (ctypes.c_char * len(blob)).from_buffer_copy(blob)
    poses = np.ascontiguousarray(poses)
    rc = queue_mirror().hostcheck_render_queued(ctypes.c_void_p(ctypes.addressof(buf)), ctypes.byref(view),
                                                ctypes.c_void_p(poses.ctypes.data), n, ctypes.c_void_p(fb.ctypes.data),
                                                ctypes.c_uint32(tics), warps, ctypes.c_uint32(words),
                                                ctypes.c_void_p(q.ctypes.data))
    assert rc == 0
    return fb, {"records": int(q[0]), "overflow": int(q[1]), "ctas": int(q[2]), "ctas_overflow": int(q[3])}


def _compare(b2d, scene, w, h, n, seed, warps, words, tics=0):
    poses = sample_poses(b2d, scene, n, seed)
    ofb = render.render(scene.blob, render.make_view(w, h), poses, threads=4, tics=tics)
    hfb, st = _queued(scene.blob, b2d.make_view(w, h), poses, warps, words, tics)
    bad = [(i, int((ofb[i] != hfb[i]).sum())) for i in range(len(poses)) if not np.array_equal(ofb[i], hfb[i])]
    assert not bad, "frames differ (index, pixels): %s" % bad[:5]
    assert st["records"] > 0
    return st


@pytest.mark.parametrize("warps", [8, 16])
@pytest.mark.parametrize("words", [0, 96, SHIPPED_WORDS])
def test_queue_any_capacity_equals_oracle(b2d, product_scene, warps, words):
    """Capacity 0 (every draw by its owner, today's order), a tiny queue (one wall piece or three spans, the rest
    overflows mid-strip) and the shipped size; widths whose CTAs straddle frames and a partial last strip."""
    for (w, h, n, seed) in ((320, 200, 12, 3), (333, 187, 6, 4), (1920, 1080, 2, 5)):
        st = _compare(b2d, product_scene, w, h, n, seed, warps, words)
        if words == 0:
            assert st["overflow"] == st["records"]
        elif words == 96:
            assert 0 < st["overflow"] < st["records"]


@pytest.mark.parametrize("words", [0, 96, SHIPPED_WORDS])
def test_queue_masked_and_sprites(b2d, words):
    """The masked passes run after the CTA's queue is drawn: they overwrite solid pixels of their strip."""
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=30, thing_pct=70, anim=True))
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    _compare(b2d, sc, 320, 200, 16, 71, 8, words, tics=9)
    _compare(b2d, sc, 1920, 1080, 2, 72, 8, words, tics=9)


def test_queue_rarely_overflows_on_the_benchmark_flythrough(b2d):
    """bench.py's c2 fly-through (synthetic E1M1, seed 1, fly poses seed 2) at 1920x1080: an evenly spaced sample of 20
    poses.  The shipped queue holds all but a few per cent of the draws (0.7 % over 100 poses)."""
    import bench
    from oracle.host import OracleScene
    sc = OracleScene(bench.build_wad("E1M1", 1, {}), 0)
    poses = bench.make_poses(sc, "fly", 1000, 2)
    poses = np.ascontiguousarray(poses[np.linspace(0, 999, 20).astype(int)])
    _, st = _queued(sc.blob, b2d.make_view(1920, 1080), poses, 8, SHIPPED_WORDS)
    assert st["records"] > 0 and st["overflow"] / st["records"] < 0.03, st
