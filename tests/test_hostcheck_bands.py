"""The raster kernel's band-major draw phase, executed on the CPU by tests/hostcheck/raster_bands.cpp: the CTA's queued
draws are drawn as (band, record) items, band by band, each record clipped to the band; a CTA whose items do not fit the
item list draws its records whole, in record order.  Whatever the band height, queue size and list capacity, the frames
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
from tests.test_hostcheck_queue import SHIPPED_WORDS

# b2d_kernels.cu kBandRows and kItemCap
SHIPPED_BAND = 256
SHIPPED_CAP = 1024

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostcheck", "raster_bands.cpp")


@functools.lru_cache(maxsize=None)
def band_mirror():
    """The band mirror, compiled into a temporary directory (the source tree may be read-only)."""
    out = os.path.join(tempfile.mkdtemp(prefix="b2d_raster_bands_"), "libb2d_raster_bands.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out, SRC])
    return ctypes.CDLL(out)


def banded(blob, view, poses, band, cap=SHIPPED_CAP, words=SHIPPED_WORDS, tics=0, frames=True, warps=8):
    """Frames (or None with frames=False) and the schedule's counts: row iterations, CTAs, CTAs that fell back to record
    order because their items exceed the list, items (total and in the largest CTA), records drawn during the clip pass,
    the line-open time's mean and 90th percentile, CTAs in record order because they deferred masked entries, and the
    mean modelled CTA makespan (row iterations)."""
    n = len(poses)
    fb = np.empty((n, view.height, view.width), np.uint8) if frames else None
    st = np.zeros(9, np.int64)
    ms = ctypes.c_double(0.0)
    buf = (ctypes.c_char * len(blob)).from_buffer_copy(blob)
    poses = np.ascontiguousarray(poses)
    rc = band_mirror().hostcheck_render_banded(
        ctypes.c_void_p(ctypes.addressof(buf)), ctypes.byref(view), ctypes.c_void_p(poses.ctypes.data), n,
        ctypes.c_void_p(fb.ctypes.data if frames else None), ctypes.c_uint32(tics), warps, ctypes.c_uint32(words), band,
        ctypes.c_uint32(cap), ctypes.c_void_p(st.ctypes.data), ctypes.byref(ms))
    assert rc == 0
    return fb, {"rows": int(st[0]), "ctas": int(st[1]), "ctas_fallback": int(st[2]), "items": int(st[3]),
                "items_max": int(st[4]), "overflow": int(st[5]), "open_mean": st[6] / 1000.0, "open_p90": st[7] / 1000.0, "ctas_masked": int(st[8]),
                "makespan": ms.value}


def _compare(b2d, scene, w, h, n, seed, band, cap, words, tics=0):
    poses = sample_poses(b2d, scene, n, seed)
    ofb = render.render(scene.blob, render.make_view(w, h), poses, threads=4, tics=tics)
    hfb, st = banded(scene.blob, b2d.make_view(w, h), poses, band, cap, words, tics)
    bad = [(i, int((ofb[i] != hfb[i]).sum())) for i in range(len(poses)) if not np.array_equal(ofb[i], hfb[i])]
    assert not bad, "frames differ (index, pixels): %s" % bad[:5]
    assert st["ctas"] > 0
    return st


BANDS = sorted({0, 32, 64, SHIPPED_BAND})


@pytest.mark.parametrize("band", BANDS)
@pytest.mark.parametrize("words", [0, 96, SHIPPED_WORDS])
def test_bands_equal_oracle(b2d, product_scene, band, words):
    """Band heights 0 (record order), 32, 64 and the shipped one; queue sizes 0 (every draw by its owner), tiny and
    shipped; widths whose CTAs straddle frames and a partial last strip."""
    for (w, h, n, seed) in ((320, 200, 12, 3), (333, 187, 6, 4), (1920, 1080, 2, 5)):
        st = _compare(b2d, product_scene, w, h, n, seed, band, SHIPPED_CAP, words)
        assert st["ctas_fallback"] == 0
        if words == 0:
            assert st["items"] == 0


@pytest.mark.parametrize("band", [b for b in BANDS if b])
def test_bands_list_fallback_equals_oracle(b2d, product_scene, band):
    """An item list one item short of the largest CTA's: that CTA draws its records whole, in record order, and the
    others band by band."""
    for (w, h, n, seed) in ((333, 187, 6, 4), (1920, 1080, 2, 5)):
        _, full = banded(product_scene.blob, b2d.make_view(w, h), sample_poses(b2d, product_scene, n, seed), band, frames=False)
        st = _compare(b2d, product_scene, w, h, n, seed, band, full["items_max"] - 1, SHIPPED_WORDS)
        assert 0 < st["ctas_fallback"] < st["ctas"], st


@pytest.mark.parametrize("band", BANDS)
def test_bands_masked_and_sprites(b2d, band):
    """The masked passes run after the banded draw phase: they overwrite solid pixels of their strip."""
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(1, ("E1M1",), cfg=synthwad.SynthConfig(mid_pct=30, thing_pct=70, anim=True))
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    _compare(b2d, sc, 320, 200, 16, 71, band, SHIPPED_CAP, SHIPPED_WORDS, tics=9)
    _compare(b2d, sc, 1920, 1080, 2, 72, band, SHIPPED_CAP, SHIPPED_WORDS, tics=9)
    _compare(b2d, sc, 1920, 1080, 2, 72, band, 40, 96, tics=9)


@functools.lru_cache(maxsize=None)
def flythrough(n):
    """bench.py's c2 fly-through (synthetic E1M1, seed 1, fly poses seed 2): n evenly spaced poses."""
    import bench
    from oracle.host import OracleScene
    sc = OracleScene(bench.build_wad("E1M1", 1, {}), 0)
    poses = bench.make_poses(sc, "fly", 1000, 2)
    return sc.blob, np.ascontiguousarray(poses[np.linspace(0, 999, n).astype(int)])


@pytest.mark.parametrize("size", [(1920, 1080), (3840, 2160)], ids=["1080p", "4k"])
def test_shipped_list_holds_every_flythrough_cta(b2d, size):
    """At the shipped band height and list capacity, no CTA of 100 poses of the benchmark's fly-through falls back to
    record order, and banding leaves the row iterations as they are."""
    blob, poses = flythrough(100)
    view = b2d.make_view(*size)
    _, st = banded(blob, view, poses, SHIPPED_BAND, frames=False)
    assert st["ctas_fallback"] == 0 and st["items_max"] <= SHIPPED_CAP, st
    _, st0 = banded(blob, view, poses, 0, frames=False)
    assert st["rows"] <= st0["rows"]
    assert st["open_mean"] < st0["open_mean"] / 4, (st, st0)
