import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def _gpu_available() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        return False


def pytest_collection_modifyitems(config, items):
    if _gpu_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def b2d():
    import rust_doom_b200
    from rust_doom_b200 import build
    build.build()
    return rust_doom_b200


@pytest.fixture(scope="session")
def synth_wad():
    """The level every generic test runs on: a generated two-map IWAD, or -- when B2D_IWAD=/path/doom1.wad is set -- that
    file, so that the whole suite (oracle, scene compiler, hostcheck, -m gpu) runs on a real IWAD's first level."""
    iwad = os.environ.get("B2D_IWAD")
    if iwad:
        with open(iwad, "rb") as f:
            return f.read()
    from rust_doom_b200 import synthwad
    return synthwad.build_iwad(1, ("E1M1", "E1M2"))


@pytest.fixture(scope="session")
def oracle_scene(synth_wad):
    from oracle import scene, wad
    a = wad.Archive(synth_wad)
    t = wad.TextureDirectory(a)
    return scene.compile_scene(a, t, 0)


@pytest.fixture(scope="session")
def product_scene(b2d, synth_wad):
    a = b2d.Archive.from_bytes(synth_wad)
    return b2d.Scene(a, 0)


HOSTCHECK_SRC = os.path.join(ROOT, "tests", "hostcheck", "hostcheck.cpp")
HOSTCHECK_SO = os.path.join(ROOT, "tests", "hostcheck", "libb2d_hostcheck.so")


@pytest.fixture(scope="session")
def hostcheck():
    """Test-only CPU execution of the product's pixel-contract maths (tests/hostcheck/hostcheck.cpp)."""
    deps = [HOSTCHECK_SRC, os.path.join(ROOT, "rust-doom_b200", "csrc", "b2d_math.cuh"),
            os.path.join(ROOT, "rust-doom_b200", "csrc", "b2d_scene.hpp")]
    if not os.path.exists(HOSTCHECK_SO) or any(os.path.getmtime(d) > os.path.getmtime(HOSTCHECK_SO) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", HOSTCHECK_SO, HOSTCHECK_SRC])
    lib = ctypes.CDLL(HOSTCHECK_SO)

    def run(blob: bytes, view, poses: np.ndarray, tics: int = 0, moves=()):
        n = len(poses)
        nsegs = int(np.frombuffer(blob, dtype="<u4", count=32)[6])
        fb = np.empty((n, view.height, view.width), np.uint8)
        counts = np.zeros(n, np.int32)
        ids = np.full((n, max(nsegs, 1)), -1, np.int32)
        buf = (ctypes.c_char * len(blob)).from_buffer_copy(blob)
        poses = np.ascontiguousarray(poses)
        mv = np.array([tuple(int(v) for v in m) for m in moves], dtype=np.int32).reshape(-1, 3)
        rc = lib.hostcheck_render_m(ctypes.c_void_p(ctypes.addressof(buf)), ctypes.byref(view),
                                    ctypes.c_void_p(poses.ctypes.data), n, ctypes.c_void_p(fb.ctypes.data),
                                    ctypes.c_void_p(counts.ctypes.data), ctypes.c_void_p(ids.ctypes.data), ids.shape[1],
                                    ctypes.c_uint32(int(tics) & 0xFFFFFFFF), ctypes.c_void_p(mv.ctypes.data if len(mv) else None), len(mv))
        assert rc == 0, "hostcheck rejected the sector moves"
        return fb, counts, ids

    run.lib = lib
    return run


def oracle_blob(wad_bytes: bytes, level: int = 0) -> bytes:
    """The scene compiled by the ORACLE's own loader + compiler (oracle/wad.py, oracle/scene.py), independent of libb2d."""
    from oracle import scene, wad
    a = wad.Archive(wad_bytes)
    return scene.compile_scene(a, wad.TextureDirectory(a), level)


def sample_poses(b2d_mod, scene, n, seed):
    """Mixed bag of poses inside the level: spawn, random, fly-through."""
    from rust_doom_b200 import poses as P
    out = [P.random_poses(scene, max(n - n // 3 - 1, 1), seed), P.flythrough_poses(scene, max(n // 3, 1), seed + 1)]
    if scene.start_pose is not None:
        out.insert(0, scene.start_pose)
    return np.concatenate(out)[:n]
