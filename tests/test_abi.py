"""C-ABI boundary: libb2d.so loads, exports exactly what include/b2d.h declares, and fails loudly
(never falls back to a CPU path) when no CUDA device is usable."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "b2d.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b2d_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported(b2d):
    from rust_doom_b200 import _lib
    lib = _lib.load()
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), "libb2d.so does not export %s" % n
    assert sorted(_lib.EXPORTS) == names, "ctypes binding and header disagree"


def test_library_is_in_tree(b2d):
    from rust_doom_b200 import _lib
    assert os.path.dirname(_lib.LIB_PATH) == os.path.join(ROOT, "rust-doom_b200")
    assert os.path.exists(_lib.LIB_PATH)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "rust-doom_b200")
    for base, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cpp", ".cu", ".cuh", ".hpp", ".h")):
                src = open(os.path.join(base, f), errors="replace").read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert "b2d_oracle" not in src and "libb2d_oracle" not in src, f


def test_invalid_arguments(b2d, product_scene):
    with pytest.raises(b2d.B2dError) as e:
        b2d.make_view(0, 200)
    assert e.value.code == b2d.ERR_INVALID_ARG
    with pytest.raises(b2d.B2dError):
        b2d.make_view(8192, 200)
    with pytest.raises(b2d.B2dError):
        b2d.make_view(320, 200, 179.5)


def test_hand_built_views_out_of_range_are_refused(b2d, product_scene):
    """b2d_renderer_create checks a view before it looks for a device: F or FY2 above 2^18, or width above 256 F."""
    from rust_doom_b200 import _lib
    for w, h, F, FY2 in ((320, 200, (1 << 18) + 1, 400), (320, 200, 300, (1 << 18) + 1), (4096, 24, 15, 20), (513, 2, 2, 2)):
        with pytest.raises(b2d.B2dError) as e:
            b2d.Renderer(product_scene, _lib.View(w, h, F, FY2))
        assert e.value.code == b2d.ERR_INVALID_ARG and "view out of range" in e.value.message, (w, h, F, FY2)


def test_no_cpu_fallback(b2d, product_scene):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(b2d.B2dError) as e:
        b2d.Renderer(product_scene, b2d.make_view(320, 200))
    assert e.value.code == b2d.ERR_CUDA
    assert "no CPU path" in e.value.message
