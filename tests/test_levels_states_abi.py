"""Per-frame states with per-frame levels on the C ABI (no GPU needed): include/b2d.h declares the three entry points,
libb2d.so exports them, the ctypes binding gives each its argument types, and Renderer has the three methods."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = {"b2d_render_levels_states": 9, "b2d_render_device_levels_states": 10, "b2d_walk_device_levels_states": 9}


def test_header_declares_level_state_calls():
    raw = open(os.path.join(ROOT, "include", "b2d.h")).read()
    text = re.sub(r"/\*.*?\*/", "", raw, flags=re.S)
    for name, arity in CALLS.items():
        m = re.search(r"\bint\s+%s\s*\(([^;]*)\)\s*;" % name, text, flags=re.S)
        assert m, "b2d.h does not declare %s" % name
        assert len(m.group(1).split(",")) == arity, "%s: %d parameters expected" % (name, arity)
    assert "per-frame states together with per-frame levels" not in raw


def test_library_exports_level_state_calls_with_argtypes(b2d):
    from rust_doom_b200 import _lib
    lib = _lib.load()
    for name, arity in CALLS.items():
        assert name in _lib.EXPORTS
        fn = getattr(lib, name)
        assert fn.argtypes and len(fn.argtypes) == arity, name


def test_renderer_has_level_state_methods(b2d):
    for name in ("render_levels_states", "render_device_levels_states", "walk_device_levels_states"):
        assert callable(getattr(b2d.Renderer, name))
