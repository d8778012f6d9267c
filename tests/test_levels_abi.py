"""Level sets on the C ABI (no GPU needed): include/b2d.h declares the five level-set entry points, libb2d.so exports
them, and the ctypes binding gives each its argument types."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVEL_CALLS = ("b2d_renderer_create_levels", "b2d_render_levels", "b2d_render_device_levels", "b2d_walk_device_levels",
               "b2d_renderer_set_level_sector_moves")


def test_header_declares_level_calls():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2d.h")).read(), flags=re.S)
    for name in LEVEL_CALLS:
        assert re.search(r"\bint\s+%s\s*\(" % name, text), "b2d.h does not declare %s" % name
    assert re.search(r"#define\s+B2D_MAX_LEVELS\s+64\b", text)


def test_library_exports_level_calls_with_argtypes(b2d):
    from rust_doom_b200 import _lib
    lib = _lib.load()
    for name in LEVEL_CALLS:
        assert name in _lib.EXPORTS
        fn = getattr(lib, name)
        assert fn.argtypes, "%s has no argtypes" % name
    assert len(lib.b2d_renderer_create_levels.argtypes) == 6
    assert len(lib.b2d_render_levels.argtypes) == 6
    assert len(lib.b2d_render_device_levels.argtypes) == 7
    assert len(lib.b2d_walk_device_levels.argtypes) == 6
    assert len(lib.b2d_renderer_set_level_sector_moves.argtypes) == 4
    assert b2d.MAX_LEVELS == 64


def test_renderer_has_level_methods(b2d):
    for name in ("render_levels", "render_device_levels", "walk_device_levels", "set_level_sector_moves"):
        assert callable(getattr(b2d.Renderer, name))
    assert callable(b2d.Renderer.from_levels)
