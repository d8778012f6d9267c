"""The resolved sharded calls on the C ABI (no GPU needed): include/b2d.h declares b2d_render_sharded_resolved and
b2d_render_sharded_levels_states_resolved, libb2d.so exports them, the ctypes binding matches the header, and both
Renderer methods take `resolve=`."""
import ctypes
import inspect
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = {"b2d_render_sharded_resolved": 11, "b2d_render_sharded_levels_states_resolved": 15}


def _declaration(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2d.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+%s\s*\(([^;]*)\)\s*;" % name, text, flags=re.S)
    assert m, "b2d.h does not declare %s" % name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def test_header_declares_the_calls():
    for name, arity in CALLS.items():
        decl = _declaration(name)
        assert len(decl) == arity, name
        # the unresolved call's parameters, with factor and format right before the mode
        base = _declaration(name[:-len("_resolved")])
        i = base.index("int mode")
        assert decl == base[:i] + ["int factor", "int format"] + base[i:], name


def test_library_exports_the_calls_with_argtypes_matching_the_header(b2d):
    from rust_doom_b200 import _lib
    lib = _lib.load()
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for name, arity in CALLS.items():
        assert name in _lib.EXPORTS and re.search(r"\bT %s$" % name, out, flags=re.M), name
        types = getattr(lib, name).argtypes
        assert types and len(types) == arity, name
        for decl, t in zip(_declaration(name), types):
            if decl.startswith("b2d_chunk_fn"):
                assert t is _lib.CHUNK_FN, (name, decl, t)
            elif "*" in decl:
                assert t is ctypes.c_void_p or hasattr(t, "_type_"), (name, decl, t)
            elif decl.startswith("size_t"):
                assert t is ctypes.c_size_t, (name, decl, t)
            else:
                assert decl.startswith("int ") and t is ctypes.c_int, (name, decl, t)
        unresolved = getattr(lib, name[:-len("_resolved")]).argtypes
        i = _declaration(name[:-len("_resolved")]).index("int mode")
        assert list(types) == list(unresolved[:i]) + [ctypes.c_int, ctypes.c_int] + list(unresolved[i:]), name


def test_renderer_methods_take_resolve(b2d):
    for name in ("render_sharded", "render_sharded_levels_states"):
        p = inspect.signature(getattr(b2d.Renderer, name)).parameters
        assert "resolve" in p and p["resolve"].default is None, name
    assert set(b2d.RESOLVE_FORMATS) == {"rgba", "rgb", "rgb_planar", "gray"}
