"""No GPU: what the level-set campaign of tests/test_gpu_campaign_levels.py reaches.  The dispatch rule of raster_go /
walk_go (csrc/b2d_kernels.cu), restated in tools/campaign_levels_gpu.py as a function of (width, RGBA, any level masked,
per-frame states, per-frame levels, a background walk of more frames than SMs), applied to the run's cases: every one of
the 40 raster and 8 walk cells is hit.  And the kernel instantiations compiled into libb2d.so are exactly the ones that
rule knows, so a new variant, or a dispatch change, shows here before it can go untested."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
import campaign_levels_gpu as C  # noqa: E402

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def short_run(b2d):
    from tests.test_gpu_campaign_levels import short_run
    todo = [c for _, c in short_run()]
    return todo, [C.case_info(c) for c in todo]


def test_matrix_sizes():
    assert len(C.ALL_RASTER) == 40 and len(C.ALL_WALK) == 8


def test_dispatch_rule():
    """raster_go: RGBA frames at 1920 columns or generic, index frames at 1920, 3840 or generic; walk_go: a persistent grid
    only for a background walk of more frames than SMs"""
    assert C.raster_cell(1920, True, True, True, True) == (True, 1920, True, True, True)
    assert C.raster_cell(3840, True, False, False, False) == (True, 0, False, False, False)
    assert C.raster_cell(3840, False, False, True, True) == (False, 3840, False, True, True)
    assert C.raster_cell(1921, False, False, False, True) == (False, 0, False, False, True)
    assert C.walk_cell(True, True, True, 133) == (True, True, True)
    assert C.walk_cell(True, True, True, 132) == (True, True, False)
    assert C.walk_cell(False, False, False, 500) == (False, False, False)
    # entry points without a level argument act on level 0: its masked content decides, and its per-frame states take the
    # plain kernels when it has no time-dependent content or dynamic sectors
    case = dict(entry="render_states", w=640, rgba=False, n=4, max_batch=4, chunk=0)
    assert C.cells(case, [(False, False), (True, True)]) == ({(False, 0, False, False, False)}, {(False, False, False)})
    assert C.cells(case, [(True, True), (False, False)]) == ({(False, 0, True, True, False)}, {(True, False, False)})
    case = dict(entry="walk_device_levels_states", w=1920, rgba=True, n=2 * 140, max_batch=141, walk_batch=140, chunk=0)
    assert C.cells(case, [(False, False), (True, True)]) == ({(True, 1920, True, True, True)}, {(True, True, True)})


def test_short_run_hits_every_cell(short_run):
    """every raster and walk kernel instantiation is launched by some case of the GPU test"""
    mr, mw = C.missing_cells(*short_run)
    assert not mr, "raster cells (rgba, kW, masked, kStates, kLevels) no case launches: %s" % sorted(mr)
    assert not mw, "walk cells (kStates, kLevels, persistent grid) no case launches: %s" % sorted(mw)


def test_short_run_has_full_size_and_unmasked_cases(short_run):
    """3840 x 2160 index frames on sets with and without masked content, with and without per-frame states, and 1920 x 1080
    frames on unmasked sets, index and RGBA, with and without states"""
    todo, infos = short_run
    seen = set()
    for c, info in zip(todo, infos):
        levels, states, _, _ = C.ENTRIES[c["entry"]]
        if levels and (c["w"], c["h"]) in ((3840, 2160), (1920, 1080)):
            seen.add((c["w"], bool(c["rgba"]), any(m for m, _ in info), states))
    for masked in (False, True):
        for states in (False, True):
            assert (3840, False, masked, states) in seen
    for rgba in (False, True):
        for states in (False, True):
            assert (1920, rgba, False, states) in seen


def kernel_instantiations(path):
    """(raster, walk) template arguments of the b2d_raster_kernel and b2d_walk_kernel instantiations in a library, from
    its ELF section names demangled as tools/sass_compare.py does"""
    txt = subprocess.run([CUOBJDUMP, "-elf", path], capture_output=True, text=True, check=True).stdout
    names = sorted(set(re.findall(r"\.text\.(\S+)", txt)))
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout
    raster, walk = set(), set()
    for line in dem.splitlines():
        m = re.search(r"b2d_raster_kernel<(\w+), (\d+), (\w+), (\w+), (\w+)>\(", line)
        if m:
            raster.add((m.group(1) == "true", int(m.group(2)), m.group(3) == "true", m.group(4) == "true", m.group(5) == "true"))
        m = re.search(r"b2d_walk_kernel<(\w+), (\w+)>\(", line)
        if m:
            walk.add((m.group(1) == "true", m.group(2) == "true"))
    return raster, walk


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="no cuobjdump")
def test_library_has_exactly_the_matrix(b2d):
    """the instantiations compiled into libb2d.so are exactly the cells of the restated dispatch rule"""
    from rust_doom_b200 import _lib
    raster, walk = kernel_instantiations(_lib.LIB_PATH)
    assert raster == C.ALL_RASTER, "in the library only: %s; in the rule only: %s" % (sorted(raster - C.ALL_RASTER),
                                                                                     sorted(C.ALL_RASTER - raster))
    assert walk == {(s, lv) for s, lv, _ in C.ALL_WALK}
