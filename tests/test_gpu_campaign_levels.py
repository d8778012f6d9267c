"""-m gpu: a short deterministic run of tools/campaign_levels_gpu.py (random level sets with per-frame levels and states,
through every entry point that renders a level set or acts on its level 0), its forced full-size cases, one small case per
walk or raster kernel instantiation the random draw misses, and a set of 64 small levels.  Each case compares every frame
with the oracle, the table sets with oracle/scene.py tables_at, the launch count with DESIGN.md §3 and the poisoned guard
bytes around every device output with what was written there.  tests/test_campaign_levels.py checks, without a GPU, that
these cases launch every instantiation the library has."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
import campaign_levels_gpu as C  # noqa: E402

pytestmark = pytest.mark.gpu

SEED, CASES = 2024, 40
# the raster cells (rgba, kW, masked, kStates, kLevels) and walk cells (kStates, kLevels, persistent grid) that the 40
# random cases of SEED and the forced cases miss: one small case each
FILL_RASTER = [(False, 0, True, False, False), (False, 1920, False, False, False), (False, 1920, False, True, False),
               (False, 1920, True, False, False), (False, 1920, True, False, True), (False, 3840, False, True, False),
               (False, 3840, True, False, False), (False, 3840, True, True, False), (True, 0, False, True, False),
               (True, 0, True, True, False), (True, 0, True, True, True), (True, 1920, False, False, False),
               (True, 1920, False, True, False), (True, 1920, True, False, True), (True, 1920, True, True, False),
               (True, 1920, True, True, True)]
FILL_WALK = [(False, False, True), (True, False, True), (True, True, True)]


def short_run():
    """[(label, case)] of the deterministic run: the random cases, the forced ones, the cell fillers"""
    out = [(k, C.draw_case(SEED, k)) for k in range(CASES)]
    out += [("forced %d" % i, c) for i, c in enumerate(C.forced_cases())]
    out += [("cell %s" % (cell,), C.cell_case(cell, 100 + i)) for i, cell in enumerate(FILL_RASTER + FILL_WALK)]
    return out


def _run(todo):
    n, bad, pixels, secs = C.run(0, SEED, todo=todo)
    print("%d cases, %d mismatching, %.1f Mpixel compared, %.1f s" % (n, bad, pixels / 1e6, secs))
    assert bad == 0, "%d of %d cases differ (printed above)" % (bad, n)


def test_campaign_levels_random(b2d):
    """the 40 random cases of SEED"""
    _run([t for t in short_run() if isinstance(t[0], int)])


def test_campaign_levels_forced_and_cells(b2d):
    """3840 x 2160 index frames on sets with and without masked content, with and without states; 1920 x 1080 index and
    RGBA frames on sets without masked content; one case per kernel instantiation the random cases miss"""
    _run([t for t in short_run() if not isinstance(t[0], int)])


def test_64_level_set(b2d):
    """A set of 64 small levels (B2D_MAX_LEVELS), frames on every one of them, level 63 included, with per-frame states
    and on the plain level path: the set adds less than 4 GB of device memory (each level's pre-lit flats take a 4 GiB
    aligned range of address space, not of memory), and every frame, table set, launch count and guard is right."""
    import torch
    rng = np.random.default_rng(64)
    specs = []
    for k in range(64):
        L = C._level_spec(rng, masked=k % 9 == 4)
        g = (2, 3) if k % 2 else (3, 2)
        L["cfg"].update(gx=g[0], gy=g[1], origin=(-128 * g[0], -128 * g[1]))
        specs.append(L)
    lvs = C.build_levels(C.prepare_case(dict(levels=specs)))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    r = b2d.Renderer.from_levels([L["scene"] for L in lvs], b2d.make_view(320, 200), max_batch=128)
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    r.close()
    assert used < 4 << 30, "a 64-level set takes %.2f GB of device memory" % (used / 1e9)
    for entry in ("render_device_levels_states", "render_levels", "walk_device_levels_states"):
        case = dict(seed=6400, levels=specs, w=320, h=200, fov=65.0, entry=entry, rgba=entry == "render_levels", lut=True,
                    lut_offset=4, chunk=0, n=128, max_batch=128, walk_batch=128)
        problems, _ = C.run_case(case, lvs)
        assert not problems, "%s: %s" % (entry, problems)


def test_guard_check_sees_one_byte(b2d):
    """the campaign's guard check reports a single byte written just past an output, and one just before it"""
    import torch
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    for at in (1000, -1):
        g = C._Guarded(1000, 1000, 4, gen)
        assert g.touched() == []
        g.buf[g.offset + at] ^= 0x5A
        assert g.touched() == [at]
