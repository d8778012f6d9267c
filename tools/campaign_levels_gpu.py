#!/usr/bin/env python3
"""Random parity campaign on the GPU over level sets and per-frame states: libb2d.so against the oracle on random sets of
1-8 generated levels (masked content in some sets and deliberately none in others, dynamic sectors on any subset, some
levels from a WAD with another palette), random views (1920 and 3840 columns drawn with fixed probability), per-frame
levels, tics and sector moves, and every entry point that renders a level set or acts on its level 0.

Every case checks each frame against the oracle's frame of its level at its (tics, moves) (RGBA from that level's own
blob), the table sets of the last batch walked with per-frame states against oracle/scene.py tables_at, the status word,
each batch's launch count (DESIGN.md §3) and, on the device paths, that the poisoned guard bytes around every output
(4 KB before and after it, and the frames past n of a batch shorter than max_batch) are untouched.

    python tools/campaign_levels_gpu.py [cases] [--seed S] [--case K]

`--case K` re-runs case K of seed S alone.  `cells()` restates which walk and raster kernel instantiation each case
launches (raster_go / walk_go in csrc/b2d_kernels.cu); tests/test_campaign_levels.py checks that the cases of
tests/test_gpu_campaign_levels.py reach all of them."""
import argparse
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

SMS = 132                           # SMs of an H100 SXM: a background walk of more frames runs as a persistent grid
GUARD = 4096                        # poisoned bytes before and after every device output
MAX_PIXELS = 48_000_000             # oracle pixels per case (n * W * H), so that a case stays around a second
NAMES = ("E1M1", "E2M3", "MAP05", "MAP15", "MAP25")

# entry points: name -> (per-frame levels, per-frame states, walk in the background (b2d_walk_device*), host frames)
ENTRIES = {
    "render_levels_states": (True, True, False, True),
    "render_device_levels_states": (True, True, False, False),
    "walk_device_levels_states": (True, True, True, False),
    "render_levels": (True, False, False, True),
    "render_device_levels": (True, False, False, False),
    "walk_device_levels": (True, False, True, False),
    "sharded_levels_states": (True, True, True, False),
    "render": (False, False, False, True),
    "walk_device": (False, False, True, False),
    "render_states": (False, True, False, True),
    "walk_device_states": (False, True, True, False),
}


# ---- the dispatch rule, restated --------------------------------------------------------------------------------------
def raster_cell(width, rgba, masked, states, levels):
    """the b2d_raster_kernel<kRgba, kW, kMasked, kStates, kLevels> raster_go launches: RGBA frames take the 1920-column
    or the generic kernel, index frames the 1920-, the 3840-column or the generic one"""
    kw = 1920 if width == 1920 else (3840 if width == 3840 and not rgba else 0)
    return (bool(rgba), kw, bool(masked), bool(states), bool(levels))


def walk_cell(states, levels, background, n, sms=SMS):
    """the b2d_walk_kernel<kStates, kLevels> walk_go launches, and whether as a persistent grid (a background walk of more
    frames than SMs) or one CTA per frame"""
    return (bool(states), bool(levels), bool(background and n > sms))


ALL_RASTER = {raster_cell(w, rgba, m, s, lv) for w in (1920, 3840, 0) for rgba in (False, True) for m in (False, True)
              for s in (False, True) for lv in (False, True) if not (rgba and w == 3840)}
ALL_WALK = {(s, lv, p) for s in (False, True) for lv in (False, True) for p in (False, True)}


def batch_sizes(case):
    """frames per walk of the case's entry point"""
    n, mb, entry = case["n"], case["max_batch"], case["entry"]
    if entry == "sharded_levels_states":
        from rust_doom_b200 import parallel
        return [c for _, c in parallel.sharded_schedule(n, 1, case["chunk"], mb)[1]]
    if ENTRIES[entry][2]:
        return [case["walk_batch"]] * (n // case["walk_batch"])
    return [min(mb, n - i) for i in range(0, n, mb)]


def cells(case, info):
    """(raster cells, walk cells) the case launches; info = [(masked, timed)] of its levels"""
    levels, states, background, _ = ENTRIES[case["entry"]]
    if not levels:
        states = states and info[0][1]          # level 0 without a state: its per-frame-state calls take the plain kernels
    masked = any(m for m, _ in info) if levels else info[0][0]
    rgba = case["rgba"] and case["entry"] != "sharded_levels_states"
    raster = {raster_cell(case["w"], rgba, masked, states, levels)}
    walk = {walk_cell(states, levels, background, b) for b in batch_sizes(case)}
    return raster, walk


# ---- the cases --------------------------------------------------------------------------------------------------------
def _level_spec(rng, masked):
    g = (int(rng.integers(4, 17)), int(rng.integers(4, 17))) if masked else (int(rng.integers(2, 17)), int(rng.integers(2, 17)))
    cfg = dict(gx=g[0], gy=g[1], origin=(-128 * g[0], -128 * g[1]),
               mid_pct=int(rng.integers(15, 50)) if masked else 0, thing_pct=int(rng.integers(15, 60)) if masked else 0,
               anim=bool(rng.integers(0, 2)), odd_tex=bool(rng.integers(0, 2)), rock_pct=int(rng.integers(5, 30)),
               sky_pct=int(rng.integers(0, 40)), door_pct=int(rng.integers(5, 40)), light_fx=bool(rng.integers(0, 2)))
    return dict(seed=int(rng.integers(100, 100000)), name=NAMES[int(rng.integers(0, len(NAMES)))], cfg=cfg,
                other_palette=bool(rng.random() < 0.3), ndyn=int(rng.integers(1, 17)) if rng.random() < 0.5 else 0)


def _view(rng, max_pixels):
    import rust_doom_b200 as b2d
    while True:
        u = rng.random()
        w = 1920 if u < 0.2 else 3840 if u < 0.35 else int(rng.integers(1, 4097))
        h = int(rng.integers(2, max(3, min(2161, max_pixels // w + 1))))
        fov = float(rng.uniform(1.0, 170.0)) if rng.random() < 0.3 else float(rng.uniform(40.0, 110.0))
        try:
            b2d.make_view(w, h, fov)
        except b2d.B2dError:
            continue                                    # outside what b2d_view_init accepts: draw again
        return w, h, fov


def draw_case(seed, k):
    """case k of a campaign seeded `seed` (a dict; the frames' levels, states and poses are drawn from case["seed"] when the
    case runs)"""
    rng = np.random.default_rng([seed, k])
    nlev = int(rng.integers(1, 9))
    masked_set = bool(rng.integers(0, 2))               # a set with masked content, or none at all
    first = int(rng.integers(0, nlev))
    levels = [_level_spec(rng, masked_set and (j == first or rng.random() < 0.4)) for j in range(nlev)]
    entry = list(ENTRIES)[int(rng.integers(0, len(ENTRIES)))]
    walked = ENTRIES[entry][2] and entry != "sharded_levels_states"
    big = walked and rng.random() < 0.3                 # more frames than SMs: the persistent background walk
    w, h, fov = _view(rng, MAX_PIXELS // (SMS + 40) if big else MAX_PIXELS)
    case = dict(seed=int(rng.integers(0, 1 << 31)), levels=levels, w=w, h=h, fov=fov, entry=entry,
                rgba=bool(rng.random() < 0.35), lut=bool(rng.random() < 0.5), lut_offset=4 * int(rng.integers(0, 4)),
                chunk=int(rng.integers(0, 12)))
    cap = max(1, MAX_PIXELS // (w * h))
    if walked:
        wb = min(int(rng.integers(SMS + 1, SMS + 40)) if big else int(rng.integers(1, 24)), cap)
        nb = max(1, min(int(rng.integers(1, 4)), cap // wb))
        case.update(walk_batch=wb, n=wb * nb, max_batch=wb + int(rng.integers(0, 3)))
    else:
        n = min(int(rng.integers(1, 24)), cap)
        mb = int(rng.integers(1, n + 1)) if rng.random() < 0.4 else n + int(rng.integers(0, 4))
        case.update(n=n, max_batch=mb)
    return case


def _set_spec(seed, masked, n_levels, timed=True):
    """n_levels levels, the first of them masked if `masked` (a forced case's set)"""
    rng = np.random.default_rng(seed)
    out = []
    for j in range(n_levels):
        L = _level_spec(rng, masked and j == 0)
        if timed and j == 0:
            L["cfg"]["light_fx"] = True
        out.append(L)
    return out


def forced_case(entry, w, h, masked, n=2, rgba=False, n_levels=3, seed=1, **kw):
    case = dict(seed=seed, levels=_set_spec(seed, masked, n_levels), w=w, h=h, fov=65.0, entry=entry, rgba=rgba, lut=False,
                lut_offset=0, chunk=0, n=n, max_batch=n)
    if ENTRIES[entry][2] and entry != "sharded_levels_states":
        case["walk_batch"] = n
    case.update(kw)
    return case


def forced_cases():
    """full-size frames the random draw reaches rarely: 3840 x 2160 index frames and 1920 x 1080 frames on sets without
    masked content"""
    out = []
    for i, (entry, masked) in enumerate([("render_device_levels_states", True), ("walk_device_levels_states", False),
                                          ("render_device_levels", True), ("render_levels", False)]):
        out.append(forced_case(entry, 3840, 2160, masked, seed=10 + i))
    for i, (entry, rgba) in enumerate([("render_device_levels_states", False), ("render_levels_states", True),
                                        ("render_device_levels", False), ("render_levels", True)]):
        out.append(forced_case(entry, 1920, 1080, False, rgba=rgba, seed=20 + i))
    return out


def missing_cells(cases, infos):
    """(raster cells, walk cells) that none of `cases` launches"""
    hit_r, hit_w = set(), set()
    for c, info in zip(cases, infos):
        r, w = cells(c, info)
        hit_r |= r
        hit_w |= w
    return ALL_RASTER - hit_r, ALL_WALK - hit_w


def cell_case(cell, seed):
    """a small case that launches raster cell (rgba, kW, masked, states, levels) or walk cell (states, levels, persistent)"""
    if len(cell) == 5:
        rgba, kw, masked, states, levels = cell
        entry = ("render_device_levels_states" if states else "render_device_levels") if levels else \
            ("render_states" if states else "render")
        return forced_case(entry, kw or 200, 24, masked, rgba=rgba, seed=seed, n=3, n_levels=2 if levels else 1)
    states, levels, persistent = cell
    entry = {(True, True): "walk_device_levels_states", (False, True): "walk_device_levels",
             (True, False): "walk_device_states", (False, False): "walk_device"}[(states, levels)]
    if not persistent:
        entry = {(True, True): "render_device_levels_states", (False, True): "render_device_levels",
                 (True, False): "render_states", (False, False): "render"}[(states, levels)]
    return forced_case(entry, 64, 40, False, n=SMS + 5 if persistent else 3, seed=seed, n_levels=2 if levels else 1)


# ---- the levels -------------------------------------------------------------------------------------------------------
def level_data(spec):
    """the WAD bytes of a level spec (a level whose walk tables are too large for the per-frame-level walk is drawn again
    at half the size)"""
    import rust_doom_b200 as b2d
    from rust_doom_b200 import synthwad
    from tests.test_gpu_levels import _other_palette
    from tests.test_scale import walk_smem_bytes
    cfg = dict(spec["cfg"])
    while True:
        data = synthwad.build_iwad(spec["seed"], (spec["name"],), cfg=synthwad.SynthConfig(**cfg))
        if spec["other_palette"]:
            data = _other_palette(data)
        if walk_smem_bytes(b2d.Scene(b2d.Archive.from_bytes(data), 0).blob) <= 200 * 1024:
            return data
        cfg["gx"], cfg["gy"] = max(2, cfg["gx"] // 2), max(2, cfg["gy"] // 2)
        cfg["origin"] = (-128 * cfg["gx"], -128 * cfg["gy"])


def blob_info(blob):
    """(masked content, timed): b2d_api.cu create_level's masked arena and scene_is_timed, restated on the blob header"""
    from oracle import scene as S
    h = S.header(blob)
    n = h[S.H_NSECTORS]
    lights = np.frombuffer(blob, "<u4", 8 * n, h[S.H_OFF_LIGHTS]).reshape(n, 8)[:, 0] if n else np.zeros(0, np.uint32)
    scrolls = bool((S.section(blob, "segs")[:, 3] & S.SEG_SCROLL).any()) if h[S.H_NSEGS] else False
    timed = h[S.H_NANIM] > 0 or h[S.H_NDYN] > 0 or bool((lights != S.LIGHT_NONE).any()) or scrolls
    return h[S.H_NMIDS] > 0 or h[S.H_NSPRITES] > 0, bool(timed)


def prepare_level(spec):
    """{data, dyn, doors, blob (oracle)} of a level spec: what a worker process builds"""
    from oracle import scene as S, wad as W
    from tests.test_scene import declare_doors
    data = level_data(spec)
    a = W.Archive(data)
    dyn, doors = declare_doors(W.Level(a, 0), spec["seed"], spec["ndyn"]) if spec["ndyn"] else ([], [])
    return dict(data=data, dyn=dyn, doors=doors, blob=S.compile_scene(a, W.TextureDirectory(a), 0, dynamic=dyn))


def prepare_case(case):
    return [prepare_level(L) for L in case["levels"]]


def build_levels(prepared):
    """the prepared levels with their oracle Level and product Scene"""
    import rust_doom_b200 as b2d
    from oracle import wad as W
    out = []
    for L in prepared:
        L = dict(L, level=W.Level(W.Archive(L["data"]), 0), scene=b2d.Scene(b2d.Archive.from_bytes(L["data"]), 0, dynamic=L["dyn"]))
        assert L["scene"].blob == L["blob"], "the product's scene compiler differs from the oracle's"
        out.append(L)
    return out


_INFO = {}


def case_info(case):
    """[(masked, timed)] of the case's levels, without a GPU"""
    import rust_doom_b200 as b2d
    from oracle import wad as W
    from tests.test_scene import declare_doors
    out = []
    for spec in case["levels"]:
        key = repr(spec)
        if key not in _INFO:
            data = level_data(spec)
            dyn = declare_doors(W.Level(W.Archive(data), 0), spec["seed"], spec["ndyn"])[0] if spec["ndyn"] else []
            _INFO[key] = blob_info(b2d.Scene(b2d.Archive.from_bytes(data), 0, dynamic=dyn).blob)
        out.append(_INFO[key])
    return out


# ---- one case ---------------------------------------------------------------------------------------------------------
def _moves_choices(L, rng):
    """move lists of a level with dynamic sectors: at rest, range endpoints, doors shut, a random state (holes allowed)"""
    from tests.refcheck import moves as MV
    secs = L["level"].sectors
    ends = []
    for (s, fmin, fmax, cmin, cmax) in L["dyn"]:
        f0, c0 = int(secs[s]["floor"]), int(secs[s]["ceil"])
        f1, c1 = (fmin, fmax)[int(rng.integers(0, 2))], (cmin, cmax)[int(rng.integers(0, 2))]
        f1 = min(f1, c1)
        if fmin <= f1 <= fmax and cmin <= c1 <= cmax:
            ends.append((s, f1 - f0, c1 - c0))
    return [[], ends, [(s, 0, f0 - c0) for (s, f0, c0) in L["doors"]],
            MV.state(L["level"], L["dyn"], int(rng.integers(0, 1 << 30)), hole_free=False)]


def _draw_frames(case, lvs, levels_arg):
    """(frame levels, tics, moves, poses, renderer time, renderer moves per level) of a case"""
    from tests.conftest import sample_poses
    from tests.test_scene import EDGE_TICS
    import rust_doom_b200 as b2d
    rng = np.random.default_rng([case["seed"], 1])
    n, nlev = case["n"], len(lvs)
    lv = rng.integers(0, nlev, n) if levels_arg else np.zeros(n, np.int64)
    if levels_arg and nlev > 1:
        lv[int(rng.integers(0, n))] = nlev - 1          # a frame on the last level
    tics, moves = [], []
    for i in range(n):
        if i and rng.random() < 0.3:                    # a repeat: frames that share a (level, state)
            j = int(rng.integers(0, i))
            lv[i] = lv[j]
            tics.append(tics[j])
            moves.append(moves[j])
            continue
        u = rng.random()
        tics.append(int(rng.integers(0, 1 << 32)) if u < 0.5 else EDGE_TICS[int(rng.integers(0, len(EDGE_TICS)))] if u < 0.8
                    else int(rng.integers(0, 200)))
        L = lvs[int(lv[i])]
        ch = _moves_choices(L, rng) if L["dyn"] else [[]]
        moves.append(ch[int(rng.integers(0, len(ch)))])
    pools = [sample_poses(b2d, L["scene"], max(1, int((lv == k).sum())), case["seed"] + 7 * k) for k, L in enumerate(lvs)]
    poses = np.empty(n, dtype=b2d.POSE_DTYPE)
    used = [0] * nlev
    for i, k in enumerate(lv):
        poses[i] = pools[k][used[k] % len(pools[k])]
        used[k] += 1
    t0 = int(rng.integers(0, 1 << 32)) if rng.random() < 0.7 else EDGE_TICS[int(rng.integers(0, len(EDGE_TICS)))]
    rmoves = {}
    for k, L in enumerate(lvs):
        if L["dyn"]:
            ch = _moves_choices(L, rng)
            rmoves[k] = ch[int(rng.integers(0, len(ch)))]
    return lv.astype(np.uint32), np.array(tics, np.uint64).astype(np.uint32), moves, poses, t0, rmoves


def compact_key(blob, tics, moves):
    """the compact state of b2d_scene.hpp (compact_state), restated: equal keys give one table set"""
    from oracle import scene as S
    h = S.header(blob)
    animates = h[S.H_NANIM] > 0
    scrolls = bool((S.section(blob, "segs")[:, 3] & S.SEG_SCROLL).any()) if h[S.H_NSEGS] else False
    t = int(tics) & 0xFFFFFFFF
    t = t if animates and scrolls else (t & ~7 if animates else (t & 0xFFFFFF if scrolls else 0))
    off = {}
    for s, f, c in moves:
        off[int(s)] = (int(f), int(c))
    moved = tuple(sorted((s, f, c) for s, (f, c) in off.items() if f or c))
    return t, moved, S.sector_lights_at(blob, tics).tobytes()


class _Oracle:
    def __init__(self, lvs, w, h, fov):
        from oracle import render
        self.lvs, self.view, self.blobs = lvs, render.make_view(w, h, fov), {}

    def blob(self, k, moves):
        from oracle import scene as S
        key = (k, tuple(map(tuple, moves)))
        if key not in self.blobs:
            self.blobs[key] = S.apply_moves(self.lvs[k]["blob"], moves) if moves else self.lvs[k]["blob"]
        return self.blobs[key]

    def frames(self, poses, lv, tics, moves, rgba):
        from oracle import render
        n = len(poses)
        idx = np.empty((n, self.view.H, self.view.W), np.uint8)
        col = np.empty((n, self.view.H, self.view.W), np.uint32) if rgba else None
        blobs = [self.blob(int(lv[i]), moves[i]) for i in range(n)]

        def one(i):
            if rgba:
                a, b = render.render(blobs[i], self.view, poses[i:i + 1], tics=int(tics[i]), rgba=True)
                idx[i], col[i] = a[0], b[0]
            else:
                render.render(blobs[i], self.view, poses[i:i + 1], tics=int(tics[i]), out=idx[i:i + 1])

        with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
            list(ex.map(one, range(n)))
        return idx, col


class _Guarded:
    """a device output of `nbytes` at byte offset `offset` inside random poison: GUARD bytes before, the rest of `cap`
    bytes and GUARD bytes after"""

    def __init__(self, nbytes, cap, offset, gen):
        import torch
        self.offset, self.nbytes = GUARD + offset, nbytes
        self.buf = torch.randint(0, 256, (GUARD + offset + max(nbytes, cap) + GUARD,), dtype=torch.uint8, device="cuda",
                                 generator=gen)
        self.ref = self.buf.clone()
        self.ptr = self.buf.data_ptr() + self.offset

    def touched(self):
        """byte offsets (relative to the output) written outside it"""
        bad = (self.buf != self.ref)
        bad[self.offset:self.offset + self.nbytes] = False
        where = bad.nonzero().flatten()
        return [int(x) - self.offset for x in where[:4].cpu()]

    def frames(self, n, h, w, dtype):
        import torch
        out = self.buf[self.offset:self.offset + self.nbytes].cpu().numpy()
        return out.view(np.uint8 if dtype == torch.uint8 else np.uint32).reshape(n, h, w)


_COMM = []


def _comm():
    from rust_doom_b200 import jobs
    if not _COMM:
        _COMM.append(jobs.single_comm(0))
    return _COMM[0]


def run_case(case, lvs=None):
    """-> (list of problems, pixels compared)"""
    import torch
    import rust_doom_b200 as b2d
    from tests.test_gpu_levels_states import check_level_sets
    entry = case["entry"]
    levels_arg, states_arg, background, host = ENTRIES[entry]
    lvs = build_levels(prepare_case(case)) if lvs is None else lvs
    info = [blob_info(L["blob"]) for L in lvs]
    timed = [t for _, t in info]
    w, h, fov, n, mb = case["w"], case["h"], case["fov"], case["n"], case["max_batch"]
    npix = w * h
    problems = []
    lv, tics, moves, poses, t0, rmoves = _draw_frames(case, lvs, levels_arg)
    r = b2d.Renderer.from_levels([L["scene"] for L in lvs], b2d.make_view(w, h, fov), max_batch=mb)
    rgba = case["rgba"] and entry != "sharded_levels_states"
    orc = _Oracle(lvs, w, h, fov)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(case["seed"])
    guards = []
    # the renderer's own state, for the entry points that read it
    if not states_arg:
        r.set_time(t0)
        if not levels_arg:                              # b2d_renderer_set_sector_moves: level 0's
            rmoves = {0: rmoves[0]} if 0 in rmoves else {}
        for k, mv in rmoves.items():
            r.set_level_sector_moves(k, mv)
        tics = np.full(n, t0, np.uint32)
        moves = [rmoves.get(int(k), []) for k in lv]
    # launches: the table set each timed level's worklist slot holds (compact_key), per slot
    slot_key = [{k: compact_key(L["blob"], 0, []) for k, L in enumerate(lvs) if timed[k]} for _ in range(2)]
    ticket = [0]

    def want_launches(sel):
        """launches of one batch (frames `sel`) by DESIGN.md §3"""
        slot = ticket[0] & 1
        ticket[0] += 1
        used = sorted({int(lv[i]) for i in sel})
        if states_arg:
            return 2 + (1 if any(timed[k] for k in used) else 0)
        stale = 0
        for k in used:
            if timed[k]:
                key = compact_key(lvs[k]["blob"], t0, rmoves.get(k, []))
                if slot_key[slot][k] != key:
                    stale += 1
                    slot_key[slot][k] = key
        return 2 + stale

    bsizes = batch_sizes(case)
    starts = np.concatenate([[0], np.cumsum(bsizes)]).astype(int)
    want_l = sum(want_launches(range(starts[b], starts[b + 1])) for b in range(len(bsizes)))
    l0 = r.launch_count
    idx = col = lut = None
    dev_poses = torch.from_numpy(np.ascontiguousarray(poses).view(np.int32).reshape(-1, 4).copy()).cuda()
    dp = dev_poses.data_ptr()
    try:
        if host:
            if entry == "render_levels_states":
                got = r.render_levels_states(poses, lv, tics, moves, rgba=rgba)
            elif entry == "render_levels":
                got = r.render_levels(poses, lv, rgba=rgba)
            elif entry == "render":
                got = r.render(poses, rgba=rgba)
            else:
                got = r.render_states(poses, tics, moves, rgba=rgba)
            idx, col = got if rgba else (got, None)
        elif entry == "sharded_levels_states":
            idx = np.empty((n, h, w), np.uint8)

            class _Dev:
                def __init__(self, ptr, nb):
                    self.__cuda_array_interface__ = {"shape": (nb,), "typestr": "|u1", "data": (ptr, False), "version": 2}

            def on_chunk(k, first, cnt, ptr, ranks, stream):
                with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
                    src = torch.as_tensor(_Dev(ptr, cnt * npix), device="cuda")
                    idx[first:first + cnt] = src.cpu().numpy().reshape(cnt, h, w)
            r.render_sharded_levels_states(_comm(), poses, lv, tics, moves, case["chunk"], on_chunk=on_chunk)
            torch.cuda.synchronize()
            want_l = None
        elif not background:
            gi = _Guarded(n * npix, max(n, mb) * npix, 0, gen)
            gc = _Guarded(n * npix * 4, max(n, mb) * npix * 4, 0, gen) if rgba else None
            guards += [("index", gi)] + ([("rgba", gc)] if gc else [])
            if entry == "render_device_levels_states":
                r.render_device_levels_states(dp, lv, tics, n, gi.ptr, gc.ptr if gc else 0, moves_per_pose=moves)
            else:
                r.render_device_levels(dp, lv, n, gi.ptr, gc.ptr if gc else 0)
            torch.cuda.synchronize()
            idx = gi.frames(n, h, w, torch.uint8)
            col = gc.frames(n, h, w, torch.int32) if gc else None
        else:                                           # walks on a walk stream, rasters alternating two streams
            s_walk, s_r = torch.cuda.Stream(priority=-1), (torch.cuda.Stream(), torch.cuda.Stream())
            outs = [(_Guarded(c * npix, mb * npix, 0, gen), _Guarded(c * npix * 4, mb * npix * 4, 0, gen) if rgba else None)
                    for c in bsizes]
            for gi, gc in outs:
                guards += [("index", gi)] + ([("rgba", gc)] if gc else [])
            torch.cuda.synchronize()

            def walk(b):
                a, c = starts[b], starts[b + 1]
                p = dp + 16 * int(a)
                if entry == "walk_device_levels_states":
                    return r.walk_device_levels_states(p, lv[a:c], tics[a:c], c - a, moves[a:c], s_walk.cuda_stream)
                if entry == "walk_device_levels":
                    return r.walk_device_levels(p, lv[a:c], c - a, s_walk.cuda_stream)
                if entry == "walk_device_states":
                    return r.walk_device_states(p, tics[a:c], c - a, moves[a:c], s_walk.cuda_stream)
                return r.walk_device(p, c - a, s_walk.cuda_stream)
            t = walk(0)
            for b in range(len(bsizes)):
                gi, gc = outs[b]
                r.raster_device(t, gi.ptr, gc.ptr if gc else 0, s_r[b % 2].cuda_stream)
                if b + 1 < len(bsizes):
                    t = walk(b + 1)
            torch.cuda.synchronize()
            idx = np.concatenate([gi.frames(c, h, w, torch.uint8) for (gi, _), c in zip(outs, bsizes)])
            col = np.concatenate([gc.frames(c, h, w, torch.int32) for (_, gc), c in zip(outs, bsizes)]) if rgba else None
        if want_l is not None and r.launch_count - l0 != want_l:
            problems.append("launches %d, DESIGN.md §3 gives %d" % (r.launch_count - l0, want_l))
        st = r.status()
        if st:
            problems.append("status %d" % st)
        # the table sets of the last batch walked with per-frame states and levels
        if levels_arg and states_arg:
            a, c = int(starts[-2]), int(starts[-1])
            check_level_sets(r, lvs, timed, lv[a:c], tics[a:c], moves[a:c], c - a)
        # the palette of each frame's level, on the device, into an output at an offset that may be unaligned
        if case["lut"] and not host and entry != "sharded_levels_states":
            src = torch.from_numpy(np.ascontiguousarray(idx)).cuda()
            gl = _Guarded(n * npix * 4, n * npix * 4, case["lut_offset"], gen)
            guards.append(("palette_lut_levels_device", gl))
            l1 = r.launch_count
            r.palette_lut_levels_device(src.data_ptr(), lv, n, gl.ptr)
            torch.cuda.synchronize()
            if r.launch_count - l1 != 1:
                problems.append("palette_lut_levels_device: %d launches" % (r.launch_count - l1))
            lut = gl.frames(n, h, w, torch.int32).view(np.uint32)
    except BaseException as e:                         # noqa: BLE001 -- a library error or check_level_sets' failure
        if isinstance(e, KeyboardInterrupt):
            raise
        problems.append("%s: %s" % (type(e).__name__, str(e).splitlines()[0] if str(e) else ""))
    if idx is not None:
        want, want_rgba = orc.frames(poses, lv, tics, moves, rgba or lut is not None)
        bad = [(i, int((want[i] != idx[i]).sum())) for i in range(n) if not np.array_equal(want[i], idx[i])]
        if bad:
            problems.append("index frames differ (frame, pixels): %s" % bad[:6])
        for what, got in (("RGBA", col), ("palette_lut_levels_device", lut)):
            if got is not None:
                got = got.view(np.uint32)
                bad = [i for i in range(n) if not np.array_equal(want_rgba[i], got[i])]
                if bad:
                    problems.append("%s frames differ: %s" % (what, bad[:6]))
    for what, g in guards:
        t = g.touched()
        if t:
            problems.append("%s: guard bytes written at offsets %s" % (what, t))
    r.close()
    return problems, n * npix


def describe(case):
    return "%s %dx%d fov %.2f n %d max_batch %d rgba %d lut %d, %d levels (%s)" % (
        case["entry"], case["w"], case["h"], case["fov"], case["n"], case["max_batch"], case["rgba"], case["lut"],
        len(case["levels"]), ", ".join("%s%s%s" % (L["name"], "+mid" if L["cfg"]["mid_pct"] else "", "+dyn" if L["ndyn"] else "")
                                       for L in case["levels"]))


def run(cases, seed=12345, only=None, verbose=False, todo=None):
    """-> (cases run, mismatching cases, pixels compared, seconds); `todo`: [(label, case)] instead of the seeded draw.
    Worker processes generate the levels and the oracle's scenes of the next cases while the GPU renders."""
    import multiprocessing
    t0 = time.time()
    if todo is None:
        todo = [(only, draw_case(seed, only))] if only is not None else [(k, draw_case(seed, k)) for k in range(cases)]
    bad = pixels = 0
    with multiprocessing.get_context("spawn").Pool(max(1, min(8, (os.cpu_count() or 2) - 1))) as pool:
        for (k, case), prepared in zip(todo, pool.imap(prepare_case, [c for _, c in todo])):
            problems, px = run_case(case, build_levels(prepared))
            pixels += px
            if problems:
                bad += 1
                print("MISMATCH --seed %d --case %s: %s" % (seed, k, describe(case)), flush=True)
                for p in problems:
                    print("    " + p, flush=True)
            elif verbose:
                print("ok  case %s: %s" % (k, describe(case)), flush=True)
    return len(todo), bad, pixels, time.time() - t0


def main(cases=None, seed=12345):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("cases", nargs="?", type=int, default=100 if cases is None else cases)
    ap.add_argument("--seed", type=int, default=seed)
    ap.add_argument("--case", type=int, default=None)
    ap.add_argument("-v", action="store_true")
    a = ap.parse_args([] if cases is not None else None)
    n, bad, pixels, secs = run(a.cases, a.seed, a.case, a.v)
    print("level-set campaign: %d cases, %d mismatching, %.1f Mpixel compared, %.1f s" % (n, bad, pixels / 1e6, secs))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
