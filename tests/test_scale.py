"""Scale without a GPU: generated levels whose BSP-walk tables need the kernel's shared-memory opt-in (or do not fit at
all), and subsectors crowded with decoration sprites.  Every level here is first shown to be a valid case -- the
product's scene compiler gives the oracle's blob, and the CPU execution of the kernels' maths (tests/hostcheck) gives
the oracle's frames -- so that tests/test_gpu_scale.py spends GPU time on cases known to be right."""
import functools
import struct

import numpy as np
import pytest

from oracle import render
from oracle import scene as S
from oracle import wad as W
from tests.conftest import oracle_blob, sample_poses

# ---- level size ------------------------------------------------------------------------------------------------------
WALK_SMEM_OPTIN = 48 * 1024      # above this the walk launch must raise cudaFuncAttributeMaxDynamicSharedMemorySize
WALK_SMEM_MAX = 227 * 1024       # the largest opt-in on sm_90a: b2d_renderer_create refuses larger levels
MASK_WORDS = 128                 # b2d_kernels.cu kMaskWords
STACK_DEPTH = 128                # b2d_kernels.cu kStackDepth


def _align16(v: int) -> int:
    return (v + 15) & ~15


def walk_smem_bytes(blob: bytes) -> int:
    """walk_layout() of b2d_kernels.cu from the blob header: the walk kernel's dynamic shared memory per CTA."""
    h = S.header(blob)
    nv, ns, nn, nss, nsp = h[S.H_NVERTS], h[S.H_NSEGS], h[S.H_NNODES], h[S.H_NSSECTORS], h[S.H_NSPRITES]
    o = 0
    for part in (4 * nv, 4 * nv,            # view-space x, z per vertex
                 4 * ns, 8 * nn,            # packed column range per seg, per node child box
                 32 * nn, 16 * nss,         # node lines + children, subsector records (the bulk-copied tables)
                 4 * nsp, 4 * nsp,          # column range and depth per sprite
                 4 * MASK_WORDS, 4 * STACK_DEPTH,
                 2 * (ns + nsp)):           # uint16 worklist indices
        o = _align16(o + part)
    return o


# grid size (gx = gy) -> what the level's walk tables must need; the sizes straddle both limits
SWEEP_GRIDS = {16: (WALK_SMEM_OPTIN, 64 * 1024),          # just over the opt-in
               24: (96 * 1024, 160 * 1024),
               32: (192 * 1024, WALK_SMEM_MAX),           # the largest generated level that still fits
               34: (WALK_SMEM_MAX, 1 << 20)}              # must be refused


@functools.lru_cache(maxsize=None)
def sweep_level(g: int):
    """(wad bytes, oracle blob) of the g x g-cell generated level with sprites and masked middles."""
    from rust_doom_b200 import synthwad
    cfg = synthwad.SynthConfig(gx=g, gy=g, origin=(-128 * g, -128 * g), thing_pct=30, mid_pct=20)
    data = synthwad.build_iwad(1, ("E1M1",), cfg=cfg)
    return data, oracle_blob(data)


def test_sweep_sizes_span_both_limits():
    from rust_doom_b200 import synthwad
    for g, (lo, hi) in SWEEP_GRIDS.items():
        smem = walk_smem_bytes(sweep_level(g)[1])
        assert lo < smem <= hi, "%dx%d level: walk shared memory %d not in (%d, %d]" % (g, g, smem, lo, hi)
    assert walk_smem_bytes(oracle_blob(synthwad.build_iwad(1, ("E1M1",)))) < WALK_SMEM_OPTIN     # the benchmark level


@pytest.mark.parametrize("g", [16, 24, 32])
def test_sweep_level_blob_and_hostcheck_match_oracle(b2d, hostcheck, g):
    data, oblob = sweep_level(g)
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    assert sc.blob == oblob
    poses = sample_poses(b2d, sc, 16, 400 + g)
    ofb = render.render(oblob, render.make_view(320, 200), poses, threads=8)
    hfb, counts, ids = hostcheck(oblob, b2d.make_view(320, 200), poses)
    bad = [(i, int((ofb[i] != hfb[i]).sum())) for i in range(len(poses)) if not np.array_equal(ofb[i], hfb[i])]
    assert not bad, "%dx%d: frames differ (index, pixels): %s" % (g, g, bad[:6])
    assert (counts > 0).all()


def test_sweep_level_over_the_limit_still_compiles(b2d):
    """The 34 x 34 level is a valid level: both compilers accept it (only the renderer refuses it, on the GPU)."""
    data, oblob = sweep_level(34)
    assert b2d.Scene(b2d.Archive.from_bytes(data), 0).blob == oblob


# ---- dense sprite clusters -------------------------------------------------------------------------------------------
DECOR_KINDS = (2035, 48, 34, 2028, 63, 46)     # the generator's decoration kinds that have sprite lumps
CLUSTER_SEED = 5


@functools.lru_cache(maxsize=None)
def _cluster_base():
    """A generated level with sprite lumps, its player-start cell (a plain room cell: one subsector) and that
    subsector's sprite count before anything is added."""
    from rust_doom_b200 import synthwad
    data = synthwad.build_iwad(CLUSTER_SEED, ("E1M1",), cfg=synthwad.SynthConfig(thing_pct=30, mid_pct=20))
    lv = W.Level(W.Archive(data), 0)
    start = next(t for t in lv.things if int(t["type"]) == 1)
    cx, cy = int(start["x"]), int(start["y"])
    ssid, _ = S.subsector_at(lv, float(cx), float(cy))
    return data, (cx, cy), ssid, subsector_sprites(oracle_blob(data), ssid)


def subsector_sprites(blob: bytes, ssid: int) -> int:
    h = S.header(blob)
    rec = np.frombuffer(blob, dtype="<u4", count=4 * h[S.H_NSSECTORS], offset=h[S.H_OFF_SSECTORS]).reshape(-1, 4)
    return int(rec[ssid, 3]) >> 24


def _with_things(data: bytes, extra) -> bytes:
    """The IWAD with 10-byte THINGS records (x, y, angle, type, flags) appended to level 0."""
    from rust_doom_b200 import synthwad
    a = W.Archive(data)
    things = a.levels[0] + 1
    lumps = []
    for k, (name, pos, size) in enumerate(a.lumps):
        body = data[pos:pos + size]
        if k == things:
            body += b"".join(struct.pack("<hhhHH", x, y, 0, kind, 7) for (x, y, kind) in extra)
        lumps.append((name.rstrip(b"\0").decode("ascii"), body))
    return synthwad.assemble_wad(lumps)


def _ties(n: int, c):
    """n things in four columns of equal x (seen from angle 0 they tie in depth).  Thing k and thing k + 32 share x, so
    ties also fall between the walk's 32-wide ranking chunks; in the second column they share y too (same position)."""
    cx, cy = c
    out = []
    for k in range(n):
        x = cx - 30 + 30 * (k % 4)
        y = cy - 90 + 24 * ((k // 4) % 8) + (0 if k % 4 == 1 else 5 * (k // 32))
        out.append((x, y, DECOR_KINDS[k % len(DECOR_KINDS)]))
    return out


def _ring(n: int, c):
    """n things on a circle of radius 80 round the cell centre (viewed from the centre every strip defers only the few
    dozen in the field of view); rounding puts some of them on the same position."""
    cx, cy = c
    return [(cx + int(round(80 * np.cos(2 * np.pi * k / n))), cy + int(round(80 * np.sin(2 * np.pi * k / n))),
             DECOR_KINDS[k % len(DECOR_KINDS)]) for k in range(n)]


def _pile(n: int, c):
    """n things in a 24 x 24 square near the cell's east wall: from the west end of the cell they all fall into the
    same few strips, more than the per-strip cap of 128."""
    cx, cy = c
    return [(cx + 78 + (k * 7) % 24, cy - 12 + (k * 5) % 24, DECOR_KINDS[k % len(DECOR_KINDS)]) for k in range(n)]


LAYOUTS = {"ties": _ties, "ring": _ring, "pile": _pile}


@functools.lru_cache(maxsize=None)
def cluster_level(total: int, layout: str = "ties"):
    """(wad bytes, oracle blob, cell centre, subsector id): the player-start subsector holds exactly `total` sprites."""
    data, c, ssid, before = _cluster_base()
    extra = LAYOUTS[layout](total - before, c)
    out = _with_things(data, extra)
    return out, oracle_blob(out), c, ssid


def cluster_poses(b2d, total: int, layout: str):
    """Poses in the cluster's cell: angle 0 exactly (sinq == 0: equal x is equal depth) and a spread of others."""
    data, blob, (cx, cy), _ = cluster_level(total, layout)
    sc = b2d.Scene(b2d.Archive.from_bytes(data), 0)
    _, floor, _ = sc.sector_at(cx, cy)
    z = floor + 41
    if layout == "ring":
        return np.concatenate([b2d.make_pose(cx + dx, cy + dy, z, a) for a in range(0, 360, 23) for (dx, dy) in ((0, 0), (7, -5))])
    if layout == "pile":
        return np.concatenate([b2d.make_pose(cx - 110, cy + dy, z, a) for dy in (-20, 0, 20) for a in (0, 3.5, -4)])
    return np.concatenate([b2d.make_pose(cx - 110, cy + dy, z, a) for dy in (-40, 0, 40) for a in (0, 15, -15)] +
                          [b2d.make_pose(cx + 110, cy, z, 180), b2d.make_pose(cx, cy - 110, z, 90)])


def test_cluster_levels_hold_the_intended_counts(b2d):
    for total, layout in ((33, "ties"), (64, "ties"), (255, "ring"), (255, "pile")):
        data, blob, _, ssid = cluster_level(total, layout)
        assert subsector_sprites(blob, ssid) == total, (total, layout)
        assert b2d.Scene(b2d.Archive.from_bytes(data), 0).blob == blob


def test_more_than_255_things_in_one_subsector_are_refused(b2d):
    """The count shares a word with the first sprite index: both compilers refuse a 256th thing as a corrupt level."""
    data, c, ssid, before = _cluster_base()
    bad = _with_things(data, _ring(256 - before, c))
    with pytest.raises(W.WadError, match="255"):
        oracle_blob(bad)
    with pytest.raises(b2d.B2dError, match="255") as e:
        b2d.Scene(b2d.Archive.from_bytes(bad), 0)
    assert e.value.code == b2d.ERR_CORRUPT_WAD


@pytest.mark.parametrize("total,layout", [(33, "ties"), (64, "ties"), (255, "ring")])
def test_cluster_hostcheck_matches_oracle(b2d, hostcheck, total, layout):
    """Nearest first with stored order on ties, across 32-wide chunks: the CPU copy of the walk's ranking."""
    _, blob, _, _ = cluster_level(total, layout)
    poses = cluster_poses(b2d, total, layout)
    ofb = render.render(blob, render.make_view(320, 200), poses, threads=8)
    hfb, counts, ids = hostcheck(blob, b2d.make_view(320, 200), poses)
    bad = [(i, int((ofb[i] != hfb[i]).sum())) for i in range(len(poses)) if not np.array_equal(ofb[i], hfb[i])]
    assert not bad, "%d sprites (%s): frames differ (index, pixels): %s" % (total, layout, bad[:6])
    nsprites = [int((ids[i, :counts[i]] < 0).sum()) for i in range(len(poses))]
    assert max(nsprites) > min(total, 40), nsprites


def test_cluster_pile_overflows_the_strip_cap_on_the_cpu(b2d, hostcheck):
    """The pile really defers more than 128 entries in one strip: the CPU copy, which keeps the first 128, differs from
    the oracle (the GPU must report this as status bit 8)."""
    _, blob, _, _ = cluster_level(255, "pile")
    poses = cluster_poses(b2d, 255, "pile")
    ofb = render.render(blob, render.make_view(320, 200), poses, threads=8)
    hfb, _, _ = hostcheck(blob, b2d.make_view(320, 200), poses)
    assert not np.array_equal(ofb, hfb)
