"""b2d -- H100-native software renderer for the Doom-WAD visibility-and-raster hot path.

Host-side mirror of the reference's renderer-facing surface over the C-ABI shared library
`libb2d.so` (include/b2d.h):

    Archive      ~ wad::Archive             (wad/src/archive.rs:36-146)
    Scene        ~ game::WadSystem's level  (game/src/wad_system.rs:18-114) compiled for the GPU
    View         ~ engine::Projection       (engine/src/projections.rs:7-13)
    Renderer     ~ engine::Renderer         (engine/src/renderer.rs:62-175)

Errors surface as B2dError carrying the library's code + message (wad::ErrorKind analogue).
All rendering runs in hand-written sm_90a CUDA kernels; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import numpy as np

from . import _lib

__version__ = "0.1.0"

POSE_DTYPE = np.dtype([("x", "<i4"), ("y", "<i4"), ("z", "<i4"), ("angle", "<u4")])
DEFAULT_FOV_DEG = 65.0          # game/src/player.rs:84

ERR_CORRUPT_WAD, ERR_IO, ERR_CUDA, ERR_INVALID_ARG, ERR_NO_MEMORY = -1, -2, -3, -4, -5


class B2dError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__("b2d error %d: %s" % (code, message))
        self.code = code
        self.message = message


def _check(rc: int) -> int:
    if rc < 0:
        raise B2dError(rc, _lib.load().b2d_last_error().decode("utf-8", "replace"))
    return rc


def wad_name(value: bytes) -> bytes:
    """WadName::from_bytes (wad/src/name.rs:41-75)."""
    out = ctypes.create_string_buffer(8)
    buf = ctypes.create_string_buffer(value, len(value)) if len(value) else ctypes.create_string_buffer(1)
    _check(_lib.load().b2d_wad_name(ctypes.addressof(buf), len(value), out))
    return out.raw


def make_pose(x: float, y: float, z: float, angle_deg: float) -> np.ndarray:
    """One pose record from map-unit floats (quantised to 16.16 / BAM on the host)."""
    p = np.zeros(1, dtype=POSE_DTYPE)
    p["x"] = int(round(x * 65536.0))
    p["y"] = int(round(y * 65536.0))
    p["z"] = int(round(z * 65536.0))
    p["angle"] = int(round(angle_deg / 360.0 * 4294967296.0)) & 0xFFFFFFFF
    return p


class Archive:
    def __init__(self, handle):
        self._h = handle

    @classmethod
    def open(cls, path: str, pwads=()) -> "Archive":
        """IWAD at `path`; `pwads`: PWAD files applied on top, in order (b2d_archive_open_files)."""
        h = ctypes.c_void_p()
        if pwads:
            paths = [path.encode()] + [p.encode() for p in pwads]
            arr = (ctypes.c_char_p * len(paths))(*paths)
            _check(_lib.load().b2d_archive_open_files(arr, len(paths), ctypes.byref(h)))
            return cls(h)
        _check(_lib.load().b2d_archive_open(path.encode(), ctypes.byref(h)))
        return cls(h)

    @classmethod
    def from_bytes(cls, data: bytes, overlays=()) -> "Archive":
        h = ctypes.c_void_p()
        if overlays:
            blobs = [bytes(data)] + [bytes(o) for o in overlays]
            bufs = [(ctypes.c_char * max(len(b), 1)).from_buffer_copy(b.ljust(1, b"\0")) for b in blobs]
            ptrs = (ctypes.c_void_p * len(bufs))(*[ctypes.addressof(b) for b in bufs])
            sizes = (ctypes.c_size_t * len(bufs))(*[len(b) for b in blobs])
            _check(_lib.load().b2d_archive_open_memory_files(ptrs, sizes, len(bufs), ctypes.byref(h)))
            return cls(h)
        buf = (ctypes.c_char * len(data)).from_buffer_copy(data) if len(data) else (ctypes.c_char * 1)()
        _check(_lib.load().b2d_archive_open_memory(ctypes.addressof(buf), len(data), ctypes.byref(h)))
        return cls(h)

    def num_levels(self) -> int:
        return _check(_lib.load().b2d_archive_num_levels(self._h))

    def level_name(self, index: int) -> str:
        out = ctypes.create_string_buffer(9)
        _check(_lib.load().b2d_archive_level_name(self._h, index, out))
        return out.value.decode("ascii")

    def level_names(self):
        return [self.level_name(i) for i in range(self.num_levels())]

    def close(self):
        if self._h:
            _lib.load().b2d_archive_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


def _dynamic_array(dynamic):
    d = list(dynamic)
    arr = (_lib.DynamicSector * max(len(d), 1))()
    for i, (sec, fmin, fmax, cmin, cmax) in enumerate(d):
        arr[i] = _lib.DynamicSector(int(sec), int(fmin), int(fmax), int(cmin), int(cmax))
    return arr, len(d)


def _moves_array(moves):
    m = list(moves)
    arr = (_lib.SectorMove * max(len(m), 1))()
    for i, (sec, dfl, dcl) in enumerate(m):
        arr[i] = _lib.SectorMove(int(sec), int(dfl), int(dcl))
    return arr, len(m)


def _frame_states(tics, moves_per_pose, n: int):
    """(b2d_frame_state array, concatenated move list, its length) for n poses: pose i at level time tics[i] with the
    sector moves moves_per_pose[i] (a list of (sector, floor_offset, ceil_offset); None = every pose at rest)."""
    t = np.ascontiguousarray(tics, dtype=np.uint64).astype(np.uint32) if not np.isscalar(tics) else np.full(n, int(tics) & 0xFFFFFFFF, np.uint32)
    assert len(t) == n, "one tic per pose"
    per = [()] * n if moves_per_pose is None else list(moves_per_pose)
    assert len(per) == n, "one move list per pose"
    states = (_lib.FrameState * max(n, 1))()
    flat = []
    for i in range(n):
        m = list(per[i])
        states[i] = _lib.FrameState(int(t[i]), len(flat), len(m))
        flat += m
    arr, nm = _moves_array(flat)
    return states, arr, nm


def _frame_arrows(arrows, n: int):
    """(b2d_arrow_range array, concatenated b2d_automap_arrow list, its length) for n frames: frame i's arrows arrows[i]
    (an (k, 4) array or a list of (x, y, angle, colour): 16.16 map units, BAM, palette colour; None = none)"""
    per = list(arrows)
    assert len(per) == n, "one arrow list per frame"
    ranges = (_lib.ArrowRange * max(n, 1))()
    flat = []
    for i in range(n):
        a = [] if per[i] is None else np.asarray(per[i], dtype=np.int64).reshape(-1, 4).tolist()
        ranges[i] = _lib.ArrowRange(len(flat), len(a))
        flat += a
    arr = (_lib.AutomapArrow * max(len(flat), 1))()
    for k, (x, y, angle, colour) in enumerate(flat):
        if not (-2 ** 31 <= x < 2 ** 31 and -2 ** 31 <= y < 2 ** 31 and 0 <= colour < 2 ** 32):
            raise B2dError(ERR_INVALID_ARG, "automap arrow out of range")
        arr[k] = _lib.AutomapArrow(int(x), int(y), int(angle) & 0xFFFFFFFF, int(colour))
    return ranges, arr, len(flat)


def _frame_marks(marks, n: int):
    """(b2d_arrow_range array, concatenated b2d_automap_mark list, its length) for n frames: frame i's marks marks[i] (an
    (k, 3) array or a list of (x, y, number): 16.16 map units, digit 0..9; None = none)"""
    per = list(marks)
    assert len(per) == n, "one mark list per frame"
    ranges = (_lib.ArrowRange * max(n, 1))()
    flat = []
    for i in range(n):
        m = [] if per[i] is None else np.asarray(per[i], dtype=np.int64).reshape(-1, 3).tolist()
        ranges[i] = _lib.ArrowRange(len(flat), len(m))
        flat += m
    arr = (_lib.AutomapMark * max(len(flat), 1))()
    for k, (x, y, number) in enumerate(flat):
        if not (-2 ** 31 <= x < 2 ** 31 and -2 ** 31 <= y < 2 ** 31 and 0 <= number < 2 ** 32):
            raise B2dError(ERR_INVALID_ARG, "automap mark out of range")
        arr[k] = _lib.AutomapMark(int(x), int(y), int(number))
    return ranges, arr, len(flat)


def _frame_lights(lights, n: int):
    """b2d_frame_light array for n poses from (fixed_colormap, extralight) pairs, one per pose (a sequence or an (n, 2)
    integer array); the values are checked by the library (fixed_colormap -1..32, extralight 0..2)."""
    a = np.asarray(lights, dtype=np.int64).reshape(-1, 2) if n else np.zeros((0, 2), np.int64)
    assert len(a) == n, "one (fixed_colormap, extralight) pair per pose"
    if n and (a[:, 0].min() < -2 ** 31 or a[:, 0].max() >= 2 ** 31 or a[:, 1].min() < 0 or a[:, 1].max() >= 2 ** 32):
        raise B2dError(ERR_INVALID_ARG, "frame light out of range")
    rec = np.zeros(max(n, 1), dtype=[("fixed_colormap", "<i4"), ("extralight", "<u4")])
    rec["fixed_colormap"][:n], rec["extralight"][:n] = a[:, 0], a[:, 1]
    return (_lib.FrameLight * max(n, 1)).from_buffer_copy(rec.tobytes())


class Scene:
    def __init__(self, archive: Optional[Archive], level_index: int = 0, _handle=None, dynamic=()):
        """`dynamic`: (sector, floor_min, floor_max, ceil_min, ceil_max) per sector that may move (b2d_scene_create_dynamic)"""
        h = _handle if _handle is not None else ctypes.c_void_p()
        if _handle is None:
            arr, n = _dynamic_array(dynamic)
            _check(_lib.load().b2d_scene_create_dynamic(archive._h, level_index, arr, n, ctypes.byref(h)))
        self._h = h
        info = _lib.SceneInfo()
        _check(_lib.load().b2d_scene_info_get(self._h, ctypes.byref(info)))
        self.info = info

    LUMP_ORDER = ("things", "linedefs", "sidedefs", "vertexes", "segs", "ssectors", "nodes", "sectors")

    @classmethod
    def from_lumps(cls, name: bytes, lumps, textures, flats, colormaps, palette: bytes, dynamic=()) -> "Scene":
        """b2d_scene_create_from_lumps: the scene from buffers a host that has already parsed the WAD owns
        (game::WadSystem's pub fields).  lumps: dict of the eight raw level lumps (bytes); textures: iterable of
        (name, uint16 array [h, w], hi byte != 0 = transparent); flats: iterable of (name, 4096 bytes); colormaps:
        iterable of 256-byte rows; palette: 768 bytes (PLAYPAL[0])."""
        keep = []                                             # buffers must outlive the call (they are copied inside)
        ll = _lib.LevelLumps()
        ll.name = name[:8]
        for key in cls.LUMP_ORDER:
            raw = bytes(lumps[key])
            buf = ctypes.create_string_buffer(raw, len(raw)) if raw else None
            keep.append(buf)
            setattr(ll, key, _lib.Lump(ctypes.addressof(buf) if buf is not None else None, len(raw)))
        tex = list(textures)
        imgs = (_lib.ImageDesc * max(len(tex), 1))()
        for i, (nm, px) in enumerate(tex):
            a = np.ascontiguousarray(px, dtype=np.uint16)
            keep.append(a)
            imgs[i].name, imgs[i].width, imgs[i].height, imgs[i].pixels = nm[:8], a.shape[1], a.shape[0], a.ctypes.data
        fl = list(flats)
        fds = (_lib.FlatDesc * max(len(fl), 1))()
        for i, (nm, data) in enumerate(fl):
            b = ctypes.create_string_buffer(bytes(data)[:4096].ljust(4096, b"\0"), 4096)
            keep.append(b)
            fds[i].name, fds[i].pixels = nm[:8], ctypes.addressof(b)
        cm = b"".join(bytes(c)[:256].ljust(256, b"\0") for c in colormaps)
        cmb = ctypes.create_string_buffer(cm, len(cm)) if cm else None
        pal = ctypes.create_string_buffer(bytes(palette)[:768].ljust(768, b"\0"), 768)
        t = _lib.Textures(imgs, len(tex), fds, len(fl), ctypes.addressof(cmb) if cmb is not None else None, len(cm) // 256,
                          ctypes.addressof(pal))
        h = ctypes.c_void_p()
        arr, n = _dynamic_array(dynamic)
        _check(_lib.load().b2d_scene_create_from_lumps_dynamic(ctypes.byref(ll), ctypes.byref(t), arr, n, ctypes.byref(h)))
        del keep
        return cls(None, 0, _handle=h)

    @property
    def num_palettes(self) -> int:
        """b2d_scene_num_palettes: the palettes the scene holds for per-frame palettes (14 for Doom's PLAYPAL)."""
        return _check(_lib.load().b2d_scene_num_palettes(self._h))

    def set_palettes(self, playpal: bytes):
        """b2d_scene_set_palettes: give a scene built from lumps the whole PLAYPAL (n x 768 bytes, n >= 1), whose palette 0
        must equal the one the scene was made with.  Renderers created afterwards see the palettes; existing ones do not."""
        raw = bytes(playpal)
        if not raw or len(raw) % 768:
            raise ValueError("a PLAYPAL is a positive multiple of 768 bytes")
        buf = ctypes.create_string_buffer(raw, len(raw))
        _check(_lib.load().b2d_scene_set_palettes(self._h, buf, len(raw) // 768))

    @property
    def automap_grid_origin(self):
        """b2d_scene_automap_grid_origin: (x, y) in map units, where the automap grid's lines cross (DESIGN.md C22): the
        level's BLOCKMAP origin for an archive scene, (0, 0) for a scene from lumps until set."""
        x, y = ctypes.c_int32(), ctypes.c_int32()
        _check(_lib.load().b2d_scene_automap_grid_origin(self._h, ctypes.byref(x), ctypes.byref(y)))
        return x.value, y.value

    def set_automap_grid_origin(self, x: int, y: int):
        """b2d_scene_set_automap_grid_origin: the grid origin in map units, e.g. the first two int16 of the level's
        BLOCKMAP lump.  Renderers created afterwards see it; existing ones do not."""
        if not (-2 ** 31 <= int(x) < 2 ** 31 and -2 ** 31 <= int(y) < 2 ** 31):
            raise ValueError("grid origin out of the int32 range")
        _check(_lib.load().b2d_scene_set_automap_grid_origin(self._h, int(x), int(y)))

    def tables_at(self, tics: int = 0, moves=()) -> bytes:
        """b2d_scene_tables_at: the state-dependent tables [textures | sectors | segs | sprites | mids] at level time `tics`
        with `moves` = (sector, floor_offset, ceil_offset) applied (host only)."""
        arr, n = _moves_array(moves)
        size = ctypes.c_size_t()
        _check(_lib.load().b2d_scene_tables_at(self._h, tics, arr, n, None, 0, ctypes.byref(size)))
        buf = ctypes.create_string_buffer(max(size.value, 1))
        _check(_lib.load().b2d_scene_tables_at(self._h, tics, arr, n, buf, size.value, ctypes.byref(size)))
        return buf.raw[:size.value]

    def automap_lines(self) -> np.ndarray:
        """b2d_scene_automap_lines: the level's automap table (DESIGN.md C19) as a structured array with fields x0, y0, x1,
        y1 (map units), colour, colour_all (palette indices, 0 = not drawn) and linedef, one record per linedef whose
        vertices exist, in LINEDEFS order."""
        n = ctypes.c_size_t()
        _check(_lib.load().b2d_scene_automap_lines(self._h, None, 0, ctypes.byref(n)))
        buf = (_lib.AutomapLine * max(n.value, 1))()
        _check(_lib.load().b2d_scene_automap_lines(self._h, buf, n.value, ctypes.byref(n)))
        return np.ctypeslib.as_array(buf)[:n.value].copy()

    @property
    def blob(self) -> bytes:
        n = ctypes.c_size_t()
        p = _lib.load().b2d_scene_blob(self._h, ctypes.byref(n))
        return ctypes.string_at(p, n.value)

    @property
    def start_pose(self) -> Optional[np.ndarray]:
        if not self.info.has_start:
            return None
        p = np.zeros(1, dtype=POSE_DTYPE)
        s = self.info.start
        p["x"], p["y"], p["z"], p["angle"] = s.x, s.y, s.z, s.angle
        return p

    def palette_rgb(self) -> np.ndarray:
        """(256, 3) uint8 RGB of PLAYPAL[0] as stored in the scene blob (header word 20 = palette offset)."""
        blob = self.blob
        off = int(np.frombuffer(blob, dtype="<u4", count=21)[20])
        rgba = np.frombuffer(blob, dtype="<u4", count=256, offset=off)
        return np.stack([rgba & 0xFF, (rgba >> 8) & 0xFF, (rgba >> 16) & 0xFF], axis=1).astype(np.uint8)

    def sector_at(self, x: float, y: float) -> Tuple[int, int, int]:
        """(sector id or -1, floor, ceiling) -- LevelWalker::sector_at."""
        f, c = ctypes.c_int32(), ctypes.c_int32()
        sec = _lib.load().b2d_scene_sector_at(self._h, float(x), float(y), ctypes.byref(f), ctypes.byref(c))
        return sec, f.value, c.value

    def close(self):
        if self._h:
            _lib.load().b2d_scene_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


class Comm:
    """One rank of a multi-GPU job: NCCL communicator + registered all-gather buffers + streams (b2d_comm)."""

    def __init__(self, unique_id: bytes, rank: int, world: int, device: int):
        assert len(unique_id) == _lib.COMM_ID_BYTES
        h = ctypes.c_void_p()
        buf = (ctypes.c_char * _lib.COMM_ID_BYTES).from_buffer_copy(unique_id)
        _check(_lib.load().b2d_comm_create(ctypes.addressof(buf), rank, world, device, ctypes.byref(h)))
        self._h = h
        self.rank, self.world, self.device = rank, world, device

    @staticmethod
    def unique_id() -> bytes:
        buf = (ctypes.c_char * _lib.COMM_ID_BYTES)()
        _check(_lib.load().b2d_comm_unique_id(ctypes.addressof(buf)))
        return bytes(buf)

    @property
    def nccl_version(self) -> int:
        v = ctypes.c_int(0)
        _check(_lib.load().b2d_comm_info(self._h, None, None, ctypes.byref(v)))
        return int(v.value)

    def close(self):
        if self._h:
            _lib.load().b2d_comm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


def frame_checksums_device(frames_ptr: int, n_frames: int, frame_bytes: int, out_ptr: int, stream: int = 0):
    """b2d_frame_checksums_device: one uint32 per frame into device memory at out_ptr (see frame_checksum)."""
    _check(_lib.load().b2d_frame_checksums_device(frames_ptr, n_frames, frame_bytes, out_ptr, stream or None))


def frame_checksum(frame: np.ndarray) -> int:
    """Host restatement of the device checksum: sum_i (p[i] + 1) * (i * 0x9E3779B1 + 0x7F4A7C15) mod 2^32."""
    p = np.ascontiguousarray(frame, dtype=np.uint8).reshape(-1).astype(np.uint64)
    i = np.arange(p.size, dtype=np.uint64)
    w = (i * np.uint64(0x9E3779B1) + np.uint64(0x7F4A7C15)) & np.uint64(0xFFFFFFFF)
    return int(((p + np.uint64(1)) * w).sum(dtype=np.uint64) & np.uint64(0xFFFFFFFF))


def make_view(width: int, height: int, fov_deg: float = DEFAULT_FOV_DEG) -> "_lib.View":
    v = _lib.View()
    _check(_lib.load().b2d_view_init(ctypes.byref(v), width, height, float(fov_deg)))
    return v


MAX_LEVELS = 64                 # B2D_MAX_LEVELS

RESOLVE_RGBA8, RESOLVE_RGB8, RESOLVE_RGB8_PLANAR, RESOLVE_GRAY8 = (_lib.RESOLVE_RGBA8, _lib.RESOLVE_RGB8, _lib.RESOLVE_RGB8_PLANAR,
                                                                   _lib.RESOLVE_GRAY8)
RESOLVE_FORMATS = {"rgba": RESOLVE_RGBA8, "rgb": RESOLVE_RGB8, "rgb_planar": RESOLVE_RGB8_PLANAR, "gray": RESOLVE_GRAY8}


AUTOMAP_ROTATE, AUTOMAP_ALL_LINES, AUTOMAP_THINGS = _lib.AUTOMAP_ROTATE, _lib.AUTOMAP_ALL_LINES, _lib.AUTOMAP_THINGS
AUTOMAP_ALLMAP, AUTOMAP_GRID = _lib.AUTOMAP_ALLMAP, _lib.AUTOMAP_GRID
AUTOMAP_FLAGS = {"rotate": AUTOMAP_ROTATE, "all": AUTOMAP_ALL_LINES, "things": AUTOMAP_THINGS, "allmap": AUTOMAP_ALLMAP,
                 "grid": AUTOMAP_GRID}
AUTOMAP_DEFAULT_SCALE_Q16 = 13107       # Doom's default automap scale, 0.2 pixels per map unit


def automap_flags(flags) -> int:
    """B2D_AUTOMAP_* bits from an int, or from names ("rotate", "all", "things", "allmap", "grid") as a list or a
    comma-separated string"""
    if isinstance(flags, int):
        return flags
    names = flags.split(",") if isinstance(flags, str) else list(flags)
    out = 0
    for name in (x.strip() for x in names):
        if name:
            if name not in AUTOMAP_FLAGS:
                raise ValueError("unknown automap flag %r (rotate, all, things, allmap, grid)" % name)
            out |= AUTOMAP_FLAGS[name]
    return out


def seen_lines(row) -> np.ndarray:
    """The linedef indices (ascending) whose bits are set in one row of seen lines (DESIGN.md C20): a numpy or torch
    array of uint32 / int32 words, bit l & 31 of word l >> 5 for linedef l."""
    if hasattr(row, "cpu"):
        row = row.cpu().numpy()
    words = np.ascontiguousarray(row).view(np.uint32).reshape(-1)
    bits = np.unpackbits(words.view(np.uint8), bitorder="little")
    return np.flatnonzero(bits).astype(np.int64)


def _levels_array(levels, n: int) -> np.ndarray:
    """the uint32 level array of n poses (the library refuses an index out of range)"""
    lv = np.asarray(levels, dtype=np.int64).reshape(-1)
    assert lv.shape == (n,), "one level per pose"
    return np.ascontiguousarray(lv & 0xFFFFFFFF, dtype=np.uint32)


def _palettes_array(palettes, n: int) -> Optional[np.ndarray]:
    """the uint32 palette array of n frames, or None (palette 0 everywhere); the library refuses a palette out of range"""
    return None if palettes is None else _levels_array(palettes, n)


def _chunk_fn(on_chunk):
    """the b2d_chunk_fn of a sharded call: on_chunk(chunk_index, first_local_pose, frames_per_rank, device_ptr, ranks, stream)"""
    def tramp(_user, k, first, cnt, ptr, ranks, stream):
        if on_chunk is not None:
            on_chunk(int(k), int(first), int(cnt), int(ptr or 0), int(ranks), int(stream or 0))
    return _lib.CHUNK_FN(tramp)


def _sharded_stats(st) -> dict:
    return {"total_ms": st.total_ms, "render_ms": st.render_ms, "gather_ms": st.gather_ms,
            "frames_local": int(st.frames_local), "frames_gathered": int(st.frames_gathered),
            "chunks": int(st.chunks), "chunk_frames": int(st.chunk_frames), "bytes_received": int(st.bytes_received),
            "registration": st.registration.decode("ascii", "replace")}


class Renderer:
    """Bound to one CUDA device; owns the scene copy in HBM and the per-batch work buffers."""

    def __init__(self, scene: Scene, view, device: int = 0, max_batch: int = 64, _scenes=None):
        h = ctypes.c_void_p()
        scenes = [scene] if _scenes is None else list(_scenes)
        if _scenes is None:
            _check(_lib.load().b2d_renderer_create(scene._h, ctypes.byref(view), device, max_batch, ctypes.byref(h)))
        else:
            arr = (ctypes.c_void_p * max(len(scenes), 1))(*[s._h for s in scenes])
            _check(_lib.load().b2d_renderer_create_levels(arr, len(scenes), ctypes.byref(view), device, max_batch, ctypes.byref(h)))
        self._h = h
        self.view = view
        self.width, self.height = view.width, view.height
        self.max_batch = max_batch
        self.device = device
        self.n_levels = len(scenes)
        self.n_segs = scenes[0].info.n_segs
        # worklist entries per frame: the library's stride, the largest of the levels
        self.worklist_stride = max(1, max(s.info.n_segs + s.info.n_sprites for s in scenes))

    @classmethod
    def from_levels(cls, scenes, view, device: int = 0, max_batch: int = 64) -> "Renderer":
        """b2d_renderer_create_levels: one renderer over a set of levels (1 .. MAX_LEVELS scenes, copied); every call
        without a level argument acts on level 0 (scenes[0])."""
        return cls(None, view, device, max_batch, _scenes=scenes)

    def set_time(self, tics: int):
        """Level time in 1/35 s for the batches walked afterwards (animated flats / walls, scrolling walls, light
        effects).  Host only: nothing is enqueued; a ticket walked before the call keeps its time."""
        _check(_lib.load().b2d_renderer_set_time(self._h, int(tics) & 0xFFFFFFFF))

    def set_time_async(self, tics: int, stream: int = 0):
        """b2d_renderer_set_time_async: the same call (`stream` is ignored)."""
        _check(_lib.load().b2d_renderer_set_time_async(self._h, int(tics) & 0xFFFFFFFF, ctypes.c_void_p(stream)))

    def set_sector_moves(self, moves=(), stream: Optional[int] = None):
        """State of the moving sectors for the batches walked afterwards: (sector, floor_offset, ceil_offset) in map
        units relative to the level lumps; sectors not listed are at rest.  Host only, like set_time; with `stream` it
        calls b2d_renderer_set_sector_moves_async, the same call."""
        arr, n = _moves_array(moves)
        if stream is None:
            _check(_lib.load().b2d_renderer_set_sector_moves(self._h, arr, n))
        else:
            _check(_lib.load().b2d_renderer_set_sector_moves_async(self._h, arr, n, ctypes.c_void_p(stream)))

    def set_level_sector_moves(self, level: int, moves=()):
        """b2d_renderer_set_level_sector_moves: the moving sectors of level `level` for the batches walked afterwards, as
        set_sector_moves does for level 0."""
        arr, n = _moves_array(moves)
        _check(_lib.load().b2d_renderer_set_level_sector_moves(self._h, int(level), arr, n))

    def status(self) -> int:
        """Sticky completeness bits of everything rendered since the last call (0 = every frame complete); synchronises
        the device and clears them.  1 stack overflow, 2 worklist overflow, 4 cyclic BSP, 8 masked-entry overflow."""
        bits = ctypes.c_int32(0)
        _check(_lib.load().b2d_renderer_status(self._h, ctypes.byref(bits)))
        return int(bits.value)

    # -- end to end: host poses in, host frames out -------------------------------------------------
    def render(self, poses: np.ndarray, rgba: bool = False, out_index: Optional[np.ndarray] = None,
               out_rgba: Optional[np.ndarray] = None):
        poses = np.ascontiguousarray(poses, dtype=POSE_DTYPE)
        n = len(poses)
        if out_index is None:
            out_index = np.empty((n, self.height, self.width), dtype=np.uint8)
        if rgba and out_rgba is None:
            out_rgba = np.empty((n, self.height, self.width), dtype=np.uint32)
        _check(_lib.load().b2d_render(self._h, poses.ctypes.data, n, out_index.ctypes.data,
                                      out_rgba.ctypes.data if rgba else None))
        return (out_index, out_rgba) if rgba else out_index

    def render_timed(self, poses: np.ndarray, tics, rgba: bool = False):
        """b2d_render_timed: pose i at level time tics[i] (per-pose time)."""
        poses = np.ascontiguousarray(poses, dtype=POSE_DTYPE)
        t = np.ascontiguousarray(tics, dtype=np.uint32)
        assert len(t) == len(poses)
        n = len(poses)
        out_index = np.empty((n, self.height, self.width), dtype=np.uint8)
        out_rgba = np.empty((n, self.height, self.width), dtype=np.uint32) if rgba else None
        _check(_lib.load().b2d_render_timed(self._h, poses.ctypes.data, t.ctypes.data, n, out_index.ctypes.data,
                                            out_rgba.ctypes.data if rgba else None))
        return (out_index, out_rgba) if rgba else out_index

    def render_device_timed(self, poses_ptr: int, tics, n: int, index_ptr: int, rgba_ptr: int = 0, stream: int = 0):
        t = np.ascontiguousarray(tics, dtype=np.uint32)
        assert len(t) == n
        _check(_lib.load().b2d_render_device_timed(self._h, poses_ptr, t.ctypes.data, n, index_ptr, rgba_ptr or None, stream or None))

    def render_states(self, poses: np.ndarray, tics, moves_per_pose=None, rgba: bool = False):
        """b2d_render_states: pose i at level time tics[i] with the sector moves moves_per_pose[i] (list of (sector,
        floor_offset, ceil_offset); None = at rest) -- a per-frame state, without touching the renderer's own time and moves."""
        poses = np.ascontiguousarray(poses, dtype=POSE_DTYPE)
        n = len(poses)
        states, arr, nm = _frame_states(tics, moves_per_pose, n)
        out_index = np.empty((n, self.height, self.width), dtype=np.uint8)
        out_rgba = np.empty((n, self.height, self.width), dtype=np.uint32) if rgba else None
        _check(_lib.load().b2d_render_states(self._h, poses.ctypes.data, states, n, arr, nm, out_index.ctypes.data,
                                             out_rgba.ctypes.data if rgba else None))
        return (out_index, out_rgba) if rgba else out_index

    def render_device_states(self, poses_ptr: int, tics, n: int, index_ptr: int, rgba_ptr: int = 0, moves_per_pose=None,
                             stream: int = 0):
        """b2d_render_device_states: device poses / frames, per-frame states as in render_states; n may exceed max_batch."""
        states, arr, nm = _frame_states(tics, moves_per_pose, n)
        _check(_lib.load().b2d_render_device_states(self._h, poses_ptr, states, n, arr, nm, index_ptr, rgba_ptr or None,
                                                    stream or None))

    def walk_device_states(self, poses_ptr: int, tics, n: int, moves_per_pose=None, stream: int = 0) -> int:
        """b2d_walk_device_states: the walk of a batch (1..max_batch) with per-frame states; returns the ticket for
        raster_device."""
        states, arr, nm = _frame_states(tics, moves_per_pose, n)
        t = ctypes.c_int64(-1)
        _check(_lib.load().b2d_walk_device_states(self._h, poses_ptr, states, n, arr, nm, stream or None, ctypes.byref(t)))
        return int(t.value)

    def render_levels(self, poses: np.ndarray, levels, rgba: bool = False):
        """b2d_render_levels: pose i rendered from level levels[i], at the renderer's time and that level's sector moves."""
        poses = np.ascontiguousarray(poses, dtype=POSE_DTYPE)
        n = len(poses)
        lv = _levels_array(levels, n)
        out_index = np.empty((n, self.height, self.width), dtype=np.uint8)
        out_rgba = np.empty((n, self.height, self.width), dtype=np.uint32) if rgba else None
        _check(_lib.load().b2d_render_levels(self._h, poses.ctypes.data, lv.ctypes.data, n, out_index.ctypes.data,
                                             out_rgba.ctypes.data if rgba else None))
        return (out_index, out_rgba) if rgba else out_index

    def render_device_levels(self, poses_ptr: int, levels, n: int, index_ptr: int, rgba_ptr: int = 0, stream: int = 0):
        """b2d_render_device_levels: device poses / frames, per-frame levels as in render_levels; n may exceed max_batch."""
        lv = _levels_array(levels, n)
        _check(_lib.load().b2d_render_device_levels(self._h, poses_ptr, lv.ctypes.data, n, index_ptr, rgba_ptr or None,
                                                    stream or None))

    def walk_device_levels(self, poses_ptr: int, levels, n: int, stream: int = 0) -> int:
        """b2d_walk_device_levels: the walk of a batch (1..max_batch) with per-frame levels; returns the ticket for
        raster_device."""
        lv = _levels_array(levels, n)
        t = ctypes.c_int64(-1)
        _check(_lib.load().b2d_walk_device_levels(self._h, poses_ptr, lv.ctypes.data, n, stream or None, ctypes.byref(t)))
        return int(t.value)

    def render_levels_states(self, poses: np.ndarray, levels, tics, moves_per_pose=None, rgba: bool = False, lights=None):
        """b2d_render_levels_states: pose i rendered from level levels[i] at level time tics[i] with the sector moves
        moves_per_pose[i] of that level (None = every pose at rest), without touching the renderer's own time and moves.
        `lights`: None, or one (fixed_colormap, extralight) pair per pose (b2d_render_levels_states_lights, DESIGN.md C18)."""
        poses = np.ascontiguousarray(poses, dtype=POSE_DTYPE)
        n = len(poses)
        lv = _levels_array(levels, n)
        states, arr, nm = _frame_states(tics, moves_per_pose, n)
        out_index = np.empty((n, self.height, self.width), dtype=np.uint8)
        out_rgba = np.empty((n, self.height, self.width), dtype=np.uint32) if rgba else None
        if lights is None:
            _check(_lib.load().b2d_render_levels_states(self._h, poses.ctypes.data, lv.ctypes.data, states, n, arr, nm,
                                                        out_index.ctypes.data, out_rgba.ctypes.data if rgba else None))
        else:
            _check(_lib.load().b2d_render_levels_states_lights(self._h, poses.ctypes.data, lv.ctypes.data, states,
                                                               _frame_lights(lights, n), n, arr, nm, out_index.ctypes.data,
                                                               out_rgba.ctypes.data if rgba else None))
        return (out_index, out_rgba) if rgba else out_index

    def render_device_levels_states(self, poses_ptr: int, levels, tics, n: int, index_ptr: int, rgba_ptr: int = 0,
                                    moves_per_pose=None, stream: int = 0, lights=None):
        """b2d_render_device_levels_states: device poses / frames, per-frame levels and states as in
        render_levels_states; n may exceed max_batch.  `lights` as in render_levels_states."""
        lv = _levels_array(levels, n)
        states, arr, nm = _frame_states(tics, moves_per_pose, n)
        if lights is None:
            _check(_lib.load().b2d_render_device_levels_states(self._h, poses_ptr, lv.ctypes.data, states, n, arr, nm, index_ptr,
                                                               rgba_ptr or None, stream or None))
        else:
            _check(_lib.load().b2d_render_device_levels_states_lights(self._h, poses_ptr, lv.ctypes.data, states,
                                                                      _frame_lights(lights, n), n, arr, nm, index_ptr,
                                                                      rgba_ptr or None, stream or None))

    def walk_device_levels_states(self, poses_ptr: int, levels, tics, n: int, moves_per_pose=None, stream: int = 0,
                                  lights=None) -> int:
        """b2d_walk_device_levels_states: the walk of a batch (1..max_batch) with per-frame levels and states; returns the
        ticket for raster_device.  `lights` as in render_levels_states."""
        lv = _levels_array(levels, n)
        states, arr, nm = _frame_states(tics, moves_per_pose, n)
        t = ctypes.c_int64(-1)
        if lights is None:
            _check(_lib.load().b2d_walk_device_levels_states(self._h, poses_ptr, lv.ctypes.data, states, n, arr, nm,
                                                             stream or None, ctypes.byref(t)))
        else:
            _check(_lib.load().b2d_walk_device_levels_states_lights(self._h, poses_ptr, lv.ctypes.data, states,
                                                                    _frame_lights(lights, n), n, arr, nm, stream or None,
                                                                    ctypes.byref(t)))
        return int(t.value)

    def render_ptr(self, poses_ptr: int, n: int, index_ptr: int, rgba_ptr: int = 0):
        """b2d_render on raw host pointers (e.g. pinned torch tensors)."""
        _check(_lib.load().b2d_render(self._h, poses_ptr, n, index_ptr, rgba_ptr or None))

    # -- device resident ----------------------------------------------------------------------------
    def render_device(self, poses_ptr: int, n: int, index_ptr: int, rgba_ptr: int = 0, stream: int = 0):
        _check(_lib.load().b2d_render_device(self._h, poses_ptr, n, index_ptr, rgba_ptr or None, stream or None))

    def walk_device(self, poses_ptr: int, n: int, stream: int = 0) -> int:
        """BSP walk of a batch on `stream`; returns the ticket to hand to raster_device (possibly on another stream)."""
        t = ctypes.c_int64(-1)
        _check(_lib.load().b2d_walk_device(self._h, poses_ptr, n, stream or None, ctypes.byref(t)))
        return int(t.value)

    def raster_device(self, ticket: int, index_ptr: int, rgba_ptr: int = 0, stream: int = 0):
        _check(_lib.load().b2d_raster_device(self._h, ticket, index_ptr, rgba_ptr or None, stream or None))

    @property
    def seen_words(self) -> int:
        """b2d_renderer_seen_words: uint32 words per row of seen lines (the largest ceil(n_linedefs / 32) of the levels)."""
        w = ctypes.c_uint32()
        _check(_lib.load().b2d_renderer_seen_words(self._h, ctypes.byref(w)))
        return int(w.value)

    def raster_device_seen(self, ticket: int, index_ptr: int, seen_ptr: int, stream: int = 0):
        """b2d_raster_device_seen: raster_device of a ticket of any walk form into index frames only, and frame f's seen
        lines (DESIGN.md C20) OR-ed into row f of the seen rows at seen_ptr (device, seen_words uint32 per row)."""
        _check(_lib.load().b2d_raster_device_seen(self._h, ticket, index_ptr, seen_ptr, stream or None))

    def render_seen(self, poses, levels=None, tics=None, moves_per_pose=None, lights=None, seen=None):
        """Index frames and seen lines of host or CUDA poses, on the current torch stream: each batch of max_batch poses
        walked by the walk its arguments ask for (plain; per-frame `tics` and `moves_per_pose`; per-frame `levels`; both;
        `lights` with both, as in render_levels_states) and rastered by raster_device_seen.  Returns (uint8 tensor
        [n, H, W], int32 tensor [n, seen_words]); with `seen` (a CUDA int32 tensor [n, seen_words]) the frames' seen lines
        are OR-ed into it, and it is returned.  seen_lines() unpacks a row."""
        import torch
        if lights is not None and (levels is None or tics is None):
            raise ValueError("lights come with per-frame levels and tics")
        if moves_per_pose is not None and tics is None:
            raise ValueError("moves_per_pose comes with per-frame tics")
        dev = torch.device("cuda", self.device)
        if isinstance(poses, torch.Tensor):
            p = poses.to(dev).contiguous()
        else:
            p = torch.from_numpy(np.ascontiguousarray(poses, dtype=POSE_DTYPE).view(np.uint8).reshape(-1)).to(dev)
        psize = ctypes.sizeof(_lib.Pose)
        n = p.numel() * p.element_size() // psize
        words = self.seen_words
        if seen is None:
            seen = torch.zeros((n, words), dtype=torch.int32, device=dev)
        elif not (seen.is_cuda and seen.dtype == torch.int32 and tuple(seen.shape) == (n, words) and seen.is_contiguous()):
            raise ValueError("seen must be a contiguous CUDA int32 tensor [%d, %d]" % (n, words))
        out = torch.empty((n, self.height, self.width), dtype=torch.uint8, device=dev)
        lv = None if levels is None else _levels_array(levels, n)
        tc = None if tics is None else np.ascontiguousarray(tics, dtype=np.uint32)
        npix = self.height * self.width
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream().cuda_stream
        for i in range(0, n, self.max_batch):
            k = min(self.max_batch, n - i)
            pp = p.data_ptr() + i * psize
            mv = None if moves_per_pose is None else list(moves_per_pose)[i:i + k]
            lt = None if lights is None else list(lights)[i:i + k]
            if lv is None and tc is None:
                ticket = self.walk_device(pp, k, stream)
            elif lv is None:
                ticket = self.walk_device_states(pp, tc[i:i + k], k, mv, stream)
            elif tc is None:
                ticket = self.walk_device_levels(pp, lv[i:i + k], k, stream)
            else:
                ticket = self.walk_device_levels_states(pp, lv[i:i + k], tc[i:i + k], k, mv, stream, lt)
            self.raster_device_seen(ticket, out.data_ptr() + i * npix, seen.data_ptr() + i * words * 4, stream)
        return out, seen

    def palette_lut_device(self, index_ptr: int, rgba_ptr: int, n_pixels: int, stream: int = 0):
        _check(_lib.load().b2d_palette_lut_device(self._h, index_ptr, rgba_ptr, n_pixels, stream or None))

    def palette_lut_levels_device(self, index_ptr: int, levels, n_frames: int, rgba_ptr: int, stream: int = 0):
        """b2d_palette_lut_levels_device: frame f of the n_frames contiguous index frames at index_ptr through the palette of
        level levels[f] (host list) into rgba_ptr (device pointers)."""
        lv = _levels_array(levels, n_frames)
        _check(_lib.load().b2d_palette_lut_levels_device(self._h, index_ptr, lv.ctypes.data, n_frames, rgba_ptr, stream or None))

    def resolve_device(self, index_ptr: int, n: int, factor: int, fmt: int, out_ptr: int, levels=None, stream: int = 0,
                       palettes=None):
        """b2d_resolve_device: frame f of the n contiguous index frames at index_ptr, box-filtered by `factor` (1..8, dividing
        the view's sides) through the palette of level levels[f] (host list; None = level 0) into out_ptr in format `fmt`
        (RESOLVE_RGBA8 / RESOLVE_RGB8 / RESOLVE_RGB8_PLANAR / RESOLVE_GRAY8; device pointers).  palettes[f] (host list):
        b2d_resolve_palettes_device, frame f through palette palettes[f] of its level (None = palette 0)."""
        lv = None if levels is None else _levels_array(levels, n)
        pv = _palettes_array(palettes, n)
        if pv is None:
            _check(_lib.load().b2d_resolve_device(self._h, index_ptr, None if lv is None else lv.ctypes.data, n, int(factor),
                                                  int(fmt), out_ptr, stream or None))
        else:
            _check(_lib.load().b2d_resolve_palettes_device(self._h, index_ptr, None if lv is None else lv.ctypes.data,
                                                           pv.ctypes.data, n, int(factor), int(fmt), out_ptr, stream or None))

    def resolve_frame_bytes(self, factor: int, fmt: int) -> int:
        """b2d_resolve_frame_bytes: bytes of one resolved frame."""
        out = ctypes.c_size_t()
        _check(_lib.load().b2d_resolve_frame_bytes(self._h, int(factor), int(fmt), ctypes.byref(out)))
        return int(out.value)

    def resolve(self, index, factor: int = 2, fmt: str = "rgb_planar", levels=None, palettes=None):
        """The resolve of a CUDA uint8 tensor [n, H, W] of index frames into a new CUDA tensor, on the current torch stream:
        fmt "rgba" -> int32 [n, H/k, W/k] (RGBA8 words), "rgb" -> uint8 [n, H/k, W/k, 3], "rgb_planar" -> uint8
        [n, 3, H/k, W/k], "gray" -> uint8 [n, H/k, W/k]; `levels` and `palettes` as in resolve_device."""
        import torch
        code = RESOLVE_FORMATS[fmt]
        if not (index.is_cuda and index.dtype == torch.uint8 and index.dim() == 3 and tuple(index.shape[1:]) == (self.height, self.width)):
            raise ValueError("resolve takes a CUDA uint8 tensor [n, %d, %d]" % (self.height, self.width))
        index = index.contiguous()
        n, k = int(index.shape[0]), int(factor)
        oh, ow = (self.height // k, self.width // k) if 1 <= k <= 8 else (0, 0)      # the library refuses other factors
        shape = {_lib.RESOLVE_RGBA8: (n, oh, ow), _lib.RESOLVE_RGB8: (n, oh, ow, 3), _lib.RESOLVE_RGB8_PLANAR: (n, 3, oh, ow),
                 _lib.RESOLVE_GRAY8: (n, oh, ow)}[code]
        out = torch.empty(shape, dtype=torch.int32 if code == _lib.RESOLVE_RGBA8 else torch.uint8, device=index.device)
        with torch.cuda.device(index.device):
            stream = torch.cuda.current_stream().cuda_stream
        self.resolve_device(index.data_ptr(), n, k, code, out.data_ptr(), levels, stream, palettes)
        return out

    def automap_device(self, poses_ptr: int, n: int, out_ptr: int, scale_q16: int = AUTOMAP_DEFAULT_SCALE_Q16,
                       flags: int = 0, levels=None, stream: int = 0, seen_ptr=None, moves_per_pose=None, arrows=None):
        """b2d_automap_device: the automap (DESIGN.md C19) of the n device poses at poses_ptr into n contiguous W x H
        palette-index frames at out_ptr, frame f of level levels[f] (host list; None = level 0), at scale_q16 pixels per map
        unit in 16.16 (256 .. 64 << 16), flags an OR of AUTOMAP_ROTATE, AUTOMAP_ALL_LINES and AUTOMAP_THINGS.  With
        `seen_ptr` (device rows of seen lines, seen_words uint32 per frame) or AUTOMAP_ALLMAP in the flags it calls
        b2d_automap_seen_device: frame f draws the lines row f has mapped (C20; seen_ptr None: every line).  With
        `moves_per_pose` (frame f's sector moves, a list of (sector, floor_offset, ceil_offset) as render_levels_states
        takes them) or `arrows` (frame f's other players' arrows, (x, y, angle, colour) each), either None for none, it
        calls b2d_automap_states_device (C21): the lines coloured at each frame's door and lift state, and the arrows
        drawn after the frame's own."""
        lv = None if levels is None else _levels_array(levels, n)
        lvp = None if lv is None else lv.ctypes.data
        if moves_per_pose is not None or arrows is not None:
            states, mv, nm = _frame_states(0, moves_per_pose, n) if moves_per_pose is not None else (None, None, 0)
            ranges, arr, na = _frame_arrows(arrows, n) if arrows is not None else (None, None, 0)
            _check(_lib.load().b2d_automap_states_device(self._h, poses_ptr, lvp, states, mv, nm, ranges, arr, na, seen_ptr or None,
                                                         n, int(scale_q16), int(flags), out_ptr, stream or None))
        elif seen_ptr is not None or int(flags) & AUTOMAP_ALLMAP:
            _check(_lib.load().b2d_automap_seen_device(self._h, poses_ptr, lvp, seen_ptr or None, n, int(scale_q16), int(flags),
                                                       out_ptr, stream or None))
        else:
            _check(_lib.load().b2d_automap_device(self._h, poses_ptr, lvp, n, int(scale_q16), int(flags), out_ptr, stream or None))

    def automap_marks_device(self, poses_ptr: int, n: int, out_ptr: int, scale_q16: int = AUTOMAP_DEFAULT_SCALE_Q16,
                             flags: int = 0, levels=None, stream: int = 0, seen_ptr=None, moves_per_pose=None, arrows=None,
                             marks=None):
        """b2d_automap_marks_device (DESIGN.md C22): automap_device's state automap, which also takes AUTOMAP_GRID (the
        grid at the level's grid origin, under everything) and `marks`: per frame None or a list of (x, y, number) rows
        (16.16 map units, digit 0..9), drawn over everything with the level's AMMNUM digit patches."""
        lv = None if levels is None else _levels_array(levels, n)
        lvp = None if lv is None else lv.ctypes.data
        states, mv, nm = _frame_states(0, moves_per_pose, n) if moves_per_pose is not None else (None, None, 0)
        ranges, arr, na = _frame_arrows(arrows, n) if arrows is not None else (None, None, 0)
        mranges, marr, nmk = _frame_marks(marks, n) if marks is not None else (None, None, 0)
        _check(_lib.load().b2d_automap_marks_device(self._h, poses_ptr, lvp, states, mv, nm, ranges, arr, na, seen_ptr or None, n,
                                                    int(scale_q16), int(flags), out_ptr, stream or None, mranges, marr, nmk))

    def automap(self, poses, levels=None, scale: float = 0.2, flags=0, seen=None, moves_per_pose=None, arrows=None,
                marks=None):
        """The automaps of host or CUDA poses as a CUDA uint8 tensor [n, H, W] of palette indices, on the current torch
        stream: `scale` in pixels per map unit (Doom's default 0.2), `flags` an int or names from "rotate", "all", "things",
        "allmap".  `seen`: a CUDA int32 tensor [n, seen_words] of seen lines (render_seen), whose mapped lines each frame
        draws (automap_device's seen_ptr).  `moves_per_pose`: each frame's sector moves, the lists render_levels_states
        takes, so each door and lift line has its colour at that frame's state; `arrows`: per frame None or an array of
        (x, y, angle, colour) rows, other players' arrows (DESIGN.md C21).  "grid" in `flags` draws the grid and `marks`
        (per frame None or (x, y, number) rows) the numbered marks (C22, automap_marks_device).  Colour the frames with
        resolve() or palette_lut_levels_device like rendered frames."""
        import torch
        flags = automap_flags(flags)
        dev = torch.device("cuda", self.device)
        if isinstance(poses, torch.Tensor):
            p = poses.to(dev).contiguous()
        else:
            arr = np.ascontiguousarray(poses)
            p = torch.from_numpy(arr.view(np.uint8).reshape(-1)).to(dev)
        n = p.numel() * p.element_size() // ctypes.sizeof(_lib.Pose)
        out = torch.empty((n, self.height, self.width), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream().cuda_stream
        seen_ptr = None
        if seen is not None:
            if not (seen.is_cuda and seen.dtype == torch.int32 and tuple(seen.shape) == (n, self.seen_words) and seen.is_contiguous()):
                raise ValueError("seen must be a contiguous CUDA int32 tensor [%d, %d]" % (n, self.seen_words))
            seen_ptr = seen.data_ptr()
        if flags & AUTOMAP_GRID or marks is not None:
            self.automap_marks_device(p.data_ptr(), n, out.data_ptr(), int(round(scale * 65536)), flags, levels, stream,
                                      seen_ptr, moves_per_pose, arrows, marks)
        else:
            self.automap_device(p.data_ptr(), n, out.data_ptr(), int(round(scale * 65536)), flags, levels, stream, seen_ptr,
                                moves_per_pose, arrows)
        return out

    def worklist(self, n: int):
        counts = np.zeros(n, dtype=np.int32)
        ids = np.full((n, self.worklist_stride), -1, dtype=np.int32)
        _check(_lib.load().b2d_debug_worklist(self._h, n, counts.ctypes.data, ids.ctypes.data, ids.shape[1]))
        return counts, ids

    def state_slots(self, n: int) -> np.ndarray:
        """b2d_debug_state_slots: table-set slot of each of the first n frames of the last batch walked with per-frame states
        (with per-frame levels as well, 0xFFFFFFFF for a frame on a level without a table set)."""
        out = np.zeros(n, dtype=np.uint32)
        _check(_lib.load().b2d_debug_state_slots(self._h, n, out.ctypes.data))
        return out

    def state_tables(self, set: int = 0) -> bytes:
        """b2d_debug_state_tables: table set `set` of the last walked batch, laid out as Scene.tables_at of the set's level
        returns it (a plain batch has the one set 0)."""
        size = ctypes.c_size_t()
        _check(_lib.load().b2d_debug_state_tables(self._h, set, None, 0, ctypes.byref(size)))
        buf = ctypes.create_string_buffer(max(size.value, 1))
        _check(_lib.load().b2d_debug_state_tables(self._h, set, buf, size.value, ctypes.byref(size)))
        return buf.raw[:size.value]

    def profile(self, enable: bool):
        _check(_lib.load().b2d_profile_enable(self._h, 1 if enable else 0))

    def profile_read(self):
        """(walk_ms, raster_ms, batches) summed since the last read; synchronises the device."""
        w, r, b = ctypes.c_double(), ctypes.c_double(), ctypes.c_int64()
        _check(_lib.load().b2d_profile_read(self._h, ctypes.byref(w), ctypes.byref(r), ctypes.byref(b)))
        return w.value, r.value, b.value

    @property
    def launch_count(self) -> int:
        return int(_lib.load().b2d_launch_count(self._h))

    # -- multi-GPU ------------------------------------------------------------------------------------
    def render_sharded(self, comm: "Comm", poses: np.ndarray, chunk_frames: int = 256, mode: int = _lib.SHARD_RENDER_GATHER,
                       on_chunk=None, resolve=None) -> dict:
        """b2d_render_sharded: collective over the communicator.  `poses` is the whole job's pose list (identical on
        every rank); on_chunk(chunk_index, first_local_pose, frames_per_rank, device_ptr, ranks, stream) is called on
        the host after each chunk has been enqueued (work it enqueues on `stream` sees the gathered frames).
        resolve=(factor, fmt), fmt a key of RESOLVE_FORMATS: b2d_render_sharded_resolved, every rank resolves its own
        frames before the exchange and the callback sees resolved frames of resolve_frame_bytes(factor, code) bytes each."""
        poses = np.ascontiguousarray(poses, dtype=POSE_DTYPE)
        st = _lib.ShardedStats()
        if resolve is None:
            _check(_lib.load().b2d_render_sharded(self._h, comm._h, poses.ctypes.data, len(poses), int(chunk_frames), int(mode),
                                                  _chunk_fn(on_chunk), None, ctypes.byref(st)))
        else:
            factor, fmt = resolve
            _check(_lib.load().b2d_render_sharded_resolved(self._h, comm._h, poses.ctypes.data, len(poses), int(chunk_frames),
                                                           int(factor), RESOLVE_FORMATS[fmt], int(mode), _chunk_fn(on_chunk), None,
                                                           ctypes.byref(st)))
        return _sharded_stats(st)

    def render_sharded_levels_states(self, comm: "Comm", poses: np.ndarray, levels, tics, moves_per_pose=None,
                                     chunk_frames: int = 256, mode: int = _lib.SHARD_RENDER_GATHER, on_chunk=None,
                                     resolve=None, palettes=None) -> dict:
        """b2d_render_sharded_levels_states: render_sharded over the renderer's level set, pose i rendered from level
        levels[i] at level time tics[i] with the sector moves moves_per_pose[i] of that level (None = every pose at rest),
        as render_levels_states renders it.  The whole job's lists, identical on every rank.  resolve=(factor, fmt):
        b2d_render_sharded_levels_states_resolved, as in render_sharded, each frame through its own level's palette.
        palettes (with resolve only): b2d_render_sharded_levels_states_resolved_palettes, pose i through palette
        palettes[i] of its level."""
        if palettes is not None and resolve is None:
            raise ValueError("palettes= colours resolved frames: pass resolve=(factor, fmt) with it")
        poses = np.ascontiguousarray(poses, dtype=POSE_DTYPE)
        n = len(poses)
        lv = _levels_array(levels, n)
        pv = _palettes_array(palettes, n)
        states, arr, nm = _frame_states(tics, moves_per_pose, n)
        st = _lib.ShardedStats()
        if pv is not None:
            factor, fmt = resolve
            _check(_lib.load().b2d_render_sharded_levels_states_resolved_palettes(
                self._h, comm._h, poses.ctypes.data, lv.ctypes.data, pv.ctypes.data, states, n, arr, nm, int(chunk_frames),
                int(factor), RESOLVE_FORMATS[fmt], int(mode), _chunk_fn(on_chunk), None, ctypes.byref(st)))
        elif resolve is None:
            _check(_lib.load().b2d_render_sharded_levels_states(self._h, comm._h, poses.ctypes.data, lv.ctypes.data, states, n, arr,
                                                                nm, int(chunk_frames), int(mode), _chunk_fn(on_chunk), None,
                                                                ctypes.byref(st)))
        else:
            factor, fmt = resolve
            _check(_lib.load().b2d_render_sharded_levels_states_resolved(self._h, comm._h, poses.ctypes.data, lv.ctypes.data, states,
                                                                         n, arr, nm, int(chunk_frames), int(factor),
                                                                         RESOLVE_FORMATS[fmt], int(mode), _chunk_fn(on_chunk),
                                                                         None, ctypes.byref(st)))
        return _sharded_stats(st)

    def close(self):
        if self._h:
            _lib.load().b2d_renderer_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass
