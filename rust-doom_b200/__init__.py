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

    def tables_at(self, tics: int = 0, moves=()) -> bytes:
        """b2d_scene_tables_at: the state-dependent tables [textures | sectors | segs | sprites | mids] at level time `tics`
        with `moves` = (sector, floor_offset, ceil_offset) applied (host only)."""
        arr, n = _moves_array(moves)
        size = ctypes.c_size_t()
        _check(_lib.load().b2d_scene_tables_at(self._h, tics, arr, n, None, 0, ctypes.byref(size)))
        buf = ctypes.create_string_buffer(max(size.value, 1))
        _check(_lib.load().b2d_scene_tables_at(self._h, tics, arr, n, buf, size.value, ctypes.byref(size)))
        return buf.raw[:size.value]

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


def _levels_array(levels, n: int) -> np.ndarray:
    """the uint32 level array of n poses (the library refuses an index out of range)"""
    lv = np.asarray(levels, dtype=np.int64).reshape(-1)
    assert lv.shape == (n,), "one level per pose"
    return np.ascontiguousarray(lv & 0xFFFFFFFF, dtype=np.uint32)


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

    def palette_lut_device(self, index_ptr: int, rgba_ptr: int, n_pixels: int, stream: int = 0):
        _check(_lib.load().b2d_palette_lut_device(self._h, index_ptr, rgba_ptr, n_pixels, stream or None))

    def worklist(self, n: int):
        counts = np.zeros(n, dtype=np.int32)
        ids = np.full((n, self.worklist_stride), -1, dtype=np.int32)
        _check(_lib.load().b2d_debug_worklist(self._h, n, counts.ctypes.data, ids.ctypes.data, ids.shape[1]))
        return counts, ids

    def state_slots(self, n: int) -> np.ndarray:
        """b2d_debug_state_slots: table-set slot of each of the first n frames of the last batch walked with per-frame states."""
        out = np.zeros(n, dtype=np.uint32)
        _check(_lib.load().b2d_debug_state_slots(self._h, n, out.ctypes.data))
        return out

    def state_tables(self, set: int = 0) -> bytes:
        """b2d_debug_state_tables: table set `set` of the last walked batch, laid out as Scene.tables_at returns it (a plain
        batch has the one set 0)."""
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
                       on_chunk=None) -> dict:
        """b2d_render_sharded: collective over the communicator.  `poses` is the whole job's pose list (identical on
        every rank); on_chunk(chunk_index, first_local_pose, frames_per_rank, device_ptr, ranks, stream) is called on
        the host after each chunk has been enqueued (work it enqueues on `stream` sees the gathered frames)."""
        poses = np.ascontiguousarray(poses, dtype=POSE_DTYPE)
        st = _lib.ShardedStats()

        def tramp(_user, k, first, cnt, ptr, ranks, stream):
            if on_chunk is not None:
                on_chunk(int(k), int(first), int(cnt), int(ptr or 0), int(ranks), int(stream or 0))

        cb = _lib.CHUNK_FN(tramp)
        _check(_lib.load().b2d_render_sharded(self._h, comm._h, poses.ctypes.data, len(poses), int(chunk_frames), int(mode),
                                              cb, None, ctypes.byref(st)))
        return {"total_ms": st.total_ms, "render_ms": st.render_ms, "gather_ms": st.gather_ms,
                "frames_local": int(st.frames_local), "frames_gathered": int(st.frames_gathered),
                "chunks": int(st.chunks), "chunk_frames": int(st.chunk_frames), "bytes_received": int(st.bytes_received),
                "registration": st.registration.decode("ascii", "replace")}

    def close(self):
        if self._h:
            _lib.load().b2d_renderer_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass
