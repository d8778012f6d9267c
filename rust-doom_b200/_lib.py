"""ctypes binding of libb2d.so (include/b2d.h).  The product has no CPU path: if the library is
missing we try to build it once with nvcc and otherwise fail loudly."""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2D_LIB") or os.path.join(_HERE, "libb2d.so")      # B2D_LIB: A/B another build of the library


class Pose(ctypes.Structure):
    _fields_ = [("x", ctypes.c_int32), ("y", ctypes.c_int32), ("z", ctypes.c_int32), ("angle", ctypes.c_uint32)]


class View(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int32), ("height", ctypes.c_int32), ("F", ctypes.c_int32), ("FY2", ctypes.c_int32)]


class SceneInfo(ctypes.Structure):
    _fields_ = [("n_verts", ctypes.c_int32), ("n_nodes", ctypes.c_int32), ("n_ssectors", ctypes.c_int32),
                ("n_segs", ctypes.c_int32), ("n_sectors", ctypes.c_int32), ("n_textures", ctypes.c_int32),
                ("n_flats", ctypes.c_int32), ("n_masked_mids", ctypes.c_int32), ("n_sprites", ctypes.c_int32),
                ("blob_bytes", ctypes.c_int32), ("has_start", ctypes.c_int32),
                ("start", Pose), ("min_height", ctypes.c_int32), ("max_height", ctypes.c_int32),
                ("n_dynamic", ctypes.c_int32)]


class DynamicSector(ctypes.Structure):
    _fields_ = [("sector", ctypes.c_int32), ("floor_min", ctypes.c_int32), ("floor_max", ctypes.c_int32),
                ("ceil_min", ctypes.c_int32), ("ceil_max", ctypes.c_int32)]


class SectorMove(ctypes.Structure):
    _fields_ = [("sector", ctypes.c_int32), ("floor_offset", ctypes.c_int32), ("ceil_offset", ctypes.c_int32)]


class FrameState(ctypes.Structure):
    """b2d_frame_state: level time + moves[first_move .. first_move + n_moves) of the call's move list"""
    _fields_ = [("tics", ctypes.c_uint32), ("first_move", ctypes.c_uint32), ("n_moves", ctypes.c_uint32)]


class FrameLight(ctypes.Structure):
    """b2d_frame_light: fixed colormap (-1, or a COLORMAP row 0..32) and extra light (0..2) of a frame"""
    _fields_ = [("fixed_colormap", ctypes.c_int32), ("extralight", ctypes.c_uint32)]


EXPORTS = [
    "b2d_last_error", "b2d_archive_open", "b2d_archive_open_memory", "b2d_archive_open_files", "b2d_archive_open_memory_files", "b2d_archive_num_levels",
    "b2d_archive_level_name", "b2d_archive_close", "b2d_wad_name", "b2d_scene_create", "b2d_scene_create_from_lumps", "b2d_scene_create_dynamic",
    "b2d_scene_create_from_lumps_dynamic", "b2d_scene_tables_at", "b2d_renderer_set_sector_moves", "b2d_renderer_set_sector_moves_async", "b2d_scene_info_get",
    "b2d_scene_blob", "b2d_scene_sector_at", "b2d_scene_destroy", "b2d_view_init", "b2d_renderer_create",
    "b2d_renderer_destroy", "b2d_renderer_set_time", "b2d_renderer_set_time_async", "b2d_renderer_status", "b2d_render", "b2d_render_device",
    "b2d_render_timed", "b2d_render_device_timed", "b2d_walk_device",
    "b2d_render_states", "b2d_render_device_states", "b2d_walk_device_states",
    "b2d_renderer_create_levels", "b2d_render_levels", "b2d_render_device_levels", "b2d_walk_device_levels",
    "b2d_renderer_set_level_sector_moves",
    "b2d_render_levels_states", "b2d_render_device_levels_states", "b2d_walk_device_levels_states",
    "b2d_raster_device", "b2d_palette_lut_device",
    "b2d_debug_worklist", "b2d_debug_state_slots", "b2d_debug_state_tables", "b2d_launch_count", "b2d_profile_enable", "b2d_profile_read",
    "b2d_comm_unique_id", "b2d_comm_create", "b2d_comm_destroy", "b2d_comm_info", "b2d_render_sharded",
    "b2d_render_sharded_levels_states", "b2d_palette_lut_levels_device",
    "b2d_frame_checksums_device", "b2d_device_alloc", "b2d_device_free", "b2d_device_upload", "b2d_device_download",
    "b2d_resolve_device", "b2d_resolve_frame_bytes", "b2d_render_sharded_resolved", "b2d_render_sharded_levels_states_resolved",
    "b2d_scene_num_palettes", "b2d_scene_set_palettes", "b2d_resolve_palettes_device",
    "b2d_render_sharded_levels_states_resolved_palettes",
    "b2d_render_levels_states_lights", "b2d_render_device_levels_states_lights", "b2d_walk_device_levels_states_lights",
    "b2d_scene_automap_lines", "b2d_automap_device", "b2d_renderer_seen_words", "b2d_raster_device_seen", "b2d_automap_seen_device",
    "b2d_automap_states_device", "b2d_scene_automap_grid_origin", "b2d_scene_set_automap_grid_origin", "b2d_automap_marks_device",
]

COMM_ID_BYTES = 128
RESOLVE_RGBA8, RESOLVE_RGB8, RESOLVE_RGB8_PLANAR, RESOLVE_GRAY8 = 0, 1, 2, 3      # B2D_RESOLVE_*
SHARD_RENDER_ONLY, SHARD_RENDER_GATHER, SHARD_GATHER_ONLY = 0, 1, 2
AUTOMAP_ROTATE, AUTOMAP_ALL_LINES, AUTOMAP_THINGS, AUTOMAP_ALLMAP, AUTOMAP_GRID = 1, 2, 4, 8, 16      # B2D_AUTOMAP_*


class AutomapLine(ctypes.Structure):
    """b2d_automap_line: a linedef's endpoints (map units), colour drawn normally and under AUTOMAP_ALL_LINES, index"""
    _fields_ = [("x0", ctypes.c_int32), ("y0", ctypes.c_int32), ("x1", ctypes.c_int32), ("y1", ctypes.c_int32),
                ("colour", ctypes.c_uint8), ("colour_all", ctypes.c_uint8), ("pad", ctypes.c_uint16), ("linedef", ctypes.c_int32)]


class AutomapArrow(ctypes.Structure):
    """b2d_automap_arrow: another player's arrow, at (x, y) in 16.16 map units, angle in BAM, palette colour 1..255"""
    _fields_ = [("x", ctypes.c_int32), ("y", ctypes.c_int32), ("angle", ctypes.c_uint32), ("colour", ctypes.c_uint32)]


class ArrowRange(ctypes.Structure):
    """b2d_arrow_range: arrows[first .. first + n) of the call's arrow list"""
    _fields_ = [("first", ctypes.c_uint32), ("n", ctypes.c_uint32)]


class AutomapMark(ctypes.Structure):
    """b2d_automap_mark: a numbered mark at (x, y) in 16.16 map units, drawn with digit patch AMMNUM<number> (0..9)"""
    _fields_ = [("x", ctypes.c_int32), ("y", ctypes.c_int32), ("number", ctypes.c_uint32)]


class ShardedStats(ctypes.Structure):
    _fields_ = [("total_ms", ctypes.c_double), ("render_ms", ctypes.c_double), ("gather_ms", ctypes.c_double),
                ("frames_local", ctypes.c_int64), ("frames_gathered", ctypes.c_int64), ("chunks", ctypes.c_int64),
                ("chunk_frames", ctypes.c_int64), ("bytes_received", ctypes.c_int64),
                ("registration", ctypes.c_char * 64)]


# void fn(void *user, int chunk, size_t first_local_pose, size_t frames_per_rank, const uint8_t *d_frames, int ranks, void *stream)
CHUNK_FN = ctypes.CFUNCTYPE(None, ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p,
                            ctypes.c_int, ctypes.c_void_p)

class Lump(ctypes.Structure):
    _fields_ = [("data", ctypes.c_void_p), ("size", ctypes.c_size_t)]


class LevelLumps(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char * 8)] + [(n, Lump) for n in ("things", "linedefs", "sidedefs", "vertexes", "segs", "ssectors", "nodes", "sectors")]


class ImageDesc(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char * 8), ("width", ctypes.c_int32), ("height", ctypes.c_int32), ("pixels", ctypes.c_void_p)]


class FlatDesc(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char * 8), ("pixels", ctypes.c_void_p)]


class Textures(ctypes.Structure):
    _fields_ = [("textures", ctypes.POINTER(ImageDesc)), ("n_textures", ctypes.c_size_t), ("flats", ctypes.POINTER(FlatDesc)),
                ("n_flats", ctypes.c_size_t), ("colormaps", ctypes.c_void_p), ("n_colormaps", ctypes.c_size_t),
                ("palette", ctypes.c_void_p)]


_lib = None


def load() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        from . import build as _build
        try:
            _build.build()
        except Exception as e:  # noqa: BLE001
            raise ImportError(
                "libb2d.so is missing and could not be built with nvcc (%s). "
                "Run `python -c 'import __graft_entry__ as g; g.build()'`. There is no CPU fallback." % e)
    L = ctypes.CDLL(LIB_PATH)
    vp, ci, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    L.b2d_last_error.restype = ctypes.c_char_p
    L.b2d_archive_open.argtypes = [ctypes.c_char_p, ctypes.POINTER(vp)]
    L.b2d_archive_open_memory.argtypes = [vp, cs, ctypes.POINTER(vp)]
    L.b2d_archive_open_files.argtypes = [ctypes.POINTER(ctypes.c_char_p), ci, ctypes.POINTER(vp)]
    L.b2d_archive_open_memory_files.argtypes = [ctypes.POINTER(vp), ctypes.POINTER(cs), ci, ctypes.POINTER(vp)]
    L.b2d_archive_num_levels.argtypes = [vp]
    L.b2d_archive_level_name.argtypes = [vp, ci, ctypes.c_char_p]
    L.b2d_archive_close.argtypes = [vp]
    L.b2d_archive_close.restype = None
    L.b2d_wad_name.argtypes = [vp, cs, ctypes.c_char_p]
    L.b2d_scene_create.argtypes = [vp, ci, ctypes.POINTER(vp)]
    L.b2d_scene_create_from_lumps.argtypes = [ctypes.POINTER(LevelLumps), ctypes.POINTER(Textures), ctypes.POINTER(vp)]
    L.b2d_scene_create_dynamic.argtypes = [vp, ci, ctypes.POINTER(DynamicSector), cs, ctypes.POINTER(vp)]
    L.b2d_scene_create_from_lumps_dynamic.argtypes = [ctypes.POINTER(LevelLumps), ctypes.POINTER(Textures), ctypes.POINTER(DynamicSector), cs,
                                                      ctypes.POINTER(vp)]
    L.b2d_scene_tables_at.argtypes = [vp, ctypes.c_uint32, ctypes.POINTER(SectorMove), cs, vp, cs, ctypes.POINTER(cs)]
    L.b2d_renderer_set_sector_moves.argtypes = [vp, ctypes.POINTER(SectorMove), cs]
    L.b2d_renderer_set_sector_moves_async.argtypes = [vp, ctypes.POINTER(SectorMove), cs, vp]
    L.b2d_scene_info_get.argtypes = [vp, ctypes.POINTER(SceneInfo)]
    L.b2d_scene_blob.argtypes = [vp, ctypes.POINTER(cs)]
    L.b2d_scene_blob.restype = vp
    L.b2d_scene_sector_at.argtypes = [vp, ctypes.c_double, ctypes.c_double, ctypes.POINTER(ctypes.c_int32),
                                      ctypes.POINTER(ctypes.c_int32)]
    L.b2d_scene_destroy.argtypes = [vp]
    L.b2d_scene_destroy.restype = None
    L.b2d_view_init.argtypes = [ctypes.POINTER(View), ci, ci, ctypes.c_double]
    L.b2d_renderer_create.argtypes = [vp, ctypes.POINTER(View), ci, ci, ctypes.POINTER(vp)]
    L.b2d_renderer_destroy.argtypes = [vp]
    L.b2d_renderer_destroy.restype = None
    L.b2d_renderer_set_time.argtypes = [vp, ctypes.c_uint32]
    L.b2d_renderer_set_time.restype = ctypes.c_int
    L.b2d_renderer_set_time_async.argtypes = [vp, ctypes.c_uint32, vp]
    L.b2d_renderer_set_time_async.restype = ctypes.c_int
    L.b2d_renderer_status.argtypes = [vp, ctypes.POINTER(ctypes.c_int32)]
    L.b2d_renderer_status.restype = ctypes.c_int
    L.b2d_render.argtypes = [vp, vp, cs, vp, vp]
    L.b2d_render_device.argtypes = [vp, vp, cs, vp, vp, vp]
    L.b2d_render_timed.argtypes = [vp, vp, vp, cs, vp, vp]
    L.b2d_render_device_timed.argtypes = [vp, vp, vp, cs, vp, vp, vp]
    L.b2d_render_states.argtypes = [vp, vp, ctypes.POINTER(FrameState), cs, ctypes.POINTER(SectorMove), cs, vp, vp]
    L.b2d_render_device_states.argtypes = [vp, vp, ctypes.POINTER(FrameState), cs, ctypes.POINTER(SectorMove), cs, vp, vp, vp]
    L.b2d_walk_device_states.argtypes = [vp, vp, ctypes.POINTER(FrameState), cs, ctypes.POINTER(SectorMove), cs, vp,
                                         ctypes.POINTER(ctypes.c_int64)]
    L.b2d_renderer_create_levels.argtypes = [ctypes.POINTER(vp), cs, ctypes.POINTER(View), ci, ci, ctypes.POINTER(vp)]
    L.b2d_render_levels.argtypes = [vp, vp, vp, cs, vp, vp]
    L.b2d_render_device_levels.argtypes = [vp, vp, vp, cs, vp, vp, vp]
    L.b2d_walk_device_levels.argtypes = [vp, vp, vp, cs, vp, ctypes.POINTER(ctypes.c_int64)]
    L.b2d_renderer_set_level_sector_moves.argtypes = [vp, ci, ctypes.POINTER(SectorMove), cs]
    L.b2d_render_levels_states.argtypes = [vp, vp, vp, ctypes.POINTER(FrameState), cs, ctypes.POINTER(SectorMove), cs, vp, vp]
    L.b2d_render_device_levels_states.argtypes = [vp, vp, vp, ctypes.POINTER(FrameState), cs, ctypes.POINTER(SectorMove), cs,
                                                  vp, vp, vp]
    L.b2d_walk_device_levels_states.argtypes = [vp, vp, vp, ctypes.POINTER(FrameState), cs, ctypes.POINTER(SectorMove), cs, vp,
                                                ctypes.POINTER(ctypes.c_int64)]
    L.b2d_render_levels_states_lights.argtypes = [vp, vp, vp, ctypes.POINTER(FrameState), ctypes.POINTER(FrameLight), cs,
                                                  ctypes.POINTER(SectorMove), cs, vp, vp]
    L.b2d_render_device_levels_states_lights.argtypes = [vp, vp, vp, ctypes.POINTER(FrameState), ctypes.POINTER(FrameLight),
                                                         cs, ctypes.POINTER(SectorMove), cs, vp, vp, vp]
    L.b2d_walk_device_levels_states_lights.argtypes = [vp, vp, vp, ctypes.POINTER(FrameState), ctypes.POINTER(FrameLight),
                                                       cs, ctypes.POINTER(SectorMove), cs, vp, ctypes.POINTER(ctypes.c_int64)]
    L.b2d_palette_lut_device.argtypes = [vp, vp, vp, cs, vp]
    L.b2d_debug_worklist.argtypes = [vp, cs, vp, vp, cs]
    L.b2d_debug_state_slots.argtypes = [vp, cs, vp]
    L.b2d_debug_state_tables.argtypes = [vp, cs, vp, cs, ctypes.POINTER(cs)]
    L.b2d_profile_enable.argtypes = [vp, ci]
    L.b2d_profile_read.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double),
                                   ctypes.POINTER(ctypes.c_int64)]
    L.b2d_walk_device.argtypes = [vp, vp, ctypes.c_size_t, vp, ctypes.POINTER(ctypes.c_int64)]
    L.b2d_walk_device.restype = ctypes.c_int
    L.b2d_raster_device.argtypes = [vp, ctypes.c_int64, vp, vp, vp]
    L.b2d_raster_device.restype = ctypes.c_int
    L.b2d_launch_count.argtypes = [vp]
    L.b2d_launch_count.restype = ctypes.c_int64
    L.b2d_comm_unique_id.argtypes = [vp]
    L.b2d_comm_create.argtypes = [vp, ci, ci, ci, ctypes.POINTER(vp)]
    L.b2d_comm_destroy.argtypes = [vp]
    L.b2d_comm_destroy.restype = None
    L.b2d_comm_info.argtypes = [vp, ctypes.POINTER(ci), ctypes.POINTER(ci), ctypes.POINTER(ci)]
    L.b2d_render_sharded.argtypes = [vp, vp, vp, cs, cs, ci, CHUNK_FN, vp, ctypes.POINTER(ShardedStats)]
    L.b2d_render_sharded_levels_states.argtypes = [vp, vp, vp, vp, ctypes.POINTER(FrameState), cs, ctypes.POINTER(SectorMove), cs, cs,
                                                   ci, CHUNK_FN, vp, ctypes.POINTER(ShardedStats)]
    L.b2d_palette_lut_levels_device.argtypes = [vp, vp, vp, cs, vp, vp]
    L.b2d_frame_checksums_device.argtypes = [vp, cs, cs, vp, vp]
    L.b2d_resolve_device.argtypes = [vp, vp, vp, cs, ci, ci, vp, vp]
    L.b2d_resolve_frame_bytes.argtypes = [vp, ci, ci, ctypes.POINTER(cs)]
    L.b2d_render_sharded_resolved.argtypes = [vp, vp, vp, cs, cs, ci, ci, ci, CHUNK_FN, vp, ctypes.POINTER(ShardedStats)]
    L.b2d_render_sharded_levels_states_resolved.argtypes = [vp, vp, vp, vp, ctypes.POINTER(FrameState), cs, ctypes.POINTER(SectorMove),
                                                            cs, cs, ci, ci, ci, CHUNK_FN, vp, ctypes.POINTER(ShardedStats)]
    L.b2d_scene_num_palettes.argtypes = [vp]
    L.b2d_scene_set_palettes.argtypes = [vp, vp, cs]
    L.b2d_resolve_palettes_device.argtypes = [vp, vp, vp, vp, cs, ci, ci, vp, vp]
    L.b2d_scene_automap_lines.argtypes = [vp, ctypes.POINTER(AutomapLine), cs, ctypes.POINTER(cs)]
    L.b2d_automap_device.argtypes = [vp, vp, vp, cs, ctypes.c_int32, ci, vp, vp]
    L.b2d_renderer_seen_words.argtypes = [vp, ctypes.POINTER(ctypes.c_uint32)]
    L.b2d_raster_device_seen.argtypes = [vp, ctypes.c_int64, vp, vp, vp]
    L.b2d_raster_device_seen.restype = ctypes.c_int
    L.b2d_automap_seen_device.argtypes = [vp, vp, vp, vp, cs, ctypes.c_int32, ci, vp, vp]
    L.b2d_automap_states_device.argtypes = [vp, vp, vp, ctypes.POINTER(FrameState), ctypes.POINTER(SectorMove), cs,
                                            ctypes.POINTER(ArrowRange), ctypes.POINTER(AutomapArrow), cs, vp, cs, ctypes.c_int32,
                                            ci, vp, vp]
    L.b2d_scene_automap_grid_origin.argtypes = [vp, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]
    L.b2d_scene_set_automap_grid_origin.argtypes = [vp, ctypes.c_int32, ctypes.c_int32]
    L.b2d_automap_marks_device.argtypes = [vp, vp, vp, ctypes.POINTER(FrameState), ctypes.POINTER(SectorMove), cs,
                                           ctypes.POINTER(ArrowRange), ctypes.POINTER(AutomapArrow), cs, vp, cs, ctypes.c_int32,
                                           ci, vp, vp, ctypes.POINTER(ArrowRange), ctypes.POINTER(AutomapMark), cs]
    L.b2d_render_sharded_levels_states_resolved_palettes.argtypes = [vp, vp, vp, vp, vp, ctypes.POINTER(FrameState), cs,
                                                                     ctypes.POINTER(SectorMove), cs, cs, ci, ci, ci, CHUNK_FN, vp,
                                                                     ctypes.POINTER(ShardedStats)]
    _lib = L
    return L
