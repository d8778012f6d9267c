/*
 * b2d.h -- C ABI of the H100-native Doom-WAD software renderer (libb2d.so).
 *
 * The reference (cristicbz/rust-doom) has no FFI or plugin ABI (100% safe Rust, README.md:39).
 * Its renderer-facing seams are Rust-level only; each entry point below names the reference
 * interface it stands in for, so that a Rust `GpuRenderer: engine::System` can bind these with
 * a plain `extern "C"` block (INTEGRATION.md shows that binding):
 *
 *   wad::Archive::open / num_levels / level_lump(i).name()      wad/src/archive.rs:36-60,108-146
 *   game::WadSystem (archive + textures + level)                game/src/wad_system.rs:18-114
 *   wad::LevelWalker::walk + game::level::Builder               wad/src/visitor.rs:541-555,
 *                                                               game/src/level.rs:330-511
 *   game::GameShaders::load_palette / load_level                game/src/game_shaders.rs:123-280
 *   engine::Renderer::update (the per-frame draw loop)          engine/src/renderer.rs:62-175
 *   engine::Projection {fov, aspect, near, far}                 engine/src/projections.rs:7-13,93-101
 *   player start marker                                         wad/src/visitor.rs:1010-1026,
 *                                                               game/src/level.rs:757-762
 *
 * Conventions (mirroring the reference's): every call returns 0 on success or a negative
 * B2D_ERR_* code (wad::ErrorKind::{CorruptWad, Io, ...}, wad/src/errors.rs:9-19); the message is
 * available from b2d_last_error() (thread-local).  Handles are owned by the library and released
 * by the matching *_destroy / *_close.  Input buffers are caller-owned and copied.  A handle may
 * be used from one thread at a time (the reference is single-threaded); distinct handles are
 * independent.  There is NO CPU rendering path in this library: every render entry point runs the
 * CUDA kernels and fails with B2D_ERR_CUDA if no device is usable.
 */
#ifndef B2D_H
#define B2D_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2D_OK 0
#define B2D_ERR_CORRUPT_WAD (-1)
#define B2D_ERR_IO (-2)
#define B2D_ERR_CUDA (-3)
#define B2D_ERR_INVALID_ARG (-4)
#define B2D_ERR_NO_MEMORY (-5)
#define B2D_ERR_NCCL (-6)

typedef struct b2d_archive b2d_archive;     /* wad::Archive */
typedef struct b2d_scene b2d_scene;         /* WadSystem's current level, compiled for the GPU */
typedef struct b2d_renderer b2d_renderer;   /* engine::Renderer replacement, bound to one device */
typedef struct b2d_comm b2d_comm;           /* one rank of a multi-GPU job (NCCL communicator + gather buffers + streams) */

/* Camera pose.  Position in 16.16 fixed-point WAD map units (z = eye height, absolute);
 * angle in BAM (2^32 = 360 deg, 0 = east / +x, counter-clockwise).  Pitch and roll are 0
 * (a column/span renderer is exact only for upright cameras; SURVEY.md 7 "Pitch"). */
typedef struct b2d_pose {
    int32_t x, y, z;
    uint32_t angle;
} b2d_pose;

/* Viewport + projection, all integers so that every consumer sees identical bits.
 * F = round(2*focal_x), FY2 = round(2*focal_y) in pixels, where focal_y = (H/2)/tan(fovy/2) and
 * focal_x = (H/2)/(1.2*tan(fovy/2))  (perspective(fovy, aspect=(W/H)*1.2): player.rs:84-89,339-343).
 * b2d_view_init accepts 1 <= width <= 4096, 2 <= height <= 2160 and 1 < fovy < 170 degrees, as long as
 * width <= 256 * F (a short view at a wide field of view: 4096 x 24 stops at 104 degrees).  The renderers accept
 * hand-built views with the same bounds and 2 <= F, FY2 <= 262144 (2^18; b2d_view_init's largest is FY2 = 247485);
 * anything else is B2D_ERR_INVALID_ARG.  DESIGN.md "Pixel contract" gives the reason for each bound. */
typedef struct b2d_view {
    int32_t width, height, F, FY2;
} b2d_view;

typedef struct b2d_scene_info {
    int32_t n_verts, n_nodes, n_ssectors, n_segs, n_sectors, n_textures, n_flats;
    int32_t n_masked_mids, n_sprites;        /* masked middle textures / decoration things compiled in */
    int32_t blob_bytes;
    int32_t has_start;                       /* player-1 start found */
    b2d_pose start;                          /* spawn camera pose (eye = floor + 62) */
    int32_t min_height, max_height;          /* level height range +-512 (visitor.rs:1173-1182) */
    int32_t n_dynamic;                       /* sectors declared dynamic at creation */
} b2d_scene_info;

const char *b2d_last_error(void);

/* ---- wad::Archive ----------------------------------------------------------------------- */
int b2d_archive_open(const char *wad_path, b2d_archive **out);
int b2d_archive_open_memory(const void *bytes, size_t size, b2d_archive **out);
/* IWAD + PWAD overlays (files[0] is the IWAD, the rest are PWADs applied in order; the reference itself opens IWADs only,
 * wad/src/archive.rs:69-72): PWAD lumps are appended to the directory, so a later lump of a name wins every by-name
 * lookup (PNAMES, TEXTUREx, patches, PLAYPAL ...); a level whose name exists replaces that level in place, new names
 * are appended; flats / sprites between a PWAD's FF_START..FF_END / SS_START..SS_END (or F_/S_) markers join the IWAD's. */
int b2d_archive_open_files(const char *const *paths, int n_paths, b2d_archive **out);
int b2d_archive_open_memory_files(const void *const *bytes, const size_t *sizes, int n_files, b2d_archive **out);
int b2d_archive_num_levels(const b2d_archive *a);
int b2d_archive_level_name(const b2d_archive *a, int level_index, char name_out[9]);
void b2d_archive_close(b2d_archive *a);

/* WadName::from_bytes (wad/src/name.rs:41-75): 0 and the padded upper-cased name, or an error. */
int b2d_wad_name(const void *bytes, size_t size, char name_out[8]);

/* ---- scene (level + textures -> GPU-ready arrays) ------------------------------------------ */
int b2d_scene_create(const b2d_archive *a, int level_index, b2d_scene **out);
/* The same scene from buffers the host already owns -- what a Rust `GpuRenderer: System` has after
 * `WadSystem::create` (game/src/wad_system.rs:18-23,72-114): the level's eight raw lumps (wad::Level keeps exactly
 * these vectors, wad/src/level.rs:22-31) and the TextureDirectory's decoded images (wad/src/tex.rs:109-135:
 * `texture(name)` -> row-major u16 image, a non-zero high byte = transparent, wad/src/image.rs:11-37; `flat(name)` ->
 * 4096 bytes; `colormap(i)`, `palette(0)`).  Nothing is parsed twice: no WAD path, no directory, no PNAMES/TEXTUREx
 * here.  Inputs are caller-owned and copied.  `textures` must hold every wall texture the level's sidedefs name, the
 * level's sky texture and the sprite images of its things (names the level uses but the list lacks render as
 * missing, as in the reference: visitor.rs:857-860); duplicates: the later entry wins (archive.rs:85). */
typedef struct b2d_lump {
    const void *data;
    size_t size;
} b2d_lump;
typedef struct b2d_level_lumps {
    char name[8];               /* level marker name ("E1M1", "MAP01"; NUL padded): selects the sky (wad/src/meta.rs:156-172) */
    b2d_lump things, linedefs, sidedefs, vertexes, segs, ssectors, nodes, sectors;
} b2d_level_lumps;
typedef struct b2d_image {
    char name[8];
    int32_t width, height;
    const uint16_t *pixels;     /* width*height, row-major */
} b2d_image;
typedef struct b2d_flat {
    char name[8];
    const uint8_t *pixels;      /* 4096 bytes */
} b2d_flat;
typedef struct b2d_textures {
    const b2d_image *textures;  /* composed wall textures, then sprites (tex.rs:81-95: one name -> image map) */
    size_t n_textures;
    const b2d_flat *flats;
    size_t n_flats;
    const uint8_t *colormaps;   /* n_colormaps x 256 (COLORMAP; rows 0..31 are used) */
    size_t n_colormaps;
    const uint8_t *palette;     /* 768 bytes: PLAYPAL[0] */
} b2d_textures;
int b2d_scene_create_from_lumps(const b2d_level_lumps *level, const b2d_textures *tex, b2d_scene **out);

/* Moving sectors (doors, lifts, crushers) as a per-batch input.  The reference finds the sectors that may move and their
 * height ranges when it loads a level (`LevelAnalysis`, wad/src/visitor.rs:316-497; ranges: `DynamicSectorInfo`,
 * :159-245), attaches every wall quad, flat and decoration to the floor or ceiling object of a sector (:733-836, :957-983,
 * :1106-1121) and moves those objects from its trigger logic (game/src/level.rs:201-245).  The analysis and the triggers
 * are gameplay and stay on the host; what the renderer takes is their result: the list of dynamic sectors with their
 * ranges at scene creation (pieces that can come into existence while a sector moves are resolved then -- the reference
 * pre-extends its quads over these ranges), and one state per batch: the offset of each moved floor and ceiling from the
 * height in the level lumps, in map units.  A range is widened to contain the sector's own heights (visitor.rs:232-245).
 * Every surface then moves rigidly with the object the reference attaches it to (DESIGN.md C16). */
typedef struct b2d_dynamic_sector {
    int32_t sector;
    int32_t floor_min, floor_max, ceil_min, ceil_max;
} b2d_dynamic_sector;
typedef struct b2d_sector_move {
    int32_t sector;
    int32_t floor_offset, ceil_offset;
} b2d_sector_move;
int b2d_scene_create_dynamic(const b2d_archive *a, int level_index, const b2d_dynamic_sector *dynamic, size_t n_dynamic,
                             b2d_scene **out);
int b2d_scene_create_from_lumps_dynamic(const b2d_level_lumps *level, const b2d_textures *tex,
                                        const b2d_dynamic_sector *dynamic, size_t n_dynamic, b2d_scene **out);
/* The state-dependent tables of a scene at level time `tics` with the given sectors moved, laid out
 * [textures | sectors | segs | sprites | mids] as in the blob (host only, no device needed: the tables a batch at that
 * state reads, which the renderer expands on the device).  out = NULL: only *size_out is set.  A move of an undeclared sector or outside its range (or with the
 * floor above the ceiling) is B2D_ERR_INVALID_ARG. */
int b2d_scene_tables_at(const b2d_scene *s, uint32_t tics, const b2d_sector_move *moves, size_t n_moves, void *out,
                        size_t capacity, size_t *size_out);

int b2d_scene_info_get(const b2d_scene *s, b2d_scene_info *out);
/* Read-only access to the compiled "B2DS" blob (layout in DESIGN.md); valid until destroy. */
const void *b2d_scene_blob(const b2d_scene *s, size_t *size_out);
/* LevelWalker::sector_at (visitor.rs:1028-1060): sector id at a map position, -1 if outside. */
int b2d_scene_sector_at(const b2d_scene *s, double x, double y, int32_t *floor_out, int32_t *ceil_out);
void b2d_scene_destroy(b2d_scene *s);

/* ---- view ------------------------------------------------------------------------------- */
int b2d_view_init(b2d_view *v, int width, int height, double fov_y_degrees);

/* ---- renderer --------------------------------------------------------------------------- */
/* Uploads the scene to `device` and sizes per-batch work buffers for up to max_batch poses. */
int b2d_renderer_create(const b2d_scene *s, const b2d_view *view, int device, int max_batch,
                        b2d_renderer **out);
void b2d_renderer_destroy(b2d_renderer *r);

/* Level time in tics (1/35 s) for every batch rendered afterwards; a new renderer is at tic 0.  Replaces the
 * reference's u_time uniform (game/src/level.rs:257-260, assets/shaders/static.vert:23-39): animated flats and
 * wall textures show frame (tics/8) mod n of their group -- whichever frame name the map uses, because the
 * reference binds every frame name to the group's first frame (wad/src/tex.rs:260, 302-306) -- and walls of
 * scrolling lines (special 0x30, wad/src/visitor.rs:922) shift their texture column by one texel per tic; sector
 * light effects (wad/src/light.rs:27-80) are re-evaluated.  A no-op for levels without time-dependent content.
 *
 * The call records the renderer's state on the host and enqueues nothing; the host never blocks on the device (this is
 * the call for a per-frame System::update loop).  A batch is rendered at the state in force when it is walked
 * (b2d_render*, b2d_walk_device): a ticket walked before the call is rastered at the old state.  The first batch of each
 * of the renderer's two worklist slots after a change costs one more launch, which expands the state's tables (a few
 * KB ... ~200 KB) on the device from a compact state of a few words.  _async is the same call; `cuda_stream` is ignored
 * (kept for compatibility). */
int b2d_renderer_set_time_async(b2d_renderer *r, uint32_t tics, void *cuda_stream);
int b2d_renderer_set_time(b2d_renderer *r, uint32_t tics);
/* The state of the moving sectors for the batches walked after this call (sectors not listed are at rest; n = 0 puts
 * everything back), recorded like b2d_renderer_set_time's; _async is the same call. */
int b2d_renderer_set_sector_moves_async(b2d_renderer *r, const b2d_sector_move *moves, size_t n, void *cuda_stream);
int b2d_renderer_set_sector_moves(b2d_renderer *r, const b2d_sector_move *moves, size_t n);

/* Sticky completeness status of everything rendered since the last call (device-resident entry points do not
 * synchronise, so they cannot report it themselves): synchronises the device, returns the OR of
 *   1 BSP traversal stack overflow   2 worklist overflow   4 BSP traversal did not terminate (cyclic node graph)
 *   8 more masked middles / sprites deferred than the renderer holds (per 32-column strip, or arena exhausted)
 * in *bits_out (0 = every frame complete) and clears it.  b2d_render reports the same bits as an error. */
int b2d_renderer_status(b2d_renderer *r, int32_t *bits_out);

/* End-to-end: HOST poses in, HOST frames out (pinned staging + copies inside).  index_fb gets
 * n*W*H palette indices, row-major, top row first; rgba_fb (nullable) gets n*W*H RGBA8
 * (R in the low byte).  n may exceed max_batch; it is processed in batches. */
int b2d_render(b2d_renderer *r, const b2d_pose *poses, size_t n, uint8_t *index_fb, uint32_t *rgba_fb);

/* Per-frame state: every pose carries its own level time and state of the moving sectors (a demo replay, a recorded
 * session where a door opens while the camera moves, a fly-through with the clock running).  Frame i is byte-identical to
 * what b2d_render_device gives after b2d_renderer_set_time(states[i].tics) and b2d_renderer_set_sector_moves(
 * moves + states[i].first_move, states[i].n_moves).  `states` and `moves` are HOST arrays; the renderer's own per-batch
 * time and moves are neither read nor changed.  A batch costs one walk, one raster and one launch that expands the
 * batch's distinct states on the device into an arena of up to max_batch table sets per worklist slot (allocated by the
 * first such call; frames with equal states share a set wherever they are in the batch; DESIGN.md §3); the host uploads a
 * compact state per distinct state (a few hundred bytes) instead of the tables.  A scene without time-dependent content
 * or dynamic sectors renders every batch as b2d_render_device does (two launches).  Moves of undeclared sectors or outside
 * their range, move ranges past n_moves and a NULL `states` are B2D_ERR_INVALID_ARG, detected before anything is enqueued.
 *
 * b2d_render_states: host poses and frames like b2d_render; b2d_render_device_states: like b2d_render_device, n may exceed
 * max_batch (split into batches).  b2d_walk_device_states: like b2d_walk_device (1..max_batch poses); the ticket is
 * rastered by b2d_raster_device, and its table sets live in the ticket's worklist slot until then.  The device-resident
 * calls do not synchronise the device, but before a batch's compact states are written into the worklist slot's pinned
 * staging, the host waits for the copy that read that staging two batches earlier (normally finished long before). */
typedef struct b2d_frame_state {
    uint32_t tics;                    /* level time */
    uint32_t first_move, n_moves;     /* moves[first_move .. first_move + n_moves) of the call's list; n_moves = 0: all at rest */
} b2d_frame_state;
int b2d_render_states(b2d_renderer *r, const b2d_pose *poses, const b2d_frame_state *states, size_t n,
                      const b2d_sector_move *moves, size_t n_moves, uint8_t *index_fb, uint32_t *rgba_fb);
int b2d_render_device_states(b2d_renderer *r, const b2d_pose *d_poses, const b2d_frame_state *states, size_t n,
                             const b2d_sector_move *moves, size_t n_moves, uint8_t *d_index_fb, uint32_t *d_rgba_fb,
                             void *cuda_stream);
int b2d_walk_device_states(b2d_renderer *r, const b2d_pose *d_poses, const b2d_frame_state *states, size_t n,
                           const b2d_sector_move *moves, size_t n_moves, void *cuda_stream, int64_t *ticket_out);

/* Per-pose level time (SURVEY 8-f2: poses (x, y, z, yaw, t)): pose i is rendered at level time tics[i] (HOST array) with
 * the renderer's current sector moves -- b2d_render_states / b2d_render_device_states with those states, so a batch costs
 * the same three launches whatever the timeline (two on a level without time-dependent content).  Leaves the renderer at
 * the last pose's time, as b2d_renderer_set_time does.  tics == NULL in b2d_render_timed is b2d_render. */
int b2d_render_timed(b2d_renderer *r, const b2d_pose *poses, const uint32_t *tics, size_t n, uint8_t *index_fb, uint32_t *rgba_fb);
int b2d_render_device_timed(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *tics, size_t n, uint8_t *d_index_fb,
                            uint32_t *d_rgba_fb, void *cuda_stream);

/* Device-resident: poses, index_fb and rgba_fb (nullable) are DEVICE pointers on the renderer's
 * device; work is enqueued on `cuda_stream` (a cudaStream_t, NULL = default stream) and NOT
 * synchronised.  n <= max_batch. */
int b2d_render_device(b2d_renderer *r, const b2d_pose *d_poses, size_t n, uint8_t *d_index_fb,
                      uint32_t *d_rgba_fb, void *cuda_stream);

/* Kernel 3 on its own: palette lookup index -> RGBA8 for n_pixels device bytes. */
int b2d_palette_lut_device(b2d_renderer *r, const uint8_t *d_index, uint32_t *d_rgba, size_t n_pixels,
                           void *cuda_stream);

/* The same work as b2d_render_device in two calls, for pipelines that have the next batch's poses early (a recorded
 * camera path, an encoder that renders ahead).  b2d_walk_device enqueues the BSP walk of a batch on `cuda_stream` into
 * one of the renderer's two worklist slots and returns a ticket; b2d_raster_device enqueues the raster of that ticket on
 * its own `cuda_stream`.  The two calls are ordered through events, not by the streams: with two streams the walk of
 * batch k+1 overlaps the raster of batch k.  b2d_walk_device launches the walk as a background grid (one CTA per SM
 * looping over the frames): it then takes several frame latencies instead of one but leaves
 * 7/8 of the registers to the raster it runs under.  Rasters of consecutive batches may go to two alternating
 * streams (and output buffers): the first CTAs of batch k+1 then fill the SMs the last CTAs of batch k leave idle.  At
 * most two batches can be walked and not yet rastered; tickets are rastered once.  d_poses is read by the walk
 * only.  Levels with masked middle textures or sprites share one arena of deferred entries per renderer: their rasters are
 * ordered one after the other through an event, whatever streams they are enqueued on.  Replaces nothing in the reference (its render loop is synchronous, engine/src/renderer.rs:62-175). */
int b2d_walk_device(b2d_renderer *r, const b2d_pose *d_poses, size_t n, void *cuda_stream, int64_t *ticket_out);
int b2d_raster_device(b2d_renderer *r, int64_t ticket, uint8_t *d_index_fb, uint32_t *d_rgba_fb, void *cuda_stream);

/* ---- level sets: frames of several levels in one batch --------------------------------------
 * The reference switches levels at run time (game/src/wad_system.rs:37-45, game/src/level.rs:188-197); many agents or
 * cameras may each be on their own map.  A renderer over a set of levels keeps every level resident (its scene, pre-lit
 * planes and walk tables; DESIGN.md §3) and renders each frame of a batch from its own level, in the same two launches per
 * batch as one level: switching levels is a per-frame index, not a new renderer.
 *
 * b2d_renderer_create_levels: a renderer over n_levels scenes (1 <= n_levels <= B2D_MAX_LEVELS) with one view, device and
 * max_batch.  Level k is scenes[k]; the scenes are copied (they may be destroyed afterwards).  Every other entry point acts
 * on level 0, so b2d_renderer_create(s, ...) behaves as a set of one.  b2d_renderer_set_time applies to every level;
 * b2d_renderer_set_sector_moves is b2d_renderer_set_level_sector_moves(r, 0, ...).
 *
 * b2d_render_levels: host poses and frames as b2d_render; frame i is rendered from level levels[i] (HOST array), at the
 * renderer's level time and that level's sector moves, byte-identical to a b2d_renderer_create renderer of that level in
 * the same state.  b2d_render_device_levels: like b2d_render_device, n may exceed max_batch (split into batches).
 * b2d_walk_device_levels: like b2d_walk_device (1..max_batch poses); the ticket is rastered by b2d_raster_device.  A batch
 * costs one walk and one raster whatever the number of levels it mixes, plus, after a change of the time or of a level's
 * moves, one launch per changed level the batch uses (the first batch of each worklist slot).  The device-resident calls
 * do not synchronise the device, but before a batch's levels are written into the worklist slot's pinned staging, the host
 * waits for the copy that read that staging two batches earlier.  A level index >= n_levels, a NULL `levels` or `scenes`
 * entry and n_levels out of range are B2D_ERR_INVALID_ARG, detected before anything is enqueued.  The per-frame-level
 * walk keeps the resident level's description in shared memory next to the walk tables: b2d_renderer_create_levels refuses
 * (B2D_ERR_INVALID_ARG) a level whose walk tables leave no room for it, a level b2d_renderer_create still accepts by a few
 * hundred bytes; the level calls on such a renderer are B2D_ERR_INVALID_ARG.
 *
 * Not covered: per-frame states together with per-frame levels (b2d_render_states & co. act on level 0), levels in
 * b2d_render_sharded, and the CLI. */
#define B2D_MAX_LEVELS 64
int b2d_renderer_create_levels(const b2d_scene *const *scenes, size_t n_levels, const b2d_view *view, int device,
                               int max_batch, b2d_renderer **out);
int b2d_render_levels(b2d_renderer *r, const b2d_pose *poses, const uint32_t *levels, size_t n, uint8_t *index_fb,
                      uint32_t *rgba_fb);
int b2d_render_device_levels(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, size_t n,
                             uint8_t *d_index_fb, uint32_t *d_rgba_fb, void *cuda_stream);
int b2d_walk_device_levels(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, size_t n, void *cuda_stream,
                           int64_t *ticket_out);
int b2d_renderer_set_level_sector_moves(b2d_renderer *r, int level, const b2d_sector_move *moves, size_t n);

/* ---- multi-GPU: pose-sharded render with a chunked, overlapped all-gather of finished frames ------------------
 * The reference has no collective and no multi-device path (SURVEY.md 2); the hand-off this replaces is the
 * per-frame `frame.finish()` of engine/src/renderer.rs:160-167.  One process per GPU.  NCCL (libnccl.so.2) is bound
 * at run time; without it these calls fail with B2D_ERR_NCCL and the rest of the library works.
 *
 * b2d_comm_unique_id: on one rank; the caller distributes the 128 bytes (MPI, torch.distributed, a file).
 * b2d_comm_create:    collective over `world` ranks (ncclCommInitRank); binds the rank to `device`. */
#define B2D_COMM_ID_BYTES 128
int b2d_comm_unique_id(uint8_t id_out[B2D_COMM_ID_BYTES]);
int b2d_comm_create(const uint8_t id[B2D_COMM_ID_BYTES], int rank, int world, int device, b2d_comm **out);
void b2d_comm_destroy(b2d_comm *c);
int b2d_comm_info(const b2d_comm *c, int *rank_out, int *world_out, int *nccl_version_out);

#define B2D_SHARD_RENDER_ONLY 0     /* render this rank's block, no exchange */
#define B2D_SHARD_RENDER_GATHER 1   /* render + all-gather of every chunk, overlapped */
#define B2D_SHARD_GATHER_ONLY 2     /* the same gathers without rendering (to time the exchange alone) */

typedef struct b2d_sharded_stats {
    double total_ms;                /* device time, first launch -> last consumer, this rank */
    double render_ms, gather_ms;    /* sums of the per-chunk kernel / ncclAllGather times (they overlap each other) */
    int64_t frames_local, frames_gathered, chunks, chunk_frames;
    int64_t bytes_received;         /* (world-1)/world of the gathered bytes */
    char registration[64];          /* exchange transport / how the gather buffers were registered with NCCL */
} b2d_sharded_stats;

/* Called on the host once per chunk, right after the chunk's work has been ENQUEUED: d_frames holds `ranks` x
 * frames_per_rank finished index frames (rank-major; frame j of rank q is pose q*per + first_local_pose + j, with
 * per = ceil(n_total/world)), valid for work enqueued on `cuda_stream`, which is ordered after the gather.  The
 * buffer is reused two chunks later, after everything the callback enqueued on that stream. */
typedef void (*b2d_chunk_fn)(void *user, int chunk_index, size_t first_local_pose, size_t frames_per_rank,
                             const uint8_t *d_frames, int ranks, void *cuda_stream);

/* Collective.  `poses` (HOST, n_total entries, identical on every rank) is split into contiguous blocks of
 * per = ceil(n_total/world); rank q renders block q (a short last block is padded by repeating the last pose) in
 * chunks of min(chunk_frames, max_batch) frames, each chunk rastered straight into this rank's slice of the
 * all-gather buffer (no staging copy) and gathered in place on a second stream while the next chunk renders; the
 * consumer callback (nullable) runs on a third.  Transport of the exchange: by default every rank pushes its slice into the
 * peers' buffers with the copy engines over CUDA-IPC mappings (ordered across ranks by two 4-byte ncclAllReduce per
 * chunk); if any rank cannot map a peer's buffer all ranks fall back, together, to an in-place ncclAllGather, which
 * B2D_GATHER=nccl also selects (buffers then from ncclMemAlloc, registered with the communicator where NCCL offers it).
 * stats_out->registration names what was used.  Synchronous: returns when this rank's part is complete. */
int b2d_render_sharded(b2d_renderer *r, b2d_comm *c, const b2d_pose *poses, size_t n_total, size_t chunk_frames,
                       int mode, b2d_chunk_fn fn, void *user, b2d_sharded_stats *stats_out);

/* One 32-bit checksum per frame on the device: sum_i (p[i] + 1) * (i * 0x9E3779B1 + 0x7F4A7C15) mod 2^32
 * (position sensitive, order independent).  Used to validate gathered frames without moving them to the host. */
int b2d_frame_checksums_device(const uint8_t *d_frames, size_t n_frames, size_t frame_bytes, uint32_t *d_out,
                               void *cuda_stream);

/* Device memory for hosts that do not link a CUDA library themselves (the compiled CLI; a Rust binding would use its
 * cuda-sys crate instead): allocate / free on `device`, and a synchronous device -> host copy. */
int b2d_device_alloc(int device, size_t bytes, void **d_out);
int b2d_device_free(int device, void *d_ptr);
int b2d_device_download(int device, void *host_dst, const void *d_src, size_t bytes);

/* Introspection for tests/profiling: copies the BSP-walk worklist of the LAST b2d_render_device
 * batch to the host.  counts_out[n], and for frame i seg ids seg_ids_out[i*stride .. +counts[i]). */
int b2d_debug_worklist(b2d_renderer *r, size_t n, int32_t *counts_out, int32_t *seg_ids_out, size_t stride);

/* Introspection for tests: the table-set slot of frames 0..n-1 of the LAST walked batch, which must have been walked with
 * per-frame states (frames with equal compact states share a slot). */
int b2d_debug_state_slots(b2d_renderer *r, size_t n, uint32_t *slots_out);

/* Introspection for tests: the expanded table set `set` of the LAST walked batch, in b2d_scene_tables_at's layout
 * [textures | sectors | segs | sprites | mids] and size (without the device copy's padding).  A batch walked with
 * per-frame states has one set per distinct state (`set` below their number, as b2d_debug_state_slots numbers them); a
 * plain batch has one, the set its worklist slot read (`set` = 0).  With out = NULL only *size_out is written.
 * Synchronises the device.  B2D_ERR_INVALID_ARG for a scene without time-dependent content or dynamic sectors, a set
 * out of range, or a renderer that has walked no batch. */
int b2d_debug_state_tables(b2d_renderer *r, size_t set, void *out, size_t capacity, size_t *size_out);

/* Per-kernel device timing for the roofline report: while enabled, every batch records CUDA events
 * around the walk and raster launches on the launching stream.  b2d_profile_read synchronises the
 * device, returns the summed milliseconds and batch count since the last read, and resets them. */
int b2d_profile_enable(b2d_renderer *r, int enable);
int b2d_profile_read(b2d_renderer *r, double *walk_ms, double *raster_ms, int64_t *batches);

/* Number of kernel launches issued by this renderer so far (bench.py's gpu_launches). */
int64_t b2d_launch_count(const b2d_renderer *r);

#ifdef __cplusplus
}
#endif
#endif /* B2D_H */
