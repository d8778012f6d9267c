// Device-side scene view + kernel launchers (implemented in b2d_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "b2d_math.cuh"
#include "b2d_scene.hpp"

namespace b2d {

// Pointers into the scene blob resident in HBM (one cudaMalloc, uploaded once per level).
struct DeviceScene {
    const int32_t *verts;
    const NodeRec *nodes;
    const SSectorRec *ssectors;
    const SegRec *segs;
    const SectorRec *sectors;
    const TexRec *tex;
    const MidRec *mids;          // masked two-sided middle textures (SegRec::mid indexes this)
    const SpriteRec *sprites;    // decoration things grouped by subsector (SSectorRec::sprites)
    const uint8_t *texels;
    const uint8_t *flats;
    const uint8_t *colormap;     // 34 x 256
    // colormap applied ahead of time (per renderer, next to the blob): plane r < 32 of a texture holds
    // colormap[r][texel] in the layout b2d_math.cuh:tex_interleaved()/lit_index() select, plane 32 the opacity of
    // textures with holes; lit_flats likewise (row-major).  A pixel is one load: no colormap lookup at run time.
    const uint8_t *lit_texels;
    const uint8_t *lit_flats;
    uint32_t lit_texel_stride, lit_flat_stride;
    const uint32_t *palette;     // 256 RGBA8
    const uint8_t *walk_static;  // the walk's traversal tables as they sit in its shared memory: {x,y,dx,dy,rchild,lchild,0,0}
                                 // per node (32 B) followed by the SSectorRec array (16 B each); one bulk copy per CTA
    const uint32_t *yslope;      // per view: H entries
    const uint16_t *skyrow;      // per view: H entries, sky texture row of each screen row
    int32_t nverts, nnodes, nss, nsegs, nsectors, ntex, nflats, sky_tex, nmids, nsprites;
    uint32_t root;
    uint32_t invF;               // floor(2^32 / F)
    int32_t *status_flag;        // device int: OR of the kStatus* bits of every frame (0 = all frames complete)
    uint32_t *masked_list;       // arena of deferred masked entries (33 words each: worklist index + 32 packed windows),
                                 // handed out in chunks of kMaskedChunk entries; nullptr = level without masked content
    uint32_t *masked_counter;    // chunks handed out by the current raster launch (reset before every launch)
    uint32_t masked_chunks;      // arena capacity in chunks (exhausted -> kStatusMaskedFull)
    int32_t masked_cap;          // strip_masked_cap(): entries one 32-column strip can defer per frame
};

constexpr int kMaskedChunk = 4;      // entries per arena chunk (528 bytes)

// The five state-dependent tables of one level at one state: an expanded table set (in a state arena, or a level's own set of
// a worklist slot), or, on a level without time-dependent content or dynamic sectors, its blob tables.  What a frame of a
// batch with per-frame states reads, and where launch_state_sets writes.
struct TableSet {
    const TexRec *tex;
    const SectorRec *sectors;
    const SegRec *segs;
    const SpriteRec *sprites;
    const MidRec *mids;
};

// Per-frame levels (b2d_render_levels): frame i of a batch is rendered from scenes[frame_level[i]], each the DeviceScene of
// one level of the renderer as the batch's worklist slot reads it.  The walk copies the frame's scene into shared memory
// and passes its level on in FrameConst::level; the raster reads the scene of that level.
// Per-frame states (b2d_render_states, b2d_render_levels_states), with or without per-frame levels: frame i reads its five
// state-dependent tables from sets[frame_set[i]] (passed on in FrameConst::set) instead of its scene's.
struct LevelTables {
    const DeviceScene *scenes;
    const uint32_t *frame_level;
    const TableSet *sets;
    const uint32_t *frame_set;
};

// One table set to expand (launch_state_sets): level `level`'s rule at the compact state at word `state` of the launch's
// states, into the tables of its TableSet.  `first`: the set's first record in the launch's numbering of all its records
// (the record counts of the sets before it, summed).  `extralight`: the player's extra light, 0..2 (DESIGN.md C18).
struct StateSet {
    uint32_t level, state, first, extralight;
};

// Fixed colormaps (b2d_*_levels_states_lights, DESIGN.md C18): the kFixed raster variant lights every wall, flat and
// masked pixel of frame i through COLORMAP row frame_fixed[i] (-1: by light and depth, as without it).  Rows 0..31 are
// the level's pre-lit planes; row 32 is planes[level of the frame], built for a level by the first call that asks for it.
struct FixedPlanes {
    const uint8_t *texels;       // row 32 of every texture, in the layout of a pre-lit texture plane
    const uint8_t *flats;        // row 32 of every flat, at an address that is a multiple of 4 GiB (as the pre-lit flats)
};
struct FixedTables {
    const int32_t *frame_fixed;
    const FixedPlanes *planes;   // per level
};

// Seen lines (b2d_raster_device_seen, DESIGN.md C20): the seen raster variant ORs bit l & 31 of word l >> 5 of row f of
// `rows` (`words` words per row) for every linedef l of which a seg owns a column of frame f in the solid pass.
// seg_line + level_off[level] is the level's seg -> linedef table (-1: no linedef).
struct SeenTables {
    uint32_t *rows;
    const int32_t *seg_line;
    const uint32_t *level_off;
    uint32_t words;
};

// Bytes of dynamic shared memory the BSP-walk kernel needs per frame (= per CTA) for this scene.
size_t walk_smem_per_warp(const DeviceScene &sc);
// Static shared memory of the per-frame-level walk (its copy of the resident level's DeviceScene and the barrier words):
// its dynamic shared memory may be at most kWalkSmemMax minus this.
size_t walk_levels_static_smem();
constexpr size_t kWalkSmemMax = 227 * 1024;      // the largest shared-memory opt-in per block on sm_90a

// The tables a batch's walk and raster read, and which of their <kStates, kLevels> variants runs.  Without per-frame levels
// every frame reads `scene` (level 0 as the batch's worklist slot reads it); with them, the scenes of `levels` (and `scene`
// is not read).  With per-frame states the five state-dependent tables come from the table sets of `levels`.
// With fixed colormaps (`fixed_rows`: some frame of the batch has one), the raster reads `fixed` (per-frame levels and
// states only).
struct BatchTables {
    DeviceScene scene;
    LevelTables levels;
    FixedTables fixed;
    bool per_frame, per_level, fixed_rows;
};

// Kernel 1: front-to-back BSP walk, one CTA per frame.  Writes frames[i] and up to `stride` worklist entries per frame at
// work[i*stride ...].  `levels_smem`: with per-frame levels, the largest walk_smem_per_warp of the levels.
cudaError_t launch_walk(const BatchTables &t, size_t levels_smem, const View &vw, const Pose *d_poses, int n,
                        FrameConst *d_frames, SegFrame *d_work, int stride, cudaStream_t stream, bool background);

// Kernel 2: wall-column / flat-span / sky rasteriser, one warp per (frame, 32-column strip), of the frames a walk of the same
// tables wrote.  Writes every pixel of d_index_fb exactly once; if d_rgba != nullptr also the palette-mapped RGBA8.
// `masked`: some level the frames read has masked content (its masked_list is set).  `seen` (nullable): the seen variant,
// which draws the same index frames (no RGBA: cudaErrorInvalidValue) and ORs each frame's seen lines into its row of
// seen->rows.
cudaError_t launch_raster(const BatchTables &t, bool masked, const View &vw, const FrameConst *d_frames, const SegFrame *d_work,
                          int stride, int n, uint8_t *d_index_fb, uint32_t *d_rgba, const SeenTables *seen,
                          cudaStream_t stream);

// Expands the `nsets` table sets of a batch in one grid: set k by the rule of level sets[k].level (srcs[level]: device
// pointers to that level's rest-state sections) into the tables of out[k].  `records`: the records of all sets together
// (sets[k].first counts them up).
cudaError_t launch_state_sets(const StateSrc *d_srcs, const StateSet *d_sets, const TableSet *d_out, const uint32_t *d_states,
                              int nsets, uint32_t records, cudaStream_t stream);

// Pre-light kernels (once per renderer).  Flats: dst[r * stride + i] = colormap[r][src[i]] for r < 32, i < n.
cudaError_t launch_prelight(const uint8_t *d_colormap, const uint8_t *d_src, uint8_t *d_dst, size_t n, size_t stride,
                            cudaStream_t stream);

// Textures: 32 pre-lit planes (+ opacity plane 32) of every texture of the table, in its per-texture layout.
cudaError_t launch_prelight_textures(const uint8_t *d_colormap, const uint8_t *d_texels, const TexRec *d_tex, int ntex,
                                     uint8_t *d_dst, size_t stride, cudaStream_t stream);

// One more pre-lit plane, of COLORMAP row `d_row` (256 bytes): the flats (dst[i] = row[src[i]], i < n) and the textures
// (in the per-texture layout of the planes above).  For fixed colormap 32 (FixedPlanes).
cudaError_t launch_prelight_row(const uint8_t *d_row, const uint8_t *d_src, uint8_t *d_dst, size_t n, cudaStream_t stream);
cudaError_t launch_prelight_textures_row(const uint8_t *d_row, const uint8_t *d_texels, const TexRec *d_tex, int ntex,
                                         uint8_t *d_dst, cudaStream_t stream);

// Kernel 3: palette LUT on its own (index -> RGBA8), 16 pixels per thread.
cudaError_t launch_palette(const uint32_t *d_palette, const uint8_t *d_index, uint32_t *d_rgba,
                           size_t n_pixels, cudaStream_t stream);
// ... with a colour table per frame: frame f of the n_frames contiguous npix-pixel frames through
// palettes[tables[f] * 256 ..] (the renderer's table layout: b2d_renderer::d_palettes).
cudaError_t launch_palette_levels(const uint32_t *d_palettes, const uint32_t *d_tables, const uint8_t *d_index, uint32_t *d_rgba,
                                  size_t n_frames, size_t npix, cudaStream_t stream);
// Kernel 4: C17 resolve of the n_frames contiguous W x H index frames at d_index, frame f through palettes[tables[f] * 256 ..]
// (d_tables NULL: table 0), box-filtered by `factor` (1..8, dividing W and H) into d_out in B2D_RESOLVE_* `format`.
cudaError_t launch_resolve(const uint32_t *d_palettes, const uint32_t *d_tables, const uint8_t *d_index, void *d_out,
                           size_t n_frames, int W, int H, int factor, int format, cudaStream_t stream);
// A frame's inputs to the state variant, staged per call: its level, the word offset of its sector offsets (floor,
// ceiling per dynamic slot of its level) in `off` (kAutomapNoSlot: at rest), and its arrows arrows[arrow_first ..
// arrow_first + n_arrows).
struct AutomapFrameIn {
    uint32_t level, off, arrow_first, n_arrows;
};
// The state variant's tables: per level its AutomapDynLine table (nullptr: no changeable lines), then the call's staging
// (frames: nullptr for every frame on level 0, at rest, without arrows).
struct AutomapStateTables {
    const AutomapDynLine *const *dyn;
    const AutomapFrameIn *frames;
    const int32_t *off;
    const AutomapArrow *arrows;
};
// The marks variant's tables: per level its grid origin and digits, then the call's staging: 2 words per frame (first,
// n) into `marks` (ranges nullptr: no marks).
struct AutomapMarkTables {
    const AutomapMarkLevel *levels;
    const uint32_t *ranges;
    const AutomapMark *marks;
};
// Kernel 5's grid: CTAs (128 x 32 tiles) per frame of view vw.
size_t automap_tiles(const View &vw);
// Kernel 5: the C19 automap of n_frames poses into contiguous W x H index frames at d_out, frame f from the items of
// levels[frame_level[f]] (d_frame_level NULL: level 0), `scale` and `flags` as checked by b2d_automap_device.
// `seen_variant`: its seen variant (C20), frame f's lines coloured by row f of d_seen (`words` per row; nullptr: every
// line mapped); d_seen and words are not read otherwise.  `states` (nullable): the state variant (C21) instead, which
// takes frame f's level from states->frames[f] (d_frame_level is not read), its sector offsets and arrows, and colours
// its lines by row f of d_seen as the seen variant does.  `marks` (nullable, with `states`): the marks variant (C22),
// the state variant with the grid under B2D_AUTOMAP_GRID and frame f's marks over everything.
cudaError_t launch_automap(const AutomapLevel *d_levels, const uint32_t *d_frame_level, const Pose *d_poses, size_t n_frames,
                           const View &vw, int32_t scale, int flags, bool seen_variant, const uint32_t *d_seen, uint32_t words,
                           uint8_t *d_out, cudaStream_t stream, const AutomapStateTables *states = nullptr,
                           const AutomapMarkTables *marks = nullptr);

}  // namespace b2d
