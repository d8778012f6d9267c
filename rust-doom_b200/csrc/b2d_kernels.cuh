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

// Per-frame states (b2d_render_states): the walk and raster variants that take it read the five state-dependent tables of
// each frame from its slot of a state arena instead of DeviceScene::{tex, sectors, segs, sprites, mids}.  Slot s holds
// [tex | sectors | segs | sprites | mids] at base + s * slot_bytes (the layout of b2d_scene_tables_at).
struct StateTables {
    const uint8_t *base;
    const uint32_t *frame_slot;      // slot of each frame of the batch: read by the walk, passed on in FrameConst::pad[0]
    uint32_t slot_bytes, off_sectors, off_segs, off_sprites, off_mids, pad;
};

// Per-frame levels (b2d_render_levels): frame i of a batch is rendered from scenes[frame_level[i]], each the DeviceScene of
// one level of the renderer as the batch's worklist slot reads it.  The walk copies the frame's scene into shared memory
// and passes its level on in FrameConst::pad[1]; the raster reads the scene of that level.  Exclusive with StateTables.
struct LevelTables {
    const DeviceScene *scenes;
    const uint32_t *frame_level;
};

// Bytes of dynamic shared memory the BSP-walk kernel needs per frame (= per CTA) for this scene.
size_t walk_smem_per_warp(const DeviceScene &sc);
// Static shared memory of the per-frame-level walk (its copy of the resident level's DeviceScene and the barrier words):
// its dynamic shared memory may be at most kWalkSmemMax minus this.
size_t walk_levels_static_smem();
constexpr size_t kWalkSmemMax = 227 * 1024;      // the largest shared-memory opt-in per block on sm_90a

// Kernel 1: front-to-back BSP walk, one CTA per frame.  Writes frames[i] and up to `stride`
// worklist entries per frame at work[i*stride ...].
// `states` (nullable): per-frame tables.
cudaError_t launch_walk(const DeviceScene &sc, const View &vw, const Pose *d_poses, int n,
                        FrameConst *d_frames, SegFrame *d_work, int stride, cudaStream_t stream, bool background = false,
                        const StateTables *states = nullptr);

// Kernel 2: wall-column / flat-span / sky rasteriser, one warp per (frame, 32-column strip).
// Writes every pixel of d_index_fb exactly once; if d_rgba != nullptr also the palette-mapped RGBA8.
// `states` (nullable): per-frame tables, the arena the walk of these frames read.
cudaError_t launch_raster(const DeviceScene &sc, const View &vw, const FrameConst *d_frames,
                          const SegFrame *d_work, int stride, int n, uint8_t *d_index_fb,
                          uint32_t *d_rgba, cudaStream_t stream, const StateTables *states = nullptr);

// The walk and the raster of a batch with per-frame levels.  `smem`: the largest walk_smem_per_warp of the levels;
// `masked`: some level has masked content (its masked_list is set).  Everything else as launch_walk / launch_raster.
cudaError_t launch_walk_levels(const LevelTables &levels, size_t smem, const View &vw, const Pose *d_poses, int n,
                               FrameConst *d_frames, SegFrame *d_work, int stride, cudaStream_t stream, bool background);
cudaError_t launch_raster_levels(const LevelTables &levels, bool masked, const View &vw, const FrameConst *d_frames,
                                 const SegFrame *d_work, int stride, int n, uint8_t *d_index_fb, uint32_t *d_rgba,
                                 cudaStream_t stream);

// Expands `nstates` compact states (StateLayout::words words each, b2d_scene.hpp) from `src` (device pointers to the
// rest-state sections) into slots 0 .. nstates-1 of `arena`: one thread per output record.
cudaError_t launch_state_tables(const StateSrc &src, const uint32_t *d_states, uint32_t words, int nstates, uint8_t *d_arena,
                                const StateTables &layout, cudaStream_t stream);

// Pre-light kernels (once per renderer).  Flats: dst[r * stride + i] = colormap[r][src[i]] for r < 32, i < n.
cudaError_t launch_prelight(const uint8_t *d_colormap, const uint8_t *d_src, uint8_t *d_dst, size_t n, size_t stride,
                            cudaStream_t stream);

// Textures: 32 pre-lit planes (+ opacity plane 32) of every texture of the table, in its per-texture layout.
cudaError_t launch_prelight_textures(const uint8_t *d_colormap, const uint8_t *d_texels, const TexRec *d_tex, int ntex,
                                     uint8_t *d_dst, size_t stride, cudaStream_t stream);

// Kernel 3: palette LUT on its own (index -> RGBA8), 16 pixels per thread.
cudaError_t launch_palette(const uint32_t *d_palette, const uint8_t *d_index, uint32_t *d_rgba,
                           size_t n_pixels, cudaStream_t stream);

}  // namespace b2d
