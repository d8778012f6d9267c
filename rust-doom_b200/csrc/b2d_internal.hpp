// Private to libb2d.so: the handle types behind include/b2d.h and the helpers its translation units share
// (b2d_api.cu: archive / scene / renderer entry points; b2d_sharded.cu: multi-GPU sharded render over NCCL).
#pragma once
#include <array>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/b2d.h"
#include "b2d_kernels.cuh"
#include "b2d_scene.hpp"
#include "b2d_wad.hpp"

namespace b2d {
int fail(int code, const std::string &msg);            // sets the thread-local message, returns code
int cuda_fail(cudaError_t e, const char *what);
// The frames of a call, or of one batch of it (HOST arrays, checked by CallFrames::prepare).  `levels`: the level of each
// frame (nullptr: every frame on level 0).  `starts`: with per-frame states, frame i's compact state is fs[starts[i] ..]
// (its level's layout.words words; none on a level without time-dependent content or dynamic sectors); nullptr: every
// level at the renderer's own state, a plain batch.  `lights`: with per-frame levels and states, each frame's fixed
// colormap and extra light (nullptr: none, as when every frame is {-1, 0}).
struct Frames {
    const uint32_t *levels = nullptr;
    const uint32_t *fs = nullptr;
    const size_t *starts = nullptr;
    const b2d_frame_light *lights = nullptr;
    Frames from(size_t first) const {
        return {levels ? levels + first : nullptr, fs, starts ? starts + first : nullptr, lights ? lights + first : nullptr};
    }
};
// What a render, walk or sharded call says about its n frames (HOST arrays), and, once prepare() has checked it, its
// `frames`, whose compact states live in `fs` / `starts`.  kFrameLevels: the call takes `levels`, a level each (refused if
// null).  kFrameStates: the call takes `states`, a time and a range of `moves` each (refused if null); or `tics` (timed
// calls), a time each with its level's current sector moves.  `palettes` and `lights` (nullable): a palette each, and a
// fixed colormap and extra light each.
constexpr unsigned kFrameLevels = 1, kFrameStates = 2;
struct CallFrames {
    CallFrames() = default;                  // no per-frame inputs: a plain call
    CallFrames(unsigned takes, const uint32_t *levels, const b2d_frame_state *states = nullptr, const b2d_sector_move *moves = nullptr,
               size_t n_moves = 0, const b2d_frame_light *lights = nullptr, const uint32_t *palettes = nullptr)
        : takes(takes), levels(levels), states(states), moves(moves), n_moves(n_moves), lights(lights), palettes(palettes) {}
    explicit CallFrames(const uint32_t *tics) : tics(tics) {}
    // The checks, in this order, each B2D_ERR_INVALID_ARG with its message: the levels (each below the renderer's number
    // of levels, on a renderer whose levels fit the per-frame-level walk -- a b2d_renderer_create renderer may not), the
    // palettes (each below the palette count of its frame's level), the lights (fixed_colormap in -1..32, extralight in
    // 0..2; lights of every frame {-1, 0} are dropped, so that such a call is the call without lights), the states (move
    // ranges inside `moves`, moves of dynamic sectors).  Then the compact states: frame i's at fs[starts[i] ..] (none on a
    // level without time-dependent content or dynamic sectors).  With every frame on level 0 and a level 0 without either,
    // the call is a plain one (frames.starts stays nullptr).  Nothing is enqueued.
    int prepare(const b2d_renderer *r, size_t n);

    unsigned takes = 0;
    const uint32_t *levels = nullptr;
    const b2d_frame_state *states = nullptr;
    const b2d_sector_move *moves = nullptr;
    size_t n_moves = 0;
    const b2d_frame_light *lights = nullptr;
    const uint32_t *palettes = nullptr;
    const uint32_t *tics = nullptr;
    std::vector<uint32_t> fs;
    std::vector<size_t> starts;
    Frames frames;
};
// The colour-table index of frame i, pal_base[levels[i]] + palettes[i] (either array nullable: 0), the levels and palettes checked.
inline uint32_t frame_table(const b2d_renderer *r, const uint32_t *levels, const uint32_t *palettes, size_t i);
// A one-call render of `batches` batches walks the first into the next worklist slot and alternates slots from there: it
// is refused (B2D_ERR_INVALID_ARG) before anything is enqueued while a slot it would use holds a walked, unrastered batch.
int check_slots_free(const b2d_renderer *r, size_t batches);
// The BSP walk of the n frames `frames` (device poses d_poses) into the next worklist slot on `stream`, and the raster of a
// ticket (b2d_walk_device* / b2d_raster_device); neither is synchronised.
int walk_batch(b2d_renderer *r, const Pose *d_poses, const Frames &frames, int n, cudaStream_t stream, bool background,
               int64_t *ticket_out);
// `d_seen`: the seen variant's rows of seen lines (b2d_raster_device_seen; index frames only), else nullptr
int raster_batch(b2d_renderer *r, int64_t ticket, uint8_t *d_index, uint32_t *d_rgba, cudaStream_t stream,
                 uint32_t *d_seen = nullptr);

// Owners of CUDA resources.  They release on the current device: ~b2d_renderer and b2d_comm_destroy select theirs first.
struct DeviceFree { void operator()(void *p) const { cudaFree(p); } };
struct HostFree { void operator()(void *p) const { cudaFreeHost(p); } };
struct StreamDestroy { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
struct EventDestroy { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
template <typename T> using DeviceBuf = std::unique_ptr<T, DeviceFree>;    // cudaMalloc
template <typename T> using PinnedBuf = std::unique_ptr<T, HostFree>;      // cudaMallocHost
using Stream = std::unique_ptr<CUstream_st, StreamDestroy>;
using Event = std::unique_ptr<CUevent_st, EventDestroy>;

// Creators: `out` holds the new resource, or is empty if the call failed (cudaMalloc for a DeviceBuf, cudaMallocHost for a PinnedBuf).
template <typename T, typename Free> cudaError_t allocate(std::unique_ptr<T, Free> &out, size_t bytes) {
    static_assert(std::is_same_v<Free, DeviceFree> || std::is_same_v<Free, HostFree>, "device or pinned host memory");
    void *p = nullptr;
    const cudaError_t e = std::is_same_v<Free, HostFree> ? cudaMallocHost(&p, bytes) : cudaMalloc(&p, bytes);
    out.reset(e == cudaSuccess ? static_cast<T *>(p) : nullptr);
    return e;
}
inline cudaError_t stream_create(Stream &out) {
    cudaStream_t s = nullptr;
    const cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    out.reset(e == cudaSuccess ? s : nullptr);
    return e;
}
inline cudaError_t event_create(Event &out, unsigned flags = cudaEventDisableTiming) {
    cudaEvent_t ev = nullptr;
    const cudaError_t e = cudaEventCreateWithFlags(&ev, flags);
    out.reset(e == cudaSuccess ? ev : nullptr);
    return e;
}

// Device memory at an address that is a multiple of 4 GiB (alloc_aligned_4g in b2d_api.cu): a VMM mapping of `mapped`
// bytes, or, with mapped == 0, the over-sized cudaMalloc `raw` that the aligned pointer lies in.
struct Aligned4GFree {
    size_t mapped = 0;
    unsigned long long handle = 0;
    void *raw = nullptr;
    void operator()(uint8_t *p) const;
};
using Aligned4G = std::unique_ptr<uint8_t, Aligned4GFree>;
}  // namespace b2d

using namespace b2d;

struct b2d_archive {
    std::unique_ptr<Archive> wad;
};

struct b2d_scene {
    std::vector<uint8_t> blob;
    Level level;
    b2d_scene_info info;
    // every palette the scene holds, at least one; palettes[0] is the one compiled into the blob (768 zero bytes when
    // the scene was made without a PLAYPAL)
    std::vector<std::array<uint8_t, 768>> palettes;
    std::vector<AutomapLine> automap;                     // automap_lines(level), built at creation
};

// A worklist slot: the BSP walk of batch k+1 may run (b2d_walk_device, another stream) while batch k is rastered.
struct WorkSlot {
    DeviceBuf<FrameConst> frames;                         // frames, worklist and events exist together (ensure_slot)
    DeviceBuf<SegFrame> work;
    Event walk_done, raster_done;
    int n = 0;                                            // frames walked into the slot
    int64_t ticket = -1;
    bool rastered = true;
    BatchTables tables{};                                 // what the batch's walk read and its raster reads
    // Per-frame states (b2d_render_states & co.): an arena of up to max_batch expanded table sets, allocated by the first
    // such call; the batch's sets are packed into it
    DeviceBuf<uint8_t> arena;
    int sets = 0;                                         // table sets of the batch in the arena (distinct states)
    std::vector<uint32_t> set_level;                      // level of each table set
    std::vector<size_t> set_off;                          // byte offset of each table set in the arena
    // The sections of a batch (StageLayout, b2d_api.cu) on the device and their pinned staging, sized at renderer creation
    // for the largest batch: what its expansions, walk and raster read besides the poses
    DeviceBuf<uint8_t> stage;
    PinnedBuf<uint8_t> h_stage;
    Event staged;                                         // h_stage has been read by its copy
};

// Host-path staging (created by the first b2d_render & co.): double-buffered frame outputs.
struct HostStaging {
    Stream render_stream, copy_stream[2];                 // one copy stream per staging buffer
    Event rendered[2], copied[2];
    DeviceBuf<uint8_t> index[2];
    PinnedBuf<Pose> poses;                                // two buffers of max_batch poses
    std::array<DeviceBuf<uint32_t>, 2> rgba;              // created by the first call that asks for RGBA frames
};

// A call's frame colour-table indices on the device, with their pinned staging (stage_tables, b2d_api.cu): grown by a
// call with more frames than they hold.
struct LevelStaging {
    DeviceBuf<uint32_t> d;
    PinnedBuf<uint32_t> h;
    size_t cap = 0;
    Event copied, done;                                   // the staging has been read by its copy; the kernel has read the copy
};

// One level of a renderer (b2d_renderer_create_levels; b2d_renderer_create makes a set of one): the scene on the device
// and what the kernels read of it.
struct LevelRes {
    DeviceBuf<uint8_t> d_blob;
    DeviceBuf<uint16_t> d_skyrow;                         // sky texture row of each screen row (the level's sky height)
    DeviceBuf<uint8_t> d_lit;       // colormap-applied copies of the texels (32 light rows + the opacity plane)
    // ... and of the flats, in a region whose address is a multiple of 4 GiB: the raster then forms a flat texel's address
    // as {high word, 32-bit offset} without a 64-bit add (one instruction per flat pixel).  Reserved + mapped through the
    // driver's virtual-memory API (cuMemAddressReserve takes an alignment); an over-sized cudaMalloc is the fall-back.
    Aligned4G d_lit_flats;
    DeviceBuf<uint8_t> d_walk_static;                     // node / subsector tables as the walk kernel's shared memory holds them
    DeviceScene ds{};
    // The state rule's inputs, for every level: a frame with extra light (DESIGN.md C18) reads a table set expanded
    // from a compact state on any level.
    StateLayout layout;
    std::vector<uint32_t> state;                          // the level's own compact state (set_time, set_*sector_moves)
    DeviceBuf<uint32_t> d_slot_maps;                      // StateLayout::sector_slots, ::mid_seg, then the light side tables
    StateSrc src{};                                       // device pointers into d_blob and d_slot_maps
    // Scenes with time-dependent content or dynamic sectors (DESIGN.md §3 "State arena"); the rest stays empty.  The
    // device blob is never written after creation: the state rule reads its rest-state sections, and every batch reads
    // its five state-dependent tables from a table set expanded on the device from a compact state.
    std::vector<uint8_t> h_blob;                          // host copy of the scene
    // per worklist slot: the table set the slot's batches read and the compact state it was expanded from
    struct Slot {
        DeviceBuf<uint8_t> tables;
        std::vector<uint32_t> state;
    } slot[2];
    // Fixed colormap 32 (C18): the row-32 texel and flat planes, built whole by the first call that asks for them on this
    // level, on that call's stream (`built` follows the build; every batch that reads them waits for it).
    struct Row32 {
        DeviceBuf<uint8_t> texels;
        Aligned4G flats;
        Event built;
    };
    std::unique_ptr<Row32> row32;
    // The automap's items (DESIGN.md C19), host copies taken at creation: the scene's automap table and the x, y of the
    // blob's sprites.  Uploaded by the first b2d_automap_device call (b2d_renderer::automap).
    std::vector<AutomapLine> automap_lines;
    std::vector<int32_t> automap_things;
    // Seen lines (DESIGN.md C20): the linedef of each seg of the level's SEGS lump (-1: none), built at creation and
    // uploaded by the first b2d_raster_device_seen call (b2d_renderer::seen)
    std::vector<int32_t> seg_line;
};

struct b2d_renderer {
    int device = 0;
    View view{};
    int max_batch = 0;
    int stride = 0;                 // worklist entries per frame (= the largest n_segs + n_sprites of the levels)
    size_t walk_smem = 0;           // the largest walk_smem_per_warp of the levels
    // the levels; every entry point without a level argument acts on level 0
    std::vector<LevelRes> lv;
    DeviceBuf<uint32_t> d_yslope;
    DeviceBuf<int32_t> d_status;
    DeviceBuf<uint32_t> d_masked;   // one arena of deferred masked entries for every level with masked content
    DeviceBuf<Pose> d_poses;
    WorkSlot slot[2];
    int64_t next_ticket = 0;
    int last_slot = 0;
    std::unique_ptr<HostStaging> host;
    uint32_t tics = 0;
    Event masked_done;                                    // last raster that used the masked-entry arena
    // every palette of every level as one colour table, [sum of the levels' palette counts][256]: level l's palette p is
    // table pal_base[l] + p.  K3-levels and K4 read a table index per frame (stage_tables, b2d_api.cu).
    DeviceBuf<uint32_t> d_palettes;
    std::vector<uint32_t> pal_base, pal_count;
    // the frame tables of a call of b2d_palette_lut_levels_device and of b2d_resolve_device / b2d_resolve_palettes_device,
    // each call kind with its own
    LevelStaging lut_levels, resolve_levels;
    // A group of tables of every level on the device, created whole by the first call that reads them: the byte image `d`,
    // uploaded from its pinned copy `h` on that call's stream (`built` follows the upload; every later call waits for it
    // on its own stream).  `off`: where the image's per-level records start.
    struct Tables {
        DeviceBuf<uint8_t> d;
        PinnedBuf<uint8_t> h;
        size_t off = 0;
        Event built;
    };
    // The automap's (first b2d_automap_device call): the lines and things of each level, then one AutomapLevel per level
    // pointing into them.  With the call's own level staging.
    std::unique_ptr<Tables> automap;
    LevelStaging automap_levels;
    // The seen raster's (first b2d_raster_device_seen call): the seg -> linedef tables one after the other, then each
    // level's offset into them.  `seen_words`: the length of a row of seen lines.
    std::unique_ptr<Tables> seen;
    uint32_t seen_words = 1;
    DeviceBuf<uint32_t> d_masked_counter;
    int64_t launches = 0;
    bool profiling = false;
    std::vector<Event> prof_events;         // pairs: before / after one kernel launch
    std::vector<int> prof_kinds;            // per pair: 0 = walk, 1 = raster

    ~b2d_renderer() { cudaSetDevice(device); }            // the members are released on the renderer's device
};

inline uint32_t b2d::frame_table(const b2d_renderer *r, const uint32_t *levels, const uint32_t *palettes, size_t i) {
    return r->pal_base[levels ? levels[i] : 0u] + (palettes ? palettes[i] : 0u);
}

#define B2D_CU(call)                                             \
    do {                                                         \
        cudaError_t e_ = (call);                                 \
        if (e_ != cudaSuccess) return b2d::cuda_fail(e_, #call); \
    } while (0)
