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
// BSP walk + raster of n device poses into d_index / d_rgba (nullable) on `stream`; not synchronised.  `frame_states`
// (nullable): n compact states (r->layout.words words each), frame i rendered at its own state.
int enqueue_frames(b2d_renderer *r, const Pose *d_poses, int n, uint8_t *d_index, uint32_t *d_rgba, cudaStream_t stream,
                   const uint32_t *frame_states = nullptr);
// A one-call render of `batches` batches walks the first into the next worklist slot and alternates slots from there: it
// is refused (B2D_ERR_INVALID_ARG) before anything is enqueued while a slot it would use holds a walked, unrastered batch.
int check_slots_free(const b2d_renderer *r, size_t batches);
// the two halves (b2d_walk_device / b2d_raster_device): a background walk into a worklist slot, the raster of a ticket
int walk_frames(b2d_renderer *r, const Pose *d_poses, int n, cudaStream_t stream, int64_t *ticket_out, bool background);
int raster_frames(b2d_renderer *r, int64_t ticket, uint8_t *d_index, uint32_t *d_rgba, cudaStream_t stream);
// per-frame states and levels (b2d_render_levels_states & co.): the n HOST levels and states checked and each frame's compact
// state built with its level's layout (frame i's from fs[starts[i]]); nothing is enqueued
int build_levels_states(const b2d_renderer *r, const uint32_t *levels, const b2d_frame_state *states, size_t n,
                        const b2d_sector_move *moves, size_t n_moves, std::vector<uint32_t> &fs, std::vector<size_t> &starts);
// the walk of such a batch (levels, fs and starts of its n frames as build_levels_states left them) into a worklist slot
int walk_levels_states_frames(b2d_renderer *r, const Pose *d_poses, const uint32_t *levels, const uint32_t *fs, const size_t *starts,
                              int n, cudaStream_t stream, int64_t *ticket_out, bool background);

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
};

// A worklist slot: the BSP walk of batch k+1 may run (b2d_walk_device, another stream) while batch k is rastered.
struct WorkSlot {
    DeviceBuf<FrameConst> frames;                         // frames, worklist and events exist together (ensure_slot)
    DeviceBuf<SegFrame> work;
    Event walk_done, raster_done;
    int n = 0;                                            // frames walked into the slot
    int64_t ticket = -1;
    bool rastered = true;
    bool per_frame = false;                               // the batch was walked with per-frame states
    bool per_level = false;                               // ... or with per-frame levels (both: b2d_render_levels_states)
    int sets = 0;                                         // ... into this many table sets of the arena (distinct states)
    // per-frame levels (b2d_render_levels & co.; allocated by the first such call): [the DeviceScene of every level as this
    // slot's batches read it | the compact states of the levels whose table sets a batch re-expands | each frame's level]
    // on the device, and its pinned staging
    DeviceBuf<uint8_t> levels;
    PinnedBuf<uint8_t> h_levels;
    Event levels_copied;                                  // h_levels has been read by its copy
    // per-frame states (b2d_render_states & co.): an arena of up to max_batch expanded table sets (allocated by the first
    // such call), and the compact states + per-frame set indices on the device and their pinned staging, shared with the
    // expansion of the slot's own table set
    DeviceBuf<uint8_t> arena;
    DeviceBuf<uint32_t> states;                           // max_batch compact states, then max_batch set indices
    PinnedBuf<uint32_t> h_states;                         // same layout
    Event states_copied;                                  // h_states has been read by its copy
    // per-frame states and levels (b2d_render_levels_states & co.): `states` and `h_states` then hold the batch's
    // LevelsStatesBatch sections (b2d_api.cu), in states_bytes bytes (grown by the first such call of the slot)
    size_t states_bytes = 0;
    std::vector<uint32_t> set_level;                      // level of each table set
    std::vector<size_t> set_off;                          // byte offset of each table set in the arena
};

// Host-path staging (created by the first b2d_render & co.): double-buffered frame outputs.
struct HostStaging {
    Stream render_stream, copy_stream[2];                 // one copy stream per staging buffer
    Event rendered[2], copied[2];
    DeviceBuf<uint8_t> index[2];
    PinnedBuf<Pose> poses;                                // two buffers of max_batch poses
    std::array<DeviceBuf<uint32_t>, 2> rgba;              // created by the first call that asks for RGBA frames
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
    // Scenes with time-dependent content or dynamic sectors (DESIGN.md §3 "State arena"); the rest stays empty.  The
    // device blob is never written after creation: the state rule reads its rest-state sections, and every batch reads
    // its five state-dependent tables from a table set expanded on the device from a compact state.
    std::vector<uint8_t> h_blob;                          // host copy of the scene
    StateLayout layout;
    std::vector<uint32_t> state;                          // the level's own compact state (set_time, set_*sector_moves)
    DeviceBuf<uint32_t> d_slot_maps;                      // StateLayout::sector_slots, then ::mid_seg
    StateSrc src{};                                       // device pointers into d_blob and d_slot_maps
    StateTables state_tables{};                           // slot size and section offsets (base / frame_slot per slot)
    size_t stage_off = 0;                                 // byte offset of its compact state in WorkSlot::levels
    // per worklist slot: the table set the slot's batches read and the compact state it was expanded from
    struct Slot {
        DeviceBuf<uint8_t> tables;
        std::vector<uint32_t> state;
    } slot[2];
};

struct b2d_renderer {
    int device = 0;
    View view{};
    int max_batch = 0;
    int stride = 0;                 // worklist entries per frame (= the largest n_segs + n_sprites of the levels)
    size_t walk_smem = 0;           // the largest walk_smem_per_warp of the levels
    // the levels; every entry point without a level argument acts on level 0
    std::vector<LevelRes> lv;
    size_t levels_frames_off = 0;   // byte offset of the frame levels in WorkSlot::levels
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
    // b2d_palette_lut_levels_device: every level's palette, [n_levels][256], and the frame levels of a call on the device
    // with their pinned staging (grown by a call with more frames than it holds)
    DeviceBuf<uint32_t> d_palettes;
    DeviceBuf<uint32_t> d_lut_levels;
    PinnedBuf<uint32_t> h_lut_levels;
    size_t lut_levels_cap = 0;
    Event lut_levels_copied, lut_done;                    // the staging has been read by its copy; the kernel has read the copy
    // b2d_resolve_device: its own frame levels on the device and their pinned staging, with the same rules
    DeviceBuf<uint32_t> d_resolve_levels;
    PinnedBuf<uint32_t> h_resolve_levels;
    size_t resolve_levels_cap = 0;
    Event resolve_levels_copied, resolve_done;
    DeviceBuf<uint32_t> d_masked_counter;
    int64_t launches = 0;
    bool profiling = false;
    std::vector<Event> prof_events;         // pairs: before / after one kernel launch
    std::vector<int> prof_kinds;            // per pair: 0 = walk, 1 = raster

    ~b2d_renderer() { cudaSetDevice(device); }            // the members are released on the renderer's device
};

#define B2D_CU(call)                                             \
    do {                                                         \
        cudaError_t e_ = (call);                                 \
        if (e_ != cudaSuccess) return b2d::cuda_fail(e_, #call); \
    } while (0)
