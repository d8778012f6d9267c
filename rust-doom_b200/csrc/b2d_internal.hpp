// Private to libb2d.so: the handle types behind include/b2d.h and the helpers its translation units share
// (b2d_api.cu: archive / scene / renderer entry points; b2d_sharded.cu: multi-GPU sharded render over NCCL).
#pragma once
#include <memory>
#include <string>
#include <vector>

#include "../../include/b2d.h"
#include "b2d_kernels.cuh"
#include "b2d_scene.hpp"
#include "b2d_wad.hpp"

using namespace b2d;

struct b2d_archive {
    std::unique_ptr<Archive> wad;
};

struct b2d_scene {
    std::vector<uint8_t> blob;
    Level level;
    b2d_scene_info info;
};

struct b2d_renderer {
    int device = 0;
    View view{};
    int max_batch = 0;
    int stride = 0;                 // worklist entries per frame (= n_segs + n_sprites)
    uint8_t *d_blob = nullptr;
    uint32_t *d_yslope = nullptr;
    uint16_t *d_skyrow = nullptr;
    int32_t *d_status = nullptr;
    uint32_t *d_masked = nullptr;
    uint8_t *d_lit = nullptr;       // colormap-applied copies of the texels (32 light rows + the opacity plane)
    // ... and of the flats, in a region whose address is a multiple of 4 GiB: the raster then forms a flat texel's address
    // as {high word, 32-bit offset} without a 64-bit add (one instruction per flat pixel).  Reserved + mapped through the
    // driver's virtual-memory API (cuMemAddressReserve takes an alignment); an over-sized cudaMalloc is the fall-back.
    uint8_t *d_lit_flats = nullptr;
    size_t lit_flats_bytes = 0;     // mapped size (VMM) or 0
    unsigned long long lit_flats_handle = 0;
    uint8_t *d_lit_flats_raw = nullptr;   // fall-back allocation the aligned pointer lies in
    DeviceScene ds{};
    Pose *d_poses = nullptr;
    // two worklist slots: the BSP walk of batch k+1 may run (b2d_walk_device, another stream) while batch k is rastered
    FrameConst *d_frames[2] = {nullptr, nullptr};
    SegFrame *d_work[2] = {nullptr, nullptr};
    cudaEvent_t walk_done[2] = {nullptr, nullptr}, raster_done[2] = {nullptr, nullptr};
    int slot_n[2] = {0, 0};          // frames walked into the slot
    int64_t slot_ticket[2] = {-1, -1};
    bool slot_rastered[2] = {true, true};
    int64_t next_ticket = 0;
    int last_slot = 0;
    // host-path staging (allocated on first b2d_render): double-buffered frame outputs
    uint8_t *d_index[2] = {nullptr, nullptr};
    uint32_t *d_rgba[2] = {nullptr, nullptr};
    Pose *h_poses = nullptr;        // pinned
    cudaStream_t render_stream = nullptr, copy_stream[2] = {nullptr, nullptr};   // one copy stream per staging buffer
    cudaEvent_t rendered[2] = {nullptr, nullptr}, copied[2] = {nullptr, nullptr};
    std::vector<uint8_t> h_blob;    // host copy of the scene, kept only when it has time-dependent content
    uint32_t tics = 0;
    // time-dependent tables (texture records, sectors, segs, sprites): rebuilt on the host into one of two pinned
    // staging buffers and copied over their sections of the device blob in stream order (b2d_renderer_set_time_async)
    uint8_t *h_timed[2] = {nullptr, nullptr};
    cudaEvent_t timed_copied[2] = {nullptr, nullptr};     // staging buffer i has been read by its copy
    cudaEvent_t tables_ready = nullptr;                   // last table upload; launches on other streams wait for it
    bool tables_pending = false;
    int timed_next = 0;
    size_t timed_bytes = 0;
    uint8_t *d_walk_static = nullptr;                     // node / subsector tables as the walk kernel's shared memory holds them
    std::vector<int32_t> floor_off, ceil_off;             // state of the moving sectors (one offset per sector; empty = at rest)
    std::vector<uint8_t> cur_tables, scratch_tables;      // host copies: tables of the last upload / of a candidate time
    // per-frame states (b2d_render_states & co., DESIGN.md §3 "State arena"): the device copy of the rest-state sections
    // the state rule reads, and per worklist slot an arena of up to max_batch expanded table sets, the batch's distinct
    // compact states + per-frame slot indices on the device and their pinned staging.  Allocated by the first such call.
    StateLayout layout;                                   // scenes with time-dependent content or dynamic sectors
    uint8_t *d_pristine = nullptr;
    StateSrc src{};                                       // device pointers into d_pristine
    StateTables state_tables{};                           // slot size and section offsets (base / frame_slot per slot)
    uint8_t *d_arena[2] = {nullptr, nullptr};
    uint32_t *d_states[2] = {nullptr, nullptr};           // max_batch compact states, then max_batch slot indices
    uint32_t *h_states[2] = {nullptr, nullptr};           // pinned, same layout
    cudaEvent_t states_copied[2] = {nullptr, nullptr};    // h_states[i] has been read by its copy
    bool slot_states[2] = {false, false};                 // the batch in worklist slot i was walked with per-frame states
    cudaEvent_t masked_done = nullptr;                    // last raster that used the masked-entry arena
    uint32_t *d_masked_counter = nullptr;
    int64_t launches = 0;
    int last_n = 0;
    bool profiling = false;
    std::vector<cudaEvent_t> prof_events;   // pairs: before / after one kernel launch
    std::vector<int> prof_kinds;            // per pair: 0 = walk, 1 = raster
};


namespace b2d {
int fail(int code, const std::string &msg);            // sets the thread-local message, returns code
int cuda_fail(cudaError_t e, const char *what);
// BSP walk + raster of n device poses into d_index / d_rgba (nullable) on `stream`; not synchronised.  `frame_states`
// (nullable): n compact states (r->layout.words words each), frame i rendered at its own state.
int enqueue_frames(b2d_renderer *r, const Pose *d_poses, int n, uint8_t *d_index, uint32_t *d_rgba, cudaStream_t stream,
                   const uint32_t *frame_states = nullptr);
// the two halves (b2d_walk_device / b2d_raster_device): a background walk into a worklist slot, the raster of a ticket
int walk_frames(b2d_renderer *r, const Pose *d_poses, int n, cudaStream_t stream, int64_t *ticket_out, bool background);
int raster_frames(b2d_renderer *r, int64_t ticket, uint8_t *d_index, uint32_t *d_rgba, cudaStream_t stream);
}  // namespace b2d

#define B2D_CU(call)                                             \
    do {                                                         \
        cudaError_t e_ = (call);                                 \
        if (e_ != cudaSuccess) return b2d::cuda_fail(e_, #call); \
    } while (0)
