// C-ABI of libb2d.so (declared in include/b2d.h).  Thin, exception-free boundary over the C++ host
// side (WAD loader, scene compiler) and the CUDA kernels.  There is deliberately no CPU rendering
// path here: every render entry point launches the sm_90a kernels or fails with B2D_ERR_CUDA.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "b2d_internal.hpp"

static_assert(sizeof(b2d_pose) == sizeof(Pose) && sizeof(b2d_view) == sizeof(View), "ABI structs");

#include <cuda.h>

namespace {
thread_local std::string g_error;

// ---- 4 GiB aligned device memory (driver VMM API, resolved through the runtime: no link-time dependency on libcuda) ----
struct Vmm {
    CUresult (*GetGranularity)(size_t *, const CUmemAllocationProp *, CUmemAllocationGranularity_flags) = nullptr;
    CUresult (*AddressReserve)(CUdeviceptr *, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
    CUresult (*Create)(CUmemGenericAllocationHandle *, size_t, const CUmemAllocationProp *, unsigned long long) = nullptr;
    CUresult (*Map)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
    CUresult (*SetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc *, size_t) = nullptr;
    CUresult (*Unmap)(CUdeviceptr, size_t) = nullptr;
    CUresult (*Release)(CUmemGenericAllocationHandle) = nullptr;
    CUresult (*AddressFree)(CUdeviceptr, size_t) = nullptr;
    bool ok = false;
};
const Vmm &vmm() {
    static Vmm v;
    static bool init = false;
    if (!init) {
        init = true;
        auto get = [](const char *name, void **fn) {
            cudaDriverEntryPointQueryResult q;
            return cudaGetDriverEntryPoint(name, fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess && *fn;
        };
        v.ok = get("cuMemGetAllocationGranularity", (void **)&v.GetGranularity) && get("cuMemAddressReserve", (void **)&v.AddressReserve) &&
               get("cuMemCreate", (void **)&v.Create) && get("cuMemMap", (void **)&v.Map) && get("cuMemSetAccess", (void **)&v.SetAccess) &&
               get("cuMemUnmap", (void **)&v.Unmap) && get("cuMemRelease", (void **)&v.Release) && get("cuMemAddressFree", (void **)&v.AddressFree);
        cudaGetLastError();
    }
    return v;
}
constexpr size_t k4G = (size_t)1 << 32;

// device memory of `bytes` bytes at an address that is a multiple of 4 GiB (empty if there is none)
Aligned4G alloc_aligned_4g(int device, size_t bytes) {
    const Vmm &v = vmm();
    if (v.ok && !getenv("B2D_NO_VMM")) {
        CUmemAllocationProp prop;
        std::memset(&prop, 0, sizeof prop);
        prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
        prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
        prop.location.id = device;
        size_t gran = 0;
        if (v.GetGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM) == CUDA_SUCCESS && gran) {
            const size_t size = (bytes + gran - 1) / gran * gran;
            CUdeviceptr ptr = 0;
            CUmemGenericAllocationHandle h = 0;
            if (v.AddressReserve(&ptr, size, k4G, 0, 0) == CUDA_SUCCESS) {
                if ((ptr & (k4G - 1)) == 0 && v.Create(&h, size, &prop, 0) == CUDA_SUCCESS) {
                    CUmemAccessDesc acc;
                    std::memset(&acc, 0, sizeof acc);
                    acc.location = prop.location;
                    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
                    if (v.Map(ptr, size, 0, h, 0) == CUDA_SUCCESS) {
                        if (v.SetAccess(ptr, size, &acc, 1) == CUDA_SUCCESS)
                            return Aligned4G(reinterpret_cast<uint8_t *>(ptr), Aligned4GFree{size, (unsigned long long)h, nullptr});
                        v.Unmap(ptr, size);
                    }
                    v.Release(h);
                }
                v.AddressFree(ptr, size);
            }
        }
    }
    // fall-back: a plain allocation 4 GiB larger than needed always contains an aligned address
    void *raw = nullptr;
    if (cudaMalloc(&raw, bytes + k4G) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return Aligned4G(reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(raw) + k4G - 1) & ~(uintptr_t)(k4G - 1)),
                     Aligned4GFree{0, 0, raw});
}
}

void b2d::Aligned4GFree::operator()(uint8_t *p) const {
    if (mapped) {
        const Vmm &v = vmm();
        v.Unmap(reinterpret_cast<CUdeviceptr>(p), mapped);
        v.Release((CUmemGenericAllocationHandle)handle);
        v.AddressFree(reinterpret_cast<CUdeviceptr>(p), mapped);
    } else {
        cudaFree(raw);
    }
}

namespace b2d {
int fail(int code, const std::string &msg) {
    g_error = msg;
    return code;
}

int cuda_fail(cudaError_t e, const char *what) {
    return fail(B2D_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}
}  // namespace b2d

namespace {

#define CU(call)                                         \
    do {                                                 \
        cudaError_t e_ = (call);                         \
        if (e_ != cudaSuccess) return cuda_fail(e_, #call); \
    } while (0)

template <typename Fn>
int guarded(Fn fn) {
    try {
        return fn();
    } catch (const WadError &e) {
        return fail(e.code == kErrIo ? B2D_ERR_IO : e.code == kErrArg ? B2D_ERR_INVALID_ARG : B2D_ERR_CORRUPT_WAD, e.what());
    } catch (const std::bad_alloc &) {
        return fail(B2D_ERR_NO_MEMORY, "out of host memory");
    } catch (const std::exception &e) {
        return fail(B2D_ERR_INVALID_ARG, e.what());
    }
}

// A worklist slot's frames, worklist and events, created together: a failed call leaves the slot without any of them.
int ensure_slot(const b2d_renderer *r, WorkSlot &s) {
    if (s.frames) return B2D_OK;
    DeviceBuf<FrameConst> frames; DeviceBuf<SegFrame> work;
    Event walk_done, raster_done;
    CU(allocate(frames, sizeof(FrameConst) * (size_t)r->max_batch));
    CU(allocate(work, sizeof(SegFrame) * (size_t)r->max_batch * (size_t)r->stride));
    CU(event_create(walk_done));
    CU(event_create(raster_done));
    s.frames = std::move(frames); s.work = std::move(work);
    s.walk_done = std::move(walk_done); s.raster_done = std::move(raster_done);
    return B2D_OK;
}

// Per-frame states: the two worklist slots' arenas of max_batch table sets, allocated together by the first such call.
int ensure_states(b2d_renderer *r) {
    if (r->slot[0].arena) return B2D_OK;
    DeviceBuf<uint8_t> arena[2];
    for (auto &a : arena) CU(allocate(a, (size_t)r->max_batch * r->lv[0].state_tables.slot_bytes));
    for (int i = 0; i < 2; i++) r->slot[i].arena = std::move(arena[i]);
    return B2D_OK;
}

// Per-frame levels: both worklist slots' scene arrays, level staging and events, allocated together by the first such call.
int ensure_levels(b2d_renderer *r) {
    if (r->slot[0].levels) return B2D_OK;
    const size_t bytes = r->levels_frames_off + 4 * (size_t)r->max_batch;
    DeviceBuf<uint8_t> d[2];
    PinnedBuf<uint8_t> h[2];
    Event ev[2];
    for (int i = 0; i < 2; i++) {
        CU(allocate(d[i], bytes));
        CU(allocate(h[i], bytes));
        CU(event_create(ev[i]));
    }
    for (int i = 0; i < 2; i++) {
        r->slot[i].levels = std::move(d[i]);
        r->slot[i].h_levels = std::move(h[i]);
        r->slot[i].levels_copied = std::move(ev[i]);
    }
    return B2D_OK;
}

// the arena view of worklist slot `slot` (after ensure_states)
StateTables slot_tables(const b2d_renderer *r, int slot) {
    StateTables t = r->lv[0].state_tables;
    t.base = r->slot[slot].arena.get();
    t.frame_slot = r->slot[slot].states.get() + (size_t)r->max_batch * r->lv[0].layout.words;
    return t;
}

// a level's scene as the kernels of worklist slot `slot` read it: on a timed scene, the five state-dependent tables are the
// level's table set of that slot
DeviceScene slot_scene(const LevelRes &lv, int slot) {
    DeviceScene d = lv.ds;
    const uint8_t *set = lv.slot[slot].tables.get();
    if (!set) return d;
    const StateTables &t = lv.state_tables;
    d.tex = reinterpret_cast<const TexRec *>(set);
    d.sectors = reinterpret_cast<const SectorRec *>(set + t.off_sectors);
    d.segs = reinterpret_cast<const SegRec *>(set + t.off_segs);
    d.sprites = reinterpret_cast<const SpriteRec *>(set + t.off_sprites);
    d.mids = reinterpret_cast<const MidRec *>(set + t.off_mids);
    return d;
}

// BSP walk of a batch into the next worklist slot, on `stream`.  The slot's previous raster (if any, on whatever
// stream) is awaited through an event, so a caller may run walks and rasters on two streams and have the walk of
// batch k+1 overlap the raster of batch k.  `frame_states` (nullable): one compact state per frame; the batch's distinct
// states are expanded into the slot's arena on `stream` first (frames with equal states share one table set).  A plain
// batch on a timed scene reads the slot's own table set, which is re-expanded on `stream` when the renderer's state
// differs from the one the set holds: the walk and the raster of a ticket read one state whatever is set in between.
int walk_into_slot(b2d_renderer *r, const Pose *d_poses, int n, cudaStream_t stream, int64_t *ticket_out, bool background = false,
                   const uint32_t *frame_states = nullptr) {
    const int slot = (int)(r->next_ticket & 1);
    WorkSlot &s = r->slot[slot];
    if (!s.rastered) return fail(B2D_ERR_INVALID_ARG, "both worklist slots hold batches that were walked but not rastered yet");
    int rc = frame_states ? ensure_states(r) : B2D_OK;
    if (rc == B2D_OK) rc = ensure_slot(r, s);
    if (rc != B2D_OK) return rc;
    LevelRes &lv = r->lv[0];
    const bool restate = !frame_states && lv.slot[slot].tables && lv.slot[slot].state != lv.state;
    const size_t words = lv.layout.words;
    int nstates = 0;
    if (frame_states || restate) {
        CU(cudaEventSynchronize(s.states_copied.get()));     // the copy issued two batches ago has read the staging
        uint32_t *hs = s.h_states.get(), *hslot = hs + (size_t)r->max_batch * words;
        if (restate) {
            std::memcpy(hs, lv.state.data(), 4 * words);
            nstates = 1;
        } else {
            // distinct states -> slots 0, 1, ... in order of first appearance, anywhere in the batch
            std::unordered_map<std::string, uint32_t> seen;
            seen.reserve((size_t)n);
            for (int f = 0; f < n; f++) {
                const uint32_t *w = frame_states + (size_t)f * words;
                auto it = seen.emplace(std::string(reinterpret_cast<const char *>(w), 4 * words), (uint32_t)nstates);
                if (it.second) std::memcpy(hs + (size_t)nstates++ * words, w, 4 * words);
                hslot[f] = it.first->second;
            }
        }
    }
    CU(cudaStreamWaitEvent(stream, s.raster_done.get(), 0));      // the raster that last read this slot
    const StateTables stt = frame_states ? slot_tables(r, slot) : StateTables{};
    if (nstates) {
        uint32_t *hs = s.h_states.get();
        CU(cudaMemcpyAsync(s.states.get(), hs, 4 * words * (size_t)nstates, cudaMemcpyHostToDevice, stream));
        if (frame_states)
            CU(cudaMemcpyAsync(const_cast<uint32_t *>(stt.frame_slot), hs + (size_t)r->max_batch * words, 4 * (size_t)n,
                               cudaMemcpyHostToDevice, stream));
        CU(cudaEventRecord(s.states_copied.get(), stream));
        uint8_t *sets = (frame_states ? s.arena : lv.slot[slot].tables).get();
        CU(launch_state_tables(lv.src, s.states.get(), (uint32_t)words, nstates, sets, lv.state_tables, stream));
        r->launches += 1;
        if (restate) lv.slot[slot].state = lv.state;
    }
    Event ev[2];
    if (r->profiling) {
        for (auto &e : ev) CU(event_create(e, cudaEventDefault));
        CU(cudaEventRecord(ev[0].get(), stream));
    }
    CU(launch_walk(slot_scene(lv, slot), r->view, d_poses, n, s.frames.get(), s.work.get(), r->stride, stream, background,
                   frame_states ? &stt : nullptr));
    if (r->profiling) {
        CU(cudaEventRecord(ev[1].get(), stream));
        for (auto &e : ev) r->prof_events.push_back(std::move(e));
        r->prof_kinds.push_back(0);
    }
    CU(cudaEventRecord(s.walk_done.get(), stream));
    s.n = n;
    s.per_frame = frame_states != nullptr;
    s.per_level = false;
    s.sets = frame_states ? nstates : 0;
    s.ticket = r->next_ticket;
    s.rastered = false;
    r->last_slot = slot;
    r->launches += 1;
    *ticket_out = r->next_ticket++;
    return B2D_OK;
}

// BSP walk of a batch with per-frame levels (levels[i] < r->lv.size(), checked by the caller) into the next worklist slot,
// as walk_into_slot.  The frame levels, the DeviceScene of every level as the slot reads it and the compact states of the
// timed levels the batch uses whose table set of the slot is stale go to the device in one copy; each stale set is then
// re-expanded (one launch per such level) before the walk.
int walk_levels_into_slot(b2d_renderer *r, const Pose *d_poses, const uint32_t *levels, int n, cudaStream_t stream,
                          int64_t *ticket_out, bool background) {
    const int slot = (int)(r->next_ticket & 1);
    WorkSlot &s = r->slot[slot];
    if (!s.rastered) return fail(B2D_ERR_INVALID_ARG, "both worklist slots hold batches that were walked but not rastered yet");
    int rc = ensure_levels(r);
    if (rc == B2D_OK) rc = ensure_slot(r, s);
    if (rc != B2D_OK) return rc;
    CU(cudaEventSynchronize(s.levels_copied.get()));     // the copy issued two batches ago has read the staging
    uint8_t *h = s.h_levels.get();
    DeviceScene *scenes = reinterpret_cast<DeviceScene *>(h);
    uint32_t *frame_level = reinterpret_cast<uint32_t *>(h + r->levels_frames_off);
    const size_t nlev = r->lv.size();
    std::vector<char> used(nlev, 0);
    for (int f = 0; f < n; f++) {
        frame_level[f] = levels[f];
        used[levels[f]] = 1;
    }
    std::vector<size_t> stale;
    for (size_t k = 0; k < nlev; k++) {
        LevelRes &lv = r->lv[k];
        scenes[k] = slot_scene(lv, slot);
        if (used[k] && lv.slot[slot].tables && lv.slot[slot].state != lv.state) {
            std::memcpy(h + lv.stage_off, lv.state.data(), 4 * lv.layout.words);
            stale.push_back(k);
        }
    }
    CU(cudaStreamWaitEvent(stream, s.raster_done.get(), 0));      // the raster that last read this slot
    CU(cudaMemcpyAsync(s.levels.get(), h, r->levels_frames_off + 4 * (size_t)n, cudaMemcpyHostToDevice, stream));
    CU(cudaEventRecord(s.levels_copied.get(), stream));
    for (size_t k : stale) {
        LevelRes &lv = r->lv[k];
        CU(launch_state_tables(lv.src, reinterpret_cast<const uint32_t *>(s.levels.get() + lv.stage_off), (uint32_t)lv.layout.words,
                               1, lv.slot[slot].tables.get(), lv.state_tables, stream));
        r->launches += 1;
        lv.slot[slot].state = lv.state;
    }
    Event ev[2];
    if (r->profiling) {
        for (auto &e : ev) CU(event_create(e, cudaEventDefault));
        CU(cudaEventRecord(ev[0].get(), stream));
    }
    const LevelTables lt{reinterpret_cast<const DeviceScene *>(s.levels.get()),
                         reinterpret_cast<const uint32_t *>(s.levels.get() + r->levels_frames_off)};
    CU(launch_walk_levels(lt, r->walk_smem, r->view, d_poses, n, s.frames.get(), s.work.get(), r->stride, stream, background));
    if (r->profiling) {
        CU(cudaEventRecord(ev[1].get(), stream));
        for (auto &e : ev) r->prof_events.push_back(std::move(e));
        r->prof_kinds.push_back(0);
    }
    CU(cudaEventRecord(s.walk_done.get(), stream));
    s.n = n;
    s.per_frame = false;
    s.per_level = true;
    s.sets = 0;
    s.ticket = r->next_ticket;
    s.rastered = false;
    r->last_slot = slot;
    r->launches += 1;
    *ticket_out = r->next_ticket++;
    return B2D_OK;
}

int raster_from_slot(b2d_renderer *r, int64_t ticket, uint8_t *d_index, uint32_t *d_rgba, cudaStream_t stream) {
    const int slot = (int)(ticket & 1);
    WorkSlot &s = r->slot[slot];
    if (ticket < 0 || s.ticket != ticket || s.rastered) return fail(B2D_ERR_INVALID_ARG, "unknown or already rastered walk ticket");
    CU(cudaStreamWaitEvent(stream, s.walk_done.get(), 0));
    if (r->d_masked) {
        // one arena of deferred masked entries per renderer: rasters that use it run one after the other (each fills the
        // machine on its own, so nothing is lost), whatever streams they were enqueued on
        CU(cudaStreamWaitEvent(stream, r->masked_done.get(), 0));
        CU(cudaMemsetAsync(r->d_masked_counter.get(), 0, sizeof(uint32_t), stream));
    }
    Event ev[2];
    if (r->profiling) {
        for (auto &e : ev) CU(event_create(e, cudaEventDefault));
        CU(cudaEventRecord(ev[0].get(), stream));
    }
    if (s.per_level) {
        const LevelTables lt{reinterpret_cast<const DeviceScene *>(s.levels.get()),
                             reinterpret_cast<const uint32_t *>(s.levels.get() + r->levels_frames_off)};
        CU(launch_raster_levels(lt, r->d_masked != nullptr, r->view, s.frames.get(), s.work.get(), r->stride, s.n, d_index,
                                d_rgba, stream));
    } else {
        const StateTables stt = s.per_frame ? slot_tables(r, slot) : StateTables{};
        CU(launch_raster(slot_scene(r->lv[0], slot), r->view, s.frames.get(), s.work.get(), r->stride, s.n, d_index, d_rgba,
                         stream, s.per_frame ? &stt : nullptr));
    }
    if (r->profiling) {
        CU(cudaEventRecord(ev[1].get(), stream));
        for (auto &e : ev) r->prof_events.push_back(std::move(e));
        r->prof_kinds.push_back(1);
    }
    CU(cudaEventRecord(s.raster_done.get(), stream));
    if (r->d_masked) CU(cudaEventRecord(r->masked_done.get(), stream));
    s.rastered = true;
    r->launches += 1;
    return B2D_OK;
}

// the state-dependent tables (level time `tics`, sector offsets), laid out [tex | sectors | segs | sprites | mids]
size_t state_table_bytes(const uint8_t *blob) {
    const uint32_t *h = reinterpret_cast<const uint32_t *>(blob);
    return h[H_NTEX] * sizeof(TexRec) + h[H_NSECTORS] * sizeof(SectorRec) + h[H_NSEGS] * sizeof(SegRec) +
           h[H_NSPRITES] * sizeof(SpriteRec) + h[H_NMIDS] * sizeof(MidRec);
}

void state_tables(const uint8_t *blob, uint32_t tics, const int32_t *floor_off, const int32_t *ceil_off, uint8_t *out) {
    const uint32_t *h = reinterpret_cast<const uint32_t *>(blob);
    TexRec *tex = reinterpret_cast<TexRec *>(out);
    SectorRec *sectors = reinterpret_cast<SectorRec *>(tex + h[H_NTEX]);
    SegRec *segs = reinterpret_cast<SegRec *>(sectors + h[H_NSECTORS]);
    SpriteRec *sprites = reinterpret_cast<SpriteRec *>(segs + h[H_NSEGS]);
    MidRec *mids = reinterpret_cast<MidRec *>(sprites + h[H_NSPRITES]);
    scene_at_time(blob, tics, tex, sectors, segs, sprites, mids, floor_off, ceil_off);
}

// The compact state of level time `tics` with the level's current sector moves into out[layout.words] (out is not
// lv.state): the moved flag and the offsets, words 1 .. 2 + 2 * ndyn, do not depend on the time.
void state_at(const LevelRes &lv, uint32_t tics, uint32_t *out) {
    compact_state(lv.h_blob.data(), lv.layout, tics, nullptr, nullptr, out);
    std::copy(lv.state.begin() + 1, lv.state.begin() + 2 + 2 * (ptrdiff_t)lv.layout.dyn_sectors.size(), out + 1);
}

// The compact state of every frame of a b2d_render_states-style call into `out` (level 0's layout.words words per frame), checking
// everything first: nothing is enqueued for a call with an invalid frame.  `out` stays empty for a scene without
// time-dependent content or dynamic sectors: its frames all render with the per-batch tables.
int build_states(const b2d_renderer *r, const b2d_frame_state *states, size_t n, const b2d_sector_move *moves, size_t n_moves,
                 std::vector<uint32_t> &out) {
    out.clear();
    if (!states || (n_moves && !moves)) return fail(B2D_ERR_INVALID_ARG, "null argument");
    for (size_t i = 0; i < n; i++)
        if (states[i].first_move > n_moves || states[i].n_moves > n_moves - states[i].first_move)
            return fail(B2D_ERR_INVALID_ARG, "a frame's move range runs past the end of the move list");
    const LevelRes &lv = r->lv[0];
    if (lv.h_blob.empty()) {
        for (size_t i = 0; i < n; i++)
            if (states[i].n_moves) return fail(B2D_ERR_INVALID_ARG, "the scene declares no dynamic sectors");
        return B2D_OK;
    }
    const size_t words = lv.layout.words;
    out.resize(n * words);
    std::vector<int32_t> fo, co;
    for (size_t i = 0; i < n; i++) {
        bool moved = false;
        if (states[i].n_moves) {
            if (const char *why = expand_moves(lv.h_blob.data(), reinterpret_cast<const SectorMove *>(moves) + states[i].first_move,
                                               states[i].n_moves, fo, co)) {
                out.clear();
                return fail(B2D_ERR_INVALID_ARG, why);
            }
            for (size_t k = 0; k < fo.size() && !moved; k++) moved = fo[k] != 0 || co[k] != 0;    // all zero: at rest
        }
        compact_state(lv.h_blob.data(), lv.layout, states[i].tics, moved ? fo.data() : nullptr, moved ? co.data() : nullptr,
                      out.data() + i * words);
    }
    return B2D_OK;
}

// b2d_render_timed: tics[i] with the renderer's current moves
void timed_states(const b2d_renderer *r, const uint32_t *tics, size_t n, std::vector<uint32_t> &out) {
    out.clear();
    const LevelRes &lv = r->lv[0];
    if (lv.h_blob.empty()) return;
    const size_t words = lv.layout.words;
    out.resize(n * words);
    for (size_t i = 0; i < n; i++) state_at(lv, tics[i], out.data() + i * words);
}

}  // namespace

int b2d::walk_frames(b2d_renderer *r, const Pose *d_poses, int n, cudaStream_t stream, int64_t *ticket_out, bool background) {
    return walk_into_slot(r, d_poses, n, stream, ticket_out, background);
}
int b2d::raster_frames(b2d_renderer *r, int64_t ticket, uint8_t *d_index, uint32_t *d_rgba, cudaStream_t stream) {
    return raster_from_slot(r, ticket, d_index, d_rgba, stream);
}

// walk -> raster on the caller's stream
int b2d::enqueue_frames(b2d_renderer *r, const Pose *d_poses, int n, uint8_t *d_index, uint32_t *d_rgba,
                        cudaStream_t stream, const uint32_t *frame_states) {
    int64_t ticket = -1;
    int rc = walk_into_slot(r, d_poses, n, stream, &ticket, false, frame_states);
    if (rc != B2D_OK) return rc;
    return raster_from_slot(r, ticket, d_index, d_rgba, stream);
}

extern "C" {

const char *b2d_last_error(void) { return g_error.c_str(); }

// ---- archive ---------------------------------------------------------------------------------
int b2d_archive_open(const char *wad_path, b2d_archive **out) {
    if (!wad_path || !out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    return guarded([&] {
        auto a = std::make_unique<b2d_archive>();
        a->wad = std::make_unique<Archive>(Archive::open(wad_path));
        *out = a.release();
        return B2D_OK;
    });
}

int b2d_archive_open_memory(const void *bytes, size_t size, b2d_archive **out) {
    if (!bytes || !out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    return guarded([&] {
        const uint8_t *p = static_cast<const uint8_t *>(bytes);
        auto a = std::make_unique<b2d_archive>();
        a->wad = std::make_unique<Archive>(std::vector<uint8_t>(p, p + size));
        *out = a.release();
        return B2D_OK;
    });
}

int b2d_archive_open_files(const char *const *paths, int n_paths, b2d_archive **out) {
    if (!paths || !out || n_paths < 1) return fail(B2D_ERR_INVALID_ARG, "null argument");
    return guarded([&] {
        std::vector<std::string> ps;
        for (int i = 0; i < n_paths; i++) {
            if (!paths[i]) throw std::invalid_argument("null path");
            ps.emplace_back(paths[i]);
        }
        auto a = std::make_unique<b2d_archive>();
        a->wad = std::make_unique<Archive>(Archive::open(ps));
        *out = a.release();
        return B2D_OK;
    });
}

int b2d_archive_open_memory_files(const void *const *bytes, const size_t *sizes, int n_files, b2d_archive **out) {
    if (!bytes || !sizes || !out || n_files < 1) return fail(B2D_ERR_INVALID_ARG, "null argument");
    return guarded([&] {
        std::vector<std::vector<uint8_t>> files;
        for (int i = 0; i < n_files; i++) {
            if (!bytes[i]) throw std::invalid_argument("null file");
            const uint8_t *p = static_cast<const uint8_t *>(bytes[i]);
            files.emplace_back(p, p + sizes[i]);
        }
        auto a = std::make_unique<b2d_archive>();
        a->wad = std::make_unique<Archive>(std::move(files));
        *out = a.release();
        return B2D_OK;
    });
}

int b2d_archive_num_levels(const b2d_archive *a) {
    if (!a) return fail(B2D_ERR_INVALID_ARG, "null archive");
    return a->wad->num_levels();
}

int b2d_archive_level_name(const b2d_archive *a, int level_index, char name_out[9]) {
    if (!a || !name_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    return guarded([&] {
        const Name &n = a->wad->level_name(level_index);
        std::memcpy(name_out, n.data(), 8);
        name_out[8] = 0;
        return B2D_OK;
    });
}

void b2d_archive_close(b2d_archive *a) { delete a; }

int b2d_wad_name(const void *bytes, size_t size, char name_out[8]) {
    if (!bytes || !name_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    return guarded([&] {
        Name n = make_name(static_cast<const uint8_t *>(bytes), size);
        std::memcpy(name_out, n.data(), 8);
        return B2D_OK;
    });
}

// ---- scene -----------------------------------------------------------------------------------
namespace {
void fill_scene_info(b2d_scene *s) {
    const uint32_t *h = reinterpret_cast<const uint32_t *>(s->blob.data());
    b2d_scene_info &i = s->info;
    i.n_verts = (int32_t)h[H_NVERTS]; i.n_nodes = (int32_t)h[H_NNODES]; i.n_ssectors = (int32_t)h[H_NSSECTORS];
    i.n_segs = (int32_t)h[H_NSEGS]; i.n_sectors = (int32_t)h[H_NSECTORS]; i.n_textures = (int32_t)h[H_NTEX];
    i.n_flats = (int32_t)h[H_NFLATS]; i.blob_bytes = (int32_t)h[H_TOTAL];
    i.n_masked_mids = (int32_t)h[H_NMIDS]; i.n_sprites = (int32_t)h[H_NSPRITES];
    i.has_start = (int32_t)h[H_HAS_START];
    i.start.x = (int32_t)h[H_START_X] * 65536; i.start.y = (int32_t)h[H_START_Y] * 65536;
    i.start.z = (int32_t)h[H_START_Z] * 65536;
    i.start.angle = (uint32_t)(((uint64_t)h[H_START_ANGLE] << 32) / 360u);
    i.min_height = (int32_t)h[H_MIN_H]; i.max_height = (int32_t)h[H_MAX_H];
    i.n_dynamic = (int32_t)h[H_NDYN];
}
}  // namespace

namespace {
std::vector<DynRec> dyn_list(const b2d_dynamic_sector *dyn, size_t n) {
    std::vector<DynRec> v(n);
    for (size_t i = 0; i < n; i++) {
        v[i] = DynRec{};
        v[i].sector = dyn[i].sector;
        v[i].floor_min = dyn[i].floor_min; v[i].floor_max = dyn[i].floor_max;
        v[i].ceil_min = dyn[i].ceil_min; v[i].ceil_max = dyn[i].ceil_max;
    }
    return v;
}
}  // namespace

int b2d_scene_create_dynamic(const b2d_archive *a, int level_index, const b2d_dynamic_sector *dyn, size_t n_dyn, b2d_scene **out) {
    if (!a || !out || (n_dyn && !dyn)) return fail(B2D_ERR_INVALID_ARG, "null argument");
    return guarded([&] {
        auto s = std::make_unique<b2d_scene>();
        TextureDirectory td = TextureDirectory::load(*a->wad);
        s->level = Level::load(*a->wad, level_index);
        s->blob = compile_scene(s->level, td, dyn_list(dyn, n_dyn));
        fill_scene_info(s.get());
        *out = s.release();
        return B2D_OK;
    });
}

int b2d_scene_create(const b2d_archive *a, int level_index, b2d_scene **out) {
    return b2d_scene_create_dynamic(a, level_index, nullptr, 0, out);
}

int b2d_scene_create_from_lumps(const b2d_level_lumps *lv, const b2d_textures *tex, b2d_scene **out) {
    return b2d_scene_create_from_lumps_dynamic(lv, tex, nullptr, 0, out);
}

int b2d_scene_tables_at(const b2d_scene *s, uint32_t tics, const b2d_sector_move *moves, size_t n_moves, void *out,
                        size_t capacity, size_t *size_out) {
    if (!s || (n_moves && !moves)) return fail(B2D_ERR_INVALID_ARG, "null argument");
    const size_t need = state_table_bytes(s->blob.data());
    if (size_out) *size_out = need;
    if (!out) return B2D_OK;
    if (capacity < need) return fail(B2D_ERR_INVALID_ARG, "buffer too small for the tables");
    std::vector<int32_t> fo, co;
    if (n_moves) {
        if (const char *why = expand_moves(s->blob.data(), reinterpret_cast<const SectorMove *>(moves), n_moves, fo, co))
            return fail(B2D_ERR_INVALID_ARG, why);
    }
    state_tables(s->blob.data(), tics, n_moves ? fo.data() : nullptr, n_moves ? co.data() : nullptr, static_cast<uint8_t *>(out));
    return B2D_OK;
}

int b2d_scene_create_from_lumps_dynamic(const b2d_level_lumps *lv, const b2d_textures *tex, const b2d_dynamic_sector *dyn,
                                        size_t n_dyn, b2d_scene **out) {
    if (!lv || !tex || !out || (n_dyn && !dyn)) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if ((tex->n_textures && !tex->textures) || (tex->n_flats && !tex->flats) || (tex->n_colormaps && !tex->colormaps))
        return fail(B2D_ERR_INVALID_ARG, "null texture table");
    return guarded([&] {
        auto s = std::make_unique<b2d_scene>();
        const b2d_lump *src[8] = {&lv->things, &lv->linedefs, &lv->sidedefs, &lv->vertexes, &lv->segs, &lv->ssectors, &lv->nodes, &lv->sectors};
        RawLump lumps[8];
        for (int k = 0; k < 8; k++) { lumps[k].data = static_cast<const uint8_t *>(src[k]->data); lumps[k].size = src[k]->size; }
        s->level = Level::from_lumps(make_name(reinterpret_cast<const uint8_t *>(lv->name), 8), lumps);
        // a TextureDirectory filled from the caller's decoded images instead of PNAMES / TEXTUREx / F_START..F_END
        TextureDirectory td;
        td.textures.reserve(tex->n_textures);
        for (size_t i = 0; i < tex->n_textures; i++) {
            const b2d_image &im = tex->textures[i];
            if (im.width < 1 || im.height < 1 || im.width > 4096 || im.height > 4096 || !im.pixels)      // image.rs:9,49-52
                throw WadError(kErrCorrupt, "texture image out of range (1..4096 x 1..4096)");
            Image img;
            img.w = im.width; img.h = im.height;
            img.px.assign(im.pixels, im.pixels + (size_t)im.width * (size_t)im.height);
            td.texture_index[make_name(reinterpret_cast<const uint8_t *>(im.name), 8)] = (int)td.textures.size();   // later wins
            td.textures.push_back(std::move(img));
        }
        td.own_flats.resize(tex->n_flats);
        for (size_t i = 0; i < tex->n_flats; i++) {
            if (!tex->flats[i].pixels) throw WadError(kErrCorrupt, "null flat");
            std::memcpy(td.own_flats[i].data(), tex->flats[i].pixels, 4096);
            td.flat_index[make_name(reinterpret_cast<const uint8_t *>(tex->flats[i].name), 8)] = (int)i;
        }
        td.colormaps.resize(tex->n_colormaps);
        for (size_t i = 0; i < tex->n_colormaps; i++) std::memcpy(td.colormaps[i].data(), tex->colormaps + 256 * i, 256);
        if (tex->palette) {
            td.palettes.resize(1);
            std::memcpy(td.palettes[0].data(), tex->palette, 768);
        }
        s->blob = compile_scene(s->level, td, dyn_list(dyn, n_dyn));
        fill_scene_info(s.get());
        *out = s.release();
        return B2D_OK;
    });
}

int b2d_scene_info_get(const b2d_scene *s, b2d_scene_info *out) {
    if (!s || !out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    *out = s->info;
    return B2D_OK;
}

const void *b2d_scene_blob(const b2d_scene *s, size_t *size_out) {
    if (!s) return nullptr;
    if (size_out) *size_out = s->blob.size();
    return s->blob.data();
}

int b2d_scene_sector_at(const b2d_scene *s, double x, double y, int32_t *floor_out, int32_t *ceil_out) {
    if (!s) return fail(B2D_ERR_INVALID_ARG, "null scene");
    int sec = sector_at(s->level, x, y);
    if (sec >= 0) {
        if (floor_out) *floor_out = s->level.sectors[(size_t)sec].floor;
        if (ceil_out) *ceil_out = s->level.sectors[(size_t)sec].ceil;
    }
    return sec;
}

void b2d_scene_destroy(b2d_scene *s) { delete s; }

// ---- view ------------------------------------------------------------------------------------
int b2d_view_init(b2d_view *v, int width, int height, double fov_y_degrees) {
    if (!v) return fail(B2D_ERR_INVALID_ARG, "null view");
    if (width < 1 || height < 2 || width > 4096 || height > 2160 || !(fov_y_degrees > 1.0 && fov_y_degrees < 170.0))
        return fail(B2D_ERR_INVALID_ARG, "view out of range (width <= 4096, height <= 2160, 1 < fov < 170)");
    const double t = std::tan(fov_y_degrees * 3.14159265358979323846 / 360.0);
    v->width = width; v->height = height;
    v->FY2 = (int32_t)((double)height / t + 0.5);
    v->F = (int32_t)((double)height / (1.2 * t) + 0.5);     // aspect_ratio_correction (player.rs:87)
    if (v->F < 2 || v->FY2 < 2) return fail(B2D_ERR_INVALID_ARG, "degenerate focal length");
    if (width > kViewWidthPerF * v->F)
        return fail(B2D_ERR_INVALID_ARG, "view too wide for its focal length (width > 256 * F: short view at a wide field of view)");
    return B2D_OK;
}

// ---- renderer --------------------------------------------------------------------------------
namespace {
// Level `lv` of renderer `r` (device, view and max_batch set) from scene `s`: the scene, its pre-lit planes and walk tables
// on the device and, for a timed scene, its table set of each worklist slot at tic 0.  The DeviceScene's per-renderer fields
// (yslope, status word, masked-entry arena) are the caller's.
int create_level(b2d_renderer *r, LevelRes &lv, const b2d_scene *s) {
    const View &view = r->view;
    const uint32_t *h = reinterpret_cast<const uint32_t *>(s->blob.data());
    CU(allocate(lv.d_blob, s->blob.size()));
    CU(cudaMemcpy(lv.d_blob.get(), s->blob.data(), s->blob.size(), cudaMemcpyHostToDevice));
    const uint8_t *db = lv.d_blob.get();
    {   // sky texture row per screen row (sky.frag:12-26 at pitch 0)
        std::vector<uint16_t> sr((size_t)view.H, 0);
        int32_t sky = (int32_t)h[H_SKY_TEX];
        if (sky >= 0) {
            const TexRec *tr = reinterpret_cast<const TexRec *>(s->blob.data() + h[H_OFF_TEX]) + sky;
            for (int y = 0; y < view.H; y++) sr[(size_t)y] = (uint16_t)sky_row(y, view.H, (int32_t)tr->h);
        }
        CU(allocate(lv.d_skyrow, sr.size() * 2));
        CU(cudaMemcpy(lv.d_skyrow.get(), sr.data(), sr.size() * 2, cudaMemcpyHostToDevice));
    }
    DeviceScene &d = lv.ds;
    d.verts = reinterpret_cast<const int32_t *>(db + h[H_OFF_VERTS]);
    d.nodes = reinterpret_cast<const NodeRec *>(db + h[H_OFF_NODES]);
    d.ssectors = reinterpret_cast<const SSectorRec *>(db + h[H_OFF_SSECTORS]);
    {   // the walk kernel's traversal tables in the layout of its shared memory (one cp.async.bulk per CTA)
        const NodeRec *nodes = reinterpret_cast<const NodeRec *>(s->blob.data() + h[H_OFF_NODES]);
        std::vector<int32_t> img(8 * (size_t)h[H_NNODES] + 4 * (size_t)h[H_NSSECTORS]);
        for (uint32_t i = 0; i < h[H_NNODES]; i++) {
            int32_t *o = &img[8 * (size_t)i];
            o[0] = nodes[i].x; o[1] = nodes[i].y; o[2] = nodes[i].dx; o[3] = nodes[i].dy;
            o[4] = (int32_t)nodes[i].child[0]; o[5] = (int32_t)nodes[i].child[1]; o[6] = 0; o[7] = 0;
        }
        if (h[H_NSSECTORS])
            std::memcpy(&img[8 * (size_t)h[H_NNODES]], s->blob.data() + h[H_OFF_SSECTORS], sizeof(SSectorRec) * h[H_NSSECTORS]);
        CU(allocate(lv.d_walk_static, img.size() * 4 + 16));
        if (!img.empty()) CU(cudaMemcpy(lv.d_walk_static.get(), img.data(), img.size() * 4, cudaMemcpyHostToDevice));
        d.walk_static = lv.d_walk_static.get();
    }
    d.segs = reinterpret_cast<const SegRec *>(db + h[H_OFF_SEGS]);
    d.sectors = reinterpret_cast<const SectorRec *>(db + h[H_OFF_SECTORS]);
    d.tex = reinterpret_cast<const TexRec *>(db + h[H_OFF_TEX]);
    d.mids = reinterpret_cast<const MidRec *>(db + h[H_OFF_MIDS]);
    d.nmids = (int32_t)h[H_NMIDS];
    d.sprites = reinterpret_cast<const SpriteRec *>(db + h[H_OFF_SPRITES]);
    d.nsprites = (int32_t)h[H_NSPRITES];
    d.masked_list = nullptr; d.masked_counter = nullptr; d.masked_chunks = 0; d.masked_cap = 0;
    if (d.nmids > 0 || d.nsprites > 0) d.masked_cap = strip_masked_cap(d.nmids, d.nsprites);
    d.texels = db + h[H_OFF_TEXELS];
    d.flats = db + h[H_OFF_FLATS];
    d.colormap = db + h[H_OFF_COLORMAP];
    d.palette = reinterpret_cast<const uint32_t *>(db + h[H_OFF_PALETTE]);
    {   // pre-lit texel and flat planes: 32 x (texel bytes + flat bytes)
        const size_t tstride = (h[H_TEXEL_BYTES] + 255u) & ~(size_t)255, fstride = (size_t)h[H_NFLATS] * 4096u;
        if (tstride * 33 > 0xFFFFFFFFull || fstride * 32 > 0xFFFFFFFFull) return fail(B2D_ERR_INVALID_ARG, "level textures too large");
        CU(allocate(lv.d_lit, 33 * tstride + 256));                    // plane 32 of the texels: opacity
        lv.d_lit_flats = alloc_aligned_4g(r->device, 32 * fstride + 256);
        if (!lv.d_lit_flats) return fail(B2D_ERR_NO_MEMORY, "no 4 GiB aligned device memory for the pre-lit flats");
        CU(launch_prelight_textures(d.colormap, d.texels, d.tex, (int)h[H_NTEX], lv.d_lit.get(), tstride, nullptr));
        CU(launch_prelight(d.colormap, d.flats, lv.d_lit_flats.get(), fstride, fstride, nullptr));
        CU(cudaDeviceSynchronize());
        d.lit_texels = lv.d_lit.get(); d.lit_flats = lv.d_lit_flats.get();     // low 32 address bits of lit_flats are zero
        d.lit_texel_stride = (uint32_t)tstride; d.lit_flat_stride = (uint32_t)fstride;
    }
    d.skyrow = lv.d_skyrow.get();
    d.nverts = (int32_t)h[H_NVERTS]; d.nnodes = (int32_t)h[H_NNODES]; d.nss = (int32_t)h[H_NSSECTORS];
    d.nsegs = (int32_t)h[H_NSEGS]; d.nsectors = (int32_t)h[H_NSECTORS]; d.ntex = (int32_t)h[H_NTEX];
    d.nflats = (int32_t)h[H_NFLATS]; d.sky_tex = (int32_t)h[H_SKY_TEX];
    d.root = h[H_ROOT];
    d.invF = (uint32_t)(4294967296ULL / (uint64_t)view.F);
    if (d.nsegs + d.nsprites > 65535) return fail(B2D_ERR_INVALID_ARG, "level has more than 65535 segs + sprites");
    if (walk_smem_per_warp(d) > 227 * 1024) return fail(B2D_ERR_INVALID_ARG, "level too large for the BSP-walk kernel's shared memory");
    if (scene_is_timed(s->blob.data())) {
        lv.h_blob = s->blob;
        try {
            lv.layout = state_layout(lv.h_blob.data());
        } catch (const std::exception &ex) {
            return fail(B2D_ERR_INVALID_ARG, ex.what());
        }
        const uint8_t *blob = lv.h_blob.data();
        const StateLayout &L = lv.layout;
        const size_t words = L.words;
        // the state rule reads the blob's rest-state sections and the two slot maps
        CU(allocate(lv.d_slot_maps, 4 * (L.sector_slots.size() + L.mid_seg.size()) + 4));
        CU(cudaMemcpy(lv.d_slot_maps.get(), L.sector_slots.data(), 4 * L.sector_slots.size(), cudaMemcpyHostToDevice));
        CU(cudaMemcpy(lv.d_slot_maps.get() + L.sector_slots.size(), L.mid_seg.data(), 4 * L.mid_seg.size(), cudaMemcpyHostToDevice));
        StateSrc &src = lv.src = state_src(blob, L);
        auto on_device = [&](auto p) { return reinterpret_cast<decltype(p)>(db + (reinterpret_cast<const uint8_t *>(p) - blob)); };
        src.tex = on_device(src.tex); src.sectors = on_device(src.sectors); src.segs = on_device(src.segs);
        src.sprites = on_device(src.sprites); src.mids = on_device(src.mids); src.anim = on_device(src.anim);
        src.flat_anim = on_device(src.flat_anim); src.segdyn = on_device(src.segdyn);
        src.sector_slots = lv.d_slot_maps.get();
        src.mid_seg = reinterpret_cast<const int32_t *>(lv.d_slot_maps.get() + L.sector_slots.size());
        StateTables &t = lv.state_tables;              // one table set: [tex | sectors | segs | sprites | mids], 256 B aligned
        t.slot_bytes = (uint32_t)((state_table_bytes(blob) + 255) & ~(size_t)255);
        t.off_sectors = (uint32_t)(h[H_NTEX] * sizeof(TexRec));
        t.off_segs = t.off_sectors + (uint32_t)(h[H_NSECTORS] * sizeof(SectorRec));
        t.off_sprites = t.off_segs + (uint32_t)(h[H_NSEGS] * sizeof(SegRec));
        t.off_mids = t.off_sprites + (uint32_t)(h[H_NSPRITES] * sizeof(SpriteRec));
        for (auto &sl : lv.slot) CU(allocate(sl.tables, t.slot_bytes));
        // tic 0 is a time like any other: a frame name with k > 0 shows its group's frame 0 (tex.rs:260, 302-306).  The
        // pre-lit planes above were built from the blob's own (per-image) records; both slots' table sets start at tic 0.
        lv.state.assign(words, 0);
        compact_state(blob, L, 0, nullptr, nullptr, lv.state.data());
        DeviceBuf<uint32_t> d_state;
        CU(allocate(d_state, 4 * words));
        CU(cudaMemcpy(d_state.get(), lv.state.data(), 4 * words, cudaMemcpyHostToDevice));
        for (auto &sl : lv.slot) {
            CU(launch_state_tables(lv.src, d_state.get(), (uint32_t)words, 1, sl.tables.get(), t, nullptr));
            sl.state = lv.state;
        }
        CU(cudaDeviceSynchronize());
    }
    return B2D_OK;
}
}  // namespace

// b2d_renderer_create_levels / b2d_renderer_create: the latter (level_walk = false) keeps accepting a level whose walk fits
// the plain walk kernel but not the per-frame-level one (whose static shared memory comes on top); its level calls then
// refuse before enqueuing anything.
static int create_renderer(const b2d_scene *const *scenes, size_t n_levels, const b2d_view *view, int device, int max_batch,
                           b2d_renderer **out, bool level_walk) {
    if (!scenes || !view || !out || max_batch < 1) return fail(B2D_ERR_INVALID_ARG, "bad renderer arguments");
    if (n_levels < 1 || n_levels > B2D_MAX_LEVELS) return fail(B2D_ERR_INVALID_ARG, "n_levels out of range (1 .. B2D_MAX_LEVELS)");
    for (size_t k = 0; k < n_levels; k++)
        if (!scenes[k]) return fail(B2D_ERR_INVALID_ARG, "null scene");
    if (view->width < 1 || view->width > 4096 || view->height < 2 || view->height > 2160 || view->F < 2 || view->FY2 < 2 ||
        view->F > kViewFocalMax || view->FY2 > kViewFocalMax || view->width > kViewWidthPerF * view->F)
        return fail(B2D_ERR_INVALID_ARG, "view out of range");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(B2D_ERR_CUDA, std::string("no usable CUDA device (this library has no CPU path): ") +
                                      (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
    if (device < 0 || device >= count) return fail(B2D_ERR_INVALID_ARG, "device index out of range");
    CU(cudaSetDevice(device));
    std::unique_ptr<b2d_renderer> r(new (std::nothrow) b2d_renderer());
    if (!r) return fail(B2D_ERR_NO_MEMORY, "out of host memory");
    r->device = device;
    r->view = View{view->width, view->height, view->F, view->FY2};
    r->max_batch = max_batch;
    int rc = guarded([&] { r->lv.resize(n_levels); return B2D_OK; });
    if (rc != B2D_OK) return rc;
    for (size_t k = 0; k < n_levels; k++) {
        rc = guarded([&] { return create_level(r.get(), r->lv[k], scenes[k]); });
        if (rc != B2D_OK) return rc;
    }
    // what the levels share: the worklist stride, the walk's shared memory, the masked-entry arena, yslope and the status word
    r->stride = 1;
    int32_t masked_cap = 0;
    for (const LevelRes &lv : r->lv) {
        r->stride = std::max(r->stride, lv.ds.nsegs + lv.ds.nsprites);            // worklist entries per frame
        r->walk_smem = std::max(r->walk_smem, walk_smem_per_warp(lv.ds));
        masked_cap = std::max(masked_cap, lv.ds.masked_cap);
    }
    if (level_walk && r->walk_smem + walk_levels_static_smem() > kWalkSmemMax)
        return fail(B2D_ERR_INVALID_ARG, "level too large for the per-frame-level BSP-walk kernel's shared memory");
    std::vector<uint32_t> ys((size_t)view->height);
    for (int y = 0; y < view->height; y++) ys[(size_t)y] = yslope_entry(y, r->view);
    CU(allocate(r->d_yslope, ys.size() * 4));
    CU(cudaMemcpy(r->d_yslope.get(), ys.data(), ys.size() * 4, cudaMemcpyHostToDevice));
    CU(allocate(r->d_status, sizeof(int32_t)));
    CU(cudaMemset(r->d_status.get(), 0, sizeof(int32_t)));
    uint32_t masked_chunks = 0;
    if (masked_cap > 0) {
        // arena of deferred masked entries: chunks of kMaskedChunk entries handed out on demand.  Sized for the worst case
        // -- every (frame, 32-column strip) of a full batch at its cap (the largest of the levels) -- whenever that takes
        // at most kMaskedArenaBudget, so that no valid batch can run out of it: a crowded subsector puts dozens of sprites
        // into every strip of a 1080p frame.  Past the budget (1080p batches of more than ~1000 frames, 4K of more than
        // ~500, with a cap of 128) two chunks per strip on average, at least 4096: frames usually defer a handful of
        // entries per strip, and a batch that needs more reports kStatusMaskedFull instead of drawing wrong pixels.
        constexpr size_t kMaskedArenaBudget = (size_t)1 << 30;
        const size_t strips = (size_t)(view->width + 31) / 32;
        const size_t per_strip = ((size_t)masked_cap + kMaskedChunk - 1) / kMaskedChunk;
        const size_t worst = strips * (size_t)max_batch * per_strip;
        size_t chunks = worst;
        if (sizeof(uint32_t) * 33 * kMaskedChunk * worst > kMaskedArenaBudget) {
            chunks = strips * (size_t)max_batch * (per_strip < 2 ? per_strip : 2);
            if (chunks < 4096) chunks = 4096;
            if (chunks > worst) chunks = worst;
        }
        if (const char *env = getenv("B2D_MASKED_CHUNKS")) chunks = (size_t)strtoull(env, nullptr, 0);   // tests: force exhaustion
        if (chunks < 1) chunks = 1;
        masked_chunks = (uint32_t)chunks;
        CU(allocate(r->d_masked, sizeof(uint32_t) * 33 * kMaskedChunk * chunks));
        CU(allocate(r->d_masked_counter, sizeof(uint32_t)));
        CU(cudaMemset(r->d_masked_counter.get(), 0, sizeof(uint32_t)));
        CU(event_create(r->masked_done));
        CU(cudaEventRecord(r->masked_done.get(), nullptr));
    }
    // per-frame levels: [DeviceScene per level | compact state per timed level | frame levels] in each slot's level buffer
    size_t off = (r->lv.size() * sizeof(DeviceScene) + 15) & ~(size_t)15;
    for (LevelRes &lv : r->lv) {
        DeviceScene &d = lv.ds;
        d.yslope = r->d_yslope.get();
        d.status_flag = r->d_status.get();
        if (d.masked_cap > 0) {
            d.masked_list = r->d_masked.get();
            d.masked_counter = r->d_masked_counter.get();
            d.masked_chunks = masked_chunks;
        }
        lv.stage_off = off;
        off += 4 * lv.layout.words;
    }
    r->levels_frames_off = (off + 15) & ~(size_t)15;
    if (!r->lv[0].h_blob.empty()) {
        // level 0's per-frame states and the restates of its plain batches: compact states + set indices and their staging
        const size_t words = r->lv[0].layout.words, mb = (size_t)max_batch;
        for (WorkSlot &sl : r->slot) {
            CU(allocate(sl.states, 4 * mb * (words + 1)));
            CU(allocate(sl.h_states, 4 * mb * (words + 1)));
            CU(event_create(sl.states_copied));
        }
    }
    CU(allocate(r->d_poses, sizeof(Pose) * (size_t)max_batch));
    rc = ensure_slot(r.get(), r->slot[0]);
    if (rc == B2D_OK) *out = r.release();
    return rc;
}

int b2d_renderer_create_levels(const b2d_scene *const *scenes, size_t n_levels, const b2d_view *view, int device, int max_batch,
                               b2d_renderer **out) {
    return create_renderer(scenes, n_levels, view, device, max_batch, out, true);
}

int b2d_renderer_create(const b2d_scene *s, const b2d_view *view, int device, int max_batch, b2d_renderer **out) {
    if (!s) return fail(B2D_ERR_INVALID_ARG, "bad renderer arguments");
    return create_renderer(&s, 1, view, device, max_batch, out, false);
}

void b2d_renderer_destroy(b2d_renderer *r) { delete r; }

// The renderer's own state is host data: the setters enqueue nothing (the stream is kept for ABI compatibility), and the
// next batch of each worklist slot that uses a level expands the level's state into the level's table set of the slot.
// The time is every level's.
int b2d_renderer_set_time(b2d_renderer *r, uint32_t tics) {
    if (!r) return fail(B2D_ERR_INVALID_ARG, "null renderer");
    return guarded([&] {
        std::vector<std::vector<uint32_t>> st(r->lv.size());
        for (size_t k = 0; k < r->lv.size(); k++) {
            if (r->lv[k].h_blob.empty()) continue;
            st[k].resize(r->lv[k].layout.words);
            state_at(r->lv[k], tics, st[k].data());
        }
        for (size_t k = 0; k < r->lv.size(); k++)
            if (!r->lv[k].h_blob.empty()) r->lv[k].state.swap(st[k]);
        r->tics = tics;
        return B2D_OK;
    });
}

int b2d_renderer_set_time_async(b2d_renderer *r, uint32_t tics, void *) { return b2d_renderer_set_time(r, tics); }

int b2d_renderer_set_level_sector_moves(b2d_renderer *r, int level, const b2d_sector_move *moves, size_t n) {
    if (!r || (n && !moves)) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (level < 0 || (size_t)level >= r->lv.size()) return fail(B2D_ERR_INVALID_ARG, "level index out of range");
    LevelRes &lv = r->lv[(size_t)level];
    if (lv.h_blob.empty()) {
        if (n == 0) return B2D_OK;
        return fail(B2D_ERR_INVALID_ARG, "the scene declares no dynamic sectors");
    }
    static_assert(sizeof(b2d_sector_move) == sizeof(SectorMove), "ABI record");
    return guarded([&] {
        std::vector<int32_t> fo, co;
        if (const char *why = expand_moves(lv.h_blob.data(), reinterpret_cast<const SectorMove *>(moves), n, fo, co))
            return fail(B2D_ERR_INVALID_ARG, why);
        bool moved = false;
        for (size_t i = 0; i < fo.size() && !moved; i++) moved = fo[i] != 0 || co[i] != 0;      // all zero: at rest
        compact_state(lv.h_blob.data(), lv.layout, r->tics, moved ? fo.data() : nullptr, moved ? co.data() : nullptr,
                      lv.state.data());
        return B2D_OK;
    });
}

int b2d_renderer_set_sector_moves(b2d_renderer *r, const b2d_sector_move *moves, size_t n) {
    return b2d_renderer_set_level_sector_moves(r, 0, moves, n);
}

int b2d_renderer_set_sector_moves_async(b2d_renderer *r, const b2d_sector_move *moves, size_t n, void *) {
    return b2d_renderer_set_sector_moves(r, moves, n);
}

int b2d_renderer_status(b2d_renderer *r, int32_t *bits_out) {
    if (!r || !bits_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    CU(cudaSetDevice(r->device));
    CU(cudaDeviceSynchronize());
    int32_t status = 0;
    CU(cudaMemcpy(&status, r->d_status.get(), sizeof status, cudaMemcpyDeviceToHost));
    if (status) CU(cudaMemset(r->d_status.get(), 0, sizeof(int32_t)));
    *bits_out = status;
    return B2D_OK;
}

int b2d_render_device(b2d_renderer *r, const b2d_pose *d_poses, size_t n, uint8_t *d_index_fb,
                      uint32_t *d_rgba_fb, void *cuda_stream) {
    if (!r || !d_poses || !d_index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (n == 0) return B2D_OK;
    if (n > (size_t)r->max_batch) return fail(B2D_ERR_INVALID_ARG, "n exceeds max_batch");
    CU(cudaSetDevice(r->device));
    return enqueue_frames(r, reinterpret_cast<const Pose *>(d_poses), (int)n, d_index_fb, d_rgba_fb,
                          static_cast<cudaStream_t>(cuda_stream));
}

// frames_states (nullable, level 0's layout.words words per frame): walk + raster of n device poses in batches of max_batch
static int enqueue_batches(b2d_renderer *r, const b2d_pose *d_poses, size_t n, const uint32_t *frame_states, uint8_t *d_index_fb,
                           uint32_t *d_rgba_fb, cudaStream_t st) {
    const size_t npix = (size_t)r->view.W * r->view.H;
    for (size_t i = 0; i < n; i += (size_t)r->max_batch) {
        const size_t cnt = n - i < (size_t)r->max_batch ? n - i : (size_t)r->max_batch;
        int rc = enqueue_frames(r, reinterpret_cast<const Pose *>(d_poses) + i, (int)cnt, d_index_fb + i * npix,
                                d_rgba_fb ? d_rgba_fb + i * npix : nullptr, st, frame_states ? frame_states + i * r->lv[0].layout.words : nullptr);
        if (rc != B2D_OK) return rc;
    }
    return B2D_OK;
}

int b2d_render_device_timed(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *tics, size_t n, uint8_t *d_index_fb,
                            uint32_t *d_rgba_fb, void *cuda_stream) {
    if (!r || !d_poses || !d_index_fb || !tics) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (n == 0) return B2D_OK;
    CU(cudaSetDevice(r->device));
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    std::vector<uint32_t> fs;
    int rc = guarded([&] { timed_states(r, tics, n, fs); return B2D_OK; });
    if (rc != B2D_OK) return rc;
    rc = enqueue_batches(r, d_poses, n, fs.empty() ? nullptr : fs.data(), d_index_fb, d_rgba_fb, st);
    if (rc != B2D_OK) return rc;
    return b2d_renderer_set_time(r, tics[n - 1]);                          // the renderer is left at the last pose's time
}

int b2d_render_device_states(b2d_renderer *r, const b2d_pose *d_poses, const b2d_frame_state *states, size_t n,
                             const b2d_sector_move *moves, size_t n_moves, uint8_t *d_index_fb, uint32_t *d_rgba_fb,
                             void *cuda_stream) {
    if (!r || !d_poses || !d_index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    std::vector<uint32_t> fs;
    int rc = guarded([&] { return build_states(r, states, n, moves, n_moves, fs); });
    if (rc != B2D_OK || n == 0) return rc;
    CU(cudaSetDevice(r->device));
    return enqueue_batches(r, d_poses, n, fs.empty() ? nullptr : fs.data(), d_index_fb, d_rgba_fb, static_cast<cudaStream_t>(cuda_stream));
}

int b2d_walk_device_states(b2d_renderer *r, const b2d_pose *d_poses, const b2d_frame_state *states, size_t n,
                           const b2d_sector_move *moves, size_t n_moves, void *cuda_stream, int64_t *ticket_out) {
    if (!r || !d_poses || !ticket_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (n == 0 || n > (size_t)r->max_batch) return fail(B2D_ERR_INVALID_ARG, "n must be in 1..max_batch");
    std::vector<uint32_t> fs;
    int rc = guarded([&] { return build_states(r, states, n, moves, n_moves, fs); });
    if (rc != B2D_OK) return rc;
    CU(cudaSetDevice(r->device));
    return walk_into_slot(r, reinterpret_cast<const Pose *>(d_poses), (int)n, static_cast<cudaStream_t>(cuda_stream), ticket_out, true,
                          fs.empty() ? nullptr : fs.data());
}

int b2d_walk_device(b2d_renderer *r, const b2d_pose *d_poses, size_t n, void *cuda_stream, int64_t *ticket_out) {
    if (!r || !d_poses || !ticket_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (n == 0 || n > (size_t)r->max_batch) return fail(B2D_ERR_INVALID_ARG, "n must be in 1..max_batch");
    CU(cudaSetDevice(r->device));
    return walk_into_slot(r, reinterpret_cast<const Pose *>(d_poses), (int)n, static_cast<cudaStream_t>(cuda_stream), ticket_out, true);
}

int b2d_raster_device(b2d_renderer *r, int64_t ticket, uint8_t *d_index_fb, uint32_t *d_rgba_fb, void *cuda_stream) {
    if (!r || !d_index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    CU(cudaSetDevice(r->device));
    return raster_from_slot(r, ticket, d_index_fb, d_rgba_fb, static_cast<cudaStream_t>(cuda_stream));
}

// Per-frame levels: n HOST levels, each below the renderer's number of levels, and a renderer whose levels fit the
// per-frame-level walk (a b2d_renderer_create renderer may not; checked before anything is enqueued)
static int check_levels(const b2d_renderer *r, const uint32_t *levels, size_t n) {
    if (!levels) return fail(B2D_ERR_INVALID_ARG, "null level array");
    if (r->walk_smem + walk_levels_static_smem() > kWalkSmemMax)
        return fail(B2D_ERR_INVALID_ARG, "level too large for the per-frame-level BSP-walk kernel's shared memory");
    for (size_t i = 0; i < n; i++)
        if (levels[i] >= r->lv.size()) return fail(B2D_ERR_INVALID_ARG, "frame level out of range (>= the renderer's number of levels)");
    return B2D_OK;
}

// walk -> raster of a batch with per-frame levels on `stream`
static int enqueue_level_frames(b2d_renderer *r, const Pose *d_poses, const uint32_t *levels, int n, uint8_t *d_index,
                                uint32_t *d_rgba, cudaStream_t stream) {
    int64_t ticket = -1;
    int rc = walk_levels_into_slot(r, d_poses, levels, n, stream, &ticket, false);
    if (rc != B2D_OK) return rc;
    return raster_from_slot(r, ticket, d_index, d_rgba, stream);
}

int b2d_render_device_levels(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, size_t n, uint8_t *d_index_fb,
                             uint32_t *d_rgba_fb, void *cuda_stream) {
    if (!r || !d_poses || !d_index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    int rc = check_levels(r, levels, n);
    if (rc != B2D_OK || n == 0) return rc;
    CU(cudaSetDevice(r->device));
    const size_t npix = (size_t)r->view.W * r->view.H;
    for (size_t i = 0; i < n; i += (size_t)r->max_batch) {
        const size_t cnt = n - i < (size_t)r->max_batch ? n - i : (size_t)r->max_batch;
        rc = enqueue_level_frames(r, reinterpret_cast<const Pose *>(d_poses) + i, levels + i, (int)cnt, d_index_fb + i * npix,
                                  d_rgba_fb ? d_rgba_fb + i * npix : nullptr, static_cast<cudaStream_t>(cuda_stream));
        if (rc != B2D_OK) return rc;
    }
    return B2D_OK;
}

int b2d_walk_device_levels(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, size_t n, void *cuda_stream,
                           int64_t *ticket_out) {
    if (!r || !d_poses || !ticket_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (n == 0 || n > (size_t)r->max_batch) return fail(B2D_ERR_INVALID_ARG, "n must be in 1..max_batch");
    int rc = check_levels(r, levels, n);
    if (rc != B2D_OK) return rc;
    CU(cudaSetDevice(r->device));
    return walk_levels_into_slot(r, reinterpret_cast<const Pose *>(d_poses), levels, (int)n, static_cast<cudaStream_t>(cuda_stream),
                                 ticket_out, true);
}

// Host poses in, host frames out; frame_states as in enqueue_frames (for all n frames), or (exclusive with it) frame_levels:
// the level of each of the n frames
static int render_host(b2d_renderer *r, const b2d_pose *poses, size_t n, const uint32_t *frame_states, uint8_t *index_fb,
                       uint32_t *rgba_fb, const uint32_t *frame_levels = nullptr) {
    if (n == 0) return B2D_OK;
    CU(cudaSetDevice(r->device));
    const size_t npix = (size_t)r->view.W * r->view.H;
    if (!r->host) {       // created whole, or not at all
        std::unique_ptr<HostStaging> staging(new (std::nothrow) HostStaging());
        if (!staging) return fail(B2D_ERR_NO_MEMORY, "out of host memory");
        CU(stream_create(staging->render_stream));
        for (int i = 0; i < 2; i++) {
            CU(stream_create(staging->copy_stream[i]));
            CU(event_create(staging->rendered[i]));
            CU(event_create(staging->copied[i]));
            CU(allocate(staging->index[i], npix * (size_t)r->max_batch));
        }
        CU(allocate(staging->poses, sizeof(Pose) * (size_t)r->max_batch * 2));
        r->host = std::move(staging);
    }
    HostStaging &hs = *r->host;
    if (rgba_fb && !hs.rgba[0]) {
        std::array<DeviceBuf<uint32_t>, 2> rgba;
        for (auto &buf : rgba) CU(allocate(buf, npix * 4 * (size_t)r->max_batch));
        hs.rgba = std::move(rgba);
    }
    // Double-buffered pipeline: batch b renders into buffer b&1 on render_stream while the copy
    // stream drains buffer (b-1)&1 to the caller's host memory.
    size_t done = 0;
    int b = 0;
    while (done < n) {
        const int cnt = (int)(n - done < (size_t)r->max_batch ? n - done : (size_t)r->max_batch);
        const int buf = b & 1;
        if (b >= 2) CU(cudaEventSynchronize(hs.copied[buf].get()));       // buffer + pose slot free again
        Pose *hp = hs.poses.get() + (size_t)buf * r->max_batch;
        std::memcpy(hp, poses + done, sizeof(Pose) * (size_t)cnt);
        cudaStream_t rs = hs.render_stream.get(), cs = hs.copy_stream[buf].get();
        CU(cudaMemcpyAsync(r->d_poses.get(), hp, sizeof(Pose) * (size_t)cnt, cudaMemcpyHostToDevice, rs));
        int rc = frame_levels
                     ? enqueue_level_frames(r, r->d_poses.get(), frame_levels + done, cnt, hs.index[buf].get(),
                                            rgba_fb ? hs.rgba[buf].get() : nullptr, rs)
                     : enqueue_frames(r, r->d_poses.get(), cnt, hs.index[buf].get(), rgba_fb ? hs.rgba[buf].get() : nullptr, rs,
                                      frame_states ? frame_states + done * r->lv[0].layout.words : nullptr);
        if (rc != B2D_OK) return rc;
        CU(cudaEventRecord(hs.rendered[buf].get(), rs));
        CU(cudaStreamWaitEvent(cs, hs.rendered[buf].get(), 0));
        CU(cudaMemcpyAsync(index_fb + done * npix, hs.index[buf].get(), npix * (size_t)cnt, cudaMemcpyDeviceToHost, cs));
        if (rgba_fb)
            CU(cudaMemcpyAsync(rgba_fb + done * npix, hs.rgba[buf].get(), npix * 4 * (size_t)cnt, cudaMemcpyDeviceToHost, cs));
        CU(cudaEventRecord(hs.copied[buf].get(), cs));
        done += (size_t)cnt;
        b++;
    }
    for (auto &st : hs.copy_stream) CU(cudaStreamSynchronize(st.get()));
    CU(cudaStreamSynchronize(hs.render_stream.get()));
    int32_t status = 0;
    CU(cudaMemcpy(&status, r->d_status.get(), sizeof status, cudaMemcpyDeviceToHost));
    if (status) {
        CU(cudaMemset(r->d_status.get(), 0, sizeof(int32_t)));
        return fail(B2D_ERR_INVALID_ARG, status & kStatusStackOverflow ? "BSP traversal stack overflow (tree deeper than 128 pending nodes): frames incomplete"
                                            : (status & kStatusNoTermination ? "BSP traversal did not terminate (cyclic node graph): frames incomplete"
                                              : (status & kStatusMaskedFull ? "more masked middle textures / sprites deferred in one 32-column strip than the renderer holds (min(level total, 128)): frames incomplete"
                                                            : "worklist overflow: frames incomplete")));
    }
    return B2D_OK;
}

int b2d_render(b2d_renderer *r, const b2d_pose *poses, size_t n, uint8_t *index_fb, uint32_t *rgba_fb) {
    if (!r || !poses || !index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    return render_host(r, poses, n, nullptr, index_fb, rgba_fb);
}

int b2d_render_timed(b2d_renderer *r, const b2d_pose *poses, const uint32_t *tics, size_t n, uint8_t *index_fb, uint32_t *rgba_fb) {
    if (!tics) return b2d_render(r, poses, n, index_fb, rgba_fb);
    if (!r || !poses || !index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (n == 0) return B2D_OK;
    std::vector<uint32_t> fs;
    int rc = guarded([&] { timed_states(r, tics, n, fs); return B2D_OK; });
    if (rc != B2D_OK) return rc;
    rc = render_host(r, poses, n, fs.empty() ? nullptr : fs.data(), index_fb, rgba_fb);
    const int trc = b2d_renderer_set_time(r, tics[n - 1]);                // the renderer is left at the last pose's time
    return rc != B2D_OK ? rc : trc;
}

int b2d_render_states(b2d_renderer *r, const b2d_pose *poses, const b2d_frame_state *states, size_t n,
                      const b2d_sector_move *moves, size_t n_moves, uint8_t *index_fb, uint32_t *rgba_fb) {
    if (!r || !poses || !index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    std::vector<uint32_t> fs;
    int rc = guarded([&] { return build_states(r, states, n, moves, n_moves, fs); });
    if (rc != B2D_OK) return rc;
    return render_host(r, poses, n, fs.empty() ? nullptr : fs.data(), index_fb, rgba_fb);
}

int b2d_render_levels(b2d_renderer *r, const b2d_pose *poses, const uint32_t *levels, size_t n, uint8_t *index_fb,
                      uint32_t *rgba_fb) {
    if (!r || !poses || !index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    int rc = check_levels(r, levels, n);
    if (rc != B2D_OK) return rc;
    return render_host(r, poses, n, nullptr, index_fb, rgba_fb, levels);
}

int b2d_palette_lut_device(b2d_renderer *r, const uint8_t *d_index, uint32_t *d_rgba, size_t n_pixels, void *cuda_stream) {
    if (!r || !d_index || !d_rgba) return fail(B2D_ERR_INVALID_ARG, "null argument");
    CU(cudaSetDevice(r->device));
    CU(launch_palette(r->lv[0].ds.palette, d_index, d_rgba, n_pixels, static_cast<cudaStream_t>(cuda_stream)));
    r->launches += 1;
    return B2D_OK;
}

int b2d_device_alloc(int device, size_t bytes, void **d_out) {
    if (!d_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    CU(cudaSetDevice(device));
    CU(cudaMalloc(d_out, bytes ? bytes : 1));
    CU(cudaMemset(*d_out, 0, bytes));
    return B2D_OK;
}

int b2d_device_free(int device, void *d_ptr) {
    CU(cudaSetDevice(device));
    CU(cudaFree(d_ptr));
    return B2D_OK;
}

int b2d_device_download(int device, void *host_dst, const void *d_src, size_t bytes) {
    if (!host_dst || !d_src) return fail(B2D_ERR_INVALID_ARG, "null argument");
    CU(cudaSetDevice(device));
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(host_dst, d_src, bytes, cudaMemcpyDeviceToHost));
    return B2D_OK;
}

int b2d_debug_worklist(b2d_renderer *r, size_t n, int32_t *counts_out, int32_t *seg_ids_out, size_t stride) {
    if (!r || !counts_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (n > (size_t)r->max_batch) return fail(B2D_ERR_INVALID_ARG, "n exceeds max_batch");
    const int slot = r->last_slot;
    if (!r->slot[slot].frames || n > (size_t)r->slot[slot].n) return fail(B2D_ERR_INVALID_ARG, "n exceeds the frames of the last walked batch");
    CU(cudaSetDevice(r->device));
    CU(cudaDeviceSynchronize());
    std::vector<FrameConst> frames(n);
    CU(cudaMemcpy(frames.data(), r->slot[slot].frames.get(), sizeof(FrameConst) * n, cudaMemcpyDeviceToHost));
    std::vector<SegFrame> work;
    for (size_t i = 0; i < n; i++) {
        counts_out[i] = frames[i].status ? -frames[i].status : frames[i].count;
        if (!seg_ids_out) continue;
        size_t c = frames[i].count > 0 ? (size_t)frames[i].count : 0;
        if (c > (size_t)r->stride) c = (size_t)r->stride;
        work.resize(c);
        if (c) CU(cudaMemcpy(work.data(), r->slot[slot].work.get() + i * (size_t)r->stride, sizeof(SegFrame) * c, cudaMemcpyDeviceToHost));
        for (size_t k = 0; k < c && k < stride; k++) seg_ids_out[i * stride + k] = work[k].seg;
    }
    return B2D_OK;
}

int b2d_debug_state_slots(b2d_renderer *r, size_t n, uint32_t *slots_out) {
    if (!r || !slots_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    const int slot = r->last_slot;
    if (!r->slot[slot].per_frame || n > (size_t)r->slot[slot].n)
        return fail(B2D_ERR_INVALID_ARG, "the last walked batch has no per-frame states or fewer than n frames");
    CU(cudaSetDevice(r->device));
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(slots_out, slot_tables(r, slot).frame_slot, 4 * n, cudaMemcpyDeviceToHost));
    return B2D_OK;
}

int b2d_debug_state_tables(b2d_renderer *r, size_t set, void *out, size_t capacity, size_t *size_out) {
    if (!r) return fail(B2D_ERR_INVALID_ARG, "null renderer");
    const LevelRes &lv = r->lv[0];
    if (lv.h_blob.empty()) return fail(B2D_ERR_INVALID_ARG, "the scene has no time-dependent content or dynamic sectors");
    const WorkSlot &s = r->slot[r->last_slot];
    if (s.ticket < 0) return fail(B2D_ERR_INVALID_ARG, "no batch has been walked");
    if (set >= (s.per_frame ? (size_t)s.sets : 1)) return fail(B2D_ERR_INVALID_ARG, "table set out of range for the last walked batch");
    const size_t need = state_table_bytes(lv.h_blob.data());
    if (size_out) *size_out = need;
    if (!out) return B2D_OK;
    if (capacity < need) return fail(B2D_ERR_INVALID_ARG, "buffer too small for the tables");
    CU(cudaSetDevice(r->device));
    CU(cudaDeviceSynchronize());
    const uint8_t *src = s.per_frame ? s.arena.get() + set * (size_t)lv.state_tables.slot_bytes : lv.slot[r->last_slot].tables.get();
    CU(cudaMemcpy(out, src, need, cudaMemcpyDeviceToHost));
    return B2D_OK;
}

int b2d_profile_enable(b2d_renderer *r, int enable) {
    if (!r) return fail(B2D_ERR_INVALID_ARG, "null renderer");
    r->profiling = enable != 0;
    return B2D_OK;
}

int b2d_profile_read(b2d_renderer *r, double *walk_ms, double *raster_ms, int64_t *batches) {
    if (!r) return fail(B2D_ERR_INVALID_ARG, "null renderer");
    CU(cudaSetDevice(r->device));
    CU(cudaDeviceSynchronize());
    // events arrive as pairs (before, after one kernel launch); prof_kinds says which kernel: 0 = walk, 1 = raster
    double w = 0.0, ra = 0.0;
    int64_t nb = 0;
    for (size_t i = 0; i + 1 < r->prof_events.size(); i += 2) {
        float a = 0.f;
        CU(cudaEventElapsedTime(&a, r->prof_events[i].get(), r->prof_events[i + 1].get()));
        if (r->prof_kinds[i / 2] == 0) w += a; else { ra += a; nb++; }
    }
    if (walk_ms) *walk_ms = w;
    if (raster_ms) *raster_ms = ra;
    if (batches) *batches = nb;
    r->prof_kinds.clear();
    r->prof_events.clear();
    return B2D_OK;
}

int64_t b2d_launch_count(const b2d_renderer *r) { return r ? r->launches : 0; }

}  // extern "C"
