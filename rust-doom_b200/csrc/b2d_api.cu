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

// device memory of `bytes` bytes at an address that is a multiple of 4 GiB
bool alloc_aligned_4g(b2d_renderer *r, size_t bytes) {
    const Vmm &v = vmm();
    if (v.ok && !getenv("B2D_NO_VMM")) {
        CUmemAllocationProp prop;
        std::memset(&prop, 0, sizeof prop);
        prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
        prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
        prop.location.id = r->device;
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
                        if (v.SetAccess(ptr, size, &acc, 1) == CUDA_SUCCESS) {
                            r->d_lit_flats = reinterpret_cast<uint8_t *>(ptr);
                            r->lit_flats_bytes = size;
                            r->lit_flats_handle = (unsigned long long)h;
                            return true;
                        }
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
    if (cudaMalloc(&raw, bytes + k4G) != cudaSuccess) { cudaGetLastError(); return false; }
    r->d_lit_flats_raw = static_cast<uint8_t *>(raw);
    r->d_lit_flats = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(raw) + k4G - 1) & ~(uintptr_t)(k4G - 1));
    r->lit_flats_bytes = 0;
    return true;
}

void free_aligned_4g(b2d_renderer *r) {
    if (r->lit_flats_bytes) {
        const Vmm &v = vmm();
        v.Unmap(reinterpret_cast<CUdeviceptr>(r->d_lit_flats), r->lit_flats_bytes);
        v.Release((CUmemGenericAllocationHandle)r->lit_flats_handle);
        v.AddressFree(reinterpret_cast<CUdeviceptr>(r->d_lit_flats), r->lit_flats_bytes);
    } else if (r->d_lit_flats_raw) {
        cudaFree(r->d_lit_flats_raw);
    }
    r->d_lit_flats = nullptr; r->d_lit_flats_raw = nullptr; r->lit_flats_bytes = 0;
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

void free_renderer(b2d_renderer *r) {
    if (!r) return;
    cudaSetDevice(r->device);
    for (int i = 0; i < 2; i++) {
        if (r->d_index[i]) cudaFree(r->d_index[i]);
        if (r->d_rgba[i]) cudaFree(r->d_rgba[i]);
        if (r->rendered[i]) cudaEventDestroy(r->rendered[i]);
        if (r->copied[i]) cudaEventDestroy(r->copied[i]);
    }
    for (cudaEvent_t e : r->prof_events) cudaEventDestroy(e);
    if (r->h_poses) cudaFreeHost(r->h_poses);
    if (r->render_stream) cudaStreamDestroy(r->render_stream);
    for (int i = 0; i < 2; i++) if (r->copy_stream[i]) cudaStreamDestroy(r->copy_stream[i]);
    for (int i = 0; i < 2; i++) {
        if (r->d_work[i]) cudaFree(r->d_work[i]);
        if (r->d_frames[i]) cudaFree(r->d_frames[i]);
        if (r->walk_done[i]) cudaEventDestroy(r->walk_done[i]);
        if (r->raster_done[i]) cudaEventDestroy(r->raster_done[i]);
    }
    if (r->d_poses) cudaFree(r->d_poses);
    if (r->d_yslope) cudaFree(r->d_yslope);
    if (r->d_skyrow) cudaFree(r->d_skyrow);
    if (r->d_status) cudaFree(r->d_status);
    if (r->d_masked) cudaFree(r->d_masked);
    if (r->d_masked_counter) cudaFree(r->d_masked_counter);
    if (r->masked_done) cudaEventDestroy(r->masked_done);
    for (int i = 0; i < 2; i++) {
        if (r->d_arena[i]) cudaFree(r->d_arena[i]);
        if (r->d_states[i]) cudaFree(r->d_states[i]);
        if (r->h_states[i]) cudaFreeHost(r->h_states[i]);
        if (r->states_copied[i]) cudaEventDestroy(r->states_copied[i]);
    }
    if (r->d_slot_tables) cudaFree(r->d_slot_tables);
    if (r->d_slot_maps) cudaFree(r->d_slot_maps);
    if (r->d_lit) cudaFree(r->d_lit);
    if (r->d_walk_static) cudaFree(r->d_walk_static);
    free_aligned_4g(r);
    if (r->d_blob) cudaFree(r->d_blob);
    delete r;
}

// Per-frame states: the two worklist slots' arenas of max_batch table sets, allocated by the first such call.
int ensure_states(b2d_renderer *r) {
    for (int i = 0; i < 2; i++)
        if (!r->d_arena[i]) CU(cudaMalloc(&r->d_arena[i], (size_t)r->max_batch * r->state_tables.slot_bytes));
    return B2D_OK;
}

// the arena view of worklist slot `slot` (after ensure_states)
StateTables slot_tables(const b2d_renderer *r, int slot) {
    StateTables t = r->state_tables;
    t.base = r->d_arena[slot];
    t.frame_slot = r->d_states[slot] + (size_t)r->max_batch * r->layout.words;
    return t;
}

// the scene as the plain kernels of worklist slot `slot` read it: on a timed scene, the five state-dependent tables are
// the slot's own table set
DeviceScene slot_scene(const b2d_renderer *r, int slot) {
    DeviceScene d = r->ds;
    if (!r->d_slot_tables) return d;
    const StateTables &t = r->state_tables;
    const uint8_t *set = r->d_slot_tables + (size_t)slot * t.slot_bytes;
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
    if (!r->slot_rastered[slot]) return fail(B2D_ERR_INVALID_ARG, "both worklist slots hold batches that were walked but not rastered yet");
    if (frame_states) {
        int rc = ensure_states(r);
        if (rc != B2D_OK) return rc;
    }
    const bool restate = !frame_states && r->d_slot_tables && r->slot_state[slot] != r->state;
    const size_t words = r->layout.words;
    int nstates = 0;
    if (frame_states || restate) {
        CU(cudaEventSynchronize(r->states_copied[slot]));      // the copy issued two batches ago has read the staging
        uint32_t *hs = r->h_states[slot], *hslot = hs + (size_t)r->max_batch * words;
        if (restate) {
            std::memcpy(hs, r->state.data(), 4 * words);
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
    if (!r->d_frames[slot]) {
        CU(cudaMalloc(&r->d_frames[slot], sizeof(FrameConst) * (size_t)r->max_batch));
        CU(cudaMalloc(&r->d_work[slot], sizeof(SegFrame) * (size_t)r->max_batch * (size_t)r->stride));
    }
    if (!r->walk_done[slot]) {
        CU(cudaEventCreateWithFlags(&r->walk_done[slot], cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&r->raster_done[slot], cudaEventDisableTiming));
    } else {
        CU(cudaStreamWaitEvent(stream, r->raster_done[slot], 0));      // the raster that last read this slot
    }
    const StateTables stt = frame_states ? slot_tables(r, slot) : StateTables{};
    if (nstates) {
        uint32_t *hs = r->h_states[slot];
        CU(cudaMemcpyAsync(r->d_states[slot], hs, 4 * words * (size_t)nstates, cudaMemcpyHostToDevice, stream));
        if (frame_states)
            CU(cudaMemcpyAsync(const_cast<uint32_t *>(stt.frame_slot), hs + (size_t)r->max_batch * words, 4 * (size_t)n,
                               cudaMemcpyHostToDevice, stream));
        CU(cudaEventRecord(r->states_copied[slot], stream));
        uint8_t *sets = frame_states ? r->d_arena[slot] : r->d_slot_tables + (size_t)slot * r->state_tables.slot_bytes;
        CU(launch_state_tables(r->src, r->d_states[slot], (uint32_t)words, nstates, sets, r->state_tables, stream));
        r->launches += 1;
        if (restate) r->slot_state[slot] = r->state;
    }
    cudaEvent_t ev[2] = {nullptr, nullptr};
    if (r->profiling) {
        for (auto &e : ev) CU(cudaEventCreate(&e));
        CU(cudaEventRecord(ev[0], stream));
    }
    CU(launch_walk(slot_scene(r, slot), r->view, d_poses, n, r->d_frames[slot], r->d_work[slot], r->stride, stream, background,
                   frame_states ? &stt : nullptr));
    if (r->profiling) {
        CU(cudaEventRecord(ev[1], stream));
        for (auto e : ev) r->prof_events.push_back(e);
        r->prof_kinds.push_back(0);
    }
    CU(cudaEventRecord(r->walk_done[slot], stream));
    r->slot_n[slot] = n;
    r->slot_states[slot] = frame_states != nullptr;
    r->slot_ticket[slot] = r->next_ticket;
    r->slot_rastered[slot] = false;
    r->last_slot = slot;
    r->launches += 1;
    *ticket_out = r->next_ticket++;
    return B2D_OK;
}

int raster_from_slot(b2d_renderer *r, int64_t ticket, uint8_t *d_index, uint32_t *d_rgba, cudaStream_t stream) {
    const int slot = (int)(ticket & 1);
    if (ticket < 0 || r->slot_ticket[slot] != ticket || r->slot_rastered[slot])
        return fail(B2D_ERR_INVALID_ARG, "unknown or already rastered walk ticket");
    CU(cudaStreamWaitEvent(stream, r->walk_done[slot], 0));
    if (r->ds.masked_list) {
        // one arena of deferred masked entries per renderer: rasters that use it run one after the other (each fills the
        // machine on its own, so nothing is lost), whatever streams they were enqueued on
        CU(cudaStreamWaitEvent(stream, r->masked_done, 0));
        CU(cudaMemsetAsync(r->d_masked_counter, 0, sizeof(uint32_t), stream));
    }
    cudaEvent_t ev[2] = {nullptr, nullptr};
    if (r->profiling) {
        for (auto &e : ev) CU(cudaEventCreate(&e));
        CU(cudaEventRecord(ev[0], stream));
    }
    const StateTables stt = r->slot_states[slot] ? slot_tables(r, slot) : StateTables{};
    CU(launch_raster(slot_scene(r, slot), r->view, r->d_frames[slot], r->d_work[slot], r->stride, r->slot_n[slot], d_index, d_rgba, stream,
                     r->slot_states[slot] ? &stt : nullptr));
    if (r->profiling) {
        CU(cudaEventRecord(ev[1], stream));
        for (auto e : ev) r->prof_events.push_back(e);
        r->prof_kinds.push_back(1);
    }
    CU(cudaEventRecord(r->raster_done[slot], stream));
    if (r->ds.masked_list) CU(cudaEventRecord(r->masked_done, stream));
    r->slot_rastered[slot] = true;
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

// The compact state of level time `tics` with the renderer's current sector moves into out[layout.words] (out is not
// r->state): the moved flag and the offsets, words 1 .. 2 + 2 * ndyn, do not depend on the time.
void state_at(const b2d_renderer *r, uint32_t tics, uint32_t *out) {
    compact_state(r->h_blob.data(), r->layout, tics, nullptr, nullptr, out);
    std::copy(r->state.begin() + 1, r->state.begin() + 2 + 2 * (ptrdiff_t)r->layout.dyn_sectors.size(), out + 1);
}

// The compact state of every frame of a b2d_render_states-style call into `out` (r->layout.words words per frame), checking
// everything first: nothing is enqueued for a call with an invalid frame.  `out` stays empty for a scene without
// time-dependent content or dynamic sectors: its frames all render with the per-batch tables.
int build_states(const b2d_renderer *r, const b2d_frame_state *states, size_t n, const b2d_sector_move *moves, size_t n_moves,
                 std::vector<uint32_t> &out) {
    out.clear();
    if (!states || (n_moves && !moves)) return fail(B2D_ERR_INVALID_ARG, "null argument");
    for (size_t i = 0; i < n; i++)
        if (states[i].first_move > n_moves || states[i].n_moves > n_moves - states[i].first_move)
            return fail(B2D_ERR_INVALID_ARG, "a frame's move range runs past the end of the move list");
    if (r->h_blob.empty()) {
        for (size_t i = 0; i < n; i++)
            if (states[i].n_moves) return fail(B2D_ERR_INVALID_ARG, "the scene declares no dynamic sectors");
        return B2D_OK;
    }
    const size_t words = r->layout.words;
    out.resize(n * words);
    std::vector<int32_t> fo, co;
    for (size_t i = 0; i < n; i++) {
        bool moved = false;
        if (states[i].n_moves) {
            if (const char *why = expand_moves(r->h_blob.data(), reinterpret_cast<const SectorMove *>(moves) + states[i].first_move,
                                               states[i].n_moves, fo, co)) {
                out.clear();
                return fail(B2D_ERR_INVALID_ARG, why);
            }
            for (size_t k = 0; k < fo.size() && !moved; k++) moved = fo[k] != 0 || co[k] != 0;    // all zero: at rest
        }
        compact_state(r->h_blob.data(), r->layout, states[i].tics, moved ? fo.data() : nullptr, moved ? co.data() : nullptr,
                      out.data() + i * words);
    }
    return B2D_OK;
}

// b2d_render_timed: tics[i] with the renderer's current moves
void timed_states(const b2d_renderer *r, const uint32_t *tics, size_t n, std::vector<uint32_t> &out) {
    out.clear();
    if (r->h_blob.empty()) return;
    const size_t words = r->layout.words;
    out.resize(n * words);
    for (size_t i = 0; i < n; i++) state_at(r, tics[i], out.data() + i * words);
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
    return B2D_OK;
}

// ---- renderer --------------------------------------------------------------------------------
int b2d_renderer_create(const b2d_scene *s, const b2d_view *view, int device, int max_batch, b2d_renderer **out) {
    if (!s || !view || !out || max_batch < 1) return fail(B2D_ERR_INVALID_ARG, "bad renderer arguments");
    if (view->width < 1 || view->width > 4096 || view->height < 2 || view->height > 2160 || view->F < 2 || view->FY2 < 2)
        return fail(B2D_ERR_INVALID_ARG, "view out of range");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(B2D_ERR_CUDA, std::string("no usable CUDA device (this library has no CPU path): ") +
                                      (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
    if (device < 0 || device >= count) return fail(B2D_ERR_INVALID_ARG, "device index out of range");
    CU(cudaSetDevice(device));
    b2d_renderer *r = new (std::nothrow) b2d_renderer();
    if (!r) return fail(B2D_ERR_NO_MEMORY, "out of host memory");
    r->device = device;
    r->view = View{view->width, view->height, view->F, view->FY2};
    r->max_batch = max_batch;
    const uint32_t *h = reinterpret_cast<const uint32_t *>(s->blob.data());
    r->stride = (int)(h[H_NSEGS] + h[H_NSPRITES]) > 0 ? (int)(h[H_NSEGS] + h[H_NSPRITES]) : 1;   // worklist entries per frame
    auto bail = [&](cudaError_t err, const char *what) { free_renderer(r); return cuda_fail(err, what); };
#define CUR(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return bail(e_, #call); } while (0)
    CUR(cudaMalloc(&r->d_blob, s->blob.size()));
    CUR(cudaMemcpy(r->d_blob, s->blob.data(), s->blob.size(), cudaMemcpyHostToDevice));
    std::vector<uint32_t> ys((size_t)view->height);
    for (int y = 0; y < view->height; y++) ys[(size_t)y] = yslope_entry(y, r->view);
    CUR(cudaMalloc(&r->d_yslope, ys.size() * 4));
    CUR(cudaMemcpy(r->d_yslope, ys.data(), ys.size() * 4, cudaMemcpyHostToDevice));
    {   // sky texture row per screen row (sky.frag:12-26 at pitch 0)
        std::vector<uint16_t> sr((size_t)view->height, 0);
        int32_t sky = (int32_t)h[H_SKY_TEX];
        if (sky >= 0) {
            const TexRec *tr = reinterpret_cast<const TexRec *>(s->blob.data() + h[H_OFF_TEX]) + sky;
            for (int y = 0; y < view->height; y++) sr[(size_t)y] = (uint16_t)sky_row(y, view->height, (int32_t)tr->h);
        }
        CUR(cudaMalloc(&r->d_skyrow, sr.size() * 2));
        CUR(cudaMemcpy(r->d_skyrow, sr.data(), sr.size() * 2, cudaMemcpyHostToDevice));
    }
    DeviceScene &d = r->ds;
    d.verts = reinterpret_cast<const int32_t *>(r->d_blob + h[H_OFF_VERTS]);
    d.nodes = reinterpret_cast<const NodeRec *>(r->d_blob + h[H_OFF_NODES]);
    d.ssectors = reinterpret_cast<const SSectorRec *>(r->d_blob + h[H_OFF_SSECTORS]);
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
        CUR(cudaMalloc(&r->d_walk_static, img.size() * 4 + 16));
        if (!img.empty()) CUR(cudaMemcpy(r->d_walk_static, img.data(), img.size() * 4, cudaMemcpyHostToDevice));
        d.walk_static = r->d_walk_static;
    }
    d.segs = reinterpret_cast<const SegRec *>(r->d_blob + h[H_OFF_SEGS]);
    d.sectors = reinterpret_cast<const SectorRec *>(r->d_blob + h[H_OFF_SECTORS]);
    d.tex = reinterpret_cast<const TexRec *>(r->d_blob + h[H_OFF_TEX]);
    d.mids = reinterpret_cast<const MidRec *>(r->d_blob + h[H_OFF_MIDS]);
    d.nmids = (int32_t)h[H_NMIDS];
    d.sprites = reinterpret_cast<const SpriteRec *>(r->d_blob + h[H_OFF_SPRITES]);
    d.nsprites = (int32_t)h[H_NSPRITES];
    d.masked_list = nullptr; d.masked_counter = nullptr; d.masked_chunks = 0; d.masked_cap = 0;
    if (d.nmids > 0 || d.nsprites > 0) {
        // arena of deferred masked entries: chunks of kMaskedChunk entries handed out on demand.  Sized for the worst case
        // -- every (frame, 32-column strip) of a full batch at its cap -- whenever that takes at most kMaskedArenaBudget, so
        // that no valid batch can run out of it: a crowded subsector puts dozens of sprites into every strip of a 1080p
        // frame.  Past the budget (1080p batches of more than ~1000 frames, 4K of more than ~500, with a cap of 128) two
        // chunks per strip on average, at least 4096: frames usually defer a handful of entries per strip, and a batch
        // that needs more reports kStatusMaskedFull instead of drawing wrong pixels.
        constexpr size_t kMaskedArenaBudget = (size_t)1 << 30;
        const size_t strips = (size_t)(view->width + 31) / 32;
        d.masked_cap = strip_masked_cap(d.nmids, d.nsprites);
        const size_t per_strip = ((size_t)d.masked_cap + kMaskedChunk - 1) / kMaskedChunk;
        const size_t worst = strips * (size_t)max_batch * per_strip;
        size_t chunks = worst;
        if (sizeof(uint32_t) * 33 * kMaskedChunk * worst > kMaskedArenaBudget) {
            chunks = strips * (size_t)max_batch * (per_strip < 2 ? per_strip : 2);
            if (chunks < 4096) chunks = 4096;
            if (chunks > worst) chunks = worst;
        }
        if (const char *env = getenv("B2D_MASKED_CHUNKS")) chunks = (size_t)strtoull(env, nullptr, 0);   // tests: force exhaustion
        if (chunks < 1) chunks = 1;
        d.masked_chunks = (uint32_t)chunks;
        CUR(cudaMalloc(&r->d_masked, sizeof(uint32_t) * 33 * kMaskedChunk * chunks));
        CUR(cudaMalloc(&r->d_masked_counter, sizeof(uint32_t)));
        CUR(cudaMemset(r->d_masked_counter, 0, sizeof(uint32_t)));
        CUR(cudaEventCreateWithFlags(&r->masked_done, cudaEventDisableTiming));
        CUR(cudaEventRecord(r->masked_done, nullptr));
        d.masked_list = r->d_masked;
        d.masked_counter = r->d_masked_counter;
    }
    d.texels = r->d_blob + h[H_OFF_TEXELS];
    d.flats = r->d_blob + h[H_OFF_FLATS];
    d.colormap = r->d_blob + h[H_OFF_COLORMAP];
    d.palette = reinterpret_cast<const uint32_t *>(r->d_blob + h[H_OFF_PALETTE]);
    {   // pre-lit texel and flat planes: 32 x (texel bytes + flat bytes)
        const size_t tstride = (h[H_TEXEL_BYTES] + 255u) & ~(size_t)255, fstride = (size_t)h[H_NFLATS] * 4096u;
        if (tstride * 33 > 0xFFFFFFFFull || fstride * 32 > 0xFFFFFFFFull) { free_renderer(r); return fail(B2D_ERR_INVALID_ARG, "level textures too large"); }
        CUR(cudaMalloc(&r->d_lit, 33 * tstride + 256));                    // plane 32 of the texels: opacity
        if (!alloc_aligned_4g(r, 32 * fstride + 256)) { free_renderer(r); return fail(B2D_ERR_NO_MEMORY, "no 4 GiB aligned device memory for the pre-lit flats"); }
        CUR(launch_prelight_textures(d.colormap, d.texels, d.tex, (int)h[H_NTEX], r->d_lit, tstride, nullptr));
        CUR(launch_prelight(d.colormap, d.flats, r->d_lit_flats, fstride, fstride, nullptr));
        CUR(cudaDeviceSynchronize());
        d.lit_texels = r->d_lit; d.lit_flats = r->d_lit_flats;           // low 32 address bits of lit_flats are zero
        d.lit_texel_stride = (uint32_t)tstride; d.lit_flat_stride = (uint32_t)fstride;
    }
    d.yslope = r->d_yslope;
    d.skyrow = r->d_skyrow;
    CUR(cudaMalloc(&r->d_status, sizeof(int32_t)));
    CUR(cudaMemset(r->d_status, 0, sizeof(int32_t)));
    d.status_flag = r->d_status;
    d.nverts = (int32_t)h[H_NVERTS]; d.nnodes = (int32_t)h[H_NNODES]; d.nss = (int32_t)h[H_NSSECTORS];
    d.nsegs = (int32_t)h[H_NSEGS]; d.nsectors = (int32_t)h[H_NSECTORS]; d.ntex = (int32_t)h[H_NTEX];
    d.nflats = (int32_t)h[H_NFLATS]; d.sky_tex = (int32_t)h[H_SKY_TEX];
    d.root = h[H_ROOT];
    d.invF = (uint32_t)(4294967296ULL / (uint64_t)view->F);
    if (d.nsegs + d.nsprites > 65535) { free_renderer(r); return fail(B2D_ERR_INVALID_ARG, "level has more than 65535 segs + sprites"); }
    if (walk_smem_per_warp(d) > 227 * 1024) { free_renderer(r); return fail(B2D_ERR_INVALID_ARG, "level too large for the BSP-walk kernel's shared memory"); }
    if (scene_is_timed(s->blob.data())) {
        r->h_blob = s->blob;
        try {
            r->layout = state_layout(r->h_blob.data());
        } catch (const std::exception &ex) {
            free_renderer(r);
            return fail(B2D_ERR_INVALID_ARG, ex.what());
        }
        const uint8_t *blob = r->h_blob.data();
        const StateLayout &L = r->layout;
        const size_t words = L.words, mb = (size_t)max_batch;
        // the state rule reads the blob's rest-state sections and the two slot maps
        CUR(cudaMalloc(&r->d_slot_maps, 4 * (L.sector_slots.size() + L.mid_seg.size()) + 4));
        CUR(cudaMemcpy(r->d_slot_maps, L.sector_slots.data(), 4 * L.sector_slots.size(), cudaMemcpyHostToDevice));
        CUR(cudaMemcpy(r->d_slot_maps + L.sector_slots.size(), L.mid_seg.data(), 4 * L.mid_seg.size(), cudaMemcpyHostToDevice));
        StateSrc &src = r->src = state_src(blob, L);
        auto on_device = [&](auto p) { return reinterpret_cast<decltype(p)>(r->d_blob + (reinterpret_cast<const uint8_t *>(p) - blob)); };
        src.tex = on_device(src.tex); src.sectors = on_device(src.sectors); src.segs = on_device(src.segs);
        src.sprites = on_device(src.sprites); src.mids = on_device(src.mids); src.anim = on_device(src.anim);
        src.flat_anim = on_device(src.flat_anim); src.segdyn = on_device(src.segdyn);
        src.sector_slots = r->d_slot_maps;
        src.mid_seg = reinterpret_cast<const int32_t *>(r->d_slot_maps + L.sector_slots.size());
        StateTables &t = r->state_tables;              // one table set: [tex | sectors | segs | sprites | mids], 256 B aligned
        t.slot_bytes = (uint32_t)((state_table_bytes(blob) + 255) & ~(size_t)255);
        t.off_sectors = (uint32_t)(h[H_NTEX] * sizeof(TexRec));
        t.off_segs = t.off_sectors + (uint32_t)(h[H_NSECTORS] * sizeof(SectorRec));
        t.off_sprites = t.off_segs + (uint32_t)(h[H_NSEGS] * sizeof(SegRec));
        t.off_mids = t.off_sprites + (uint32_t)(h[H_NSPRITES] * sizeof(SpriteRec));
        CUR(cudaMalloc(&r->d_slot_tables, 2 * (size_t)t.slot_bytes));
        for (int i = 0; i < 2; i++) {
            CUR(cudaMalloc(&r->d_states[i], 4 * mb * (words + 1)));
            CUR(cudaMallocHost(&r->h_states[i], 4 * mb * (words + 1)));
            CUR(cudaEventCreateWithFlags(&r->states_copied[i], cudaEventDisableTiming));
        }
        // tic 0 is a time like any other: a frame name with k > 0 shows its group's frame 0 (tex.rs:260, 302-306).  The
        // pre-lit planes above were built from the blob's own (per-image) records; both slots' table sets start at tic 0.
        r->state.assign(words, 0);
        compact_state(blob, L, 0, nullptr, nullptr, r->state.data());
        CUR(cudaMemcpy(r->d_states[0], r->state.data(), 4 * words, cudaMemcpyHostToDevice));
        for (int i = 0; i < 2; i++) {
            CUR(launch_state_tables(r->src, r->d_states[0], (uint32_t)words, 1, r->d_slot_tables + i * (size_t)t.slot_bytes, t, nullptr));
            r->slot_state[i] = r->state;
        }
        CUR(cudaDeviceSynchronize());
    }
    CUR(cudaMalloc(&r->d_poses, sizeof(Pose) * (size_t)max_batch));
    CUR(cudaMalloc(&r->d_frames[0], sizeof(FrameConst) * (size_t)max_batch));
    CUR(cudaMalloc(&r->d_work[0], sizeof(SegFrame) * (size_t)max_batch * (size_t)r->stride));
#undef CUR
    *out = r;
    return B2D_OK;
}

void b2d_renderer_destroy(b2d_renderer *r) { free_renderer(r); }

// The renderer's own state is host data: the setters enqueue nothing (the stream is kept for ABI compatibility), and the
// next plain batch of each worklist slot expands it into the slot's table set.
int b2d_renderer_set_time(b2d_renderer *r, uint32_t tics) {
    if (!r) return fail(B2D_ERR_INVALID_ARG, "null renderer");
    if (r->h_blob.empty()) { r->tics = tics; return B2D_OK; }
    return guarded([&] {
        std::vector<uint32_t> s(r->layout.words);
        state_at(r, tics, s.data());
        r->state.swap(s);
        r->tics = tics;
        return B2D_OK;
    });
}

int b2d_renderer_set_time_async(b2d_renderer *r, uint32_t tics, void *) { return b2d_renderer_set_time(r, tics); }

int b2d_renderer_set_sector_moves(b2d_renderer *r, const b2d_sector_move *moves, size_t n) {
    if (!r || (n && !moves)) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (r->h_blob.empty()) {
        if (n == 0) return B2D_OK;
        return fail(B2D_ERR_INVALID_ARG, "the scene declares no dynamic sectors");
    }
    static_assert(sizeof(b2d_sector_move) == sizeof(SectorMove), "ABI record");
    return guarded([&] {
        std::vector<int32_t> fo, co;
        if (const char *why = expand_moves(r->h_blob.data(), reinterpret_cast<const SectorMove *>(moves), n, fo, co))
            return fail(B2D_ERR_INVALID_ARG, why);
        bool moved = false;
        for (size_t i = 0; i < fo.size() && !moved; i++) moved = fo[i] != 0 || co[i] != 0;      // all zero: at rest
        compact_state(r->h_blob.data(), r->layout, r->tics, moved ? fo.data() : nullptr, moved ? co.data() : nullptr,
                      r->state.data());
        return B2D_OK;
    });
}

int b2d_renderer_set_sector_moves_async(b2d_renderer *r, const b2d_sector_move *moves, size_t n, void *) {
    return b2d_renderer_set_sector_moves(r, moves, n);
}

int b2d_renderer_status(b2d_renderer *r, int32_t *bits_out) {
    if (!r || !bits_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    CU(cudaSetDevice(r->device));
    CU(cudaDeviceSynchronize());
    int32_t status = 0;
    CU(cudaMemcpy(&status, r->d_status, sizeof status, cudaMemcpyDeviceToHost));
    if (status) CU(cudaMemset(r->d_status, 0, sizeof(int32_t)));
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

// frames_states (nullable, r->layout.words words per frame): walk + raster of n device poses in batches of max_batch
static int enqueue_batches(b2d_renderer *r, const b2d_pose *d_poses, size_t n, const uint32_t *frame_states, uint8_t *d_index_fb,
                           uint32_t *d_rgba_fb, cudaStream_t st) {
    const size_t npix = (size_t)r->view.W * r->view.H;
    for (size_t i = 0; i < n; i += (size_t)r->max_batch) {
        const size_t cnt = n - i < (size_t)r->max_batch ? n - i : (size_t)r->max_batch;
        int rc = enqueue_frames(r, reinterpret_cast<const Pose *>(d_poses) + i, (int)cnt, d_index_fb + i * npix,
                                d_rgba_fb ? d_rgba_fb + i * npix : nullptr, st, frame_states ? frame_states + i * r->layout.words : nullptr);
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

// Host poses in, host frames out; frame_states as in enqueue_frames (for all n frames)
static int render_host(b2d_renderer *r, const b2d_pose *poses, size_t n, const uint32_t *frame_states, uint8_t *index_fb,
                       uint32_t *rgba_fb) {
    if (n == 0) return B2D_OK;
    CU(cudaSetDevice(r->device));
    const size_t npix = (size_t)r->view.W * r->view.H;
    if (!r->render_stream) {
        CU(cudaStreamCreateWithFlags(&r->render_stream, cudaStreamNonBlocking));
        for (int i = 0; i < 2; i++) CU(cudaStreamCreateWithFlags(&r->copy_stream[i], cudaStreamNonBlocking));
        for (int i = 0; i < 2; i++) {
            CU(cudaEventCreateWithFlags(&r->rendered[i], cudaEventDisableTiming));
            CU(cudaEventCreateWithFlags(&r->copied[i], cudaEventDisableTiming));
            CU(cudaMalloc(&r->d_index[i], npix * (size_t)r->max_batch));
        }
        CU(cudaMallocHost(&r->h_poses, sizeof(Pose) * (size_t)r->max_batch * 2));
    }
    if (rgba_fb && !r->d_rgba[0])
        for (int i = 0; i < 2; i++) CU(cudaMalloc(&r->d_rgba[i], npix * 4 * (size_t)r->max_batch));
    // Double-buffered pipeline: batch b renders into buffer b&1 on render_stream while the copy
    // stream drains buffer (b-1)&1 to the caller's host memory.
    size_t done = 0;
    int b = 0;
    while (done < n) {
        const int cnt = (int)(n - done < (size_t)r->max_batch ? n - done : (size_t)r->max_batch);
        const int buf = b & 1;
        if (b >= 2) CU(cudaEventSynchronize(r->copied[buf]));       // buffer + pose slot free again
        Pose *hp = r->h_poses + (size_t)buf * r->max_batch;
        std::memcpy(hp, poses + done, sizeof(Pose) * (size_t)cnt);
        CU(cudaMemcpyAsync(r->d_poses, hp, sizeof(Pose) * (size_t)cnt, cudaMemcpyHostToDevice, r->render_stream));
        int rc = enqueue_frames(r, r->d_poses, cnt, r->d_index[buf], rgba_fb ? r->d_rgba[buf] : nullptr, r->render_stream,
                                frame_states ? frame_states + done * r->layout.words : nullptr);
        if (rc != B2D_OK) return rc;
        CU(cudaEventRecord(r->rendered[buf], r->render_stream));
        CU(cudaStreamWaitEvent(r->copy_stream[buf], r->rendered[buf], 0));
        CU(cudaMemcpyAsync(index_fb + done * npix, r->d_index[buf], npix * (size_t)cnt, cudaMemcpyDeviceToHost, r->copy_stream[buf]));
        if (rgba_fb)
            CU(cudaMemcpyAsync(rgba_fb + done * npix, r->d_rgba[buf], npix * 4 * (size_t)cnt, cudaMemcpyDeviceToHost, r->copy_stream[buf]));
        CU(cudaEventRecord(r->copied[buf], r->copy_stream[buf]));
        done += (size_t)cnt;
        b++;
    }
    for (int i = 0; i < 2; i++) CU(cudaStreamSynchronize(r->copy_stream[i]));
    CU(cudaStreamSynchronize(r->render_stream));
    int32_t status = 0;
    CU(cudaMemcpy(&status, r->d_status, sizeof status, cudaMemcpyDeviceToHost));
    if (status) {
        CU(cudaMemset(r->d_status, 0, sizeof(int32_t)));
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

int b2d_palette_lut_device(b2d_renderer *r, const uint8_t *d_index, uint32_t *d_rgba, size_t n_pixels, void *cuda_stream) {
    if (!r || !d_index || !d_rgba) return fail(B2D_ERR_INVALID_ARG, "null argument");
    CU(cudaSetDevice(r->device));
    CU(launch_palette(r->ds.palette, d_index, d_rgba, n_pixels, static_cast<cudaStream_t>(cuda_stream)));
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
    if (!r->d_frames[slot] || n > (size_t)r->slot_n[slot]) return fail(B2D_ERR_INVALID_ARG, "n exceeds the frames of the last walked batch");
    CU(cudaSetDevice(r->device));
    CU(cudaDeviceSynchronize());
    std::vector<FrameConst> frames(n);
    CU(cudaMemcpy(frames.data(), r->d_frames[slot], sizeof(FrameConst) * n, cudaMemcpyDeviceToHost));
    std::vector<SegFrame> work;
    for (size_t i = 0; i < n; i++) {
        counts_out[i] = frames[i].status ? -frames[i].status : frames[i].count;
        if (!seg_ids_out) continue;
        size_t c = frames[i].count > 0 ? (size_t)frames[i].count : 0;
        if (c > (size_t)r->stride) c = (size_t)r->stride;
        work.resize(c);
        if (c) CU(cudaMemcpy(work.data(), r->d_work[slot] + i * (size_t)r->stride, sizeof(SegFrame) * c, cudaMemcpyDeviceToHost));
        for (size_t k = 0; k < c && k < stride; k++) seg_ids_out[i * stride + k] = work[k].seg;
    }
    return B2D_OK;
}

int b2d_debug_state_slots(b2d_renderer *r, size_t n, uint32_t *slots_out) {
    if (!r || !slots_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    const int slot = r->last_slot;
    if (!r->slot_states[slot] || n > (size_t)r->slot_n[slot])
        return fail(B2D_ERR_INVALID_ARG, "the last walked batch has no per-frame states or fewer than n frames");
    CU(cudaSetDevice(r->device));
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(slots_out, slot_tables(r, slot).frame_slot, 4 * n, cudaMemcpyDeviceToHost));
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
        CU(cudaEventElapsedTime(&a, r->prof_events[i], r->prof_events[i + 1]));
        if (r->prof_kinds[i / 2] == 0) w += a; else { ra += a; nb++; }
    }
    if (walk_ms) *walk_ms = w;
    if (raster_ms) *raster_ms = ra;
    if (batches) *batches = nb;
    r->prof_kinds.clear();
    for (cudaEvent_t e : r->prof_events) cudaEventDestroy(e);
    r->prof_events.clear();
    return B2D_OK;
}

int64_t b2d_launch_count(const b2d_renderer *r) { return r ? r->launches : 0; }

}  // extern "C"
