// C-ABI of libb2d.so (declared in include/b2d.h).  Thin, exception-free boundary over the C++ host
// side (WAD loader, scene compiler) and the CUDA kernels.  There is deliberately no CPU rendering
// path here: every render entry point launches the sm_90a kernels or fails with B2D_ERR_CUDA.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
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
    if (r->tables_ready) cudaEventDestroy(r->tables_ready);
    for (int i = 0; i < 2; i++) {
        if (r->h_timed[i]) cudaFreeHost(r->h_timed[i]);
        if (r->timed_copied[i]) cudaEventDestroy(r->timed_copied[i]);
    }
    if (r->d_lit) cudaFree(r->d_lit);
    if (r->d_walk_static) cudaFree(r->d_walk_static);
    free_aligned_4g(r);
    if (r->d_blob) cudaFree(r->d_blob);
    delete r;
}

// BSP walk of a batch into the next worklist slot, on `stream`.  The slot's previous raster (if any, on whatever
// stream) is awaited through an event, so a caller may run walks and rasters on two streams and have the walk of
// batch k+1 overlap the raster of batch k.
int walk_into_slot(b2d_renderer *r, const Pose *d_poses, int n, cudaStream_t stream, int64_t *ticket_out, bool background = false) {
    const int slot = (int)(r->next_ticket & 1);
    if (!r->slot_rastered[slot]) return fail(B2D_ERR_INVALID_ARG, "both worklist slots hold batches that were walked but not rastered yet");
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
    if (r->tables_pending) CU(cudaStreamWaitEvent(stream, r->tables_ready, 0));   // a table upload on another stream
    cudaEvent_t ev[2] = {nullptr, nullptr};
    if (r->profiling) {
        for (auto &e : ev) CU(cudaEventCreate(&e));
        CU(cudaEventRecord(ev[0], stream));
    }
    CU(launch_walk(r->ds, r->view, d_poses, n, r->d_frames[slot], r->d_work[slot], r->stride, stream, background));
    if (r->profiling) {
        CU(cudaEventRecord(ev[1], stream));
        for (auto e : ev) r->prof_events.push_back(e);
        r->prof_kinds.push_back(0);
    }
    CU(cudaEventRecord(r->walk_done[slot], stream));
    r->slot_n[slot] = n;
    r->slot_ticket[slot] = r->next_ticket;
    r->slot_rastered[slot] = false;
    r->last_slot = slot;
    r->last_n = n;
    r->launches += 1;
    *ticket_out = r->next_ticket++;
    return B2D_OK;
}

int raster_from_slot(b2d_renderer *r, int64_t ticket, uint8_t *d_index, uint32_t *d_rgba, cudaStream_t stream) {
    const int slot = (int)(ticket & 1);
    if (ticket < 0 || r->slot_ticket[slot] != ticket || r->slot_rastered[slot])
        return fail(B2D_ERR_INVALID_ARG, "unknown or already rastered walk ticket");
    CU(cudaStreamWaitEvent(stream, r->walk_done[slot], 0));
    if (r->tables_pending) CU(cudaStreamWaitEvent(stream, r->tables_ready, 0));
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
    CU(launch_raster(r->ds, r->view, r->d_frames[slot], r->d_work[slot], r->stride, r->slot_n[slot], d_index, d_rgba, stream));
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

// Rebuild the time-dependent tables for `tics` on the host (scene_at_time) and copy them over their sections of the
// device blob in stream order.  Everything this renderer has enqueued so far -- on any stream -- is awaited by `stream`
// first (the walk/raster events of both worklist slots), and later launches on other streams wait for the upload, so the
// host never blocks on the device: no cudaDeviceSynchronize in the System::update loop this stands in for.
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

void tables_at(const b2d_renderer *r, uint32_t tics, uint8_t *out) {
    const bool moved = !r->floor_off.empty();
    state_tables(r->h_blob.data(), tics, moved ? r->floor_off.data() : nullptr, moved ? r->ceil_off.data() : nullptr, out);
}

int upload_tables(b2d_renderer *r, const uint8_t *tables, cudaStream_t stream) {
    const uint32_t *h = reinterpret_cast<const uint32_t *>(r->h_blob.data());
    const int buf = r->timed_next;
    r->timed_next ^= 1;
    CU(cudaEventSynchronize(r->timed_copied[buf]));          // the copy issued two uploads ago has read this buffer
    uint8_t *p = r->h_timed[buf];
    std::memcpy(p, tables, r->timed_bytes);
    const uint8_t *tex = p, *sectors = tex + h[H_NTEX] * sizeof(TexRec), *segs = sectors + h[H_NSECTORS] * sizeof(SectorRec),
                  *sprites = segs + h[H_NSEGS] * sizeof(SegRec), *mids = sprites + h[H_NSPRITES] * sizeof(SpriteRec);
    for (int i = 0; i < 2; i++) {
        if (r->walk_done[i]) CU(cudaStreamWaitEvent(stream, r->walk_done[i], 0));
        if (r->raster_done[i]) CU(cudaStreamWaitEvent(stream, r->raster_done[i], 0));
    }
    CU(cudaMemcpyAsync(r->d_blob + h[H_OFF_TEX], tex, h[H_NTEX] * sizeof(TexRec), cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(r->d_blob + h[H_OFF_SECTORS], sectors, h[H_NSECTORS] * sizeof(SectorRec), cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(r->d_blob + h[H_OFF_SEGS], segs, h[H_NSEGS] * sizeof(SegRec), cudaMemcpyHostToDevice, stream));
    if (h[H_NSPRITES])
        CU(cudaMemcpyAsync(r->d_blob + h[H_OFF_SPRITES], sprites, h[H_NSPRITES] * sizeof(SpriteRec), cudaMemcpyHostToDevice, stream));
    if (h[H_NMIDS] && h[H_NDYN])        // masked middle textures only move with their sector
        CU(cudaMemcpyAsync(r->d_blob + h[H_OFF_MIDS], mids, h[H_NMIDS] * sizeof(MidRec), cudaMemcpyHostToDevice, stream));
    CU(cudaEventRecord(r->timed_copied[buf], stream));
    CU(cudaEventRecord(r->tables_ready, stream));
    r->tables_pending = true;
    r->cur_tables.assign(tables, tables + r->timed_bytes);
    return B2D_OK;
}

int upload_timed_tables(b2d_renderer *r, uint32_t tics, cudaStream_t stream) {
    r->scratch_tables.resize(r->timed_bytes);
    tables_at(r, tics, r->scratch_tables.data());
    return upload_tables(r, r->scratch_tables.data(), stream);
}

// Per-pose time: poses [i, n) with their tics; makes the tables of tics[i] current on `stream` (uploading only if they
// differ from what is there) and returns in *end the end of the run of poses that can share this launch: consecutive
// poses whose tables are byte-identical (equal tics, or different tics that change nothing -- e.g. inside one 8-tic
// animation frame of a level without light effects or scrolling walls).
int timed_run(b2d_renderer *r, const uint32_t *tics, size_t i, size_t n, size_t limit, cudaStream_t stream, size_t *end) {
    if (r->h_blob.empty() || !tics) { *end = n < i + limit ? n : i + limit; return B2D_OK; }
    r->scratch_tables.resize(r->timed_bytes);
    tables_at(r, tics[i], r->scratch_tables.data());
    if (r->cur_tables.size() != r->timed_bytes || std::memcmp(r->cur_tables.data(), r->scratch_tables.data(), r->timed_bytes) != 0) {
        int rc = upload_tables(r, r->scratch_tables.data(), stream);
        if (rc != B2D_OK) return rc;
    }
    r->tics = tics[i];
    size_t j = i + 1;
    uint32_t same = tics[i];
    while (j < n && j < i + limit) {
        if (tics[j] != same) {
            tables_at(r, tics[j], r->scratch_tables.data());
            if (std::memcmp(r->cur_tables.data(), r->scratch_tables.data(), r->timed_bytes) != 0) break;
            same = tics[j];
            r->tics = same;
        }
        j++;
    }
    *end = j;
    return B2D_OK;
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
                        cudaStream_t stream) {
    int64_t ticket = -1;
    int rc = walk_into_slot(r, d_poses, n, stream, &ticket);
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
        // arena of deferred masked entries: chunks of kMaskedChunk entries handed out on demand.  Sized for two chunks per
        // (frame, 32-column strip) of a full batch -- frames defer a handful of entries per strip -- and never more than the
        // worst case (every strip at its cap).  1000 x 1080p: 63 MB instead of the 1 GB a fixed per-strip list takes.
        const size_t strips = (size_t)(view->width + 31) / 32;
        d.masked_cap = strip_masked_cap(d.nmids, d.nsprites);
        const size_t per_strip = ((size_t)d.masked_cap + kMaskedChunk - 1) / kMaskedChunk;
        size_t chunks = strips * (size_t)max_batch * (per_strip < 2 ? per_strip : 2);
        if (chunks < 4096) chunks = 4096;
        const size_t worst = strips * (size_t)max_batch * per_strip;
        if (chunks > worst) chunks = worst;
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
        r->timed_bytes = state_table_bytes(r->h_blob.data());
        for (int i = 0; i < 2; i++) {
            CUR(cudaMallocHost(&r->h_timed[i], r->timed_bytes ? r->timed_bytes : 1));
            CUR(cudaEventCreateWithFlags(&r->timed_copied[i], cudaEventDisableTiming));
        }
        CUR(cudaEventCreateWithFlags(&r->tables_ready, cudaEventDisableTiming));
        // tic 0 is a time like any other: a frame name with k > 0 shows its group's frame 0 (tex.rs:260, 302-306).  The
        // pre-lit planes above were built from the blob's own (per-image) records; from here on the records are re-pointed.
        int rc = upload_timed_tables(r, 0, nullptr);
        if (rc != B2D_OK) { free_renderer(r); return rc; }
        CUR(cudaStreamSynchronize(nullptr));
        r->tables_pending = false;
    }
    CUR(cudaMalloc(&r->d_poses, sizeof(Pose) * (size_t)max_batch));
    CUR(cudaMalloc(&r->d_frames[0], sizeof(FrameConst) * (size_t)max_batch));
    CUR(cudaMalloc(&r->d_work[0], sizeof(SegFrame) * (size_t)max_batch * (size_t)r->stride));
#undef CUR
    *out = r;
    return B2D_OK;
}

void b2d_renderer_destroy(b2d_renderer *r) { free_renderer(r); }

int b2d_renderer_set_time_async(b2d_renderer *r, uint32_t tics, void *cuda_stream) {
    if (!r) return fail(B2D_ERR_INVALID_ARG, "null renderer");
    if (r->h_blob.empty() || tics == r->tics) { r->tics = tics; return B2D_OK; }
    CU(cudaSetDevice(r->device));
    int rc = upload_timed_tables(r, tics, static_cast<cudaStream_t>(cuda_stream));
    if (rc == B2D_OK) r->tics = tics;
    return rc;
}

int b2d_renderer_set_sector_moves_async(b2d_renderer *r, const b2d_sector_move *moves, size_t n, void *cuda_stream) {
    if (!r || (n && !moves)) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (r->h_blob.empty()) {
        if (n == 0) return B2D_OK;
        return fail(B2D_ERR_INVALID_ARG, "the scene declares no dynamic sectors");
    }
    static_assert(sizeof(b2d_sector_move) == sizeof(SectorMove), "ABI record");
    std::vector<int32_t> fo, co;
    if (const char *why = expand_moves(r->h_blob.data(), reinterpret_cast<const SectorMove *>(moves), n, fo, co))
        return fail(B2D_ERR_INVALID_ARG, why);
    bool any = false;
    for (size_t i = 0; i < fo.size(); i++) any |= fo[i] != 0 || co[i] != 0;
    if (!any) { fo.clear(); co.clear(); }
    if (fo == r->floor_off && co == r->ceil_off) return B2D_OK;
    r->floor_off.swap(fo);
    r->ceil_off.swap(co);
    CU(cudaSetDevice(r->device));
    return upload_timed_tables(r, r->tics, static_cast<cudaStream_t>(cuda_stream));
}

int b2d_renderer_set_sector_moves(b2d_renderer *r, const b2d_sector_move *moves, size_t n) {
    int rc = b2d_renderer_set_sector_moves_async(r, moves, n, nullptr);
    if (rc != B2D_OK) return rc;
    if (r->tables_pending) {
        CU(cudaEventSynchronize(r->tables_ready));
        r->tables_pending = false;
    }
    return B2D_OK;
}

int b2d_renderer_set_time(b2d_renderer *r, uint32_t tics) {
    int rc = b2d_renderer_set_time_async(r, tics, nullptr);
    if (rc != B2D_OK) return rc;
    if (r->tables_pending) {
        CU(cudaEventSynchronize(r->tables_ready));
        r->tables_pending = false;
    }
    return B2D_OK;
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

int b2d_render_device_timed(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *tics, size_t n, uint8_t *d_index_fb,
                            uint32_t *d_rgba_fb, void *cuda_stream) {
    if (!r || !d_poses || !d_index_fb || !tics) return fail(B2D_ERR_INVALID_ARG, "null argument");
    CU(cudaSetDevice(r->device));
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    const size_t npix = (size_t)r->view.W * r->view.H;
    size_t i = 0;
    while (i < n) {
        size_t j = i;
        int rc = timed_run(r, tics, i, n, (size_t)r->max_batch, st, &j);
        if (rc != B2D_OK) return rc;
        rc = enqueue_frames(r, reinterpret_cast<const Pose *>(d_poses) + i, (int)(j - i), d_index_fb + i * npix,
                            d_rgba_fb ? d_rgba_fb + i * npix : nullptr, st);
        if (rc != B2D_OK) return rc;
        i = j;
    }
    return B2D_OK;
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

int b2d_render(b2d_renderer *r, const b2d_pose *poses, size_t n, uint8_t *index_fb, uint32_t *rgba_fb) {
    return b2d_render_timed(r, poses, nullptr, n, index_fb, rgba_fb);
}

int b2d_render_timed(b2d_renderer *r, const b2d_pose *poses, const uint32_t *tics, size_t n, uint8_t *index_fb, uint32_t *rgba_fb) {
    if (!r || !poses || !index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
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
        size_t run_end = done;                                      // per-pose time: a batch ends where the tables change
        int trc = timed_run(r, tics, done, n, (size_t)r->max_batch, r->render_stream, &run_end);
        if (trc != B2D_OK) return trc;
        const int cnt = (int)(run_end - done);
        const int buf = b & 1;
        if (b >= 2) CU(cudaEventSynchronize(r->copied[buf]));       // buffer + pose slot free again
        Pose *hp = r->h_poses + (size_t)buf * r->max_batch;
        std::memcpy(hp, poses + done, sizeof(Pose) * (size_t)cnt);
        CU(cudaMemcpyAsync(r->d_poses, hp, sizeof(Pose) * (size_t)cnt, cudaMemcpyHostToDevice, r->render_stream));
        int rc = enqueue_frames(r, r->d_poses, cnt, r->d_index[buf], rgba_fb ? r->d_rgba[buf] : nullptr, r->render_stream);
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
