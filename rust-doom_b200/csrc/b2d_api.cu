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

// The layout of one table set of a level, [tex | sectors | segs | sprites | mids] (b2d_scene_tables_at's), from its five
// record counts: the byte offsets of the sections after the first, the set's bytes, and `slot`, those rounded up to 256
// (the space a set takes in an arena or as a worklist slot's own set).
struct SetLayout {
    size_t sectors, segs, sprites, mids, bytes, slot;
    SetLayout(size_t ntex, size_t nsectors, size_t nsegs, size_t nsprites, size_t nmids)
        : sectors(ntex * sizeof(TexRec)), segs(sectors + nsectors * sizeof(SectorRec)), sprites(segs + nsegs * sizeof(SegRec)),
          mids(sprites + nsprites * sizeof(SpriteRec)), bytes(mids + nmids * sizeof(MidRec)), slot((bytes + 255) & ~(size_t)255) {}
    explicit SetLayout(const StateSrc &s) : SetLayout(s.ntex, s.nsectors, s.nsegs, s.nsprites, s.nmids) {}
    explicit SetLayout(const uint8_t *blob)      // a scene blob's, from its header
        : SetLayout(hdr(blob)[H_NTEX], hdr(blob)[H_NSECTORS], hdr(blob)[H_NSEGS], hdr(blob)[H_NSPRITES], hdr(blob)[H_NMIDS]) {}
    // the five tables of the set at `base`
    TableSet at(const uint8_t *base) const {
        return TableSet{reinterpret_cast<const TexRec *>(base), reinterpret_cast<const SectorRec *>(base + sectors),
                        reinterpret_cast<const SegRec *>(base + segs), reinterpret_cast<const SpriteRec *>(base + sprites),
                        reinterpret_cast<const MidRec *>(base + mids)};
    }
  private:
    static const uint32_t *hdr(const uint8_t *blob) { return reinterpret_cast<const uint32_t *>(blob); }
};

// Per-frame states: the two worklist slots' arenas of max_batch table sets, allocated together by the first such call.  A
// set takes its level's SetLayout::slot; the arena is sized by the largest of the levels, so that it holds max_batch sets
// of any mix of levels.
int ensure_states(b2d_renderer *r) {
    if (r->slot[0].arena) return B2D_OK;
    size_t slot_bytes = 0;
    for (const LevelRes &lv : r->lv) slot_bytes = std::max(slot_bytes, SetLayout(lv.src).slot);
    DeviceBuf<uint8_t> arena[2];
    for (auto &a : arena) CU(allocate(a, (size_t)r->max_batch * slot_bytes));
    for (int i = 0; i < 2; i++) r->slot[i].arena = std::move(arena[i]);
    return B2D_OK;
}

// The sections of a batch in its worklist slot's staging (WorkSlot::stage, h_stage), copied to the device in one piece:
// what the batch's expansions, walk and raster read.  Byte offsets, each section 16-byte aligned; a section the batch
// does not use is empty.
struct StageLayout {
    size_t scenes = 0;         // with per-frame levels: the DeviceScene of every level
    size_t srcs, sets, descs;  // StateSrc of every level | TableSet of every set to expand, then, with per-frame states, of
                               // every level's blob tables | StateSet of every set to expand
    size_t frame_level, frame_set;  // per frame: level | TableSet index (per-frame states)
    size_t frame_fixed, planes;     // with fixed colormaps: per frame its row | per level its FixedPlanes
    size_t states, end;             // the sets' states
    StageLayout(size_t nlev, size_t nsets, size_t n, size_t state_words, bool per_frame, bool per_level, bool fixed_rows = false) {
        auto up = [](size_t x) { return (x + 15) & ~(size_t)15; };
        srcs = up((per_level ? nlev : 0) * sizeof(DeviceScene));
        sets = up(srcs + nlev * sizeof(StateSrc));
        descs = up(sets + (nsets + (per_frame ? nlev : 0)) * sizeof(TableSet));
        frame_level = up(descs + nsets * sizeof(StateSet));
        frame_set = up(frame_level + (per_level ? 4 * n : 0));
        frame_fixed = up(frame_set + (per_frame ? 4 * n : 0));
        planes = up(frame_fixed + (fixed_rows ? 4 * n : 0));
        states = up(planes + (fixed_rows ? nlev * sizeof(FixedPlanes) : 0));
        end = states + 4 * state_words;
    }
};

// records of one table set of a level (the threads of its expansion)
size_t set_records(const LevelRes &lv) { return (size_t)lv.src.ntex + lv.src.nsectors + lv.src.nsegs + lv.src.nsprites + lv.src.nmids; }

// a level's scene as the kernels of worklist slot `slot` read it: on a timed scene, the five state-dependent tables are the
// level's table set of that slot
DeviceScene slot_scene(const LevelRes &lv, int slot) {
    DeviceScene d = lv.ds;
    if (const uint8_t *set = lv.slot[slot].tables.get()) {
        const TableSet t = SetLayout(lv.src).at(set);
        d.tex = t.tex; d.sectors = t.sectors; d.segs = t.segs; d.sprites = t.sprites; d.mids = t.mids;
    }
    return d;
}

// `launch` on `stream`, between two timing events while the renderer profiles (b2d_profile_read): kind 0 = walk, 1 = raster
template <typename Launch>
int profiled(b2d_renderer *r, cudaStream_t stream, int kind, Launch launch) {
    Event ev[2];
    if (r->profiling) {
        for (auto &e : ev) CU(event_create(e, cudaEventDefault));
        CU(cudaEventRecord(ev[0].get(), stream));
    }
    CU(launch());
    if (r->profiling) {
        CU(cudaEventRecord(ev[1].get(), stream));
        for (auto &e : ev) r->prof_events.push_back(std::move(e));
        r->prof_kinds.push_back(kind);
    }
    return B2D_OK;
}

// A table set a batch expands: level `level` at the compact state `state` (host) with extra light `extralight` into the
// tables at `tables`.
struct Expansion {
    uint32_t level;
    const uint32_t *state;
    uint8_t *tables;
    uint32_t extralight;
};

// Level `lv`'s row-32 planes (fixed colormap 32, DESIGN.md C18), built on `stream` by the first batch that needs them: the
// group is created whole, or not at all.
int ensure_row32(b2d_renderer *r, LevelRes &lv, cudaStream_t stream) {
    if (lv.row32) return B2D_OK;
    std::unique_ptr<LevelRes::Row32> g(new (std::nothrow) LevelRes::Row32());
    if (!g) return fail(B2D_ERR_NO_MEMORY, "out of host memory");
    const DeviceScene &d = lv.ds;
    CU(allocate(g->texels, (size_t)d.lit_texel_stride + 256));
    g->flats = alloc_aligned_4g(r->device, (size_t)d.lit_flat_stride + 256);
    if (!g->flats) return fail(B2D_ERR_NO_MEMORY, "no 4 GiB aligned device memory for the row-32 flats");
    CU(event_create(g->built));
    const uint8_t *row = d.colormap + 32 * 256;
    CU(launch_prelight_textures_row(row, d.texels, d.tex, d.ntex, g->texels.get(), stream));
    CU(launch_prelight_row(row, d.flats, g->flats.get(), d.lit_flat_stride, stream));
    CU(cudaEventRecord(g->built.get(), stream));
    r->launches += (d.ntex > 0) + (d.lit_flat_stride > 0);
    lv.row32 = std::move(g);
    return B2D_OK;
}

// the state-dependent tables (level time `tics`, sector offsets) as a table set at `out` (SetLayout(blob))
void state_tables(const uint8_t *blob, uint32_t tics, const int32_t *floor_off, const int32_t *ceil_off, uint8_t *out) {
    const SetLayout L(blob);
    scene_at_time(blob, tics, reinterpret_cast<TexRec *>(out), reinterpret_cast<SectorRec *>(out + L.sectors),
                  reinterpret_cast<SegRec *>(out + L.segs), reinterpret_cast<SpriteRec *>(out + L.sprites),
                  reinterpret_cast<MidRec *>(out + L.mids), floor_off, ceil_off);
}

// The compact state of level time `tics` with the level's current sector moves into out[layout.words] (out is not
// lv.state): the moved flag and the offsets, words 1 .. 2 + 2 * ndyn, do not depend on the time.
void state_at(const LevelRes &lv, uint32_t tics, uint32_t *out) {
    compact_state(lv.h_blob.data(), lv.layout, tics, nullptr, nullptr, out);
    std::copy(lv.state.begin() + 1, lv.state.begin() + 2 + 2 * (ptrdiff_t)lv.layout.dyn_sectors.size(), out + 1);
}

// The state automap's changeable lines (C21) of a level: each two-sided line that is neither special 39 nor ML_SECRET and
// has a dynamic sector (layout's slots) on a side gets kAutomapChangeable in its device copy and, in dyn (one record per
// line, left empty when no line changes), its sectors' rest heights and dynamic slots.
void automap_dyn_lines(const Level &lv, const StateLayout &layout, std::vector<AutomapLine> &lines, std::vector<AutomapDynLine> &dyn) {
    auto side_sector = [&](int side) -> int {            // as automap_lines finds a side's sector
        if (side < 0 || (size_t)side >= lv.sidedefs.size()) return -1;
        const int sec = lv.sidedefs[(size_t)side].sector;
        return (size_t)sec < lv.sectors.size() ? sec : -1;
    };
    auto slot = [&](int sec) -> uint32_t {
        const uint32_t d = (size_t)sec < layout.sector_slots.size() ? layout.sector_slots[(size_t)sec] >> 16 : kNoSlot;
        return d == kNoSlot ? kAutomapNoSlot : d;
    };
    for (size_t i = 0; i < lines.size(); i++) {
        const Linedef &l = lv.linedefs[(size_t)lines[i].linedef];
        const int front = side_sector(l.right), back = side_sector(l.left);
        if (front < 0 || back < 0 || l.special == 39 || (l.flags & 0x20)) continue;
        const AutomapDynLine d{{lv.sectors[(size_t)front].floor, lv.sectors[(size_t)back].floor},
                               {lv.sectors[(size_t)front].ceil, lv.sectors[(size_t)back].ceil},
                               {slot(front), slot(back)}};
        if (d.slot[0] == kAutomapNoSlot && d.slot[1] == kAutomapNoSlot) continue;
        dyn.resize(lines.size(), AutomapDynLine{});
        dyn[i] = d;
        lines[i].dev_flags |= kAutomapChangeable;
    }
}

// Per-frame levels (HOST, nullable = level 0): each below the renderer's number of levels; B2D_ERR_INVALID_ARG otherwise.
int check_levels(const b2d_renderer *r, const uint32_t *levels, size_t n) {
    if (levels)
        for (size_t i = 0; i < n; i++)
            if (levels[i] >= r->lv.size()) return fail(B2D_ERR_INVALID_ARG, "frame level out of range (>= the renderer's number of levels)");
    return B2D_OK;
}

// Per-frame palettes (HOST, nullable = palette 0): frame i's palette below the palette count of its level (levels[i],
// nullable = level 0), the levels already checked; B2D_ERR_INVALID_ARG otherwise.
int check_palettes(const b2d_renderer *r, const uint32_t *levels, const uint32_t *palettes, size_t n) {
    if (palettes)
        for (size_t i = 0; i < n; i++)
            if (palettes[i] >= r->pal_count[levels ? levels[i] : 0u])
                return fail(B2D_ERR_INVALID_ARG, "frame palette out of range (>= the palette count of the frame's level)");
    return B2D_OK;
}

}  // namespace

int b2d::CallFrames::prepare(const b2d_renderer *r, size_t n) {
    if (takes & kFrameLevels) {
        if (!levels) return fail(B2D_ERR_INVALID_ARG, "null level array");
        if (r->walk_smem + walk_levels_static_smem() > kWalkSmemMax)
            return fail(B2D_ERR_INVALID_ARG, "level too large for the per-frame-level BSP-walk kernel's shared memory");
        if (int rc = check_levels(r, levels, n)) return rc;
    }
    if (int rc = check_palettes(r, levels, palettes, n)) return rc;
    if (lights) {
        bool any = false;
        for (size_t i = 0; i < n; i++) {
            if (lights[i].fixed_colormap < -1 || lights[i].fixed_colormap > 32)
                return fail(B2D_ERR_INVALID_ARG, "frame fixed colormap out of range (-1 .. 32)");
            if (lights[i].extralight > 2) return fail(B2D_ERR_INVALID_ARG, "frame extra light out of range (0 .. 2)");
            any = any || lights[i].fixed_colormap != -1 || lights[i].extralight != 0;
        }
        if (!any) lights = nullptr;
    }
    frames = Frames{levels, nullptr, nullptr, lights};
    if (!(takes & kFrameStates) && !tics) return B2D_OK;
    if (!tics) {
        if (!states || (n_moves && !moves)) return fail(B2D_ERR_INVALID_ARG, "null argument");
        for (size_t i = 0; i < n; i++)
            if (states[i].first_move > n_moves || states[i].n_moves > n_moves - states[i].first_move)
                return fail(B2D_ERR_INVALID_ARG, "a frame's move range runs past the end of the move list");
    }
    return guarded([&] {
        size_t total = 0;
        starts.assign(n, 0);
        for (size_t i = 0; i < n; i++) {
            const LevelRes &lv = r->lv[levels ? levels[i] : 0];
            if (lv.h_blob.empty()) {
                if (!tics && states[i].n_moves) return fail(B2D_ERR_INVALID_ARG, "the scene declares no dynamic sectors");
                continue;
            }
            starts[i] = total;
            total += lv.layout.words;
        }
        fs.assign(total, 0);
        std::vector<int32_t> fo, co;
        for (size_t i = 0; i < n; i++) {
            const LevelRes &lv = r->lv[levels ? levels[i] : 0];
            if (lv.h_blob.empty()) continue;
            if (tics) {
                state_at(lv, tics[i], fs.data() + starts[i]);
                continue;
            }
            bool moved = false;
            if (states[i].n_moves) {
                if (const char *why = expand_moves(lv.h_blob.data(), reinterpret_cast<const SectorMove *>(moves) + states[i].first_move,
                                                   states[i].n_moves, fo, co))
                    return fail(B2D_ERR_INVALID_ARG, why);
                for (size_t k = 0; k < fo.size() && !moved; k++) moved = fo[k] != 0 || co[k] != 0;    // all zero: at rest
            }
            compact_state(lv.h_blob.data(), lv.layout, states[i].tics, moved ? fo.data() : nullptr, moved ? co.data() : nullptr,
                          fs.data() + starts[i], lights ? lights[i].extralight : 0u);
        }
        frames.fs = fs.data();
        frames.starts = !levels && r->lv[0].h_blob.empty() ? nullptr : starts.data();
        return B2D_OK;
    });
}

int b2d::check_slots_free(const b2d_renderer *r, size_t batches) {
    for (size_t k = 0; k < batches && k < 2; k++)
        if (!r->slot[(r->next_ticket + (int64_t)k) & 1].rastered)
            return fail(B2D_ERR_INVALID_ARG, "a worklist slot this call needs holds a batch that was walked but not rastered yet");
    return B2D_OK;
}

// BSP walk of a batch into the next worklist slot, on `stream`.  The slot's previous raster (if any, on whatever stream) is
// awaited through an event, so a caller may run walks and rasters on two streams and have the walk of batch k+1 overlap the
// raster of batch k.  The batch's table sets are expanded on `stream` first.  With per-frame states: frames whose (level,
// compact state) are equal share a set; sets are numbered in order of first appearance and packed into the slot's arena,
// and one launch expands them all.  Without: the slot's own table set of each timed level the batch
// uses is re-expanded, one launch per level, when the level's state differs from the one the set holds, so the walk and
// the raster of a ticket read one state whatever is set in between.  What the batch stages (StageLayout) goes to the device
// in one copy; a plain batch at an unchanged state stages nothing and does not wait on the host.
int b2d::walk_batch(b2d_renderer *r, const Pose *d_poses, const Frames &fr, int n, cudaStream_t stream, bool background,
                    int64_t *ticket_out) {
    const int slot = (int)(r->next_ticket & 1);
    WorkSlot &s = r->slot[slot];
    if (!s.rastered) return fail(B2D_ERR_INVALID_ARG, "both worklist slots hold batches that were walked but not rastered yet");
    const bool per_frame = fr.starts != nullptr, per_level = fr.levels != nullptr;
    int rc = per_frame ? ensure_states(r) : B2D_OK;
    if (rc == B2D_OK) rc = ensure_slot(r, s);
    if (rc != B2D_OK) return rc;
    const size_t nlev = r->lv.size();
    auto level = [&](int f) { return per_level ? fr.levels[f] : 0u; };
    // fixed colormaps (per-frame levels and states only): the row-32 planes of every level a frame asks for them on,
    // built on this stream the first time, and awaited by this batch's walk (and so by its raster)
    bool fixed_rows = false;
    for (int f = 0; f < n && fr.lights && per_frame && per_level; f++) {
        const int32_t row = fr.lights[f].fixed_colormap;
        fixed_rows = fixed_rows || row >= 0;
        if (row != 32) continue;
        LevelRes &lv = r->lv[level(f)];
        const bool built = lv.row32 != nullptr;
        rc = ensure_row32(r, lv, stream);
        if (rc != B2D_OK) return rc;
        if (built) CU(cudaStreamWaitEvent(stream, lv.row32->built.get(), 0));
    }
    std::vector<Expansion> plan;
    std::vector<uint32_t> frame_set;
    size_t state_words = 0;
    if (per_frame) {
        frame_set.resize((size_t)n);
        std::unordered_map<std::string, uint32_t> seen;
        seen.reserve((size_t)n);
        size_t aoff = 0;
        for (int f = 0; f < n; f++) {
            const uint32_t k = level(f), e = fr.lights ? fr.lights[f].extralight : 0u;
            const LevelRes &lv = r->lv[k];
            if (lv.h_blob.empty() && e == 0) {        // no set: the frame reads its level's blob tables
                frame_set[(size_t)f] = (uint32_t)-1;
                continue;
            }
            // a level without time-dependent content has one state, its rest state
            const uint32_t *w = lv.h_blob.empty() ? lv.state.data() : fr.fs + fr.starts[f];
            std::string key(reinterpret_cast<const char *>(&k), 4);
            key.append(reinterpret_cast<const char *>(&e), 4);
            key.append(reinterpret_cast<const char *>(w), 4 * lv.layout.words);
            auto it = seen.emplace(std::move(key), (uint32_t)plan.size());
            if (it.second) {
                plan.push_back(Expansion{k, w, s.arena.get() + aoff, e});
                aoff += SetLayout(lv.src).slot;
                state_words += lv.layout.words;
            }
            frame_set[(size_t)f] = it.first->second;
        }
    } else {
        for (uint32_t k = 0; k < nlev; k++) {
            LevelRes &lv = r->lv[k];
            if (lv.slot[slot].tables && lv.slot[slot].state != lv.state &&
                (per_level ? std::find(fr.levels, fr.levels + n, k) != fr.levels + n : k == 0)) {
                plan.push_back(Expansion{k, lv.state.data(), lv.slot[slot].tables.get(), 0});
                state_words += lv.layout.words;
            }
        }
    }
    const size_t nsets = plan.size();
    const StageLayout L(nlev, nsets, (size_t)n, state_words, per_frame, per_level, fixed_rows);
    const bool stage = per_level || nsets > 0;
    size_t records = 0;
    if (stage) {
        CU(cudaEventSynchronize(s.staged.get()));     // the copy issued two batches ago has read the staging
        uint8_t *h = s.h_stage.get();
        StateSrc *srcs = reinterpret_cast<StateSrc *>(h + L.srcs);
        TableSet *sets = reinterpret_cast<TableSet *>(h + L.sets);
        StateSet *descs = reinterpret_cast<StateSet *>(h + L.descs);
        uint32_t *words = reinterpret_cast<uint32_t *>(h + L.states);
        for (size_t k = 0; k < nlev; k++) {
            const LevelRes &lv = r->lv[k];
            if (per_level) reinterpret_cast<DeviceScene *>(h + L.scenes)[k] = per_frame ? lv.ds : slot_scene(lv, slot);
            srcs[k] = lv.src;
            if (per_frame) sets[nsets + k] = TableSet{lv.ds.tex, lv.ds.sectors, lv.ds.segs, lv.ds.sprites, lv.ds.mids};
        }
        size_t woff = 0;
        for (size_t k = 0; k < nsets; k++) {
            const LevelRes &lv = r->lv[plan[k].level];
            sets[k] = SetLayout(lv.src).at(plan[k].tables);
            // one launch numbers the records of all per-frame sets; a launch of its own per stale set starts at 0
            descs[k] = StateSet{plan[k].level, (uint32_t)woff, per_frame ? (uint32_t)records : 0u, plan[k].extralight};
            std::memcpy(words + woff, plan[k].state, 4 * lv.layout.words);
            woff += lv.layout.words;
            records += set_records(lv);
        }
        if (records > 0x7FFFFFFFu) return fail(B2D_ERR_INVALID_ARG, "the batch's table sets hold more than 2^31 records");
        for (int f = 0; f < n && per_level; f++) reinterpret_cast<uint32_t *>(h + L.frame_level)[f] = fr.levels[f];
        for (int f = 0; f < n && per_frame; f++)
            reinterpret_cast<uint32_t *>(h + L.frame_set)[f] =
                frame_set[(size_t)f] == (uint32_t)-1 ? (uint32_t)(nsets + level(f)) : frame_set[(size_t)f];
        for (int f = 0; f < n && fixed_rows; f++) reinterpret_cast<int32_t *>(h + L.frame_fixed)[f] = fr.lights[f].fixed_colormap;
        for (size_t k = 0; k < nlev && fixed_rows; k++) {
            const LevelRes &lv = r->lv[k];
            reinterpret_cast<FixedPlanes *>(h + L.planes)[k] =
                lv.row32 ? FixedPlanes{lv.row32->texels.get(), lv.row32->flats.get()} : FixedPlanes{nullptr, nullptr};
        }
    }
    CU(cudaStreamWaitEvent(stream, s.raster_done.get(), 0));      // the raster that last read this slot
    const uint8_t *d = s.stage.get();
    if (stage) {
        CU(cudaMemcpyAsync(s.stage.get(), s.h_stage.get(), L.end, cudaMemcpyHostToDevice, stream));
        CU(cudaEventRecord(s.staged.get(), stream));
    }
    const StateSrc *d_srcs = reinterpret_cast<const StateSrc *>(d + L.srcs);
    const TableSet *d_sets = reinterpret_cast<const TableSet *>(d + L.sets);
    const StateSet *d_descs = reinterpret_cast<const StateSet *>(d + L.descs);
    const uint32_t *d_words = reinterpret_cast<const uint32_t *>(d + L.states);
    if (per_frame && nsets) {
        CU(launch_state_sets(d_srcs, d_descs, d_sets, d_words, (int)nsets, (uint32_t)records, stream));
        r->launches += 1;
    }
    for (size_t k = 0; k < nsets && !per_frame; k++) {
        LevelRes &lv = r->lv[plan[k].level];
        CU(launch_state_sets(d_srcs, d_descs + k, d_sets + k, d_words, 1, (uint32_t)set_records(lv), stream));
        r->launches += 1;
        lv.slot[slot].state = lv.state;
    }
    BatchTables t{};
    t.per_frame = per_frame;
    t.per_level = per_level;
    t.fixed_rows = fixed_rows;
    if (fixed_rows)
        t.fixed = FixedTables{reinterpret_cast<const int32_t *>(d + L.frame_fixed), reinterpret_cast<const FixedPlanes *>(d + L.planes)};
    if (!per_level) t.scene = slot_scene(r->lv[0], slot);
    t.levels = LevelTables{per_level ? reinterpret_cast<const DeviceScene *>(d + L.scenes) : nullptr,
                           per_level ? reinterpret_cast<const uint32_t *>(d + L.frame_level) : nullptr,
                           per_frame ? d_sets : nullptr, per_frame ? reinterpret_cast<const uint32_t *>(d + L.frame_set) : nullptr};
    rc = profiled(r, stream, 0, [&] {
        return launch_walk(t, r->walk_smem, r->view, d_poses, n, s.frames.get(), s.work.get(), r->stride, stream, background);
    });
    if (rc != B2D_OK) return rc;
    CU(cudaEventRecord(s.walk_done.get(), stream));
    s.n = n;
    s.tables = t;
    s.sets = per_frame ? (int)nsets : 0;
    s.set_level.resize(s.sets);
    s.set_off.resize(s.sets);
    for (int k = 0; k < s.sets; k++) {
        s.set_level[k] = plan[k].level;
        s.set_off[k] = (size_t)(plan[k].tables - s.arena.get());
    }
    s.ticket = r->next_ticket;
    s.rastered = false;
    r->last_slot = slot;
    r->launches += 1;
    *ticket_out = r->next_ticket++;
    return B2D_OK;
}

// Creates the table group `g` whole (or not at all): `bytes` of device memory and of pinned memory, whose image
// lay_out(h, d) writes (d: the device copy, which pointers in the image point into), uploaded on `st`; `built` follows the
// upload.  `off`: where the image's per-level records start.
template <typename LayOut>
static int build_tables(std::unique_ptr<b2d_renderer::Tables> &g, size_t bytes, size_t off, cudaStream_t st, LayOut lay_out) {
    auto a = std::make_unique<b2d_renderer::Tables>();
    CU(allocate(a->d, bytes));
    CU(allocate(a->h, bytes));
    CU(event_create(a->built));
    lay_out(a->h.get(), a->d.get());
    a->off = off;
    CU(cudaMemcpyAsync(a->d.get(), a->h.get(), bytes, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(a->built.get(), st));
    g = std::move(a);
    return B2D_OK;
}

// The table group `g` of r for work enqueued on `st`: a wait for the first call's upload, or, at the first call,
// build(r, st), which creates it with its upload on `st`.
static int tables_on(b2d_renderer *r, const std::unique_ptr<b2d_renderer::Tables> &g, cudaStream_t st,
                     int (*build)(b2d_renderer *, cudaStream_t)) {
    if (!g) return guarded([&] { return build(r, st); });
    CU(cudaStreamWaitEvent(st, g->built.get(), 0));
    return B2D_OK;
}

// The seg -> linedef tables of every level (b2d_renderer::seen): the tables one after the other, then each level's
// offset into them.
static int ensure_seen(b2d_renderer *r, cudaStream_t st) {
    std::vector<int32_t> words;
    std::vector<uint32_t> off;
    for (const LevelRes &lv : r->lv) {
        off.push_back((uint32_t)words.size());
        words.insert(words.end(), lv.seg_line.begin(), lv.seg_line.end());
    }
    const size_t tables = words.size() * sizeof(int32_t);
    for (uint32_t o : off) words.push_back((int32_t)o);
    const size_t bytes = words.size() * sizeof(int32_t);
    return build_tables(r->seen, bytes, tables, st, [&](uint8_t *h, const uint8_t *) { std::memcpy(h, words.data(), bytes); });
}

int b2d::raster_batch(b2d_renderer *r, int64_t ticket, uint8_t *d_index, uint32_t *d_rgba, cudaStream_t stream,
                      uint32_t *d_seen) {
    const int slot = (int)(ticket & 1);
    WorkSlot &s = r->slot[slot];
    if (ticket < 0 || s.ticket != ticket || s.rastered) return fail(B2D_ERR_INVALID_ARG, "unknown or already rastered walk ticket");
    SeenTables seen{};
    if (d_seen) {
        if (int rc = tables_on(r, r->seen, stream, ensure_seen)) return rc;
        const uint8_t *d = r->seen->d.get();
        seen = SeenTables{d_seen, reinterpret_cast<const int32_t *>(d), reinterpret_cast<const uint32_t *>(d + r->seen->off),
                          r->seen_words};
    }
    CU(cudaStreamWaitEvent(stream, s.walk_done.get(), 0));
    if (r->d_masked) {
        // one arena of deferred masked entries per renderer: rasters that use it run one after the other (each fills the
        // machine on its own, so nothing is lost), whatever streams they were enqueued on
        CU(cudaStreamWaitEvent(stream, r->masked_done.get(), 0));
        CU(cudaMemsetAsync(r->d_masked_counter.get(), 0, sizeof(uint32_t), stream));
    }
    // masked content in a level the frames read: with per-frame levels, any level's
    const bool masked = r->d_masked && (s.tables.per_level || s.tables.scene.masked_list);
    const int rc = profiled(r, stream, 1, [&] {
        return launch_raster(s.tables, masked, r->view, s.frames.get(), s.work.get(), r->stride, s.n, d_index, d_rgba,
                             d_seen ? &seen : nullptr, stream);
    });
    if (rc != B2D_OK) return rc;
    CU(cudaEventRecord(s.raster_done.get(), stream));
    if (r->d_masked) CU(cudaEventRecord(r->masked_done.get(), stream));
    s.rastered = true;
    r->launches += 1;
    return B2D_OK;
}

// batches of at most max_batch frames in n frames
static size_t batch_count(const b2d_renderer *r, size_t n) { return (n + (size_t)r->max_batch - 1) / (size_t)r->max_batch; }

// walk -> raster of one batch on `stream`
static int enqueue_frames(b2d_renderer *r, const Pose *d_poses, const Frames &fr, int n, uint8_t *d_index, uint32_t *d_rgba,
                          cudaStream_t stream) {
    int64_t ticket = -1;
    int rc = walk_batch(r, d_poses, fr, n, stream, false, &ticket);
    if (rc != B2D_OK) return rc;
    return raster_batch(r, ticket, d_index, d_rgba, stream);
}

// The n words word(i) of a call staged in `s` on `st` (stage_tables: the colour-table indices of its frames, frame_table
// of its checked levels and palettes; b2d_automap_device: its levels): into staging grown to hold them (created whole, or
// not at all; the old buffers go once the last call's kernel has read them), or into the present staging once the
// previous call's copy has read it and, on `st`, its kernel the device copy.  The caller records s.done after its kernel.
template <typename Word>
static int stage_words(LevelStaging &s, size_t n, cudaStream_t st, Word word) {
    if (s.cap < n) {
        LevelStaging g;
        g.cap = s.cap ? s.cap : 1024;
        while (g.cap < n) g.cap *= 2;
        CU(allocate(g.d, g.cap * sizeof(uint32_t)));
        CU(allocate(g.h, g.cap * sizeof(uint32_t)));
        CU(event_create(g.copied));
        CU(event_create(g.done));
        if (s.done) CU(cudaEventSynchronize(s.done.get()));
        s = std::move(g);
    } else {
        CU(cudaEventSynchronize(s.copied.get()));     // the previous call's copy has read the staging
        CU(cudaStreamWaitEvent(st, s.done.get(), 0));        // ... and its kernel the device copy
    }
    for (size_t i = 0; i < n; i++) s.h.get()[i] = word(i);
    CU(cudaMemcpyAsync(s.d.get(), s.h.get(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(s.copied.get(), st));
    return B2D_OK;
}

static int stage_tables(const b2d_renderer *r, LevelStaging &s, const uint32_t *levels, const uint32_t *palettes, size_t n,
                        cudaStream_t st) {
    return stage_words(s, n, st, [&](size_t i) { return frame_table(r, levels, palettes, i); });
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

// The automap digit names AMMNUM0 .. AMMNUM9 (C22)
Name digit_name(int d) {
    char name[8] = {'A', 'M', 'M', 'N', 'U', 'M', (char)('0' + d), 0};
    return make_name(reinterpret_cast<const uint8_t *>(name), 8);
}

// An archive scene's grid origin and digits (C22): the origin from the header of the lump at marker + 10 (ML_BLOCKMAP)
// when it is named BLOCKMAP and holds at least 8 bytes inside the file, else (0, 0); each digit the picture of its lump
// name (a later lump wins), offsets included, or missing when absent, outside the file or undecodable.  Neither fails
// the scene: the level renders without them.
void archive_marks(const Archive &wad, int level_index, b2d_scene *s) {
    const int bm = wad.level_lump_index(level_index) + 10;
    if ((size_t)bm < wad.num_lumps() && wad.lump(bm).name == make_name("BLOCKMAP") && wad.lump(bm).size >= 8) {
        try {
            const uint8_t *p = wad.lump_data(bm);
            s->grid_origin[0] = (int16_t)(p[0] | p[1] << 8);
            s->grid_origin[1] = (int16_t)(p[2] | p[3] << 8);
        } catch (const WadError &) {
        }
    }
    for (int d = 0; d < kAutomapDigits; d++) {
        const int i = wad.find(digit_name(d));
        if (i < 0 || wad.lump(i).size <= 0) continue;
        try {
            s->digits[(size_t)d] = Image::decode(wad.lump_data(i), (size_t)wad.lump(i).size);
        } catch (const WadError &) {
            s->digits[(size_t)d] = Image{};
        }
    }
}
}  // namespace

int b2d_scene_create_dynamic(const b2d_archive *a, int level_index, const b2d_dynamic_sector *dyn, size_t n_dyn, b2d_scene **out) {
    if (!a || !out || (n_dyn && !dyn)) return fail(B2D_ERR_INVALID_ARG, "null argument");
    return guarded([&] {
        auto s = std::make_unique<b2d_scene>();
        TextureDirectory td = TextureDirectory::load(*a->wad);
        s->level = Level::load(*a->wad, level_index);
        s->blob = compile_scene(s->level, td, dyn_list(dyn, n_dyn));
        s->automap = automap_lines(s->level);
        archive_marks(*a->wad, level_index, s.get());
        fill_scene_info(s.get());
        s->palettes = td.palettes;
        if (s->palettes.empty()) s->palettes.push_back({});
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
    const size_t need = SetLayout(s->blob.data()).bytes;
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
        s->automap = automap_lines(s->level);
        for (int d = 0; d < kAutomapDigits; d++)      // the digits among the caller's images, at offsets 0 (C22)
            if (const Image *im = td.texture(digit_name(d))) s->digits[(size_t)d] = *im;
        fill_scene_info(s.get());
        s->palettes.assign(1, td.palettes.empty() ? std::array<uint8_t, 768>{} : td.palettes[0]);
        *out = s.release();
        return B2D_OK;
    });
}

int b2d_scene_num_palettes(const b2d_scene *s) {
    if (!s) return fail(B2D_ERR_INVALID_ARG, "null scene");
    return (int)s->palettes.size();
}

int b2d_scene_set_palettes(b2d_scene *s, const uint8_t *playpal, size_t n_palettes) {
    if (!s || !playpal || n_palettes == 0) return fail(B2D_ERR_INVALID_ARG, "null argument or no palettes");
    if (n_palettes > (size_t)INT32_MAX / 768) return fail(B2D_ERR_INVALID_ARG, "too many palettes");
    if (std::memcmp(playpal, s->palettes[0].data(), 768) != 0)
        return fail(B2D_ERR_INVALID_ARG, "palette 0 differs from the palette the scene was made with");
    return guarded([&] {
        std::vector<std::array<uint8_t, 768>> p(n_palettes);
        for (size_t i = 0; i < n_palettes; i++) std::memcpy(p[i].data(), playpal + 768 * i, 768);
        s->palettes = std::move(p);
        return B2D_OK;
    });
}

static_assert(sizeof(b2d_automap_line) == sizeof(AutomapLine) && offsetof(b2d_automap_line, colour) == offsetof(AutomapLine, colour) &&
                  offsetof(b2d_automap_line, linedef) == offsetof(AutomapLine, linedef), "b2d_automap_line");
static_assert(B2D_AUTOMAP_ROTATE == kAutomapRotate && B2D_AUTOMAP_ALL_LINES == kAutomapAllLines && B2D_AUTOMAP_THINGS == kAutomapThings &&
                  B2D_AUTOMAP_ALLMAP == kAutomapAllmap,
              "automap flags");

int b2d_scene_automap_lines(const b2d_scene *s, b2d_automap_line *out, size_t capacity, size_t *n_out) {
    if (!s || !n_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    *n_out = s->automap.size();
    if (!out) return B2D_OK;
    if (capacity < s->automap.size()) return fail(B2D_ERR_INVALID_ARG, "buffer too small for the automap lines");
    if (!s->automap.empty()) std::memcpy(out, s->automap.data(), s->automap.size() * sizeof(AutomapLine));
    return B2D_OK;
}

int b2d_scene_automap_grid_origin(const b2d_scene *s, int32_t *x_out, int32_t *y_out) {
    if (!s || !x_out || !y_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    *x_out = s->grid_origin[0];
    *y_out = s->grid_origin[1];
    return B2D_OK;
}

int b2d_scene_set_automap_grid_origin(b2d_scene *s, int32_t x, int32_t y) {
    if (!s) return fail(B2D_ERR_INVALID_ARG, "null scene");
    s->grid_origin[0] = x;
    s->grid_origin[1] = y;
    return B2D_OK;
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
    {   // the state rule's inputs, on every level (a frame with extra light reads a table set on any level): the blob's
        // rest-state sections, the two slot maps and the light side tables
        const uint8_t *blob = s->blob.data();
        try {
            lv.layout = state_layout(blob);
        } catch (const std::exception &ex) {
            return fail(B2D_ERR_INVALID_ARG, ex.what());
        }
        const StateLayout &L = lv.layout;
        std::vector<int16_t> steps;
        std::vector<int8_t> contrast;
        light_steps(blob, steps, contrast);
        const size_t maps = L.sector_slots.size() + L.mid_seg.size();         // words
        CU(allocate(lv.d_slot_maps, 4 * maps + 2 * steps.size() + contrast.size() + 4));
        uint8_t *dm = reinterpret_cast<uint8_t *>(lv.d_slot_maps.get());
        CU(cudaMemcpy(dm, L.sector_slots.data(), 4 * L.sector_slots.size(), cudaMemcpyHostToDevice));
        CU(cudaMemcpy(dm + 4 * L.sector_slots.size(), L.mid_seg.data(), 4 * L.mid_seg.size(), cudaMemcpyHostToDevice));
        CU(cudaMemcpy(dm + 4 * maps, steps.data(), 2 * steps.size(), cudaMemcpyHostToDevice));
        CU(cudaMemcpy(dm + 4 * maps + 2 * steps.size(), contrast.data(), contrast.size(), cudaMemcpyHostToDevice));
        StateSrc &src = lv.src = state_src(blob, L);
        auto on_device = [&](auto p) { return reinterpret_cast<decltype(p)>(db + (reinterpret_cast<const uint8_t *>(p) - blob)); };
        src.tex = on_device(src.tex); src.sectors = on_device(src.sectors); src.segs = on_device(src.segs);
        src.sprites = on_device(src.sprites); src.mids = on_device(src.mids); src.anim = on_device(src.anim);
        src.flat_anim = on_device(src.flat_anim); src.segdyn = on_device(src.segdyn);
        src.sector_slots = lv.d_slot_maps.get();
        src.mid_seg = reinterpret_cast<const int32_t *>(lv.d_slot_maps.get() + L.sector_slots.size());
        src.sector_steps = reinterpret_cast<const int16_t *>(dm + 4 * maps);
        src.seg_contrast = reinterpret_cast<const int8_t *>(dm + 4 * maps + 2 * steps.size());
        // tic 0 is a time like any other: a frame name with k > 0 shows its group's frame 0 (tex.rs:260, 302-306)
        lv.state.assign(L.words, 0);
        compact_state(blob, L, 0, nullptr, nullptr, lv.state.data());
    }
    if (scene_is_timed(s->blob.data())) {
        lv.h_blob = s->blob;
        const uint8_t *blob = lv.h_blob.data();
        const size_t words = lv.layout.words;
        const SetLayout t(lv.src);
        for (auto &sl : lv.slot) CU(allocate(sl.tables, t.slot));
        // The pre-lit planes above were built from the blob's own (per-image) records; both slots' table sets start at tic
        // 0, expanded by one launch.
        const StageLayout S(1, 2, 0, words, false, false);
        const uint32_t records = (uint32_t)set_records(lv);
        std::vector<uint8_t> stage(S.end);
        *reinterpret_cast<StateSrc *>(stage.data() + S.srcs) = lv.src;
        for (uint32_t k = 0; k < 2; k++) {
            reinterpret_cast<TableSet *>(stage.data() + S.sets)[k] = t.at(lv.slot[k].tables.get());
            reinterpret_cast<StateSet *>(stage.data() + S.descs)[k] = StateSet{0, 0, k * records, 0};
            lv.slot[k].state = lv.state;
        }
        std::memcpy(stage.data() + S.states, lv.state.data(), 4 * words);
        DeviceBuf<uint8_t> d;
        CU(allocate(d, S.end));
        CU(cudaMemcpy(d.get(), stage.data(), S.end, cudaMemcpyHostToDevice));
        CU(launch_state_sets(reinterpret_cast<const StateSrc *>(d.get() + S.srcs), reinterpret_cast<const StateSet *>(d.get() + S.descs),
                             reinterpret_cast<const TableSet *>(d.get() + S.sets), reinterpret_cast<const uint32_t *>(d.get() + S.states),
                             2, 2 * records, nullptr));
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
    size_t words = 0;
    for (LevelRes &lv : r->lv) {
        DeviceScene &d = lv.ds;
        d.yslope = r->d_yslope.get();
        d.status_flag = r->d_status.get();
        if (d.masked_cap > 0) {
            d.masked_list = r->d_masked.get();
            d.masked_counter = r->d_masked_counter.get();
            d.masked_chunks = masked_chunks;
        }
        words = std::max(words, (size_t)lv.layout.words);
    }
    // the automap's items of every level (host copies; the device tables come with the first automap call)
    rc = guarded([&] {
        for (size_t k = 0; k < n_levels; k++) {
            const uint32_t *h = reinterpret_cast<const uint32_t *>(scenes[k]->blob.data());
            const SpriteRec *sp = reinterpret_cast<const SpriteRec *>(scenes[k]->blob.data() + h[H_OFF_SPRITES]);
            r->lv[k].automap_lines = scenes[k]->automap;
            for (AutomapLine &l : r->lv[k].automap_lines)      // the device copy's don't-draw bit (the seen automap's ALLMAP rule)
                if (scenes[k]->level.linedefs[(size_t)l.linedef].flags & 0x80) l.dev_flags = kAutomapDontDraw;
            automap_dyn_lines(scenes[k]->level, r->lv[k].layout, r->lv[k].automap_lines, r->lv[k].automap_dyn);
            r->lv[k].grid_origin[0] = scenes[k]->grid_origin[0];
            r->lv[k].grid_origin[1] = scenes[k]->grid_origin[1];
            r->lv[k].digits = scenes[k]->digits;
            for (uint32_t i = 0; i < h[H_NSPRITES]; i++) {
                r->lv[k].automap_things.push_back(sp[i].x);
                r->lv[k].automap_things.push_back(sp[i].y);
            }
            // seen lines (C20): compiled segs are 1:1 with the SEGS lump
            const Level &lvl = scenes[k]->level;
            for (const Seg &sg : lvl.segs) r->lv[k].seg_line.push_back(sg.linedef < lvl.linedefs.size() ? (int32_t)sg.linedef : -1);
            r->seen_words = std::max(r->seen_words, (uint32_t)((lvl.linedefs.size() + 31) / 32));
        }
        return B2D_OK;
    });
    if (rc != B2D_OK) return rc;
    // every palette of every level in one colour table (K3-levels, K4), copied from the scenes now: 14 KB per PLAYPAL
    std::vector<uint32_t> table;
    for (size_t k = 0; k < n_levels; k++) {
        r->pal_base.push_back((uint32_t)(table.size() / 256));
        r->pal_count.push_back((uint32_t)scenes[k]->palettes.size());
        for (const auto &p : scenes[k]->palettes)
            for (int i = 0; i < 256; i++) table.push_back(palette_word(&p[(size_t)i * 3]));
    }
    CU(allocate(r->d_palettes, table.size() * sizeof(uint32_t)));
    CU(cudaMemcpy(r->d_palettes.get(), table.data(), table.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    // each worklist slot's staging, for the largest batch: max_batch frames with a table set each, or a stale set per level
    const size_t sets = std::max((size_t)max_batch, r->lv.size());
    const size_t stage_bytes = StageLayout(r->lv.size(), sets, (size_t)max_batch, sets * words, true, true, true).end;
    for (WorkSlot &sl : r->slot) {
        CU(allocate(sl.stage, stage_bytes));
        CU(allocate(sl.h_stage, stage_bytes));
        CU(event_create(sl.staged));
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
    return enqueue_frames(r, reinterpret_cast<const Pose *>(d_poses), Frames{}, (int)n, d_index_fb, d_rgba_fb,
                          static_cast<cudaStream_t>(cuda_stream));
}

// b2d_render_device_*: the null checks, then walk + raster of the n frames `c` describes (device poses), prepared, in
// batches of max_batch on `cuda_stream`
static int enqueue_batches(b2d_renderer *r, const b2d_pose *d_poses, CallFrames c, size_t n, uint8_t *d_index_fb,
                           uint32_t *d_rgba_fb, void *cuda_stream) {
    if (!r || !d_poses || !d_index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    int rc = c.prepare(r, n);
    if (rc != B2D_OK || n == 0) return rc;
    CU(cudaSetDevice(r->device));
    rc = check_slots_free(r, batch_count(r, n));
    if (rc != B2D_OK) return rc;
    const size_t npix = (size_t)r->view.W * r->view.H;
    for (size_t i = 0; i < n; i += (size_t)r->max_batch) {
        const size_t cnt = n - i < (size_t)r->max_batch ? n - i : (size_t)r->max_batch;
        rc = enqueue_frames(r, reinterpret_cast<const Pose *>(d_poses) + i, c.frames.from(i), (int)cnt, d_index_fb + i * npix,
                            d_rgba_fb ? d_rgba_fb + i * npix : nullptr, static_cast<cudaStream_t>(cuda_stream));
        if (rc != B2D_OK) return rc;
    }
    return B2D_OK;
}

// b2d_walk_device*: the null checks and 1 <= n <= max_batch, then the walk of the n frames `c` describes (device poses),
// prepared, as one batch in a background grid on `cuda_stream`
static int walk_device(b2d_renderer *r, const b2d_pose *d_poses, CallFrames c, size_t n, void *cuda_stream, int64_t *ticket_out) {
    if (!r || !d_poses || !ticket_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (n == 0 || n > (size_t)r->max_batch) return fail(B2D_ERR_INVALID_ARG, "n must be in 1..max_batch");
    if (int rc = c.prepare(r, n)) return rc;
    CU(cudaSetDevice(r->device));
    return walk_batch(r, reinterpret_cast<const Pose *>(d_poses), c.frames, (int)n, static_cast<cudaStream_t>(cuda_stream), true,
                      ticket_out);
}

int b2d_render_device_timed(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *tics, size_t n, uint8_t *d_index_fb,
                            uint32_t *d_rgba_fb, void *cuda_stream) {
    if (!r || !d_poses || !d_index_fb || !tics) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (n == 0) return B2D_OK;
    int rc = check_slots_free(r, batch_count(r, n));                       // refused before the states are built
    if (rc == B2D_OK) rc = enqueue_batches(r, d_poses, CallFrames(tics), n, d_index_fb, d_rgba_fb, cuda_stream);
    if (rc != B2D_OK) return rc;
    return b2d_renderer_set_time(r, tics[n - 1]);                          // the renderer is left at the last pose's time
}

int b2d_render_device_states(b2d_renderer *r, const b2d_pose *d_poses, const b2d_frame_state *states, size_t n,
                             const b2d_sector_move *moves, size_t n_moves, uint8_t *d_index_fb, uint32_t *d_rgba_fb,
                             void *cuda_stream) {
    return enqueue_batches(r, d_poses, CallFrames(kFrameStates, nullptr, states, moves, n_moves), n, d_index_fb, d_rgba_fb,
                           cuda_stream);
}

int b2d_walk_device_states(b2d_renderer *r, const b2d_pose *d_poses, const b2d_frame_state *states, size_t n,
                           const b2d_sector_move *moves, size_t n_moves, void *cuda_stream, int64_t *ticket_out) {
    return walk_device(r, d_poses, CallFrames(kFrameStates, nullptr, states, moves, n_moves), n, cuda_stream, ticket_out);
}

int b2d_walk_device(b2d_renderer *r, const b2d_pose *d_poses, size_t n, void *cuda_stream, int64_t *ticket_out) {
    return walk_device(r, d_poses, CallFrames(), n, cuda_stream, ticket_out);
}

int b2d_raster_device(b2d_renderer *r, int64_t ticket, uint8_t *d_index_fb, uint32_t *d_rgba_fb, void *cuda_stream) {
    if (!r || !d_index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    CU(cudaSetDevice(r->device));
    return raster_batch(r, ticket, d_index_fb, d_rgba_fb, static_cast<cudaStream_t>(cuda_stream));
}

int b2d_render_device_levels(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, size_t n, uint8_t *d_index_fb,
                             uint32_t *d_rgba_fb, void *cuda_stream) {
    return enqueue_batches(r, d_poses, CallFrames(kFrameLevels, levels), n, d_index_fb, d_rgba_fb, cuda_stream);
}

int b2d_walk_device_levels(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, size_t n, void *cuda_stream,
                           int64_t *ticket_out) {
    return walk_device(r, d_poses, CallFrames(kFrameLevels, levels), n, cuda_stream, ticket_out);
}

int b2d_render_device_levels_states(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, const b2d_frame_state *states,
                                    size_t n, const b2d_sector_move *moves, size_t n_moves, uint8_t *d_index_fb,
                                    uint32_t *d_rgba_fb, void *cuda_stream) {
    return enqueue_batches(r, d_poses, CallFrames(kFrameLevels | kFrameStates, levels, states, moves, n_moves), n, d_index_fb,
                           d_rgba_fb, cuda_stream);
}

int b2d_walk_device_levels_states(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, const b2d_frame_state *states,
                                  size_t n, const b2d_sector_move *moves, size_t n_moves, void *cuda_stream, int64_t *ticket_out) {
    return walk_device(r, d_poses, CallFrames(kFrameLevels | kFrameStates, levels, states, moves, n_moves), n, cuda_stream,
                       ticket_out);
}

int b2d_render_device_levels_states_lights(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels,
                                           const b2d_frame_state *states, const b2d_frame_light *lights, size_t n,
                                           const b2d_sector_move *moves, size_t n_moves, uint8_t *d_index_fb,
                                           uint32_t *d_rgba_fb, void *cuda_stream) {
    return enqueue_batches(r, d_poses, CallFrames(kFrameLevels | kFrameStates, levels, states, moves, n_moves, lights), n,
                           d_index_fb, d_rgba_fb, cuda_stream);
}

int b2d_walk_device_levels_states_lights(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels,
                                         const b2d_frame_state *states, const b2d_frame_light *lights, size_t n,
                                         const b2d_sector_move *moves, size_t n_moves, void *cuda_stream,
                                         int64_t *ticket_out) {
    return walk_device(r, d_poses, CallFrames(kFrameLevels | kFrameStates, levels, states, moves, n_moves, lights), n, cuda_stream,
                       ticket_out);
}

// b2d_render*: the null checks, then host poses in, host frames out: the n frames `c` describes, prepared, in batches of
// max_batch.
static int render_host(b2d_renderer *r, const b2d_pose *poses, CallFrames c, size_t n, uint8_t *index_fb, uint32_t *rgba_fb) {
    if (!r || !poses || !index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (int rc = c.prepare(r, n)) return rc;
    if (n == 0) return B2D_OK;
    if (check_slots_free(r, batch_count(r, n)) != B2D_OK) return B2D_ERR_INVALID_ARG;
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
        int rc = enqueue_frames(r, r->d_poses.get(), c.frames.from(done), cnt, hs.index[buf].get(), rgba_fb ? hs.rgba[buf].get() : nullptr, rs);
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
    return render_host(r, poses, CallFrames(), n, index_fb, rgba_fb);
}

int b2d_render_timed(b2d_renderer *r, const b2d_pose *poses, const uint32_t *tics, size_t n, uint8_t *index_fb, uint32_t *rgba_fb) {
    if (!tics) return b2d_render(r, poses, n, index_fb, rgba_fb);
    if (!r || !poses || !index_fb) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (n == 0) return B2D_OK;
    int rc = check_slots_free(r, batch_count(r, n));          // refused before the states are built and the time changes
    if (rc != B2D_OK) return rc;
    rc = render_host(r, poses, CallFrames(tics), n, index_fb, rgba_fb);
    const int trc = b2d_renderer_set_time(r, tics[n - 1]);                // the renderer is left at the last pose's time
    return rc != B2D_OK ? rc : trc;
}

int b2d_render_states(b2d_renderer *r, const b2d_pose *poses, const b2d_frame_state *states, size_t n,
                      const b2d_sector_move *moves, size_t n_moves, uint8_t *index_fb, uint32_t *rgba_fb) {
    return render_host(r, poses, CallFrames(kFrameStates, nullptr, states, moves, n_moves), n, index_fb, rgba_fb);
}

int b2d_render_levels(b2d_renderer *r, const b2d_pose *poses, const uint32_t *levels, size_t n, uint8_t *index_fb,
                      uint32_t *rgba_fb) {
    return render_host(r, poses, CallFrames(kFrameLevels, levels), n, index_fb, rgba_fb);
}

int b2d_render_levels_states(b2d_renderer *r, const b2d_pose *poses, const uint32_t *levels, const b2d_frame_state *states, size_t n,
                             const b2d_sector_move *moves, size_t n_moves, uint8_t *index_fb, uint32_t *rgba_fb) {
    return render_host(r, poses, CallFrames(kFrameLevels | kFrameStates, levels, states, moves, n_moves), n, index_fb, rgba_fb);
}

int b2d_render_levels_states_lights(b2d_renderer *r, const b2d_pose *poses, const uint32_t *levels,
                                    const b2d_frame_state *states, const b2d_frame_light *lights, size_t n,
                                    const b2d_sector_move *moves, size_t n_moves, uint8_t *index_fb, uint32_t *rgba_fb) {
    return render_host(r, poses, CallFrames(kFrameLevels | kFrameStates, levels, states, moves, n_moves, lights), n, index_fb,
                       rgba_fb);
}

int b2d_palette_lut_device(b2d_renderer *r, const uint8_t *d_index, uint32_t *d_rgba, size_t n_pixels, void *cuda_stream) {
    if (!r || !d_index || !d_rgba) return fail(B2D_ERR_INVALID_ARG, "null argument");
    CU(cudaSetDevice(r->device));
    CU(launch_palette(r->lv[0].ds.palette, d_index, d_rgba, n_pixels, static_cast<cudaStream_t>(cuda_stream)));
    r->launches += 1;
    return B2D_OK;
}

int b2d_palette_lut_levels_device(b2d_renderer *r, const uint8_t *d_index, const uint32_t *levels, size_t n_frames, uint32_t *d_rgba,
                                  void *cuda_stream) {
    if (!r || !d_index || !levels || !d_rgba) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (int rc = check_levels(r, levels, n_frames)) return rc;
    if (n_frames == 0) return B2D_OK;
    CU(cudaSetDevice(r->device));
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    if (int rc = stage_tables(r, r->lut_levels, levels, nullptr, n_frames, st)) return rc;
    CU(launch_palette_levels(r->d_palettes.get(), r->lut_levels.d.get(), d_index, d_rgba, n_frames, (size_t)r->view.W * r->view.H, st));
    CU(cudaEventRecord(r->lut_levels.done.get(), st));
    r->launches += 1;
    return B2D_OK;
}

// the resolve's arguments against the renderer's view: B2D_OK or B2D_ERR_INVALID_ARG with the message set
static int check_resolve(const b2d_renderer *r, int factor, int format) {
    if (factor < 1 || factor > 8 || r->view.W % factor || r->view.H % factor)
        return fail(B2D_ERR_INVALID_ARG, "resolve factor must be in 1..8 and divide the view's width and height");
    if (format < B2D_RESOLVE_RGBA8 || format > B2D_RESOLVE_GRAY8) return fail(B2D_ERR_INVALID_ARG, "unknown resolve format");
    return B2D_OK;
}

int b2d_resolve_frame_bytes(const b2d_renderer *r, int factor, int format, size_t *bytes_out) {
    if (!r || !bytes_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (int rc = check_resolve(r, factor, format)) return rc;
    const size_t bpp = format == B2D_RESOLVE_RGBA8 ? 4 : format == B2D_RESOLVE_GRAY8 ? 1 : 3;
    *bytes_out = (size_t)(r->view.W / factor) * (size_t)(r->view.H / factor) * bpp;
    return B2D_OK;
}

int b2d_resolve_palettes_device(b2d_renderer *r, const uint8_t *d_index, const uint32_t *levels, const uint32_t *palettes,
                                size_t n_frames, int factor, int format, void *d_out, void *cuda_stream) {
    if (!r || !d_index || !d_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (int rc = check_resolve(r, factor, format)) return rc;
    if (int rc = check_levels(r, levels, n_frames)) return rc;
    if (int rc = check_palettes(r, levels, palettes, n_frames)) return rc;
    if (n_frames == 0) return B2D_OK;
    CU(cudaSetDevice(r->device));
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    const bool staged = levels || palettes;      // neither: every frame through table 0 (level 0, palette 0), nothing to stage
    if (staged)
        if (int rc = stage_tables(r, r->resolve_levels, levels, palettes, n_frames, st)) return rc;
    CU(launch_resolve(r->d_palettes.get(), staged ? r->resolve_levels.d.get() : nullptr, d_index, d_out, n_frames, r->view.W,
                      r->view.H, factor, format, st));
    if (staged) CU(cudaEventRecord(r->resolve_levels.done.get(), st));
    r->launches += 1;
    return B2D_OK;
}

int b2d_resolve_device(b2d_renderer *r, const uint8_t *d_index, const uint32_t *levels, size_t n_frames, int factor, int format,
                       void *d_out, void *cuda_stream) {
    return b2d_resolve_palettes_device(r, d_index, levels, nullptr, n_frames, factor, format, d_out, cuda_stream);
}

// The automap tables of every level (b2d_renderer::automap): the lines and things of each level in one buffer, then an
// AutomapLevel per level pointing into it, then each level's AutomapDynLine table pointer (automap_dyn_records) and the
// tables, then an AutomapMarkLevel per level (automap_mark_records: the grid origin and digits, C22) and the digits' texels.
static size_t automap_dyn_records(const b2d_renderer *r) { return r->automap->off + r->lv.size() * sizeof(AutomapLevel); }
// `items`: where the AutomapLevel records start (b2d_renderer::Tables::off).
static size_t automap_mark_records(const b2d_renderer *r, size_t items) {
    size_t bytes = items + r->lv.size() * (sizeof(AutomapLevel) + sizeof(const AutomapDynLine *));
    for (const LevelRes &lv : r->lv) bytes += lv.automap_dyn.size() * sizeof(AutomapDynLine);
    return (bytes + 15) & ~(size_t)15;
}
static int ensure_automap(b2d_renderer *r, cudaStream_t st) {
    size_t items = 0;
    std::vector<size_t> line_off, thing_off, dyn_off, digit_off;
    for (const LevelRes &lv : r->lv) {
        line_off.push_back(items);
        items += lv.automap_lines.size() * sizeof(AutomapLine);
        thing_off.push_back(items);
        items += lv.automap_things.size() * sizeof(int32_t);
    }
    items = (items + 15) & ~(size_t)15;                   // the AutomapLevel records follow, aligned
    const size_t dyn_records = items + r->lv.size() * sizeof(AutomapLevel);     // 8-byte aligned
    size_t bytes = dyn_records + r->lv.size() * sizeof(const AutomapDynLine *);
    for (const LevelRes &lv : r->lv) {
        dyn_off.push_back(bytes);
        bytes += lv.automap_dyn.size() * sizeof(AutomapDynLine);
    }
    const size_t mark_records = automap_mark_records(r, items);
    bytes = mark_records + r->lv.size() * sizeof(AutomapMarkLevel);
    for (const LevelRes &lv : r->lv)
        for (const Image &im : lv.digits) {
            digit_off.push_back(bytes);
            bytes += im.px.size() * sizeof(uint16_t);
        }
    return build_tables(r->automap, bytes, items, st, [&](uint8_t *h, const uint8_t *d) {
        for (size_t k = 0; k < r->lv.size(); k++) {
            const LevelRes &lv = r->lv[k];
            AutomapMarkLevel m{lv.grid_origin[0], lv.grid_origin[1], {}};
            for (int g = 0; g < kAutomapDigits; g++) {
                const Image &im = lv.digits[(size_t)g];
                const size_t at = digit_off[k * kAutomapDigits + (size_t)g];
                if (im.px.empty()) continue;          // missing, or 0 x h / w x 0: nothing to draw
                std::memcpy(h + at, im.px.data(), im.px.size() * sizeof(uint16_t));
                m.digit[g] = AutomapDigit{reinterpret_cast<const uint16_t *>(d + at), im.w, im.h, im.xoff, im.yoff};
            }
            std::memcpy(h + mark_records + k * sizeof(AutomapMarkLevel), &m, sizeof m);
        }
        for (size_t k = 0; k < r->lv.size(); k++) {
            const LevelRes &lv = r->lv[k];
            if (!lv.automap_lines.empty()) std::memcpy(h + line_off[k], lv.automap_lines.data(), lv.automap_lines.size() * sizeof(AutomapLine));
            if (!lv.automap_things.empty()) std::memcpy(h + thing_off[k], lv.automap_things.data(), lv.automap_things.size() * sizeof(int32_t));
            const AutomapLevel L{reinterpret_cast<const AutomapLine *>(d + line_off[k]), reinterpret_cast<const int32_t *>(d + thing_off[k]),
                                 (int32_t)lv.automap_lines.size(), (int32_t)(lv.automap_things.size() / 2)};
            std::memcpy(h + items + k * sizeof(AutomapLevel), &L, sizeof L);
            const AutomapDynLine *dyn = lv.automap_dyn.empty() ? nullptr : reinterpret_cast<const AutomapDynLine *>(d + dyn_off[k]);
            std::memcpy(h + dyn_records + k * sizeof dyn, &dyn, sizeof dyn);
            if (dyn) std::memcpy(h + dyn_off[k], lv.automap_dyn.data(), lv.automap_dyn.size() * sizeof(AutomapDynLine));
        }
    });
}

int b2d_renderer_seen_words(const b2d_renderer *r, uint32_t *words_out) {
    if (!r || !words_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    *words_out = r->seen_words;
    return B2D_OK;
}

int b2d_raster_device_seen(b2d_renderer *r, int64_t ticket, uint8_t *d_index_fb, uint32_t *d_seen, void *cuda_stream) {
    if (!r || !d_index_fb || !d_seen) return fail(B2D_ERR_INVALID_ARG, "null argument");
    if (reinterpret_cast<uintptr_t>(d_seen) & 3) return fail(B2D_ERR_INVALID_ARG, "seen rows not 4-byte aligned");
    CU(cudaSetDevice(r->device));
    return raster_batch(r, ticket, d_index_fb, nullptr, static_cast<cudaStream_t>(cuda_stream), d_seen);
}

static_assert(sizeof(b2d_automap_arrow) == sizeof(AutomapArrow) && offsetof(b2d_automap_arrow, colour) == offsetof(AutomapArrow, colour),
              "b2d_automap_arrow");

// What b2d_automap_states_device adds to the seen automap (HOST arrays, each nullable; C21).
struct AutomapStates {
    const b2d_frame_state *states;
    const b2d_sector_move *moves;
    size_t n_moves;
    const b2d_arrow_range *ranges;
    const b2d_automap_arrow *arrows;
    size_t n_arrows;
};

// The state automap's per-frame inputs as one staged image of words: an AutomapFrameIn per frame, the arrows, then the
// distinct sector offsets (2 words per dynamic slot of the level) of the moved frames, shared by frames of equal level and
// offsets.  `c` holds the frames' compact states (CallFrames::prepare), whose words 2 .. 2 + 2 * ndyn are the offsets.
static int automap_states_image(const b2d_renderer *r, const uint32_t *levels, const AutomapStates &a, const CallFrames &c,
                                size_t n, std::vector<uint32_t> &img) {
    return guarded([&] {
        const size_t arrow_words = a.ranges ? 4 * a.n_arrows : 0, pool = 4 * n + arrow_words;
        img.assign(pool, 0);
        if (arrow_words) std::memcpy(img.data() + 4 * n, a.arrows, 4 * arrow_words);
        std::unordered_map<std::string, uint32_t> seen;
        for (size_t i = 0; i < n; i++) {
            const uint32_t level = levels ? levels[i] : 0u;
            const LevelRes &lv = r->lv[level];
            const uint32_t ndyn = (uint32_t)lv.layout.dyn_sectors.size();
            AutomapFrameIn in{level, kAutomapNoSlot, a.ranges ? a.ranges[i].first : 0u, a.ranges ? a.ranges[i].n : 0u};
            if (a.states && !c.starts.empty() && !lv.h_blob.empty() && ndyn && c.fs[c.starts[i] + 1]) {      // moved
                const uint32_t *w = c.fs.data() + c.starts[i] + 2;
                std::string key(reinterpret_cast<const char *>(&level), 4);
                key.append(reinterpret_cast<const char *>(w), 8 * ndyn);
                auto it = seen.emplace(std::move(key), (uint32_t)(img.size() - pool));
                if (it.second) img.insert(img.end(), w, w + 2 * ndyn);
                in.off = it.first->second;
            }
            std::memcpy(img.data() + 4 * i, &in, sizeof in);
        }
        if (img.size() - pool >= kAutomapNoSlot) return fail(B2D_ERR_INVALID_ARG, "too many distinct sector states for one call");
        return B2D_OK;
    });
}

static_assert(sizeof(b2d_automap_mark) == sizeof(AutomapMark) && offsetof(b2d_automap_mark, number) == offsetof(AutomapMark, number),
              "b2d_automap_mark");
static_assert(B2D_AUTOMAP_GRID == kAutomapGrid, "automap flags");

// What b2d_automap_marks_device adds to the state automap (HOST arrays, nullable; C22).
struct AutomapMarks {
    const b2d_arrow_range *ranges;
    const b2d_automap_mark *marks;
    size_t n_marks;
};

// b2d_automap_device (seen_variant false, states nullptr: K5), b2d_automap_seen_device (its seen variant, which also takes
// ALLMAP), b2d_automap_states_device (states: the state variant) and b2d_automap_marks_device (states and marks: the
// marks variant, which also takes GRID)
static int automap_call(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, const uint32_t *d_seen, size_t n_frames,
                        int32_t scale_q16, int flags, uint8_t *d_out, void *cuda_stream, bool seen_variant,
                        const AutomapStates *states = nullptr, const AutomapMarks *marks = nullptr) {
    if (!r || !d_poses || !d_out) return fail(B2D_ERR_INVALID_ARG, "null argument");
    const int known = B2D_AUTOMAP_ROTATE | B2D_AUTOMAP_ALL_LINES | B2D_AUTOMAP_THINGS | (seen_variant ? B2D_AUTOMAP_ALLMAP : 0) |
                      (marks ? B2D_AUTOMAP_GRID : 0);
    if (flags & ~known) return fail(B2D_ERR_INVALID_ARG, "unknown automap flags");
    if (reinterpret_cast<uintptr_t>(d_seen) & 3) return fail(B2D_ERR_INVALID_ARG, "seen rows not 4-byte aligned");
    if (scale_q16 < kAutomapScaleMin || scale_q16 > kAutomapScaleMax)
        return fail(B2D_ERR_INVALID_ARG, "automap scale out of range (256 .. 64 << 16, 16.16 pixels per map unit)");
    if (int rc = check_levels(r, levels, n_frames)) return rc;
    for (const LevelRes &lv : r->lv)      // the key of an item is (item + 1) << 8 | colour
        if (lv.automap_lines.size() + kAutomapArrowSegs + kAutomapThingSegs * lv.automap_things.size() / 2 >= (1u << 24))
            return fail(B2D_ERR_INVALID_ARG, "level has too many automap items (2^24)");
    if (n_frames > 0x7FFFFFFFull / automap_tiles(r->view)) return fail(B2D_ERR_INVALID_ARG, "too many frames for one grid (2^31 - 1 tiles)");
    // the state variant: the states as the walk checks them (without its shared-memory limit: nothing is walked), then
    // the arrows, then each frame's items
    CallFrames c(kFrameStates, levels, states ? states->states : nullptr, states ? states->moves : nullptr, states ? states->n_moves : 0);
    std::vector<uint32_t> img;
    if (states) {
        if (states->states)
            if (int rc = c.prepare(r, n_frames)) return rc;
        if (states->ranges) {
            if (states->n_arrows && !states->arrows) return fail(B2D_ERR_INVALID_ARG, "null argument");
            for (size_t k = 0; k < states->n_arrows; k++)
                if (states->arrows[k].colour == 0 || states->arrows[k].colour > 255)
                    return fail(B2D_ERR_INVALID_ARG, "automap arrow colour out of range (1 .. 255)");
            for (size_t i = 0; i < n_frames; i++) {
                const b2d_arrow_range &g = states->ranges[i];
                if (g.first > states->n_arrows || g.n > states->n_arrows - g.first)
                    return fail(B2D_ERR_INVALID_ARG, "a frame's arrow range runs past the end of the arrow list");
                const LevelRes &lv = r->lv[levels ? levels[i] : 0];
                if (lv.automap_lines.size() + kAutomapArrowSegs * (1 + (uint64_t)g.n) + kAutomapThingSegs * lv.automap_things.size() / 2 >=
                    (1u << 24))
                    return fail(B2D_ERR_INVALID_ARG, "a frame has too many automap items (2^24)");
            }
        }
        if (marks && marks->ranges) {
            if (marks->n_marks && !marks->marks) return fail(B2D_ERR_INVALID_ARG, "null argument");
            for (size_t k = 0; k < marks->n_marks; k++)
                if (marks->marks[k].number > 9) return fail(B2D_ERR_INVALID_ARG, "automap mark number out of range (0 .. 9)");
            for (size_t i = 0; i < n_frames; i++) {
                const b2d_arrow_range &g = marks->ranges[i];
                if (g.first > marks->n_marks || g.n > marks->n_marks - g.first)
                    return fail(B2D_ERR_INVALID_ARG, "a frame's mark range runs past the end of the mark list");
                const LevelRes &lv = r->lv[levels ? levels[i] : 0];
                const uint64_t arrows = states->ranges ? states->ranges[i].n : 0;
                if (lv.automap_lines.size() + kAutomapArrowSegs * (1 + arrows) + kAutomapThingSegs * lv.automap_things.size() / 2 + g.n >=
                    (1u << 24))
                    return fail(B2D_ERR_INVALID_ARG, "a frame has too many automap items (2^24)");
            }
        }
        if (int rc = automap_states_image(r, levels, *states, c, n_frames, img)) return rc;
    }
    // the marks variant's staging follows the state variant's: 2 words (first, n) per frame, then the marks
    const size_t mark_at = img.size();
    if (marks && marks->ranges) {
        if (int rc = guarded([&] {
                img.resize(mark_at + 2 * n_frames + 3 * marks->n_marks);
                if (n_frames) std::memcpy(img.data() + mark_at, marks->ranges, 8 * n_frames);
                if (marks->n_marks) std::memcpy(img.data() + mark_at + 2 * n_frames, marks->marks, 12 * marks->n_marks);
                return B2D_OK;
            }))
            return rc;
    }
    if (n_frames == 0) return B2D_OK;
    CU(cudaSetDevice(r->device));
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    if (int rc = tables_on(r, r->automap, st, ensure_automap)) return rc;
    const AutomapLevel *d_levels = reinterpret_cast<const AutomapLevel *>(r->automap->d.get() + r->automap->off);
    if (states) {
        // nothing per frame (level 0, at rest, no arrows): nothing to stage
        const bool marked = marks && marks->ranges;
        const bool staged = levels || c.frames.starts || states->ranges || marked;
        if (staged)
            if (int rc = stage_words(r->automap_states, img.size(), st, [&](size_t i) { return img[i]; })) return rc;
        const uint32_t *d = r->automap_states.d.get();
        const size_t pool = 4 * n_frames + (states->ranges ? 4 * states->n_arrows : 0);
        const AutomapStateTables t{reinterpret_cast<const AutomapDynLine *const *>(r->automap->d.get() + automap_dyn_records(r)),
                                   staged ? reinterpret_cast<const AutomapFrameIn *>(d) : nullptr,
                                   staged ? reinterpret_cast<const int32_t *>(d + pool) : nullptr,
                                   staged ? reinterpret_cast<const AutomapArrow *>(d + 4 * n_frames) : nullptr};
        const AutomapMarkTables m{
            reinterpret_cast<const AutomapMarkLevel *>(r->automap->d.get() + automap_mark_records(r, r->automap->off)),
            marked ? d + mark_at : nullptr, marked ? reinterpret_cast<const AutomapMark *>(d + mark_at + 2 * n_frames) : nullptr};
        CU(launch_automap(d_levels, nullptr, reinterpret_cast<const Pose *>(d_poses), n_frames, r->view, scale_q16, flags, true,
                          d_seen, r->seen_words, d_out, st, &t, marks ? &m : nullptr));
        if (staged) CU(cudaEventRecord(r->automap_states.done.get(), st));
        r->launches += 1;
        return B2D_OK;
    }
    if (levels)
        if (int rc = stage_words(r->automap_levels, n_frames, st, [&](size_t i) { return levels[i]; })) return rc;
    const uint32_t *d_frame_level = levels ? r->automap_levels.d.get() : nullptr;
    CU(launch_automap(d_levels, d_frame_level, reinterpret_cast<const Pose *>(d_poses), n_frames, r->view, scale_q16, flags,
                      seen_variant, d_seen, r->seen_words, d_out, st));
    if (levels) CU(cudaEventRecord(r->automap_levels.done.get(), st));
    r->launches += 1;
    return B2D_OK;
}

int b2d_automap_device(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, size_t n_frames, int32_t scale_q16,
                       int flags, uint8_t *d_out, void *cuda_stream) {
    return automap_call(r, d_poses, levels, nullptr, n_frames, scale_q16, flags, d_out, cuda_stream, false);
}

int b2d_automap_seen_device(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, const uint32_t *d_seen,
                            size_t n_frames, int32_t scale_q16, int flags, uint8_t *d_out, void *cuda_stream) {
    return automap_call(r, d_poses, levels, d_seen, n_frames, scale_q16, flags, d_out, cuda_stream, true);
}

int b2d_automap_states_device(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, const b2d_frame_state *states,
                              const b2d_sector_move *moves, size_t n_moves, const b2d_arrow_range *arrow_ranges,
                              const b2d_automap_arrow *arrows, size_t n_arrows, const uint32_t *d_seen, size_t n_frames,
                              int32_t scale_q16, int flags, uint8_t *d_out, void *cuda_stream) {
    const AutomapStates a{states, moves, n_moves, arrow_ranges, arrows, n_arrows};
    return automap_call(r, d_poses, levels, d_seen, n_frames, scale_q16, flags, d_out, cuda_stream, true, &a);
}

int b2d_automap_marks_device(b2d_renderer *r, const b2d_pose *d_poses, const uint32_t *levels, const b2d_frame_state *states,
                             const b2d_sector_move *moves, size_t n_moves, const b2d_arrow_range *arrow_ranges,
                             const b2d_automap_arrow *arrows, size_t n_arrows, const uint32_t *d_seen, size_t n_frames,
                             int32_t scale_q16, int flags, uint8_t *d_out, void *cuda_stream, const b2d_arrow_range *mark_ranges,
                             const b2d_automap_mark *marks, size_t n_marks) {
    const AutomapStates a{states, moves, n_moves, arrow_ranges, arrows, n_arrows};
    const AutomapMarks m{mark_ranges, marks, n_marks};
    return automap_call(r, d_poses, levels, d_seen, n_frames, scale_q16, flags, d_out, cuda_stream, true, &a, &m);
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

int b2d_device_upload(int device, void *d_dst, const void *host_src, size_t bytes) {
    if (!d_dst || !host_src) return fail(B2D_ERR_INVALID_ARG, "null argument");
    CU(cudaSetDevice(device));
    CU(cudaMemcpy(d_dst, host_src, bytes, cudaMemcpyHostToDevice));
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
    const WorkSlot &s = r->slot[r->last_slot];
    if (!s.tables.per_frame || n > (size_t)s.n)
        return fail(B2D_ERR_INVALID_ARG, "the last walked batch has no per-frame states or fewer than n frames");
    CU(cudaSetDevice(r->device));
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(slots_out, s.tables.levels.frame_set, 4 * n, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; i++)      // a frame on a level without a table set (TableSet index >= sets) has none
        if (slots_out[i] >= (uint32_t)s.sets) slots_out[i] = 0xFFFFFFFFu;
    return B2D_OK;
}

int b2d_debug_state_tables(b2d_renderer *r, size_t set, void *out, size_t capacity, size_t *size_out) {
    if (!r) return fail(B2D_ERR_INVALID_ARG, "null renderer");
    const WorkSlot &s = r->slot[r->last_slot];
    const bool per_frame = s.tables.per_frame;        // a per-frame set of the arena, or the slot's own set of level 0
    const LevelRes &lv = r->lv[per_frame && set < (size_t)s.sets ? s.set_level[set] : 0];
    if (!per_frame && lv.h_blob.empty()) return fail(B2D_ERR_INVALID_ARG, "the scene has no time-dependent content or dynamic sectors");
    if (s.ticket < 0) return fail(B2D_ERR_INVALID_ARG, "no batch has been walked");
    if (set >= (per_frame ? (size_t)s.sets : 1)) return fail(B2D_ERR_INVALID_ARG, "table set out of range for the last walked batch");
    const size_t need = SetLayout(lv.src).bytes;
    if (size_out) *size_out = need;
    if (!out) return B2D_OK;
    if (capacity < need) return fail(B2D_ERR_INVALID_ARG, "buffer too small for the tables");
    CU(cudaSetDevice(r->device));
    CU(cudaDeviceSynchronize());
    const uint8_t *src = per_frame ? s.arena.get() + s.set_off[set] : lv.slot[r->last_slot].tables.get();
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
