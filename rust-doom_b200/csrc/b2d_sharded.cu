// Multi-GPU sharded render (include/b2d.h: b2d_comm_*, b2d_render_sharded, b2d_frame_checksums_device).
//
// One process per GPU.  Poses are independent, so rank r renders the contiguous block r of the pose list with the scene
// replicated; the only exchange the path has is BASELINE.json's "all-gather of finished frames".  It is built so that it
// costs no extra pass over HBM and hides under rendering:
//   * a chunk of frames is rastered straight into this rank's slice of the all-gather receive buffer (the buffer IS the
//     NCCL send buffer: in-place ncclAllGather, no staging copy); the resolved calls raster it into a rank-local staging
//     buffer instead and resolve it (K4) from there into the slice, so the exchange carries the smaller resolved frames;
//   * the gather of chunk k runs on its own stream while chunk k+1 is rendered into the other buffer; a third stream
//     runs the consumer of gathered chunk k (the caller's callback: checksum, encoder, sink), so the gather stream goes
//     back to back;
//   * the buffers come from ncclMemAlloc and are registered with the communicator (symmetric window if the library has
//     it, else ncclCommRegister) so that NCCL can use zero-copy / NVLS paths over NVSwitch.
// 100 k index frames are 207 GB -- more than one GPU's HBM -- hence chunks and a consumer instead of one big buffer.
//
// NCCL is bound at run time (dlopen "libnccl.so.2"): libb2d.so loads and renders on machines without it, and inside a
// PyTorch process it picks up the copy torch has already loaded.  The reference has no collective (SURVEY.md 2); the
// hand-off this stands in for is `frame.finish()` in engine/src/renderer.rs:160-167.
#include <dlfcn.h>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "b2d_internal.hpp"

namespace {

// ---- the slice of the NCCL API used here (matches nccl.h 2.19+; checked against /usr/include/nccl.h 2.27.3) ----
typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef void *ncclWindow_t;
constexpr int kNcclUint8 = 1;        // ncclUint8 / ncclChar enum value
constexpr int kNcclInt32 = 2, kNcclSum = 0;
constexpr int kWinCollSymmetric = 1; // NCCL_WIN_COLL_SYMMETRIC

struct Nccl {
    void *lib = nullptr;
    int version = 0;
    const char *(*GetErrorString)(int) = nullptr;
    int (*GetVersion)(int *) = nullptr;
    int (*GetUniqueId)(ncclUniqueId *) = nullptr;
    int (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    int (*CommDestroy)(ncclComm_t) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*AllReduce)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*MemAlloc)(void **, size_t) = nullptr;                       // optional
    int (*MemFree)(void *) = nullptr;
    int (*CommRegister)(ncclComm_t, void *, size_t, void **) = nullptr;
    int (*CommDeregister)(ncclComm_t, void *) = nullptr;
    int (*CommWindowRegister)(ncclComm_t, void *, size_t, ncclWindow_t *, int) = nullptr;
    int (*CommWindowDeregister)(ncclComm_t, ncclWindow_t) = nullptr;
    std::string error;
};

Nccl &nccl() {
    static Nccl n;
    static std::once_flag once;
    std::call_once(once, [] {
        const char *names[] = {getenv("B2D_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char *nm : names) {
            if (!nm || !*nm) continue;
            n.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (n.lib) break;
        }
        if (!n.lib) { n.error = std::string("libnccl.so.2 not found: ") + (dlerror() ? dlerror() : "?"); return; }
        auto sym = [&](const char *s) { return dlsym(n.lib, s); };
#define B2D_NCCL_SYM(field, name) n.field = reinterpret_cast<decltype(n.field)>(sym(name))
        B2D_NCCL_SYM(GetErrorString, "ncclGetErrorString");
        B2D_NCCL_SYM(GetVersion, "ncclGetVersion");
        B2D_NCCL_SYM(GetUniqueId, "ncclGetUniqueId");
        B2D_NCCL_SYM(CommInitRank, "ncclCommInitRank");
        B2D_NCCL_SYM(CommDestroy, "ncclCommDestroy");
        B2D_NCCL_SYM(AllGather, "ncclAllGather");
        B2D_NCCL_SYM(AllReduce, "ncclAllReduce");
        B2D_NCCL_SYM(MemAlloc, "ncclMemAlloc");
        B2D_NCCL_SYM(MemFree, "ncclMemFree");
        B2D_NCCL_SYM(CommRegister, "ncclCommRegister");
        B2D_NCCL_SYM(CommDeregister, "ncclCommDeregister");
        B2D_NCCL_SYM(CommWindowRegister, "ncclCommWindowRegister");
        B2D_NCCL_SYM(CommWindowDeregister, "ncclCommWindowDeregister");
#undef B2D_NCCL_SYM
        if (!n.GetUniqueId || !n.CommInitRank || !n.CommDestroy || !n.AllGather || !n.GetErrorString) {
            n.error = "libnccl.so.2 lacks a required symbol";
            return;
        }
        if (n.GetVersion) n.GetVersion(&n.version);
    });
    return n;
}

int nccl_fail(int rc, const char *what) {
    Nccl &n = nccl();
    return b2d::fail(B2D_ERR_NCCL, std::string(what) + ": " + (n.GetErrorString ? n.GetErrorString(rc) : "nccl error"));
}
#define B2D_NC(call)                                   \
    do {                                               \
        int rc_ = (call);                              \
        if (rc_ != 0) return nccl_fail(rc_, #call);    \
    } while (0)

// one checksum per frame: sum over pixels of (p + 1) * (i * 0x9E3779B1 + 0x7F4A7C15) mod 2^32 -- position sensitive,
// order independent (so any reduction tree gives the same word), cheap to restate on the host for sampled frames
__global__ void __launch_bounds__(256)
b2d_checksum_kernel(const uint8_t *__restrict__ frames, size_t npix, int parts, uint32_t *__restrict__ out) {
    const size_t frame = blockIdx.x / parts;
    const int part = blockIdx.x % parts;
    const uint8_t *p = frames + frame * npix;
    const size_t nvec = npix / 16;                       // 128-bit loads; a frame starts 16-byte aligned iff npix % 16 == 0
    const bool aligned = (npix % 16 == 0) && ((reinterpret_cast<uintptr_t>(frames) & 15) == 0);
    uint32_t acc = 0;
    if (aligned) {
        const uint4 *v = reinterpret_cast<const uint4 *>(p);
        for (size_t i = (size_t)part * blockDim.x + threadIdx.x; i < nvec; i += (size_t)parts * blockDim.x) {
            const uint4 q = __ldcs(v + i);
            const uint32_t w[4] = {q.x, q.y, q.z, q.w};
            uint32_t idx = (uint32_t)(i * 16);
#pragma unroll
            for (int k = 0; k < 4; k++)
#pragma unroll
                for (int b = 0; b < 4; b++, idx++)
                    acc += (((w[k] >> (8 * b)) & 0xFFu) + 1u) * (idx * 0x9E3779B1u + 0x7F4A7C15u);
        }
    } else {
        for (size_t i = (size_t)part * blockDim.x + threadIdx.x; i < npix; i += (size_t)parts * blockDim.x)
            acc += ((uint32_t)p[i] + 1u) * ((uint32_t)i * 0x9E3779B1u + 0x7F4A7C15u);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xFFFFFFFFu, acc, o);
    __shared__ uint32_t s[8];
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int i = 0; i < 8; i++) t += s[i];
        atomicAdd(out + frame, t);
    }
}

}  // namespace

struct b2d_comm {
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1, device = 0;
    // two all-gather receive buffers (world x chunk x W*H bytes each), allocated on first use / when the shape grows
    uint8_t *buf[2] = {nullptr, nullptr};
    size_t buf_bytes = 0;
    bool nccl_mem = false;
    void *reg[2] = {nullptr, nullptr};
    ncclWindow_t win[2] = {nullptr, nullptr};
    const char *registration = "none";
    Stream render_stream, gather_stream, consume_stream, walk_stream;
    // copy-engine transport (B2D_GATHER=ce): every rank pushes its slice into the peers' buffers with cudaMemcpyAsync over
    // CUDA-IPC mappings -- no SM is used for the exchange; two tiny NCCL all-reduces per chunk order it across ranks
    bool ce = false;
    std::vector<uint8_t *> peer[2];                 // [buffer][rank]: that rank's buffer as mapped here (own rank: buf[b])
    std::vector<Stream> push_stream;                // one per peer
    std::vector<Event> push_done;
    Event push_go;
    DeviceBuf<int32_t> d_token;
    DeviceBuf<Pose> d_poses; PinnedBuf<Pose> h_poses;
    size_t poses_cap = 0;
    // resolved calls (b2d_render_sharded*_resolved*): the rank-local index frames of one chunk, which K4 reads, and the
    // frame colour-table indices of the rank's block with their pinned staging, uploaded once per call next to the poses
    DeviceBuf<uint8_t> d_stage;
    size_t stage_bytes = 0;
    DeviceBuf<uint32_t> d_tables; PinnedBuf<uint32_t> h_tables;
    size_t tables_cap = 0;
};

namespace {

void release_buffers(b2d_comm *c) {
    Nccl &n = nccl();
    for (int i = 0; i < 2; i++) {
        for (size_t q = 0; q < c->peer[i].size(); q++)
            if ((int)q != c->rank && c->peer[i][q]) cudaIpcCloseMemHandle(c->peer[i][q]);
        c->peer[i].clear();
    }
    for (int i = 0; i < 2; i++) {
        if (!c->buf[i]) continue;
        if (c->win[i] && n.CommWindowDeregister) n.CommWindowDeregister(c->comm, c->win[i]);
        if (c->reg[i] && n.CommDeregister) n.CommDeregister(c->comm, c->reg[i]);
        if (c->nccl_mem && n.MemFree) n.MemFree(c->buf[i]); else cudaFree(c->buf[i]);
        c->buf[i] = nullptr; c->win[i] = nullptr; c->reg[i] = nullptr;
    }
    c->buf_bytes = 0;
}

int ensure_buffers(b2d_comm *c, size_t bytes) {
    if (c->buf_bytes >= bytes) return B2D_OK;
    Nccl &n = nccl();
    release_buffers(c);
    // exchange transport: the copy engines over CUDA-IPC peer mappings (no SM or L2 taken from the raster beside it)
    // unless B2D_GATHER=nccl asks for ncclAllGather; if any rank cannot map a peer's buffer, all ranks agree to fall back to NCCL below
    const char *tr = getenv("B2D_GATHER");
    c->ce = !(tr && std::strcmp(tr, "nccl") == 0) && c->world > 1 && n.AllReduce;
    const bool want_reg = !getenv("B2D_NCCL_NO_REGISTER") && !c->ce;      // IPC needs plain cudaMalloc memory
    c->nccl_mem = want_reg && n.MemAlloc && n.MemFree;
    c->registration = "none";
    for (int i = 0; i < 2; i++) {
        void *p = nullptr;
        if (c->nccl_mem) {
            if (n.MemAlloc(&p, bytes) != 0) { c->nccl_mem = false; p = nullptr; cudaGetLastError(); }
        }
        if (!p) B2D_CU(cudaMalloc(&p, bytes));
        c->buf[i] = static_cast<uint8_t *>(p);
    }
    if (c->nccl_mem) {
        // collective calls: every rank reaches them with the same sizes
        bool ok = false;
        if (n.CommWindowRegister && n.CommWindowDeregister && !getenv("B2D_NCCL_NO_WINDOW")) {
            ok = true;
            for (int i = 0; i < 2 && ok; i++) ok = n.CommWindowRegister(c->comm, c->buf[i], bytes, &c->win[i], kWinCollSymmetric) == 0 && c->win[i];
            if (ok) c->registration = "ncclCommWindowRegister(NCCL_WIN_COLL_SYMMETRIC)";
            else for (int i = 0; i < 2; i++) c->win[i] = nullptr;
        }
        if (!ok && n.CommRegister && n.CommDeregister) {
            ok = true;
            for (int i = 0; i < 2 && ok; i++) ok = n.CommRegister(c->comm, c->buf[i], bytes, &c->reg[i]) == 0;
            if (ok) c->registration = "ncclCommRegister";
        }
        cudaGetLastError();
    }
    if (c->ce) {
        // exchange the IPC handles of both buffers (NCCL all-gather of 2 x 64 bytes per rank) and map the peers' buffers
        const size_t hb = sizeof(cudaIpcMemHandle_t);
        std::vector<uint8_t> mine(2 * hb), all(2 * hb * (size_t)c->world);
        for (int i = 0; i < 2; i++) {
            cudaIpcMemHandle_t h;
            B2D_CU(cudaIpcGetMemHandle(&h, c->buf[i]));
            std::memcpy(&mine[(size_t)i * hb], &h, hb);
        }
        DeviceBuf<uint8_t> d_h;
        B2D_CU(allocate(d_h, all.size()));
        B2D_CU(cudaMemcpy(d_h.get() + (size_t)c->rank * 2 * hb, mine.data(), 2 * hb, cudaMemcpyHostToDevice));
        int nrc = n.AllGather(d_h.get() + (size_t)c->rank * 2 * hb, d_h.get(), 2 * hb, kNcclUint8, c->comm, c->gather_stream.get());
        if (nrc != 0) return nccl_fail(nrc, "ncclAllGather (ipc handles)");
        B2D_CU(cudaStreamSynchronize(c->gather_stream.get()));
        B2D_CU(cudaMemcpy(all.data(), d_h.get(), all.size(), cudaMemcpyDeviceToHost));
        int32_t mapped = 1;
        for (int i = 0; i < 2; i++) {
            c->peer[i].assign((size_t)c->world, nullptr);
            for (int q = 0; q < c->world && mapped; q++) {
                if (q == c->rank) { c->peer[i][(size_t)q] = c->buf[i]; continue; }
                cudaIpcMemHandle_t h;
                std::memcpy(&h, &all[((size_t)q * 2 + (size_t)i) * hb], hb);
                void *p = nullptr;
                if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { mapped = 0; cudaGetLastError(); break; }
                c->peer[i][(size_t)q] = static_cast<uint8_t *>(p);
            }
        }
        // every rank must have mapped every peer, or nobody uses the mappings (minimum over ranks = sum of the failures == 0)
        int32_t failures = mapped ? 0 : 1;
        DeviceBuf<int32_t> d_flag;
        B2D_CU(allocate(d_flag, sizeof(int32_t)));
        B2D_CU(cudaMemcpy(d_flag.get(), &failures, sizeof failures, cudaMemcpyHostToDevice));
        nrc = n.AllReduce(d_flag.get(), d_flag.get(), 1, kNcclInt32, kNcclSum, c->comm, c->gather_stream.get());
        if (nrc != 0) return nccl_fail(nrc, "ncclAllReduce (ipc agreement)");
        B2D_CU(cudaStreamSynchronize(c->gather_stream.get()));
        B2D_CU(cudaMemcpy(&failures, d_flag.get(), sizeof failures, cudaMemcpyDeviceToHost));
        if (failures) {
            for (int i = 0; i < 2; i++) {
                for (size_t q = 0; q < c->peer[i].size(); q++)
                    if ((int)q != c->rank && c->peer[i][q]) cudaIpcCloseMemHandle(c->peer[i][q]);
                c->peer[i].clear();
            }
            c->ce = false;
            c->registration = "none (peers not mappable: ncclAllGather, plain buffers)";
            c->buf_bytes = bytes;
            return B2D_OK;
        }
        if (c->push_stream.empty()) {       // created whole, or not at all
            std::vector<Stream> push_stream((size_t)c->world);
            std::vector<Event> push_done((size_t)c->world);
            Event push_go; DeviceBuf<int32_t> d_token;
            for (int q = 0; q < c->world; q++) {
                if (q == c->rank) continue;
                B2D_CU(stream_create(push_stream[(size_t)q]));
                B2D_CU(event_create(push_done[(size_t)q]));
            }
            B2D_CU(event_create(push_go));
            B2D_CU(allocate(d_token, sizeof(int32_t)));
            B2D_CU(cudaMemset(d_token.get(), 0, sizeof(int32_t)));
            c->push_stream = std::move(push_stream); c->push_done = std::move(push_done);
            c->push_go = std::move(push_go); c->d_token = std::move(d_token);
        }
        c->registration = "copy engines: cudaMemcpyAsync over CUDA-IPC peer mappings";
    }
    c->buf_bytes = bytes;
    return B2D_OK;
}

// copy-engine all-gather of one chunk (see b2d_comm::ce).  Enqueued on the gather stream after `rendered`.
int ce_gather(b2d_comm *c, int b, size_t slice_off, size_t bytes) {
    Nccl &n = nccl();
    // 1. every rank's buffer b is free again (each rank enqueues this after the event that says so locally)
    B2D_NC(n.AllReduce(c->d_token.get(), c->d_token.get(), 1, kNcclInt32, kNcclSum, c->comm, c->gather_stream.get()));
    B2D_CU(cudaEventRecord(c->push_go.get(), c->gather_stream.get()));
    // 2. push my slice into every peer's buffer, one stream (one copy engine queue) per peer
    for (int k = 1; k < c->world; k++) {
        const int q = (c->rank + k) % c->world;                        // stagger the targets across ranks
        cudaStream_t ps = c->push_stream[(size_t)q].get();
        B2D_CU(cudaStreamWaitEvent(ps, c->push_go.get(), 0));
        B2D_CU(cudaMemcpyAsync(c->peer[b][(size_t)q] + slice_off, c->buf[b] + slice_off, bytes, cudaMemcpyDeviceToDevice, ps));
        B2D_CU(cudaEventRecord(c->push_done[(size_t)q].get(), ps));
        B2D_CU(cudaStreamWaitEvent(c->gather_stream.get(), c->push_done[(size_t)q].get(), 0));
    }
    // 3. everybody's pushes have landed
    B2D_NC(n.AllReduce(c->d_token.get(), c->d_token.get(), 1, kNcclInt32, kNcclSum, c->comm, c->gather_stream.get()));
    return B2D_OK;
}

}  // namespace

extern "C" {

int b2d_comm_unique_id(uint8_t id_out[B2D_COMM_ID_BYTES]) {
    if (!id_out) return b2d::fail(B2D_ERR_INVALID_ARG, "null argument");
    Nccl &n = nccl();
    if (!n.error.empty()) return b2d::fail(B2D_ERR_NCCL, n.error);
    ncclUniqueId id;
    B2D_NC(n.GetUniqueId(&id));
    static_assert(sizeof(ncclUniqueId) == B2D_COMM_ID_BYTES, "unique id size");
    std::memcpy(id_out, &id, sizeof id);
    return B2D_OK;
}

int b2d_comm_create(const uint8_t id[B2D_COMM_ID_BYTES], int rank, int world, int device, b2d_comm **out) {
    if (!id || !out || world < 1 || rank < 0 || rank >= world) return b2d::fail(B2D_ERR_INVALID_ARG, "bad communicator arguments");
    Nccl &n = nccl();
    if (!n.error.empty()) return b2d::fail(B2D_ERR_NCCL, n.error);
    B2D_CU(cudaSetDevice(device));
    b2d_comm *c = new (std::nothrow) b2d_comm();
    if (!c) return b2d::fail(B2D_ERR_NO_MEMORY, "out of host memory");
    c->rank = rank; c->world = world; c->device = device;
    ncclUniqueId uid;
    std::memcpy(&uid, id, sizeof uid);
    int rc = n.CommInitRank(&c->comm, world, uid, rank);
    if (rc != 0) { delete c; return nccl_fail(rc, "ncclCommInitRank"); }
    cudaError_t e = stream_create(c->render_stream);
    if (e == cudaSuccess) e = stream_create(c->gather_stream);
    if (e == cudaSuccess) e = stream_create(c->consume_stream);
    if (e == cudaSuccess) e = stream_create(c->walk_stream);
    if (e != cudaSuccess) { b2d_comm_destroy(c); return b2d::cuda_fail(e, "cudaStreamCreate"); }
    *out = c;
    return B2D_OK;
}

void b2d_comm_destroy(b2d_comm *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    release_buffers(c);
    if (c->comm) nccl().CommDestroy(c->comm);
    delete c;                               // the streams, events and pose buffers, on this device
}

int b2d_comm_info(const b2d_comm *c, int *rank_out, int *world_out, int *nccl_version_out) {
    if (!c) return b2d::fail(B2D_ERR_INVALID_ARG, "null communicator");
    if (rank_out) *rank_out = c->rank;
    if (world_out) *world_out = c->world;
    if (nccl_version_out) *nccl_version_out = nccl().version;
    return B2D_OK;
}

int b2d_frame_checksums_device(const uint8_t *d_frames, size_t n_frames, size_t frame_bytes, uint32_t *d_out, void *cuda_stream) {
    if (!d_frames || !d_out) return b2d::fail(B2D_ERR_INVALID_ARG, "null argument");
    if (n_frames == 0 || frame_bytes == 0) return B2D_OK;
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    B2D_CU(cudaMemsetAsync(d_out, 0, n_frames * sizeof(uint32_t), st));
    int parts = (int)((frame_bytes + 65535) / 65536);                 // ~64 KB of a frame per CTA
    if (parts < 1) parts = 1;
    if (parts > 64) parts = 64;
    if (n_frames * (size_t)parts > 0x7FFFFFFFull) return b2d::fail(B2D_ERR_INVALID_ARG, "too many frames for one checksum launch");
    b2d_checksum_kernel<<<(unsigned)(n_frames * parts), 256, 0, st>>>(d_frames, frame_bytes, parts, d_out);
    B2D_CU(cudaGetLastError());
    return B2D_OK;
}

}  // extern "C"

namespace {

int check_sharded(const b2d_renderer *r, const b2d_comm *c, const b2d_pose *poses, int mode) {
    if (!r || !c || !poses) return b2d::fail(B2D_ERR_INVALID_ARG, "null argument");
    if (mode < B2D_SHARD_RENDER_ONLY || mode > B2D_SHARD_GATHER_ONLY) return b2d::fail(B2D_ERR_INVALID_ARG, "unknown mode");
    if (r->device != c->device) return b2d::fail(B2D_ERR_INVALID_ARG, "renderer and communicator are on different devices");
    return B2D_OK;
}

// The resolve step of a resolved sharded call: K4 by `factor` into `format`, frame_bytes bytes per resolved frame;
// block_tables (HOST, nullable = table 0 on every frame) holds the colour-table index (frame_table) of each entry of this
// rank's padded block.
struct ShardResolve {
    int factor = 1, format = B2D_RESOLVE_RGBA8;
    size_t frame_bytes = 0;
    const uint32_t *block_tables = nullptr;
};

// The chunk loop of the sharded calls, after their arguments have been checked (check_sharded and the caller's checks of
// the whole job: a rank that refused its input here would leave its peers waiting in a collective).  `block`: the frames
// of this rank's padded block (its poses are padded here the same way); each chunk of it is walked as a background grid
// on the walk stream.  With `res` (nullable) each chunk is rastered into the comm's index staging and
// resolved from there into this rank's slice of the exchange buffer, on the render stream: the raster of chunk k+1 follows
// the resolve of chunk k there, so one staging buffer serves every chunk.  Without it, chunks are rastered into the slice.
int sharded_loop(b2d_renderer *r, b2d_comm *c, const b2d_pose *poses, size_t n_total, size_t chunk_frames, int mode, b2d_chunk_fn fn,
                 void *user, b2d_sharded_stats *stats_out, const Frames &block, const ShardResolve *res = nullptr) {
    B2D_CU(cudaSetDevice(c->device));
    Nccl &n = nccl();
    const size_t world = (size_t)c->world, rank = (size_t)c->rank;
    const size_t per = (n_total + world - 1) / world;                    // poses per rank; short last block padded
    size_t chunk = chunk_frames ? chunk_frames : 256;
    if (chunk > (size_t)r->max_batch) chunk = (size_t)r->max_batch;
    if (chunk > per) chunk = per;
    const size_t nchunks = (per + chunk - 1) / chunk;
    const size_t npix = (size_t)r->view.W * r->view.H;
    const size_t frame_bytes = res ? res->frame_bytes : npix;            // of one frame in the exchange buffers
    const bool do_render = mode != B2D_SHARD_GATHER_ONLY, do_gather = mode != B2D_SHARD_RENDER_ONLY;
    const bool do_resolve = res && do_render;

    int rc = do_render ? b2d::check_slots_free(r, nchunks) : B2D_OK;
    if (rc == B2D_OK) rc = ensure_buffers(c, world * chunk * frame_bytes);
    if (rc != B2D_OK) return rc;
    if (do_resolve && c->stage_bytes < chunk * npix) {
        c->stage_bytes = 0; c->d_stage.reset();
        B2D_CU(allocate(c->d_stage, chunk * npix));
        c->stage_bytes = chunk * npix;
    }
    if (do_resolve && res->block_tables && c->tables_cap < per) {
        c->tables_cap = 0; c->d_tables.reset(); c->h_tables.reset();
        B2D_CU(allocate(c->d_tables, per * sizeof(uint32_t)));
        B2D_CU(allocate(c->h_tables, per * sizeof(uint32_t)));
        c->tables_cap = per;
    }
    // this rank's block of poses, padded by repeating the last pose of the list, on the device in one copy
    if (c->poses_cap < per) {
        c->poses_cap = 0; c->d_poses.reset(); c->h_poses.reset();
        B2D_CU(allocate(c->d_poses, per * sizeof(Pose)));
        B2D_CU(allocate(c->h_poses, per * sizeof(Pose)));
        c->poses_cap = per;
    }
    for (size_t i = 0; i < per; i++) {
        size_t g = rank * per + i;
        if (g >= n_total) g = n_total - 1;
        std::memcpy(&c->h_poses.get()[i], &poses[g], sizeof(Pose));
    }
    cudaStream_t render_stream = c->render_stream.get(), gather_stream = c->gather_stream.get(),
                 consume_stream = c->consume_stream.get(), walk_stream = c->walk_stream.get();
    B2D_CU(cudaMemcpyAsync(c->d_poses.get(), c->h_poses.get(), per * sizeof(Pose), cudaMemcpyHostToDevice, render_stream));
    Event poses_up;
    B2D_CU(event_create(poses_up));
    B2D_CU(cudaEventRecord(poses_up.get(), render_stream));
    B2D_CU(cudaStreamWaitEvent(walk_stream, poses_up.get(), 0));
    const uint32_t *d_tables = nullptr;                                  // the resolve's frame tables; NULL: table 0
    if (do_resolve && res->block_tables) {
        std::memcpy(c->h_tables.get(), res->block_tables, per * sizeof(uint32_t));
        B2D_CU(cudaMemcpyAsync(c->d_tables.get(), c->h_tables.get(), per * sizeof(uint32_t), cudaMemcpyHostToDevice, render_stream));
        d_tables = c->d_tables.get();
    }
    // the BSP walk of chunk k+1 runs as a background grid on its own stream under the raster of chunk k
    auto walk = [&](size_t k, int64_t *ticket) {
        const size_t f = k * chunk;
        return b2d::walk_batch(r, c->d_poses.get() + f, block.from(f), (int)((per - f) < chunk ? (per - f) : chunk), walk_stream,
                               true, ticket);
    };
    int64_t ticket = -1;
    if (do_render) {
        int wrc = walk(0, &ticket);
        if (wrc != B2D_OK) return wrc;
    }

    // events: per buffer "rendered", "gathered", "consumed"; timing pairs per chunk
    Event rendered[2], gathered[2], consumed[2], t_begin, t_end;
    for (int i = 0; i < 2; i++) {
        B2D_CU(event_create(rendered[i]));
        B2D_CU(event_create(gathered[i]));
        B2D_CU(event_create(consumed[i]));
    }
    B2D_CU(event_create(t_begin, cudaEventDefault));
    B2D_CU(event_create(t_end, cudaEventDefault));
    std::vector<Event> rt(2 * nchunks), gt(2 * nchunks);
    for (auto &e : rt) B2D_CU(event_create(e, cudaEventDefault));
    for (auto &e : gt) B2D_CU(event_create(e, cudaEventDefault));

    B2D_CU(cudaEventRecord(t_begin.get(), render_stream));
    int result = B2D_OK;
    for (size_t k = 0; k < nchunks && result == B2D_OK; k++) {
        const int b = (int)(k & 1);
        const size_t first = k * chunk;
        const size_t cnt = (per - first) < chunk ? (per - first) : chunk;
        uint8_t *slice = c->buf[b] + rank * cnt * frame_bytes;           // in-place all-gather: rank-major slices of cnt frames
        if (k >= 2) B2D_CU(cudaStreamWaitEvent(render_stream, consumed[b].get(), 0));     // chunk k-2 has left this buffer
        B2D_CU(cudaEventRecord(rt[2 * k].get(), render_stream));
        if (do_render) {
            result = b2d::raster_batch(r, ticket, do_resolve ? c->d_stage.get() : slice, nullptr, render_stream);
            if (result != B2D_OK) break;
            if (do_resolve) {
                B2D_CU(launch_resolve(r->d_palettes.get(), d_tables ? d_tables + first : nullptr, c->d_stage.get(), slice, cnt,
                                      r->view.W, r->view.H, res->factor, res->format, render_stream));
                r->launches += 1;
            }
            if (k + 1 < nchunks) {
                result = walk(k + 1, &ticket);
                if (result != B2D_OK) break;
            }
        }
        B2D_CU(cudaEventRecord(rt[2 * k + 1].get(), render_stream));
        B2D_CU(cudaEventRecord(rendered[b].get(), render_stream));
        if (do_gather) {
            B2D_CU(cudaStreamWaitEvent(gather_stream, rendered[b].get(), 0));
            B2D_CU(cudaEventRecord(gt[2 * k].get(), gather_stream));
            if (c->ce) {
                result = ce_gather(c, b, rank * cnt * frame_bytes, cnt * frame_bytes);
                if (result != B2D_OK) break;
            } else {
                int nrc = n.AllGather(slice, c->buf[b], cnt * frame_bytes, kNcclUint8, c->comm, gather_stream);
                if (nrc != 0) { result = nccl_fail(nrc, "ncclAllGather"); break; }
            }
            B2D_CU(cudaEventRecord(gt[2 * k + 1].get(), gather_stream));
            B2D_CU(cudaEventRecord(gathered[b].get(), gather_stream));
        }
        // consumer of the chunk (gathered: world x cnt frames, rank-major; render only: this rank's cnt frames)
        B2D_CU(cudaStreamWaitEvent(consume_stream, (do_gather ? gathered[b] : rendered[b]).get(), 0));
        if (fn) fn(user, (int)k, first, cnt, do_gather ? c->buf[b] : slice, do_gather ? c->world : 1, consume_stream);
        B2D_CU(cudaEventRecord(consumed[b].get(), consume_stream));
    }
    // the end of the job on this rank: everything on the three streams
    B2D_CU(cudaStreamWaitEvent(consume_stream, rendered[(nchunks - 1) & 1].get(), 0));
    B2D_CU(cudaEventRecord(t_end.get(), consume_stream));
    cudaError_t se = cudaStreamSynchronize(consume_stream);
    if (se == cudaSuccess) se = cudaStreamSynchronize(gather_stream);
    if (se == cudaSuccess) se = cudaStreamSynchronize(render_stream);
    if (se != cudaSuccess && result == B2D_OK) result = b2d::cuda_fail(se, "cudaStreamSynchronize");
    if (result == B2D_OK && stats_out) {
        b2d_sharded_stats st;
        std::memset(&st, 0, sizeof st);
        float ms = 0.f;
        cudaEventElapsedTime(&ms, t_begin.get(), t_end.get());
        st.total_ms = ms;
        for (size_t k = 0; k < nchunks; k++) {
            cudaEventElapsedTime(&ms, rt[2 * k].get(), rt[2 * k + 1].get()); st.render_ms += ms;
            if (do_gather) { cudaEventElapsedTime(&ms, gt[2 * k].get(), gt[2 * k + 1].get()); st.gather_ms += ms; }
        }
        st.frames_local = (int64_t)per;
        st.frames_gathered = do_gather ? (int64_t)(per * world) : 0;
        st.chunks = (int64_t)nchunks;
        st.chunk_frames = (int64_t)chunk;
        st.bytes_received = do_gather ? (int64_t)((world - 1) * per * frame_bytes) : 0;
        std::strncpy(st.registration, c->registration, sizeof st.registration - 1);
        *stats_out = st;
    }
    return result;
}

// The two sharded calls, unresolved (res = NULL) or resolved (res: factor and format set).  A resolved call's factor and
// format are checked by the rule of b2d_resolve_device with the other whole-job checks, before any collective or launch.
int render_sharded(b2d_renderer *r, b2d_comm *c, const b2d_pose *poses, size_t n_total, size_t chunk_frames, int mode,
                   b2d_chunk_fn fn, void *user, b2d_sharded_stats *stats_out, ShardResolve *res) {
    int rc = check_sharded(r, c, poses, mode);
    if (rc == B2D_OK && res) rc = b2d_resolve_frame_bytes(r, res->factor, res->format, &res->frame_bytes);
    if (rc != B2D_OK || n_total == 0) return rc;
    return sharded_loop(r, c, poses, n_total, chunk_frames, mode, fn, user, stats_out, Frames{}, res);
}

int render_sharded_levels_states(b2d_renderer *r, b2d_comm *c, const b2d_pose *poses, const uint32_t *levels,
                                 const uint32_t *palettes, const b2d_frame_state *states, size_t n_total,
                                 const b2d_sector_move *moves, size_t n_moves, size_t chunk_frames, int mode, b2d_chunk_fn fn,
                                 void *user, b2d_sharded_stats *stats_out, ShardResolve *res) {
    int rc = check_sharded(r, c, poses, mode);
    if (rc == B2D_OK && res) rc = b2d_resolve_frame_bytes(r, res->factor, res->format, &res->frame_bytes);
    if (rc != B2D_OK) return rc;
    // the whole list, identical on every rank, is checked and its compact states built before anything else: every rank
    // then refuses the same input, before any collective
    CallFrames all(kFrameLevels | kFrameStates, levels, states, moves, n_moves, nullptr, palettes);
    rc = all.prepare(r, n_total);
    if (rc != B2D_OK || n_total == 0) return rc;
    // this rank's block, padded like its poses by repeating the last entry (level, palette and state with it); its
    // states stay where prepare put them
    const size_t world = (size_t)c->world, rank = (size_t)c->rank, per = (n_total + world - 1) / world;
    std::vector<uint32_t> block_levels(per), block_tables(per);
    std::vector<size_t> block_starts(per);
    for (size_t i = 0; i < per; i++) {
        const size_t g = std::min(rank * per + i, n_total - 1);
        block_levels[i] = levels[g];
        block_tables[i] = b2d::frame_table(r, levels, palettes, g);
        block_starts[i] = all.starts[g];
    }
    if (res) res->block_tables = block_tables.data();
    return sharded_loop(r, c, poses, n_total, chunk_frames, mode, fn, user, stats_out,
                        Frames{block_levels.data(), all.fs.data(), block_starts.data()}, res);
}

}  // namespace

extern "C" {

int b2d_render_sharded(b2d_renderer *r, b2d_comm *c, const b2d_pose *poses, size_t n_total, size_t chunk_frames, int mode,
                       b2d_chunk_fn fn, void *user, b2d_sharded_stats *stats_out) {
    return render_sharded(r, c, poses, n_total, chunk_frames, mode, fn, user, stats_out, nullptr);
}

int b2d_render_sharded_levels_states(b2d_renderer *r, b2d_comm *c, const b2d_pose *poses, const uint32_t *levels,
                                     const b2d_frame_state *states, size_t n_total, const b2d_sector_move *moves, size_t n_moves,
                                     size_t chunk_frames, int mode, b2d_chunk_fn fn, void *user, b2d_sharded_stats *stats_out) {
    return render_sharded_levels_states(r, c, poses, levels, nullptr, states, n_total, moves, n_moves, chunk_frames, mode, fn,
                                        user, stats_out, nullptr);
}

int b2d_render_sharded_resolved(b2d_renderer *r, b2d_comm *c, const b2d_pose *poses, size_t n_total, size_t chunk_frames,
                                int factor, int format, int mode, b2d_chunk_fn fn, void *user, b2d_sharded_stats *stats_out) {
    ShardResolve res;
    res.factor = factor; res.format = format;
    return render_sharded(r, c, poses, n_total, chunk_frames, mode, fn, user, stats_out, &res);
}

int b2d_render_sharded_levels_states_resolved(b2d_renderer *r, b2d_comm *c, const b2d_pose *poses, const uint32_t *levels,
                                              const b2d_frame_state *states, size_t n_total, const b2d_sector_move *moves,
                                              size_t n_moves, size_t chunk_frames, int factor, int format, int mode,
                                              b2d_chunk_fn fn, void *user, b2d_sharded_stats *stats_out) {
    return b2d_render_sharded_levels_states_resolved_palettes(r, c, poses, levels, nullptr, states, n_total, moves, n_moves,
                                                              chunk_frames, factor, format, mode, fn, user, stats_out);
}

int b2d_render_sharded_levels_states_resolved_palettes(b2d_renderer *r, b2d_comm *c, const b2d_pose *poses,
                                                       const uint32_t *levels, const uint32_t *palettes,
                                                       const b2d_frame_state *states, size_t n_total,
                                                       const b2d_sector_move *moves, size_t n_moves, size_t chunk_frames,
                                                       int factor, int format, int mode, b2d_chunk_fn fn, void *user,
                                                       b2d_sharded_stats *stats_out) {
    ShardResolve res;
    res.factor = factor; res.format = format;
    return render_sharded_levels_states(r, c, poses, levels, palettes, states, n_total, moves, n_moves, chunk_frames, mode, fn,
                                        user, stats_out, &res);
}

}  // extern "C"
