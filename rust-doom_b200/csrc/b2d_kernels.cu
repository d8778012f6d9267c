// sm_90a kernels of the Doom-WAD software renderer.
//
//   b2d_walk_kernel    : one CTA per frame.  Thread-parallel view transform of all vertices, per-seg
//                        projection setup and per-node-child bounding-box ranges into shared memory,
//                        then (warp 0) a front-to-back BSP walk with a warp-wide solid-column bitmask
//                        (ballot / lane-striped words) that emits the compact seg worklist.
//   b2d_raster_kernel  : one warp per (frame, 32-column strip); lane = screen column.  Consumes the
//                        worklist front to back, keeps the per-column clip window in registers,
//                        draws wall columns, floor/ceiling spans and sky from texel planes that already
//                        carry the light->colormap lookup; every pixel is written exactly once.
//   b2d_prelight_*     : build those planes once per renderer (32 light rows x texels / flats).
//   b2d_palette_kernel : index -> RGBA8 with the 256-entry palette in shared memory, 128-bit I/O;
//   b2d_palette_levels_kernel the same with a colour table per frame (a level set's frames).
//   b2d_resolve_kernel : k x k box filter of index frames through a colour table (or its luma) per frame into RGBA, RGB,
//                        planar RGB or grey frames at 1/k of the size (C17).
//
// There is no dense contraction anywhere on this path, so no tensor-core (wgmma) work: the
// kernels are integer/LSU/latency bound and are tuned against the HBM write roofline (DESIGN.md).
#include <type_traits>

#include "b2d_kernels.cuh"

namespace b2d {

namespace {

constexpr unsigned kFull = 0xFFFFFFFFu;

constexpr int kMaskWords = 128;      // up to 4096 columns
constexpr int kStackDepth = 128;

// packed per-seg / per-box visibility word in shared memory
constexpr uint32_t kVisBit = 1u << 25, kSolidBit = 1u << 24;
__device__ __forceinline__ uint32_t pack_range(int lo, int hi, uint32_t bits) {
    return (uint32_t)lo | ((uint32_t)hi << 12) | bits;
}
__device__ __forceinline__ int range_lo(uint32_t r) { return (int)(r & 0xFFFu); }
__device__ __forceinline__ int range_hi(uint32_t r) { return (int)((r >> 12) & 0xFFFu); }

// bits of columns [lo, hi] that fall into mask word w
__device__ __forceinline__ uint32_t word_bits(int w, int lo, int hi) {
    int a = max(lo, w * 32), b = min(hi, w * 32 + 31);
    if (a > b) return 0u;
    uint32_t m = 0xFFFFFFFFu >> (31 - (b - w * 32));
    return m & (0xFFFFFFFFu << (a - w * 32));
}

// warp-wide: is any column of [lo, hi] still open?  (lane-striped words + ballot)
__device__ __forceinline__ bool range_open(const uint32_t *mask, int lane, int lo, int hi, int passes) {
    bool open = false;
#pragma unroll
    for (int k = 0; k < kMaskWords / 32; k++) {
        if (k >= passes) break;              // only ceil(W / 1024) lane passes carry columns
        int w = lane + 32 * k;
        uint32_t bits = word_bits(w, lo, hi);
        if (bits & ~mask[w]) open = true;
    }
    return __any_sync(kFull, open);
}

// single lane: same test over its own range (used for per-seg culling)
__device__ __forceinline__ bool lane_range_open(const uint32_t *mask, int lo, int hi) {
    for (int w = lo >> 5; w <= (hi >> 5); w++)
        if (word_bits(w, lo, hi) & ~mask[w]) return true;
    return false;
}

__device__ __forceinline__ void mark_solid(uint32_t *mask, int lane, int lo, int hi, int passes) {
#pragma unroll
    for (int k = 0; k < kMaskWords / 32; k++) {
        if (k >= passes) break;
        int w = lane + 32 * k;
        uint32_t bits = word_bits(w, lo, hi);
        if (bits) mask[w] |= bits;
    }
}

__host__ __device__ inline size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

struct WalkSmem {
    size_t off_tx, off_tz, off_segr, off_boxr, off_node, off_ssec, off_sprr, off_sprz, off_mask, off_stack, off_list, total;
};
__host__ __device__ inline WalkSmem walk_layout(int nverts, int nsegs, int nnodes, int nss, int nsprites) {
    WalkSmem L;
    size_t o = 0;
    L.off_tx = o; o = align16(o + 4 * (size_t)nverts);
    L.off_tz = o; o = align16(o + 4 * (size_t)nverts);
    L.off_segr = o; o = align16(o + 4 * (size_t)nsegs);
    L.off_boxr = o; o = align16(o + 8 * (size_t)nnodes);
    L.off_node = o; o = align16(o + 32 * (size_t)nnodes);     // {x,y,dx,dy,rchild,lchild,-,-} per node
    L.off_ssec = o; o = align16(o + 16 * (size_t)nss);        // SSectorRec copies
    L.off_sprr = o; o = align16(o + 4 * (size_t)nsprites);    // packed column range per sprite
    L.off_sprz = o; o = align16(o + 4 * (size_t)nsprites);    // view depth per sprite (ordering inside a subsector)
    L.off_mask = o; o = align16(o + 4 * kMaskWords);
    L.off_stack = o; o = align16(o + 4 * kStackDepth);
    L.off_list = o; o = align16(o + 2 * ((size_t)nsegs + (size_t)nsprites));
    L.total = o;
    return L;
}

// 1-D bulk copy global -> shared memory through the TMA unit (cp.async.bulk, SASS UBLKCP), completion on an mbarrier.
__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t arrivals) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(arrivals));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_wait(uint64_t *bar, uint32_t parity) {      // bounded: a lost copy must not hang the GPU
    for (int spin = 0; spin < (1 << 24); spin++) {
        uint32_t done;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(smem_addr(bar)), "r"(parity) : "memory");
        if (done) return true;
    }
    return false;
}

// ------------------------------------------------------------------------------------------------
// Kernel 1: BSP walk -> worklist
// ------------------------------------------------------------------------------------------------
template <bool kStates, bool kLevels>
__global__ void __launch_bounds__(128, 7)     // 7 CTAs/SM (72 registers): 924 frames resident on an H100's 132 SMs
b2d_walk_kernel(const __grid_constant__ DeviceScene scene, const __grid_constant__ View vw, const Pose *__restrict__ poses, int n,
                FrameConst *__restrict__ frames, SegFrame *__restrict__ work, int stride, const __grid_constant__ LevelTables lt) {
    // One CTA per frame.  The per-frame setup (steps 1-3) and the worklist records (step 5) are data-parallel and
    // use all 128 threads; the traversal itself (step 4) is sequential and runs in warp 0 with the lanes working
    // on the segs of a subsector / the words of the column mask.  The kernel is latency-bound (one frame = one
    // dependent chain), so spreading the parallel phases over four warps shortens the chain directly.
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tid = threadIdx.x, nthr = blockDim.x;
    // Per-frame levels: the scene of the level resident in this CTA (copied from lt.scenes when a frame's level differs
    // from it); the shared-memory layout below and the traversal tables in it are that level's.
    DeviceScene *s_level = nullptr;
    if constexpr (kLevels) {
        __shared__ DeviceScene s_lv;
        s_level = &s_lv;
    }
    const DeviceScene &sc = kLevels ? *s_level : scene;
    WalkSmem L = kLevels ? WalkSmem{} : walk_layout(sc.nverts, sc.nsegs, sc.nnodes, sc.nss, sc.nsprites);   // levels: per frame
    uint8_t *base = smem;
    __shared__ int s_count, s_status;
    __shared__ __align__(8) uint64_t s_bar;
    int32_t *tx = reinterpret_cast<int32_t *>(base + L.off_tx);
    int32_t *tz = reinterpret_cast<int32_t *>(base + L.off_tz);
    uint32_t *segr = reinterpret_cast<uint32_t *>(base + L.off_segr);
    uint32_t *boxr = reinterpret_cast<uint32_t *>(base + L.off_boxr);
    int4 *node_s = reinterpret_cast<int4 *>(base + L.off_node);       // traversal reads shared memory, not L2
    int4 *ssec_s = reinterpret_cast<int4 *>(base + L.off_ssec);
    uint32_t *sprr = reinterpret_cast<uint32_t *>(base + L.off_sprr);
    int32_t *sprz = reinterpret_cast<int32_t *>(base + L.off_sprz);
    uint32_t *mask = reinterpret_cast<uint32_t *>(base + L.off_mask);
    uint32_t *stack = reinterpret_cast<uint32_t *>(base + L.off_stack);
    uint16_t *list = reinterpret_cast<uint16_t *>(base + L.off_list);

    // One frame per CTA when the grid has a CTA per frame; a smaller (persistent) grid loops: that is the form for running
    // under another batch's raster -- a CTA per SM keeps the walk's footprint at 1/8 of the register file while it takes
    // a few frame latencies, all hidden behind the raster (launch_walk).
    // The traversal tables (node partition lines + children, subsector records) do not depend on the frame: one bulk copy
    // per CTA brings them into shared memory while the threads are busy with steps 1-3 of the first frame.  With per-frame
    // levels they are copied again whenever a frame's level differs from the resident one (each copy completes one phase
    // of the mbarrier: `parity` is the phase the next wait is for).
    uint32_t static_bytes = 0, parity = 0, resident = 0xFFFFFFFFu;
    bool static_pending = false;
    if constexpr (kLevels) {
        if (tid == 0) mbar_init(&s_bar, 1);
    } else {
        static_bytes = 32u * (uint32_t)sc.nnodes + 16u * (uint32_t)sc.nss;
    }
    if (static_bytes) {
        if (tid == 0) mbar_init(&s_bar, 1);
        __syncthreads();
        if (tid == 0) bulk_copy_g2s(node_s, sc.walk_static, static_bytes, &s_bar);
        static_pending = true;
    }
    for (int frame = blockIdx.x; frame < n; frame += gridDim.x) {
    if constexpr (kLevels) {
        const uint32_t level = lt.frame_level[frame];
        if (level != resident) {
            // The previous frame ended in __syncthreads(): nothing reads the old scene or tables any more.  Generic-proxy
            // accesses to the shared memory the bulk copy overwrites are ordered before it (fence.proxy.async).
            const uint32_t *src = reinterpret_cast<const uint32_t *>(lt.scenes + level);
            uint32_t *dst = reinterpret_cast<uint32_t *>(s_level);
            for (int i = tid; i < (int)(sizeof(DeviceScene) / 4); i += nthr) dst[i] = src[i];
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            L = walk_layout(sc.nverts, sc.nsegs, sc.nnodes, sc.nss, sc.nsprites);
            tx = reinterpret_cast<int32_t *>(base + L.off_tx);
            tz = reinterpret_cast<int32_t *>(base + L.off_tz);
            segr = reinterpret_cast<uint32_t *>(base + L.off_segr);
            boxr = reinterpret_cast<uint32_t *>(base + L.off_boxr);
            node_s = reinterpret_cast<int4 *>(base + L.off_node);
            ssec_s = reinterpret_cast<int4 *>(base + L.off_ssec);
            sprr = reinterpret_cast<uint32_t *>(base + L.off_sprr);
            sprz = reinterpret_cast<int32_t *>(base + L.off_sprz);
            mask = reinterpret_cast<uint32_t *>(base + L.off_mask);
            stack = reinterpret_cast<uint32_t *>(base + L.off_stack);
            list = reinterpret_cast<uint16_t *>(base + L.off_list);
            static_bytes = 32u * (uint32_t)sc.nnodes + 16u * (uint32_t)sc.nss;
            if (static_bytes) {
                if (tid == 0) bulk_copy_g2s(node_s, sc.walk_static, static_bytes, &s_bar);
                static_pending = true;
            }
            resident = level;
        }
    }
    FrameConst fc;
    frame_setup(poses[frame], fc);
    uint32_t set = 0;                   // per-frame states: this frame's table set, and its tables
    TableSet fs{};
    if (kStates) {
        set = lt.frame_set[frame];
        fs = lt.sets[set];
    }

    // 1. all vertices into view space (lane-parallel)
    for (int i = tid; i < sc.nverts; i += nthr) {
        int32_t vx = sc.verts[2 * i], vy = sc.verts[2 * i + 1];
        int32_t a, b;
        to_view(fc, vx, vy, a, b);
        tx[i] = a; tz[i] = b;
    }
    __syncthreads();

    // 2. per-seg exact column interval + static/solid flags (lane-parallel, 64-bit setup)
    for (int i = tid; i < sc.nsegs; i += nthr) {
        const SegRec &S = (kStates ? fs.segs : sc.segs)[i];
        uint32_t packed = 0;
        int32_t flags = S.flags;
        if (!(flags & kSegInvalid)) {
            SegFrame sf;
            const bool closes = seg_closes(flags & kSegTwoSided, S.otop, S.obot);
            if (seg_frame_setup(vw, tx[S.v1], tz[S.v1], tx[S.v2], tz[S.v2], sf, closes))
                packed = pack_range(sf.xlo, sf.xhi, kVisBit | (seg_solid(closes, sf) ? kSolidBit : 0u));
        }
        segr[i] = packed;
    }
    // 3. conservative column range of both child boxes of every node
    for (int i = tid; i < 2 * sc.nnodes; i += nthr) {
        const NodeRec &N = sc.nodes[i >> 1];
        const int32_t *box = (i & 1) ? N.lbox : N.rbox;
        int32_t b4[4] = {box[0], box[1], box[2], box[3]};
        int lo, hi;
        boxr[i] = box_range(fc, vw, b4, lo, hi) ? pack_range(lo, hi, kVisBit) : 0u;
    }
    if (static_pending) {                        // first frame of this CTA (or level): the bulk copy has had steps 1-3 to land
        if (!mbar_wait(&s_bar, kLevels ? parity : 0u)) __trap();
        static_pending = false;
        if (kLevels) parity ^= 1u;
    }
    for (int i = tid; i < sc.nsprites; i += nthr) {          // decoration sprites: exact column interval
        const SpriteRec &P = (kStates ? fs.sprites : sc.sprites)[i];
        SpriteFrame sp;
        uint32_t packed = 0;
        sp.cz = 0;
        if (P.tex >= 0 && P.tex < sc.ntex && sprite_setup(fc, vw, P.x, P.y, (int32_t)(kStates ? fs.tex : sc.tex)[P.tex].w, sp))
            packed = pack_range(sp.lo, sp.hi, kVisBit);
        sprr[i] = packed;
        sprz[i] = (int32_t)sp.cz;
    }
    // solid-column mask: columns >= W start out solid
    for (int w = tid; w < kMaskWords; w += nthr) mask[w] = ~word_bits(w, 0, vw.W - 1);
    if (tid == 0) stack[0] = sc.root;
    __syncthreads();

    // 4. front-to-back traversal in warp 0 (control flow is warp-uniform)
    const int passes = (vw.W + 1023) / 1024;
    int sp = warp == 0 ? 1 : 0, count = 0, status = 0;
    int budget = 2 * (sc.nnodes + sc.nss) + 64;      // a corrupt BSP with a cycle must not hang the GPU
    while (sp > 0) {
        if (--budget < 0) { status |= kStatusNoTermination; break; }
        uint32_t child = stack[--sp];
        __syncwarp();
        if (child & kLeaf) {
            uint32_t id = child & 0x7FFFFFFFu;
            if (id >= (uint32_t)sc.nss) continue;
            const int4 ssv = ssec_s[id];
            SSectorRec ss;
            ss.first_seg = ssv.x; ss.num_segs = ssv.y; ss.sector = ssv.z; ss.sprites = ssv.w;
            if (ss.sector < 0) continue;
            {   // the subsector's decoration sprites come first: they stand in front of its far segs.  Among themselves
                // nearest first (drawn back to front, the nearer billboard ends up on top); ties keep the stored order.
                // A lane's slot = the number of visible sprites of the subsector that sort before its own.
                const int sfirst = ss.sprites & 0xFFFFFF;
                int scnt = (ss.sprites >> 24) & 0xFF;
                if (sfirst + scnt > sc.nsprites) scnt = sc.nsprites > sfirst ? sc.nsprites - sfirst : 0;
                int nvis = 0;
                for (int k0 = 0; k0 < scnt; k0 += 32) {
                    const int k = k0 + lane, pi = sfirst + k;
                    const uint32_t r = k < scnt ? sprr[pi] : 0u;
                    const bool vis = (r & kVisBit) && lane_range_open(mask, range_lo(r), range_hi(r));
                    int rank = 0, total = 0;
                    const int32_t myz = vis ? sprz[pi] : 0;
                    for (int j0 = 0; j0 < scnt; j0 += 32) {                 // warp-uniform loop over all sprites of the subsector
                        const int j = j0 + lane, pj = sfirst + j;
                        const uint32_t rj = j < scnt ? sprr[pj] : 0u;
                        const bool vj = (rj & kVisBit) && lane_range_open(mask, range_lo(rj), range_hi(rj));
                        const int32_t zj = vj ? sprz[pj] : 0;
                        unsigned mj = __ballot_sync(kFull, vj);
                        total += __popc(mj);
                        while (mj) {
                            const int b = __ffs(mj) - 1;
                            mj &= mj - 1;
                            const int32_t zb = __shfl_sync(kFull, zj, b);
                            const int jb = j0 + b;
                            if (vis && (zb < myz || (zb == myz && jb < k))) rank++;
                        }
                    }
                    const int pos = count + rank;
                    if (vis && pos < sc.nsegs + sc.nsprites) list[pos] = (uint16_t)(sc.nsegs + pi);
                    nvis = total;
                }
                count = min(count + nvis, sc.nsegs + sc.nsprites);
                __syncwarp();
            }
            for (int k0 = 0; k0 < ss.num_segs; k0 += 32) {
                int k = k0 + lane;
                int si = ss.first_seg + k;
                uint32_t r = k < ss.num_segs ? segr[si] : 0u;
                bool vis = (r & kVisBit) && lane_range_open(mask, range_lo(r), range_hi(r));
                unsigned m = __ballot_sync(kFull, vis);
                int pos = count + __popc(m & ((1u << lane) - 1u));
                if (vis && pos < sc.nsegs + sc.nsprites) list[pos] = (uint16_t)si;
                count = min(count + __popc(m), sc.nsegs + sc.nsprites);
                unsigned sm = __ballot_sync(kFull, vis && (r & kSolidBit));
                __syncwarp();
                while (sm) {
                    int j = __ffs(sm) - 1;
                    sm &= sm - 1;
                    uint32_t rj = __shfl_sync(kFull, r, j);
                    mark_solid(mask, lane, range_lo(rj), range_hi(rj), passes);
                }
                __syncwarp();
            }
            if (!range_open(mask, lane, 0, vw.W - 1, passes)) break;     // every column is closed
        } else {
            if (child >= (uint32_t)sc.nnodes) continue;
            const int4 nl = node_s[2 * child], nc = node_s[2 * child + 1];
            int side = node_side(fc.pose, nl.x, nl.y, nl.z, nl.w);   // 1: left child is near
            uint32_t near_c = (uint32_t)(side ? nc.y : nc.x), far_c = (uint32_t)(side ? nc.x : nc.y);
            uint32_t rn = boxr[2 * child + side], rf = boxr[2 * child + (side ^ 1)];
            bool far_vis = (rf & kVisBit) && range_open(mask, lane, range_lo(rf), range_hi(rf), passes);
            bool near_vis = (rn & kVisBit) && range_open(mask, lane, range_lo(rn), range_hi(rn), passes);
            int need = (far_vis ? 1 : 0) + (near_vis ? 1 : 0);
            if (sp + need > kStackDepth) { status = kStatusStackOverflow; break; }
            if (lane == 0) {
                int p = sp;
                if (far_vis) stack[p++] = far_c;
                if (near_vis) stack[p++] = near_c;
            }
            sp += need;
            __syncwarp();
        }
    }
    __syncwarp();
    if (warp == 0 && lane == 0) {
        if (count > stride) { count = stride; status |= kStatusWorklistFull; }
        s_count = count; s_status = status;
    }
    __syncthreads();
    count = s_count; status = s_status;

    // 5. worklist records (thread-parallel): the projection coefficients of each emitted seg
    for (int k = tid; k < count; k += nthr) {
        int si = list[k];
        SegFrame sf;
        if (si >= sc.nsegs) {
            const int pi = si - sc.nsegs;
            const SpriteRec &P = (kStates ? fs.sprites : sc.sprites)[pi];
            SpriteFrame sp;
            sprite_setup(fc, vw, P.x, P.y, (int32_t)(kStates ? fs.tex : sc.tex)[P.tex].w, sp);
            sprite_entry(pi, sp, sf);
            work[(size_t)frame * stride + k] = sf;
            continue;
        }
        const SegRec &S = (kStates ? fs.segs : sc.segs)[si];
        seg_frame_setup(vw, tx[S.v1], tz[S.v1], tx[S.v2], tz[S.v2], sf, false);
        sf.seg = si;
        work[(size_t)frame * stride + k] = sf;
    }
    if (tid == 0) {
        if (status) atomicOr(sc.status_flag, status);
        fc.count = count;
        fc.status = status;
#pragma unroll
        for (int i = 0; i < 4; i++) fc.pad[i] = 0;
        fc.set = kStates ? (int32_t)set : 0;           // the raster reads the frame's tables from the same set
        fc.level = kLevels ? (int32_t)resident : 0;    // ... and the frame's scene from its level
        frames[frame] = fc;
    }
    __syncthreads();                              // the next frame of this CTA reuses the shared-memory tables
    }
}

// ------------------------------------------------------------------------------------------------
// Kernel 2: raster
// ------------------------------------------------------------------------------------------------
// shared-memory accesses by 32-bit shared-window address: keeps the per-pixel address arithmetic to one
// add (the generic-pointer form re-derives the window base for every access)
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}

// A frame's fixed colormap (kFixed raster variant, FixedTables): COLORMAP row `row` (-1: none) and the row-32 planes
// of its level.
struct FixedWarp {
    const uint8_t *texels, *flats;
    int row;
};

struct RasterCtx {
    const DeviceScene *sc;
    FixedWarp fix;             // kFixed variant only
    uint32_t pal_s;            // ... of the palette (rgba only)
    uint2 *rowz;               // this warp's 32-entry staging of per-row plane constants {depth Q8, plane offset / 64}
    PlaneDir dir;              // direction of this lane's column ray (Q18), for the flat texel
    uint8_t *fb;               // &index_fb[frame][0][x]
    uint32_t *rgba;            // &rgba_fb[frame][0][x] or nullptr
    int W, H, x, lane;
    uint32_t skycol;
};

template <bool kRgba>
__device__ __forceinline__ void put_px(const RasterCtx &c, uint8_t *p8, uint32_t *p32, bool on, uint32_t v) {
    if (on) {
        // Index-only kernels store with st.global.cs (streaming: evict-first in L1 and L2).  The raster writes every
        // index byte once and never reads it back, while every warp re-reads the pre-lit texel and flat planes; the frames
        // in flight are larger than the L2, and default stores push those planes out.  With RGBA output, whose lines
        // are four times as many, evict-first index lines leave L2 before they are complete and the kernel is slower,
        // so those kernels keep default stores (DESIGN.md §6).
        if (kRgba) {
            *p8 = (uint8_t)v;
            *p32 = lds_u32(c.pal_s + 4u * v);
        } else {
            __stcs(p8, (uint8_t)v);
        }
    }
}

__host__ __device__ __forceinline__ bool tex_interleaved(const TexRec &T) { return b2d::tex_interleaved(T.h, T.texel_off); }

// Rows are produced in batches of kBatch: all texel loads first, then all colormap lookups, then the stores.
// Issuing the independent loads back to back keeps kBatch of them in flight per warp (the one-row-at-a-time
// form serialises load -> lookup -> store and leaves the LSU idle while each warp waits).  `full` (warp-uniform)
// says every lane owns all rows of the batch, so the stores need no predicate.
constexpr int kBatch = 8;

template <bool kRgba, int kW>
__device__ __forceinline__ void store_batch(const RasterCtx &c, uint8_t *p8, uint32_t *p32, const uint32_t (&v)[kBatch],
                                            int y, int ya, int yb, bool full) {
    const int Wc = kW ? kW : c.W;
    if (full) {
#pragma unroll
        for (int k = 0; k < kBatch; k++) put_px<kRgba>(c, p8 + (size_t)k * Wc, kRgba ? p32 + (size_t)k * Wc : nullptr, true, v[k]);
    } else {
        const uint32_t m = row_mask(y, ya, yb, kBatch);      // one bit test per row instead of two compares
#pragma unroll
        for (int k = 0; k < kBatch; k++)
            put_px<kRgba>(c, p8 + (size_t)k * Wc, kRgba ? p32 + (size_t)k * Wc : nullptr, (m >> k) & 1u, v[k]);
    }
}

// rows [ya, yb) of this lane's column := void (index 0); lanes with ya >= yb idle
template <bool kRgba, int kW>
__device__ __forceinline__ void fill_void_warp(const RasterCtx &c, int ya, int yb) {
    bool act = ya < yb;
    int y0 = __reduce_min_sync(kFull, act ? ya : 0x7FFFFFFF);
    int y1 = __reduce_max_sync(kFull, act ? yb : 0);
    if (y0 >= y1) return;
    const int Wc = kW ? kW : c.W;
    uint8_t *p8 = c.fb + (size_t)y0 * Wc;
    uint32_t *p32 = kRgba ? c.rgba + (size_t)y0 * Wc : nullptr;
#pragma unroll 1
    for (int y = y0; y < y1; y++, p8 += Wc, p32 += Wc) put_px<kRgba>(c, p8, p32, y >= ya && y < yb, 0u);
}

template <bool kRgba, int kW>
__device__ __forceinline__ void draw_sky_warp(const RasterCtx &c, int ya, int yb) {
    const DeviceScene &sc = *c.sc;
    if (sc.sky_tex < 0) { fill_void_warp<kRgba, kW>(c, ya, yb); return; }
    const TexRec T = sc.tex[sc.sky_tex];
    const bool inter = tex_interleaved(T);
    const uint8_t *px = sc.lit_texels + T.texel_off + (inter ? 4u * c.skycol : c.skycol);   // light row 0
    const uint32_t w4 = 4u * T.w;
    bool act = ya < yb;
    int y0 = __reduce_min_sync(kFull, act ? ya : 0x7FFFFFFF);
    int y1 = __reduce_max_sync(kFull, act ? yb : 0);
    if (y0 >= y1) return;
    const int Wc = kW ? kW : c.W;
    uint8_t *p8 = c.fb + (size_t)y0 * Wc;
    uint32_t *p32 = kRgba ? c.rgba + (size_t)y0 * Wc : nullptr;
#pragma unroll 2
    for (int y = y0; y < y1; y++, p8 += Wc, p32 += Wc) {
        const uint32_t r = sc.skyrow[y];                                   // warp-uniform table entry
        put_px<kRgba>(c, p8, p32, y >= ya && y < yb, __ldg(px + (inter ? (r >> 2) * w4 + (r & 3u) : r * T.w)));
    }
}

template <bool kRgba, int kW, bool kFixed = false>
__device__ __forceinline__ void draw_plane_warp(const RasterCtx &c, const FrameConst &fc, const View &vw,
                                                int ya, int yb, int32_t h, int32_t flat, int lightb,
                                                bool visible) {
    const DeviceScene &sc = *c.sc;
    if (!__any_sync(kFull, ya < yb)) return;
    if (!visible) { fill_void_warp<kRgba, kW>(c, ya, yb); return; }
    if (flat == kFlatSky) { draw_sky_warp<kRgba, kW>(c, ya, yb); return; }
    if (flat < 0 || flat >= sc.nflats) { fill_void_warp<kRgba, kW>(c, ya, yb); return; }
    // the pre-lit flats start at a multiple of 4 GiB (b2d_api.cu alloc_aligned_4g): a texel's address is {high word,
    // 32-bit offset} -- no 64-bit add per pixel
    const uint8_t *lit_flats = sc.lit_flats;
    int fixed_row = -1;
    if constexpr (kFixed) {      // a fixed colormap: every row of the plane on one pre-lit plane (row 32: the level's own)
        lit_flats = c.fix.row == 32 ? c.fix.flats : lit_flats;
        fixed_row = c.fix.row == 32 ? 0 : c.fix.row;
    }
    const uint64_t px_hi = reinterpret_cast<uint64_t>(lit_flats) & 0xFFFFFFFF00000000ull;   // low word is zero: tell the compiler
    const uint32_t habs = plane_habs(h, fc.pose.z);
    bool act = ya < yb;
    int y0 = __reduce_min_sync(kFull, act ? ya : 0x7FFFFFFF);
    int y1 = __reduce_max_sync(kFull, act ? yb : 0);
    const int full_lo = __reduce_max_sync(kFull, act ? ya : 0x7FFFFFFF);
    const int full_hi = __reduce_min_sync(kFull, act ? yb : 0);
    const int Wc = kW ? kW : c.W;
    uint8_t *p8 = c.fb + (size_t)y0 * Wc;
    uint32_t *p32 = kRgba ? c.rgba + (size_t)y0 * Wc : nullptr;
    const uint32_t bu = (uint32_t)fc.pose.x << 10, bv = (uint32_t)fc.pose.y << 10;
    const uint32_t ax = (uint32_t)c.dir.ax, ay = (uint32_t)c.dir.ay;
    for (int yc = y0; yc < y1; yc += 32) {
        // lane j prepares the constants of row yc+j (64-bit maths, once per row per warp): view depth and plane offset
        int yy = yc + c.lane;
        if (yy < y1) {
            const PlaneRow pr = plane_row(habs, sc.yslope[yy]);
            // plane + flat offset / 64: the texel offset is then two instructions, LEA.HI (cm6 + (U >> 26)) and a funnel
            // shift ((.) << 6 | V >> 26)
            c.rowz[c.lane] = make_uint2(pr.z8q, (sc.lit_flat_stride >> 6) * (uint32_t)(kFixed && fixed_row >= 0 ? fixed_row : light_row(lightb, pr.z8)) + 64u * (uint32_t)flat);
        }
        __syncwarp();
        const int rows = min(32, y1 - yc);
        int j = 0;
        for (; j + kBatch <= rows; j += kBatch, p8 += (size_t)kBatch * Wc, p32 += (size_t)kBatch * Wc) {
            uint32_t v[kBatch];
#pragma unroll
            for (int k = 0; k < kBatch; k++) {
                const uint2 rz = c.rowz[j + k];                               // shared-memory broadcast: one 64-bit word per row
                v[k] = __ldg(reinterpret_cast<const uint8_t *>(px_hi | flat_offset(rz.y, bu + rz.x * ax, bv + rz.x * ay)));   // always in bounds
            }
            const int y = yc + j;
            store_batch<kRgba, kW>(c, p8, p32, v, y, ya, yb, y >= full_lo && y + kBatch <= full_hi);
        }
        for (; j < rows; j++, p8 += Wc, p32 += Wc) {
            const uint2 rz = c.rowz[j];
            const int y = yc + j;
            put_px<kRgba>(c, p8, p32, y >= ya && y < yb,
                          __ldg(reinterpret_cast<const uint8_t *>(px_hi | flat_offset(rz.y, bu + rz.x * ax, bv + rz.x * ay))));
        }
        __syncwarp();
    }
}

// Magnified wall columns (every lane's texture step <= kWallFast8 / kWallFast16, b2d_math.cuh): R rows per batch from
// two aligned word loads, the row quad tracked incrementally -- per pixel one IMAD + one shift (byte index), one PRMT, one store.
template <bool kRgba, int kW, int R>
__device__ __forceinline__ void wall_fast_loop(const RasterCtx &c, const uint8_t *plq, uint32_t w4, uint32_t nq, uint32_t q,
                                               uint32_t acc, uint32_t ts29, int y0, int y1, int ya, int yb,
                                               int full_lo, int full_hi) {
    const int Wc = kW ? kW : c.W;
    uint8_t *p8 = c.fb + (size_t)y0 * Wc;
    uint32_t *p32 = kRgba ? c.rgba + (size_t)y0 * Wc : nullptr;
    asm("" : "+l"(plq));       // keep the column's plane pointer whole: one IMAD.WIDE per load instead of re-adding the base
#pragma unroll 1
    for (int y = y0; y < y1; y += R, p8 += (size_t)R * Wc, p32 += (size_t)R * Wc) {
        const uint32_t q1 = q + 1u == nq ? 0u : q + 1u;
        const uint32_t w0 = __ldg(reinterpret_cast<const uint32_t *>(plq + (size_t)q * w4));
        const uint32_t w1 = __ldg(reinterpret_cast<const uint32_t *>(plq + (size_t)q1 * w4));
        if (y >= full_lo && y + R <= full_hi) {
#pragma unroll
            for (int k = 0; k < R; k++) {
                uint32_t v = pick_byte(w0, w1, wall_sel(acc, ts29, (uint32_t)k));
                if (kRgba) v &= 0xFFu;
                put_px<kRgba>(c, p8 + (size_t)k * Wc, kRgba ? p32 + (size_t)k * Wc : nullptr, true, v);
            }
        } else {
            const uint32_t m = row_mask(y, ya, yb, R);
#pragma unroll
            for (int k = 0; k < R; k++) {
                uint32_t v = pick_byte(w0, w1, wall_sel(acc, ts29, (uint32_t)k));
                if (kRgba) v &= 0xFFu;
                put_px<kRgba>(c, p8 + (size_t)k * Wc, kRgba ? p32 + (size_t)k * Wc : nullptr, (m >> k) & 1u, v);
            }
        }
        wall_advance(acc, q, ts29, (uint32_t)R, nq);
    }
}

// `row`: the lane's light row; with a fixed colormap (kFixed) its row, 32 meaning the level's row-32 plane
template <bool kRgba, int kW, bool kFixed = false>
__device__ __forceinline__ void draw_wall_warp(const RasterCtx &c, const FrameConst &fc, int ya, int yb,
                                               int32_t tex, int32_t tA, int32_t hA, int32_t ucol,
                                               int32_t iscale, int row) {
    const DeviceScene &sc = *c.sc;
    if (!__any_sync(kFull, ya < yb)) return;
    if (tex < 0 || tex >= sc.ntex) { fill_void_warp<kRgba, kW>(c, ya, yb); return; }
    const TexRec T = sc.tex[tex];
    bool act = ya < yb;
    const uint32_t col = (uint32_t)floormod32(ucol, (int32_t)T.w);
    const uint8_t *pl = sc.lit_texels + (size_t)row * sc.lit_texel_stride + T.texel_off;   // this lane's light plane
    if constexpr (kFixed) {
        if (row == 32) pl = c.fix.texels + T.texel_off;
    }
    const uint32_t tstep = (uint32_t)(iscale >> 4);
    int y0 = __reduce_min_sync(kFull, act ? ya : 0x7FFFFFFF);
    int y1 = __reduce_max_sync(kFull, act ? yb : 0);
    const int full_lo = __reduce_max_sync(kFull, act ? ya : 0x7FFFFFFF);
    const int full_hi = __reduce_min_sync(kFull, act ? yb : 0);
    uint32_t t = (uint32_t)wall_tbase(tA, hA, fc.pose.z, c.H, iscale) + (uint32_t)y0 * tstep;
    const int Wc = kW ? kW : c.W;
    uint8_t *p8 = c.fb + (size_t)y0 * Wc;
    uint32_t *p32 = kRgba ? c.rgba + (size_t)y0 * Wc : nullptr;
    // Texel loads are unconditional (t is a bounded linear function of y for every lane, so the row index
    // is always inside the texture); only the store is predicated.  That keeps the loops branch-free.
    if (tex_interleaved(T) && T.h >= 8u) {
        // magnified columns: the whole piece runs on the incremental path when every lane qualifies (inactive lanes step 0)
        const uint32_t ts = act ? tstep : 0u;
        const bool f16 = __all_sync(kFull, ts <= kWallFast16);
        if (f16 || __all_sync(kFull, ts <= kWallFast8)) {
            const uint32_t tt = act ? t : 0u;
            const uint32_t r0 = wall_row((int32_t)tt, T.h, T.hmagic, T.hbias);
            const uint8_t *plq = pl + 4u * col;
            if (f16) wall_fast_loop<kRgba, kW, 16>(c, plq, 4u * T.w, T.h >> 2, r0 >> 2, wall_acc29(tt, r0), ts << 13, y0, y1, ya, yb, full_lo, full_hi);
            else wall_fast_loop<kRgba, kW, 8>(c, plq, 4u * T.w, T.h >> 2, r0 >> 2, wall_acc29(tt, r0), ts << 13, y0, y1, ya, yb, full_lo, full_hi);
            return;
        }
    }
    if (tex_interleaved(T)) {
        // 4-row interleaved plane.  Rows of a batch: u_k = asr(t + k*tstep, 16), texture row = floormod(u_k, h).
        // With r0 the row of the first pixel, pixel k reads byte (r0 & 3) + u_k - u_0 of the 8 bytes made of row
        // quad r0 >> 2 and the next one (wrapping at h, a multiple of 4).  If that byte index stays below 8 for
        // every lane -- the column is magnified -- two aligned word loads serve the whole batch.
        const uint32_t colb = 4u * col, w4 = 4u * T.w;
        for (int y = y0; y < y1; y += kBatch, p8 += (size_t)kBatch * Wc, p32 += (size_t)kBatch * Wc, t += (uint32_t)kBatch * tstep) {
            const uint32_t r0 = wall_row((int32_t)t, T.h, T.hmagic, T.hbias);
            // acc = t with its integer part replaced by r0 & 3: byte index of pixel k = (acc + k*tstep) >> 16
            const uint32_t acc = wall_acc(t, r0);
            const uint32_t b7 = (acc + 7u * tstep) >> 16;
            uint32_t v[kBatch];
            if (__all_sync(kFull, b7 < 8u)) {
                const uint32_t q0 = r0 >> 2, q1 = next_quad(q0, T.h);
                const uint32_t w0 = __ldg(reinterpret_cast<const uint32_t *>(pl + (q0 * w4 + colb)));
                const uint32_t w1 = __ldg(reinterpret_cast<const uint32_t *>(pl + (q1 * w4 + colb)));
#pragma unroll
                for (int k = 0; k < kBatch; k++) {
                    v[k] = pick_byte(w0, w1, (acc + (uint32_t)k * tstep) >> 16);
                    if (kRgba) v[k] &= 0xFFu;
                }
            } else {
                // less magnified: re-anchor after 4 rows -- two word pairs serve the batch as long as each half
                // stays inside two row quads (up to ~1.3 texture rows per screen row); byte loads otherwise
                const uint32_t t4 = t + 4u * tstep;
                const uint32_t r4 = wall_row((int32_t)t4, T.h, T.hmagic, T.hbias);
                const uint32_t acc4 = wall_acc(t4, r4);
                if (__all_sync(kFull, ((acc + 3u * tstep) >> 16) < 8u && ((acc4 + 3u * tstep) >> 16) < 8u)) {
                    const uint32_t q0 = r0 >> 2, q4 = r4 >> 2;
                    const uint32_t a0 = __ldg(reinterpret_cast<const uint32_t *>(pl + (q0 * w4 + colb)));
                    const uint32_t a1 = __ldg(reinterpret_cast<const uint32_t *>(pl + (next_quad(q0, T.h) * w4 + colb)));
                    const uint32_t b0 = __ldg(reinterpret_cast<const uint32_t *>(pl + (q4 * w4 + colb)));
                    const uint32_t b1 = __ldg(reinterpret_cast<const uint32_t *>(pl + (next_quad(q4, T.h) * w4 + colb)));
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        v[k] = pick_byte(a0, a1, (acc + (uint32_t)k * tstep) >> 16);
                        v[k + 4] = pick_byte(b0, b1, (acc4 + (uint32_t)k * tstep) >> 16);
                        if (kRgba) { v[k] &= 0xFFu; v[k + 4] &= 0xFFu; }
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < kBatch; k++) {
                        const uint32_t rk = wall_row((int32_t)(t + (uint32_t)k * tstep), T.h, T.hmagic, T.hbias);
                        v[k] = __ldg(pl + ((rk >> 2) * w4 + colb + (rk & 3u)));
                    }
                }
            }
            // rows past y1 belong to no lane: the predicated form drops them, so there is no tail loop
            store_batch<kRgba, kW>(c, p8, p32, v, y, ya, yb, y >= full_lo && y + kBatch <= full_hi);
        }
    } else {
        // heights that are not a multiple of 4 (patches used as textures, odd PWAD content): rare, kept small
        const uint8_t *px = pl + col;
#pragma unroll 1
        for (int y = y0; y < y1; y++, p8 += Wc, p32 += Wc, t += tstep)
            put_px<kRgba>(c, p8, p32, y >= ya && y < yb, __ldg(px + wall_row((int32_t)t, T.h, T.hmagic, T.hbias) * T.w));
    }
}

// Deferred masked entries (33 words: worklist index + one packed window per lane) live in a per-launch arena of
// kMaskedChunk-entry chunks handed out by an atomic counter; a warp keeps the ids of its chunks in shared memory.  Memory
// follows what frames actually defer (a few entries per strip) instead of strips x cap x batch.
__device__ __forceinline__ uint32_t *masked_entry(const DeviceScene &sc, const uint32_t *chunks, int e) {
    return sc.masked_list + ((size_t)chunks[e / kMaskedChunk] * kMaskedChunk + (size_t)(e % kMaskedChunk)) * 33u;
}
// next entry of this warp, or nullptr when the strip's cap or the arena is exhausted (frames incomplete)
__device__ __forceinline__ uint32_t *masked_push(const DeviceScene &sc, uint32_t *chunks, int &mcount, int lane) {
    bool ok = mcount < sc.masked_cap;
    if (ok && mcount % kMaskedChunk == 0) {
        uint32_t id = 0;
        if (lane == 0) id = atomicAdd(sc.masked_counter, 1u);
        id = __shfl_sync(kFull, id, 0);
        ok = id < sc.masked_chunks;
        if (ok && lane == 0) chunks[mcount / kMaskedChunk] = id;
        __syncwarp();
    }
    if (!ok) {
        if (lane == 0) atomicOr(sc.status_flag, kStatusMaskedFull);
        return nullptr;
    }
    return masked_entry(sc, chunks, mcount++);
}

// Back-to-front pass over the masked middle textures this strip deferred during the solid pass.  Each entry
// holds the worklist index and, per lane, the clip window [ya, yb) that was open behind the seg when the
// front-to-back walk reached it (the per-column silhouette of everything nearer).  Texels whose opacity plane
// is 0 leave the pixel as the solid pass drew it (static.frag:21-22).  Kept out of line so that the
// register allocation of the solid pass is not affected.  kStates and kLevels only give each raster variant its own copy
// (one caller each, so that what the compiler propagates into it from its caller stays as it is).  The kFixed variant
// takes the frame's fixed colormap as two more arguments, its row-32 texel plane and its row (`fix`: empty in the others,
// whose arguments stay as they are).
template <bool kRgba, int kW, bool kStates, bool kLevels, typename... Fix>
__device__ __noinline__ void masked_pass(const DeviceScene &sc, const View &vw, int32_t pose_z, uint8_t *fb,
                                         uint32_t *rgba, uint32_t pal_s, int x, int lane,
                                         const SegFrame *wl, const uint32_t *chunks, int count, Fix... fix) {
    constexpr bool kFixed = sizeof...(Fix) != 0;
    static_assert(sizeof...(Fix) == 0 || sizeof...(Fix) == 2, "the fixed colormap: the row-32 texel plane and the row");
    struct { const uint8_t *texels; int row; } const fw{fix...};     // the row-32 texel plane and the row
    // everything arrives by value (or points at kernel parameters): taking the address of the solid pass's
    // register-resident context would force it into local memory
    RasterCtx c;
    c.sc = &sc; c.pal_s = pal_s; c.fb = fb; c.rgba = rgba;
    c.W = vw.W; c.H = vw.H; c.x = x; c.lane = lane;
    const int Wc = kW ? kW : c.W;
    for (int e = count - 1; e >= 0; e--) {
        const uint32_t *ml = masked_entry(sc, chunks, e);
        const uint32_t k = ml[0];
        const uint32_t packed = ml[1 + c.lane];
        int ya = (int)(packed & 0xFFFFu), yb = (int)(packed >> 16);
        const SegFrame sf = wl[k];
        int32_t tex, tA, hA, ucol = 0, iscale = 1, row = 0;
        if (is_sprite_entry(sf)) {
            // decoration sprite (billboard at constant depth): everything but the column is warp-uniform
            SpriteFrame sp;
            const SpriteRec P = sc.sprites[entry_sprite(sf, sp)];
            if (P.tex < 0 || P.tex >= sc.ntex) continue;
            const int32_t sw = (int32_t)sc.tex[P.tex].w, sh = (int32_t)sc.tex[P.tex].h;
            const int64_t scale = sprite_scale(vw, sp.cz);      // >= 1: the walk's sprite_setup accepted the sprite
            int32_t z8;
            scale_depth(vw, scale, iscale, z8);
            row = kFixed && fw.row >= 0 ? fw.row : light_row_sprite(P.light, z8);
            tex = P.tex; tA = 0; hA = P.low + sh;
            if (ya < yb) {
                clip_rows(P.low + sh, P.low, row_scale(scale), pose_z, c.H, ya, yb);
                ucol = sprite_column(sp, vw, c.x, sw);
            }
        } else {
            const SegRec S = sc.segs[sf.seg];
            if (S.mid < 0 || S.mid >= sc.nmids) continue;
            const MidRec M = sc.mids[S.mid];
            tex = M.tex; tA = M.t_high; hA = M.high;
            ColumnEval ce = {0u, 1, 1, 0};
            if (ya < yb && column_eval(sf, vw, c.x, ce)) {
                clip_rows(M.high, M.low, ce.scale, pose_z, c.H, ya, yb);
                ucol = wall_column(S.uoff, S.len_q12, ce.s24);
                iscale = ce.iscale;
                row = kFixed && fw.row >= 0 ? fw.row : light_row(S.light, ce.z8);
            } else {
                ya = yb = 0;
            }
        }
        if (tex < 0 || tex >= sc.ntex) continue;
        const TexRec T = sc.tex[tex];
        const bool act = ya < yb;
        int y0 = __reduce_min_sync(kFull, act ? ya : 0x7FFFFFFF);
        int y1 = __reduce_max_sync(kFull, act ? yb : 0);
        if (y0 >= y1) continue;
        const uint32_t col = (uint32_t)floormod32(ucol, (int32_t)T.w);
        // colour from this lane's pre-lit plane, opacity from plane 32 (same layout, written by the pre-light kernel
        // for textures with holes)
        const bool inter = tex_interleaved(T);
        const bool has_mask = T.mask_off != 0xFFFFFFFFu;
        const uint8_t *pl = sc.lit_texels + (size_t)row * sc.lit_texel_stride + T.texel_off;
        if constexpr (kFixed) {
            if (row == 32) pl = fw.texels + T.texel_off;
        }
        const uint8_t *pm = sc.lit_texels + (size_t)32 * sc.lit_texel_stride + T.texel_off;
        const uint32_t tstep = (uint32_t)(iscale >> 4);
        uint32_t t = (uint32_t)wall_tbase(tA, hA, pose_z, c.H, iscale) + (uint32_t)y0 * tstep;
        uint8_t *p8 = c.fb + (size_t)y0 * Wc;
        uint32_t *p32 = kRgba ? c.rgba + (size_t)y0 * Wc : nullptr;
        const uint32_t len = act ? (uint32_t)(yb - ya) : 0u;   // the clipped window can be inverted (ya > yb): no rows then
        if (inter) {
            // batches of 8 rows as in draw_wall_warp: magnified columns (sprites nearly always are) read two colour
            // words and two opacity words per batch
            const uint32_t colb = 4u * col, w4 = 4u * T.w;
#pragma unroll 1
            for (int y = y0; y < y1; y += kBatch, p8 += (size_t)kBatch * Wc, p32 += (size_t)kBatch * Wc, t += (uint32_t)kBatch * tstep) {
                const uint32_t r0 = wall_row((int32_t)t, T.h, T.hmagic, T.hbias);
                const uint32_t acc = wall_acc(t, r0);
                const uint32_t d = (uint32_t)(y - ya);
                uint32_t v[kBatch], o[kBatch];
                if (__all_sync(kFull, ((acc + 7u * tstep) >> 16) < 8u)) {
                    const uint32_t o0 = (r0 >> 2) * w4 + colb, o1 = next_quad(r0 >> 2, T.h) * w4 + colb;
                    const uint32_t w0 = __ldg(reinterpret_cast<const uint32_t *>(pl + o0));
                    const uint32_t w1 = __ldg(reinterpret_cast<const uint32_t *>(pl + o1));
                    uint32_t m0 = 0x01010101u, m1 = 0x01010101u;
                    if (has_mask) {
                        m0 = __ldg(reinterpret_cast<const uint32_t *>(pm + o0));
                        m1 = __ldg(reinterpret_cast<const uint32_t *>(pm + o1));
                    }
#pragma unroll
                    for (int k = 0; k < kBatch; k++) {
                        const uint32_t bk = (acc + (uint32_t)k * tstep) >> 16;
                        v[k] = pick_byte(w0, w1, bk) & 0xFFu;
                        o[k] = pick_byte(m0, m1, bk) & 0xFFu;
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < kBatch; k++) {
                        const uint32_t rk = wall_row((int32_t)(t + (uint32_t)k * tstep), T.h, T.hmagic, T.hbias);
                        const uint32_t off = (rk >> 2) * w4 + colb + (rk & 3u);
                        v[k] = __ldg(pl + off);
                        o[k] = has_mask ? (uint32_t)__ldg(pm + off) : 1u;
                    }
                }
#pragma unroll
                for (int k = 0; k < kBatch; k++)
                    put_px<kRgba>(c, p8 + (size_t)k * Wc, kRgba ? p32 + (size_t)k * Wc : nullptr, d + (uint32_t)k < len && o[k] != 0u, v[k]);
            }
        } else {
#pragma unroll 1
            for (int y = y0; y < y1; y++, p8 += Wc, p32 += Wc, t += tstep) {
                const uint32_t off = wall_row((int32_t)t, T.h, T.hmagic, T.hbias) * T.w + col;
                const bool on = (uint32_t)(y - ya) < len && (!has_mask || __ldg(pm + off) != 0);
                put_px<kRgba>(c, p8, p32, on, __ldg(pl + off));
            }
        }
    }
}

// Warps per raster CTA: the eight 32-column strips of two adjacent 128-column line groups (for widths that are a multiple
// of 256; at 1920 columns every other CTA straddles two frames).
constexpr int kRasterWarps = 8;

// The CTA's draw queue (DESIGN.md §5).  Each warp's front-to-back clip pass turns its strip's draws into records instead
// of drawing them; after a barrier every warp of the CTA pops records and draws them, so a CTA lasts about as long as its
// average strip instead of its longest one.  A record is a header {meta, three warp-uniform arguments} and, per lane, the
// packed window [ya, yb) -- for a wall piece also the texture column and iscale | light row << 24 (iscale <= 2^23).
// meta = pool offset (words) | kind << 16 | visible << 17 | owner warp << 18.  Flat spans and the closing void fill are
// plane records (void: not visible).  A record that does not fit is drawn by its owner at once, as without the queue.
constexpr uint32_t kQueueWords = 6144;                 // per-lane record words per CTA (24 KB)
constexpr uint32_t kQueueRecs = kQueueWords / 32;      // headers: every record has at least 32 per-lane words
constexpr uint32_t kRecWall = 1u << 16, kRecVisible = 1u << 17;

// The queue is drawn in row bands (DESIGN.md §5): a work item is (band, record) with the record's windows clipped to the
// band, and items go out band by band, so the CTA's stores sweep down its frame rows and a 128-byte line is finished soon
// after it is started.  Every pixel depends only on its absolute row, so clipping changes no byte.  kBandRows is a
// multiple of 32: band starts fall on the flat spans' 32-row constant chunks and on the wall batches of 8 and 16 rows.
// The item list holds kItemCap items {record | band << 8}; a CTA with more draws its records whole, in record order, and
// so does a CTA with a deferred masked entry: its masked pass rewrites pixels of lines that banding has already finished
// and streamed out of L2 (DESIGN.md §6).
constexpr int kBandRows = 256;
constexpr int kMaxBands = (2160 + kBandRows - 1) / kBandRows;   // b2d_view_init accepts at most 2160 rows
constexpr uint32_t kItemCap = 1024;
static_assert(kBandRows % 32 == 0 && kMaxBands <= 256 && kQueueRecs <= 256, "an item is record | band << 8 in 16 bits");

struct DrawQueue {
    uint4 *head;                 // [kQueueRecs]
    uint32_t *ext;               // [kQueueRecs] the record's warp extent y0 | y1 << 16 (min ya, max yb over active lanes)
    uint32_t *pool;              // [kQueueWords]
    uint32_t *nrec, *nwords;     // records and words handed out (the words of a record that found no header are lost)
};

// warp-wide: append one record, or return false when it does not fit; a draw that no lane owns needs no record
__device__ __forceinline__ bool queue_push(const DrawQueue &q, int lane, uint32_t meta, int32_t a, int32_t b, int32_t c,
                                           int ya, int yb, int32_t ucol, uint32_t iscale_row) {
    const bool act = ya < yb;
    if (!__any_sync(kFull, act)) return true;
    const uint32_t y0 = __reduce_min_sync(kFull, act ? (uint32_t)ya : 0xFFFFu);
    const uint32_t y1 = __reduce_max_sync(kFull, act ? (uint32_t)yb : 0u);
    const bool wall = meta & kRecWall;
    const uint32_t words = wall ? 96u : 32u;
    uint32_t off = 0, i = kQueueRecs;
    if (lane == 0) {
        off = atomicAdd(q.nwords, words);
        if (off + words <= kQueueWords) i = atomicAdd(q.nrec, 1u);
    }
    i = __shfl_sync(kFull, i, 0);
    if (i >= kQueueRecs) return false;
    off = __shfl_sync(kFull, off, 0);
    q.pool[off + lane] = act ? (uint32_t)ya | ((uint32_t)yb << 16) : 0u;
    if (wall) {
        q.pool[off + 32 + lane] = (uint32_t)ucol;
        q.pool[off + 64 + lane] = iscale_row;
    }
    if (lane == 0) {
        q.head[i] = make_uint4(meta | off, (uint32_t)a, (uint32_t)b, (uint32_t)c);
        q.ext[i] = y0 | y1 << 16;
    }
    return true;
}

// the element of type T of a raster variant's appended tables
template <typename T, typename A, typename... P>
__device__ __forceinline__ const T &extra_tables(const A &a, const P &...p) {
    if constexpr (std::is_same_v<T, A>) return a;
    else return extra_tables<T>(p...);
}

// `Extra`: the variant's appended tables, each appended as a parameter of `fx` -- FixedTables for the fixed-colormap
// variant (kFixed, DESIGN.md C18; per-frame levels and states only), whose frames may have a fixed colormap, then
// SeenTables for the seen variant (kSeen, DESIGN.md C20; index frames only), which marks the lines each frame sees.  An
// empty pack leaves the other variants' names, parameters and code as they are.
template <bool kRgba, int kW, bool kMasked, bool kStates, bool kLevels, typename... Extra>
__global__ void __launch_bounds__(32 * kRasterWarps, 16 / kRasterWarps)
b2d_raster_kernel(const __grid_constant__ DeviceScene sc, const __grid_constant__ View vw, const FrameConst *__restrict__ frames,
                  const SegFrame *__restrict__ work, int stride, int n, int strips,
                  uint8_t *__restrict__ index_fb, uint32_t *__restrict__ rgba_fb, const __grid_constant__ LevelTables lt,
                  const Extra... fx) {
    constexpr bool kFixed = (std::is_same_v<Extra, FixedTables> || ...);
    constexpr bool kSeen = (std::is_same_v<Extra, SeenTables> || ...);
    static_assert(sizeof...(Extra) == (int)kFixed + (int)kSeen, "appended tables: FixedTables, SeenTables, each at most once");
    static_assert(!kFixed || (kStates && kLevels), "fixed colormaps come with per-frame levels and states");
    static_assert(!kSeen || !kRgba, "the seen variant draws index frames only");
    // per-frame levels: a palette per warp (the warps of a CTA may draw frames of levels from different WADs)
    __shared__ uint32_t s_pal[kRgba ? (kLevels ? 256 * kRasterWarps : 256) : 1];
    __shared__ uint2 s_rowz[kRasterWarps][32];
    __shared__ uint32_t s_chunks[kRasterWarps][kMasked ? kMaskedCapMax / kMaskedChunk : 1];
    // what a warp drawing another warp's record needs of its strip: per lane {plane direction, sky column, x}, and the frame
    __shared__ int4 s_lanes[kRasterWarps][32];
    __shared__ int s_frame[kRasterWarps];
    __shared__ uint4 s_qhead[kQueueRecs];
    __shared__ uint32_t s_qext[kQueueRecs];
    __shared__ uint32_t s_qpool[kQueueWords];
    __shared__ uint16_t s_items[kItemCap];       // band-major work items: record | band << 8
    __shared__ uint32_t s_band[kMaxBands];       // items per band, then each band's next slot in s_items
    __shared__ uint32_t s_qn[5];                  // records, words, items popped, items, a warp deferred masked entries
    // per-frame states or levels: each warp's copy of its frame's scene description (see below)
    __shared__ DeviceScene s_scn[kStates || kLevels ? kRasterWarps : 1];
    __shared__ FixedWarp s_fix[kFixed ? kRasterWarps : 1];      // each warp's fixed colormap
    if (threadIdx.x < 5) s_qn[threadIdx.x] = 0;
    for (int b = threadIdx.x; b < kMaxBands; b += blockDim.x) s_band[b] = 0;
    if (kRgba && !kLevels) {   // the palette into shared memory (colours come pre-lit from global memory: no colormap here)
        for (int i = threadIdx.x; i < 256; i += blockDim.x) s_pal[i] = sc.palette[i];
    }
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long gw = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
    // The grid's last CTA may hold warps without a strip: they skip the clip pass but take part in every barrier and
    // in the draw phase.
    const bool has_strip = gw < (long long)n * strips;
    const int frame = has_strip ? (int)(gw / strips) : 0, strip = has_strip ? (int)(gw % strips) : 0;
    const int W = kW ? kW : vw.W, H = vw.H;
    const int x0 = strip * 32, x = x0 + lane;
    const bool inside = has_strip && x < W;
    const DrawQueue q{s_qhead, s_qext, s_qpool, &s_qn[0], &s_qn[1]};

    FrameConst fc{};
    if (has_strip) fc = frames[frame];
    const DeviceScene *scp = &sc;
    if constexpr (kStates || kLevels) {
        // per-frame states or levels: this warp's copy of the scene description of its frame -- with per-frame levels, of
        // the frame's level (the walk passed the level on in FrameConst::level), with that level's palette; with per-frame
        // states, its five state-dependent tables pointed at the frame's TableSet (FrameConst::set).  Every table read
        // below goes through it.
        DeviceScene *d = &s_scn[warp];
        if (has_strip) {
            const DeviceScene *lsrc = kLevels ? lt.scenes + (uint32_t)fc.level : &sc;
            const uint32_t *src = reinterpret_cast<const uint32_t *>(lsrc);
            uint32_t *dst = reinterpret_cast<uint32_t *>(d);
            for (int i = lane; i < (int)(sizeof(DeviceScene) / 4); i += 32) dst[i] = src[i];
            if (kLevels && kRgba) {
                const uint32_t *pal = lsrc->palette;
                for (int i = lane; i < 256; i += 32) s_pal[256 * warp + i] = pal[i];
            }
            __syncwarp();
            if constexpr (kStates) {
                if (lane == 0) {
                    const TableSet t = lt.sets[(uint32_t)fc.set];
                    d->tex = t.tex; d->sectors = t.sectors; d->segs = t.segs; d->sprites = t.sprites; d->mids = t.mids;
                }
                __syncwarp();
            }
        }
        scp = d;
    }
    if constexpr (kFixed) {
        if (has_strip && lane == 0) {
            const FixedTables &t = extra_tables<FixedTables>(fx...);
            const FixedPlanes p = t.planes[(uint32_t)fc.level];
            s_fix[warp] = FixedWarp{p.texels, p.flats, t.frame_fixed[frame]};
        }
        __syncwarp();
    }
    const DeviceScene &ts = *scp;      // = sc without per-frame states or levels
    const DeviceScene &ls = kLevels ? ts : sc;     // the level's own fields (sky, masked-entry cap): = sc but per-frame levels
    RasterCtx c;
    c.sc = &ts;
    if constexpr (kFixed) c.fix = s_fix[warp];
    c.pal_s = (uint32_t)__cvta_generic_to_shared(kLevels ? s_pal + 256 * warp : s_pal);
    c.rowz = s_rowz[warp];
    c.W = W; c.H = H; c.x = x; c.lane = lane;
    int mcount = 0;
    uint32_t *chunks = s_chunks[warp];
    asm("" : "+l"(chunks));        // a run-time value: propagated into masked_pass as a constant, it makes that pass spill more
    const SegFrame *wl = work + (size_t)frame * stride;

    if (has_strip) {
    c.dir = plane_dir(fc, vw, inside ? x : 0, ls.invF);
    c.fb = index_fb + (size_t)frame * W * H + (inside ? x : 0);
    c.rgba = kRgba ? rgba_fb + (size_t)frame * W * H + (inside ? x : 0) : nullptr;
    c.skycol = 0;
    if (ls.sky_tex >= 0 && inside) c.skycol = umulhi32(sky_u32(x, vw, fc.pose.angle), ts.tex[ls.sky_tex].w);
    s_lanes[warp][lane] = make_int4(c.dir.ax, c.dir.ay, (int)c.skycol, inside ? x : 0);
    if (lane == 0) s_frame[warp] = frame;

    int ct = 0, cb = inside ? H : 0;              // open window [ct, cb) of this lane's column
    const bool defer = kMasked && ls.masked_list != nullptr;
    const int count = fc.count;
    const uint32_t owner = (uint32_t)warp << 18;
    bool done = false;
    // the seen variant: this frame's row of seen lines and its level's seg -> linedef table (lane 0 marks)
    uint32_t *seen_row = nullptr;
    const int32_t *seen_line = nullptr;
    int32_t seen_last = -1;
    if constexpr (kSeen) {
        const SeenTables &st = extra_tables<SeenTables>(fx...);
        seen_row = st.rows + (size_t)frame * st.words;
        seen_line = st.seg_line + st.level_off[kLevels ? (uint32_t)fc.level : 0u];
    }

    for (int k0 = 0; k0 < count && !done; k0 += 32) {
        int k = k0 + lane;
        bool overlap = false;
        if (k < count) {
            int xlo = wl[k].xlo, xhi = wl[k].xhi;
            overlap = xhi >= x0 && xlo <= x0 + 31;
        }
        unsigned m = __ballot_sync(kFull, overlap);
        while (m) {
            int j = __ffs(m) - 1;
            m &= m - 1;
            if (!__any_sync(kFull, ct < cb)) { done = true; break; }
            const SegFrame sf = wl[k0 + j];                              // warp-uniform 64 B
            bool in = inside && ct < cb && x >= sf.xlo && x <= sf.xhi;
            if (!__any_sync(kFull, in)) continue;
            if (is_sprite_entry(sf)) {
                // decoration sprite: remember the windows open right now; it is drawn in the masked pass
                if (defer) {
                    uint32_t *ml = masked_push(ls, chunks, mcount, lane);
                    if (ml) {
                        if (lane == 0) ml[0] = (uint32_t)(k0 + j);
                        ml[1 + lane] = in ? ((uint32_t)ct | ((uint32_t)cb << 16)) : 0u;
                    }
                }
                continue;
            }
            ColumnEval ce = {0u, 1, 1, 0};
            bool ok = in && column_eval(sf, vw, x, ce);
            if (!__any_sync(kFull, ok)) continue;
            if constexpr (kSeen) {
                // C20: the seg owns a column of the frame.  Consecutive entries are often segs of one linedef: a warp
                // marks a linedef once per run.
                if (lane == 0) {
                    const int32_t l = __ldg(seen_line + sf.seg);
                    if (l >= 0 && l != seen_last) {
                        atomicOr(seen_row + (l >> 5), 1u << (l & 31));
                        seen_last = l;
                    }
                }
            }

            const SegRec S = ts.segs[sf.seg];
            const SectorRec SF = ts.sectors[S.front];
            const int32_t fcl = SF.ceil, ffl = SF.floor;
            const bool two = S.flags & kSegTwoSided;
            const bool ceil_vis = plane_visible(true, fcl, SF.ceil_flat == kFlatSky, fc.pose.z);
            const bool floor_vis = plane_visible(false, ffl, SF.floor_flat == kFlatSky, fc.pose.z);

            WallRows wr = {ct, ct, ct, ct};          // per lane
            int yend = ct, row = 0;
            int32_t ucol = 0;
            if (ok) {
                row = kFixed && c.fix.row >= 0 ? c.fix.row : light_row(S.light, ce.z8);
                ucol = wall_column(S.uoff, S.len_q12, ce.s24);
                wr = wall_rows(fcl, ffl, two, S.otop, S.obot, ce.scale, fc.pose.z, H, ct, cb);
                yend = cb;
            }
            // The two flat spans (ceiling [ct, y1), floor [y4, cb)) and the two wall pieces go through ONE inlined
            // copy of each span routine (loops kept rolled): the routines are large, and the kernel's speed depends
            // on its hot code staying resident in the instruction cache.
#pragma unroll 1
            for (int pz = 0; pz < 2; pz++) {
                const bool top = pz == 0;
                const int ya = ok ? (top ? ct : wr.y4) : 0, yb = ok ? (top ? wr.y1 : yend) : 0;
                const int32_t h = top ? fcl : ffl, flat = top ? SF.ceil_flat : SF.floor_flat;
                const bool vis = top ? ceil_vis : floor_vis;
                if (!queue_push(q, lane, owner | (vis ? kRecVisible : 0u), h, flat, SF.light, ya, yb, 0, 0u))
                    draw_plane_warp<kRgba, kW, kFixed>(c, fc, vw, ya, yb, h, flat, SF.light, vis);
            }
#pragma unroll 1
            for (int pw = 0; pw < 2; pw++) {
                const bool upper = pw == 0;            // piece A, then piece B
                if (!wall_piece(upper, two, fcl, ffl, S.otop, S.obot)) continue;
                const int ya = ok ? (upper ? wr.y1 : wr.y3) : 0, yb = ok ? (upper ? wr.y2 : wr.y4) : 0;
                const int32_t tex = upper ? S.texA : S.texB, tA = upper ? S.tA : S.tB, hA = upper ? S.hA : S.hB;
                if (!queue_push(q, lane, owner | kRecWall, tex, tA, hA, ya, yb, ucol, (uint32_t)ce.iscale | ((uint32_t)row << 24)))
                    draw_wall_warp<kRgba, kW, kFixed>(c, fc, ya, yb, tex, tA, hA, ucol, ce.iscale, row);
            }
            if (ok) wall_window(two, wr, H, ct, cb);
            if (defer && two && S.mid >= 0) {
                // defer the masked middle texture: remember the window that is open behind this seg
                const bool keep = ok && wr.y2 < wr.y3;
                if (__any_sync(kFull, keep)) {
                    uint32_t *ml = masked_push(ls, chunks, mcount, lane);
                    if (ml) {
                        if (lane == 0) ml[0] = (uint32_t)(k0 + j);
                        ml[1 + lane] = keep ? ((uint32_t)wr.y2 | ((uint32_t)wr.y3 << 16)) : 0u;
                    }
                }
            }
        }
    }
    // whatever is still open is void
    if (!queue_push(q, lane, owner, 0, 0, 0, inside ? ct : 0, inside ? cb : 0, 0, 0u))
        fill_void_warp<kRgba, kW>(c, inside ? ct : 0, inside ? cb : 0);
    }

    if (kMasked && mcount > 0 && lane == 0) s_qn[4] = 1;
    // Draw phase: every warp of the CTA pops work items until the list is empty.  Correctness does not depend on the
    // order: the clip windows of a strip's draws are disjoint, so every byte is still written once.
    __syncthreads();
    const uint32_t nrec = min(s_qn[0], kQueueRecs);
    // the band-major item list, a counting sort: items per band, an exclusive scan, then each record scattered to its bands
    for (uint32_t r = threadIdx.x; r < nrec; r += blockDim.x) {
        const uint32_t e = s_qext[r];
        for (uint32_t b = (e & 0xFFFFu) / kBandRows; b <= ((e >> 16) - 1u) / kBandRows; b++) atomicAdd(&s_band[b], 1u);
    }
    __syncthreads();
    if (warp == 0) {
        constexpr int kPer = (kMaxBands + 31) / 32;
        uint32_t v[kPer], sum = 0;
#pragma unroll
        for (int k = 0; k < kPer; k++) {
            const int b = lane * kPer + k;
            v[k] = b < kMaxBands ? s_band[b] : 0u;
            sum += v[k];
        }
        uint32_t incl = sum;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t u = __shfl_up_sync(kFull, incl, d);
            if (lane >= d) incl += u;
        }
        uint32_t at = incl - sum;
#pragma unroll
        for (int k = 0; k < kPer; k++) {
            const int b = lane * kPer + k;
            if (b < kMaxBands) s_band[b] = at;
            at += v[k];
        }
        if (lane == 31) s_qn[3] = incl;
    }
    __syncthreads();
    const bool banded = s_qn[3] <= kItemCap && !(kMasked && s_qn[4]);
    if (banded) {
        for (uint32_t r = threadIdx.x; r < nrec; r += blockDim.x) {
            const uint32_t e = s_qext[r];
            for (uint32_t b = (e & 0xFFFFu) / kBandRows; b <= ((e >> 16) - 1u) / kBandRows; b++)
                s_items[atomicAdd(&s_band[b], 1u)] = (uint16_t)(r | b << 8);
        }
        __syncthreads();
    }
    const uint32_t nitems = banded ? s_qn[3] : nrec;
    for (;;) {
        uint32_t i = 0;
        if (lane == 0) i = atomicAdd(&s_qn[2], 1u);
        i = __shfl_sync(kFull, i, 0);
        if (i >= nitems) break;
        int lo = 0, hi = H;
        if (banded) {
            const uint32_t it = s_items[i];
            i = it & 0xFFu;
            lo = (int)(it >> 8) * kBandRows;
            hi = lo + kBandRows;
        }
        const uint4 hd = s_qhead[i];
        const uint32_t off = hd.x & 0xFFFFu, o = hd.x >> 18;
        const int4 ln = s_lanes[o][lane];
        const int f = s_frame[o];
        const FrameConst fo = frames[f];
        RasterCtx d;
        d.sc = kStates || kLevels ? &s_scn[o] : &sc;      // the owner's scene description
        if constexpr (kFixed) d.fix = s_fix[o];
        d.pal_s = (uint32_t)__cvta_generic_to_shared(kLevels ? s_pal + 256 * o : s_pal);
        d.rowz = s_rowz[warp];
        d.dir = PlaneDir{ln.x, ln.y};
        d.fb = index_fb + (size_t)f * W * H + ln.w;
        d.rgba = kRgba ? rgba_fb + (size_t)f * W * H + ln.w : nullptr;
        d.W = W; d.H = H; d.x = ln.w; d.lane = lane;
        d.skycol = (uint32_t)ln.z;
        const uint32_t win = s_qpool[off + lane];
        const int ya = max((int)(win & 0xFFFFu), lo), yb = min((int)(win >> 16), hi);
        if (hd.x & kRecWall) {
            const uint32_t isr = s_qpool[off + 64 + lane];
            draw_wall_warp<kRgba, kW, kFixed>(d, fo, ya, yb, (int32_t)hd.y, (int32_t)hd.z, (int32_t)hd.w, (int32_t)s_qpool[off + 32 + lane],
                                      (int32_t)(isr & 0xFFFFFFu), (int)(isr >> 24));
        } else {
            draw_plane_warp<kRgba, kW, kFixed>(d, fo, vw, ya, yb, (int32_t)hd.y, (int32_t)hd.z, (int)hd.w, hd.x & kRecVisible);
        }
    }
    if constexpr (kMasked) {
        // the masked pass overwrites solid pixels of its own strip: every draw of the CTA must be done first
        __syncthreads();
        if constexpr (kFixed) {
            if (mcount > 0) masked_pass<kRgba, kW, kStates, kLevels>(ts, vw, fc.pose.z, c.fb, c.rgba, c.pal_s, x, lane, wl, chunks, mcount, c.fix.texels, c.fix.row);
        } else {
            if (mcount > 0) masked_pass<kRgba, kW, kStates, kLevels>(ts, vw, fc.pose.z, c.fb, c.rgba, c.pal_s, x, lane, wl, chunks, mcount);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Kernel 3: palette LUT
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
b2d_palette_kernel(const uint32_t *__restrict__ palette, const uint8_t *__restrict__ index,
                   uint32_t *__restrict__ rgba, size_t n_pixels) {
    __shared__ uint32_t s_pal[256];
    s_pal[threadIdx.x] = palette[threadIdx.x];
    __syncthreads();
    // 128-bit path only for 16-byte aligned buffers (a caller may pass &index_fb[i*W*H] with W*H % 16 != 0)
    const bool aligned = ((reinterpret_cast<uintptr_t>(index) | reinterpret_cast<uintptr_t>(rgba)) & 15) == 0;
    const size_t nvec = aligned ? n_pixels / 16 : 0;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride) {
        uint4 in = __ldcs(reinterpret_cast<const uint4 *>(index) + i);
        uint32_t wds[4] = {in.x, in.y, in.z, in.w};
        uint4 *out = reinterpret_cast<uint4 *>(rgba) + 4 * i;
#pragma unroll
        for (int q = 0; q < 4; q++) {
            uint4 o;
            o.x = s_pal[wds[q] & 0xFF];
            o.y = s_pal[(wds[q] >> 8) & 0xFF];
            o.z = s_pal[(wds[q] >> 16) & 0xFF];
            o.w = s_pal[wds[q] >> 24];
            __stcs(out + q, o);
        }
    }
    // tail (n_pixels not a multiple of 16)
    for (size_t p = nvec * 16 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < n_pixels; p += stride)
        rgba[p] = s_pal[index[p]];
}

// Kernel 3 with a colour table per frame: `parts` CTAs per frame (blockIdx.x = frame * parts + part), each loading its
// frame's table, palettes[tables[frame]] (a palette of the frame's level), into shared memory and streaming a contiguous
// 1/parts of the frame.
__global__ void __launch_bounds__(256)
b2d_palette_levels_kernel(const uint32_t *__restrict__ palettes, const uint32_t *__restrict__ tables,
                          const uint8_t *__restrict__ index, uint32_t *__restrict__ rgba, size_t npix, int parts) {
    __shared__ uint32_t s_pal[256];
    const size_t frame = blockIdx.x / parts;
    const int part = blockIdx.x % parts;
    s_pal[threadIdx.x] = palettes[(size_t)tables[frame] * 256 + threadIdx.x];
    __syncthreads();
    const uint8_t *in = index + frame * npix;
    uint32_t *out = rgba + frame * npix;
    // 128-bit path when every frame starts 16-byte aligned in both buffers
    const bool aligned = npix % 16 == 0 && ((reinterpret_cast<uintptr_t>(index) | reinterpret_cast<uintptr_t>(rgba)) & 15) == 0;
    const size_t n = aligned ? npix / 16 : npix;
    const size_t per = (n + parts - 1) / parts, lo = (size_t)part * per, hi = lo + per < n ? lo + per : n;
    if (aligned) {
        for (size_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
            const uint4 q = __ldcs(reinterpret_cast<const uint4 *>(in) + i);
            const uint32_t wds[4] = {q.x, q.y, q.z, q.w};
            uint4 *o4 = reinterpret_cast<uint4 *>(out) + 4 * i;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                uint4 o;
                o.x = s_pal[wds[k] & 0xFF];
                o.y = s_pal[(wds[k] >> 8) & 0xFF];
                o.z = s_pal[(wds[k] >> 16) & 0xFF];
                o.w = s_pal[wds[k] >> 24];
                __stcs(o4 + k, o);
            }
        }
    } else {
        for (size_t p = lo + threadIdx.x; p < hi; p += blockDim.x) out[p] = s_pal[in[p]];
    }
}

// ------------------------------------------------------------------------------------------------
// Kernel 4: resolve (C17) -- k x k box filter of index frames through a palette per frame
// ------------------------------------------------------------------------------------------------
// Output formats, the values of B2D_RESOLVE_* in include/b2d.h.
constexpr int kResolveRgba = 0, kResolveRgb = 1, kResolvePlanar = 2, kResolveGray = 3;

// `N` bytes, packed little-endian in w[], to dst with the widest stores its alignment allows.
template <int N>
__device__ __forceinline__ void store_run(uint8_t *dst, const uint32_t (&w)[(N + 3) / 4]) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(dst);
    if constexpr (N % 16 == 0) {
        if ((a & 15) == 0) {
#pragma unroll
            for (int q = 0; q < N / 16; q++) __stcs(reinterpret_cast<uint4 *>(dst) + q, make_uint4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]));
            return;
        }
    }
    if constexpr (N % 8 == 0) {
        if ((a & 7) == 0) {
#pragma unroll
            for (int q = 0; q < N / 8; q++) __stcs(reinterpret_cast<uint2 *>(dst) + q, make_uint2(w[2 * q], w[2 * q + 1]));
            return;
        }
    }
    if constexpr (N % 4 == 0) {
        if ((a & 3) == 0) {
#pragma unroll
            for (int q = 0; q < N / 4; q++) __stcs(reinterpret_cast<unsigned int *>(dst) + q, w[q]);
            return;
        }
    }
    if constexpr (N % 2 == 0) {
        if ((a & 1) == 0) {
#pragma unroll
            for (int q = 0; q < N / 2; q++) reinterpret_cast<uint16_t *>(dst)[q] = (uint16_t)(w[q / 2] >> (16 * (q % 2)));
            return;
        }
    }
#pragma unroll
    for (int b = 0; b < N; b++) dst[b] = (uint8_t)(w[b / 4] >> (8 * (b % 4)));
}

// Writes the P output pixels (x0 .. x0+P-1, y) of one frame from their k x k sums: acc0 = {R | B << 16} (grey: Y) and
// acc1 = G, each rounded half up, (sum + k*k/2) / (k*k).  `o` is the frame's output, OW x OH pixels.
template <int K, int FMT, int P>
__device__ __forceinline__ void resolve_emit(uint8_t *o, size_t opix, int OW, int y, int x0, const uint32_t (&acc0)[P],
                                             const uint32_t (&acc1)[P]) {
    constexpr uint32_t kk = K * K, half = K * K / 2;
    const size_t at = (size_t)y * OW + x0;
    if constexpr (FMT == kResolveGray) {
        uint32_t w[(P + 3) / 4] = {};
#pragma unroll
        for (int p = 0; p < P; p++) w[p / 4] |= ((acc0[p] + half) / kk) << (8 * (p % 4));
        store_run<P>(o + at, w);
    } else {
        uint32_t r[P], g[P], b[P];
#pragma unroll
        for (int p = 0; p < P; p++) {
            r[p] = ((acc0[p] & 0xFFFFu) + half) / kk;
            b[p] = ((acc0[p] >> 16) + half) / kk;
            g[p] = (acc1[p] + half) / kk;
        }
        if constexpr (FMT == kResolveRgba) {
            uint32_t w[P];
#pragma unroll
            for (int p = 0; p < P; p++) w[p] = r[p] | (g[p] << 8) | (b[p] << 16) | 0xFF000000u;
            store_run<4 * P>(o + 4 * at, w);
        } else if constexpr (FMT == kResolveRgb) {
            uint32_t w[(3 * P + 3) / 4] = {};
#pragma unroll
            for (int p = 0; p < P; p++) {
                w[(3 * p) / 4] |= r[p] << (8 * ((3 * p) % 4));
                w[(3 * p + 1) / 4] |= g[p] << (8 * ((3 * p + 1) % 4));
                w[(3 * p + 2) / 4] |= b[p] << (8 * ((3 * p + 2) % 4));
            }
            store_run<3 * P>(o + 3 * at, w);
        } else {   // planar: R plane, G plane, B plane
            uint32_t wr[(P + 3) / 4] = {}, wg[(P + 3) / 4] = {}, wb[(P + 3) / 4] = {};
#pragma unroll
            for (int p = 0; p < P; p++) {
                wr[p / 4] |= r[p] << (8 * (p % 4));
                wg[p / 4] |= g[p] << (8 * (p % 4));
                wb[p / 4] |= b[p] << (8 * (p % 4));
            }
            store_run<P>(o + at, wr);
            store_run<P>(o + opix + at, wg);
            store_run<P>(o + 2 * opix + at, wb);
        }
    }
}

// `parts` CTAs per frame (blockIdx.x = frame * parts + part), each loading its frame's colour table, palettes[tables[frame]]
// (NULL tables: table 0) -- as {R | B << 16, G}, or
// the luma Y = (77 R + 150 G + 29 B + 128) >> 8 for grey -- into shared memory and resolving a contiguous 1/parts of the
// frame's work items (sums of up to 64 entries stay below 2^14, so R and B share a word).  Vector path (`vec`: W a
// multiple of P * K and the index frames 16-byte aligned): an item is P = 16 / gcd(K, 16) output pixels of one output row,
// read as P * K / 16 128-bit streaming loads from each of its K input rows, so every byte's output pixel is a
// compile-time constant.  Otherwise an item is one output pixel, read byte by byte.  Stores: store_run.
template <int K, int FMT>
__global__ void __launch_bounds__(256)
b2d_resolve_kernel(const uint32_t *__restrict__ palettes, const uint32_t *__restrict__ tables, const uint8_t *__restrict__ index,
                   uint8_t *__restrict__ out, int W, int H, int parts, bool vec) {
    constexpr int P = K == 1 ? 16 : K == 2 ? 8 : K == 4 ? 4 : K == 6 ? 8 : K == 8 ? 2 : 16;     // 16 / gcd(K, 16)
    constexpr int kBpp = FMT == kResolveRgba ? 4 : FMT == kResolveGray ? 1 : 3;
    __shared__ uint2 s_tab[256];
    const size_t frame = blockIdx.x / parts;
    const int part = blockIdx.x % parts;
    {
        const uint32_t c = palettes[(size_t)(tables ? tables[frame] : 0u) * 256 + threadIdx.x];
        const uint32_t R = c & 0xFF, G = (c >> 8) & 0xFF, B = (c >> 16) & 0xFF;
        s_tab[threadIdx.x] = FMT == kResolveGray ? make_uint2((77 * R + 150 * G + 29 * B + 128) >> 8, 0u) : make_uint2(R | (B << 16), G);
    }
    __syncthreads();
    const int OW = W / K, OH = H / K;
    const size_t opix = (size_t)OW * OH;
    const uint8_t *in = index + frame * (size_t)W * H;
    uint8_t *o = out + frame * opix * kBpp;
    if (vec) {
        const int groups = OW / P;
        const size_t n = (size_t)OH * groups, per = (n + parts - 1) / parts, lo = (size_t)part * per, hi = lo + per < n ? lo + per : n;
        for (size_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
            const int y = (int)(i / groups), x0 = (int)(i % groups) * P;
            const uint8_t *src = in + (size_t)y * K * W + (size_t)x0 * K;
            uint32_t acc0[P], acc1[P];
#pragma unroll
            for (int p = 0; p < P; p++) acc0[p] = acc1[p] = 0;
#pragma unroll
            for (int j = 0; j < K; j++) {
#pragma unroll
                for (int q = 0; q < P * K / 16; q++) {
                    const uint4 v = __ldcs(reinterpret_cast<const uint4 *>(src + (size_t)j * W) + q);
                    const uint32_t wds[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (int b = 0; b < 16; b++) {
                        const uint2 t = s_tab[(wds[b / 4] >> (8 * (b % 4))) & 0xFF];
                        acc0[(16 * q + b) / K] += t.x;
                        if (FMT != kResolveGray) acc1[(16 * q + b) / K] += t.y;
                    }
                }
            }
            resolve_emit<K, FMT, P>(o, opix, OW, y, x0, acc0, acc1);
        }
    } else {
        const size_t n = opix, per = (n + parts - 1) / parts, lo = (size_t)part * per, hi = lo + per < n ? lo + per : n;
        for (size_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
            const int y = (int)(i / OW), x = (int)(i % OW);
            const uint8_t *src = in + (size_t)y * K * W + (size_t)x * K;
            uint32_t acc0[1] = {0}, acc1[1] = {0};
#pragma unroll
            for (int j = 0; j < K; j++) {
#pragma unroll
                for (int b = 0; b < K; b++) {
                    const uint2 t = s_tab[__ldcs(src + (size_t)j * W + b)];
                    acc0[0] += t.x;
                    if (FMT != kResolveGray) acc1[0] += t.y;
                }
            }
            resolve_emit<K, FMT, 1>(o, opix, OW, y, x, acc0, acc1);
        }
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------
size_t walk_smem_per_warp(const DeviceScene &sc) { return walk_layout(sc.nverts, sc.nsegs, sc.nnodes, sc.nss, sc.nsprites).total; }

// SMs of the current device (132 on an H100 SXM): the persistent and capped grids below are sized per SM
static int device_sms() {
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms > 0 ? sms : 1;
}

// The walk's launch: `smem` bytes of dynamic shared memory per CTA (one frame per CTA).
template <bool kStates, bool kLevels>
static cudaError_t walk_go(const BatchTables &t, size_t smem, const View &vw, const Pose *d_poses, int n, FrameConst *d_frames,
                           SegFrame *d_work, int stride, cudaStream_t stream, bool background) {
    if (n <= 0) return cudaSuccess;
    if (smem > 227 * 1024) return cudaErrorInvalidValue;
    if (smem > 48 * 1024) {   // per device and cheap: set it on every launch that needs the opt-in
        cudaError_t e = cudaFuncSetAttribute(b2d_walk_kernel<kStates, kLevels>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    // background (b2d_walk_device: the walk of the NEXT batch, meant to run under another batch's raster): a persistent grid
    // of one CTA per SM.  It takes n/SMs frame latencies instead of one, but holds 1/8 of the register file instead of
    // 7/8, so the raster keeps 16 of its 19 warps per SM while the walk hides behind it.
    const int sms = device_sms();
    const int blocks = (background && n > sms) ? sms : n, warps = 4;
    b2d_walk_kernel<kStates, kLevels><<<blocks, warps * 32, smem, stream>>>(t.scene, vw, d_poses, n, d_frames, d_work, stride,
                                                                            t.levels);
    return cudaGetLastError();
}

size_t walk_levels_static_smem() {
    static const size_t bytes = [] {
        // the larger of the two per-frame-level walks (with and without per-frame states)
        cudaFuncAttributes a{}, b{};
        if (cudaFuncGetAttributes(&a, b2d_walk_kernel<false, true>) == cudaSuccess &&
            cudaFuncGetAttributes(&b, b2d_walk_kernel<true, true>) == cudaSuccess)
            return a.sharedSizeBytes > b.sharedSizeBytes ? a.sharedSizeBytes : b.sharedSizeBytes;
        cudaGetLastError();
        return sizeof(DeviceScene) + 16;       // s_lv, s_count, s_status, s_bar
    }();
    return bytes;
}

cudaError_t launch_walk(const BatchTables &t, size_t levels_smem, const View &vw, const Pose *d_poses, int n,
                        FrameConst *d_frames, SegFrame *d_work, int stride, cudaStream_t stream, bool background) {
    if (t.per_level && levels_smem + walk_levels_static_smem() > kWalkSmemMax) return cudaErrorInvalidValue;
    const size_t smem = t.per_level ? levels_smem : walk_smem_per_warp(t.scene);
    auto go = t.per_level ? (t.per_frame ? walk_go<true, true> : walk_go<false, true>)
                          : (t.per_frame ? walk_go<true, false> : walk_go<false, false>);
    return go(t, smem, vw, d_poses, n, d_frames, d_work, stride, stream, background);
}

// The raster's launch for every frame shape.  Launch shape: one warp per (frame, 32-column strip), kRasterWarps = 8 warps
// per CTA, so a CTA holds the eight strips of two adjacent 128-column line groups (a CTA may straddle two frames at 1920
// columns and at other widths).  The warps that write the sectors of the same 128-byte frame lines, and of the next lines
// of the same rows, then start together on one SM and finish those lines close together in time, so fewer partly written
// lines sit in L2.  Against four-warp CTAs (one line group) that is worth 3.8 % of the bench.py c2 step and 5.9 % at 4K,
// although residency falls from 20 to 16 warps per SM.  The CTA's draw queue shares the strips' draws among its warps, so
// a finished strip's warp draws for its slower siblings instead of idling.  The registers are left to the compiler (cap
// 128): 94 for the 1080p and 4K index-only kernels, i.e. 2 CTAs = 16 warps per SM (DESIGN.md §5, §6).
// The frame width is a compile-time constant for the benchmark resolutions (immediate store offsets).  `fx`: the variant's
// appended tables (b2d_raster_kernel's `Extra`); a seen variant draws index frames only.
template <bool kStates, bool kLevels, typename... Extra>
static cudaError_t raster_go(const BatchTables &t, bool masked, const View &vw, const FrameConst *d_frames,
                             const SegFrame *d_work, int stride, int n, uint8_t *d_index_fb, uint32_t *d_rgba,
                             cudaStream_t stream, const Extra &...fx) {
    constexpr bool kSeen = (std::is_same_v<Extra, SeenTables> || ...);
    if (n <= 0) return cudaSuccess;
    const int strips = (vw.W + 31) / 32;
    const int nblocks = (int)(((long long)n * strips + kRasterWarps - 1) / kRasterWarps);
    // the kernel of one frame shape; rgba and kw are std::integral_constant
    const auto go = [&](auto rgba, auto kw) {
        constexpr bool kRgba = decltype(rgba)::value;
        constexpr int kW = decltype(kw)::value;
        if (masked)
            b2d_raster_kernel<kRgba, kW, true, kStates, kLevels, Extra...><<<nblocks, 32 * kRasterWarps, 0, stream>>>(
                t.scene, vw, d_frames, d_work, stride, n, strips, d_index_fb, d_rgba, t.levels, fx...);
        else
            b2d_raster_kernel<kRgba, kW, false, kStates, kLevels, Extra...><<<nblocks, 32 * kRasterWarps, 0, stream>>>(
                t.scene, vw, d_frames, d_work, stride, n, strips, d_index_fb, d_rgba, t.levels, fx...);
    };
    using Index = std::false_type;
    using Rgba = std::true_type;
    if (d_rgba) {
        if constexpr (kSeen) return cudaErrorInvalidValue;
        else if (vw.W == 1920) go(Rgba{}, std::integral_constant<int, 1920>{});
        else go(Rgba{}, std::integral_constant<int, 0>{});
    } else if (vw.W == 1920) go(Index{}, std::integral_constant<int, 1920>{});
    else if (vw.W == 3840) go(Index{}, std::integral_constant<int, 3840>{});  // BASELINE.json's 4K configuration (index frames only)
    else go(Index{}, std::integral_constant<int, 0>{});
    return cudaGetLastError();
}

// The appended tables of a <kStates, kLevels> variant: FixedTables for kFixed, then SeenTables for a seen raster.
template <bool kStates, bool kLevels, bool kFixed>
static cudaError_t raster_tables_go(const BatchTables &t, bool masked, const View &vw, const FrameConst *d_frames,
                                    const SegFrame *d_work, int stride, int n, uint8_t *d_index_fb, uint32_t *d_rgba,
                                    const SeenTables *seen, cudaStream_t stream) {
    const auto go = [&](const auto &...fx) {
        return seen ? raster_go<kStates, kLevels>(t, masked, vw, d_frames, d_work, stride, n, d_index_fb, d_rgba, stream, fx..., *seen)
                    : raster_go<kStates, kLevels>(t, masked, vw, d_frames, d_work, stride, n, d_index_fb, d_rgba, stream, fx...);
    };
    if constexpr (kFixed) return go(t.fixed);
    else return go();
}

// Per-frame states take the kStates variant of each shape; the frames are the same pixel for pixel.  A batch of per-frame
// levels and states with a fixed colormap takes the kFixed variant.
cudaError_t launch_raster(const BatchTables &t, bool masked, const View &vw, const FrameConst *d_frames, const SegFrame *d_work,
                          int stride, int n, uint8_t *d_index_fb, uint32_t *d_rgba, const SeenTables *seen,
                          cudaStream_t stream) {
    if (t.fixed_rows && !(t.per_level && t.per_frame)) return cudaErrorInvalidValue;
    auto go = t.per_level ? (t.per_frame ? (t.fixed_rows ? raster_tables_go<true, true, true> : raster_tables_go<true, true, false>)
                                         : raster_tables_go<false, true, false>)
                          : (t.per_frame ? raster_tables_go<true, false, false> : raster_tables_go<false, false, false>);
    return go(t, masked, vw, d_frames, d_work, stride, n, d_index_fb, d_rgba, seen, stream);
}

namespace {
__global__ void __launch_bounds__(256)
b2d_prelight_kernel(const uint8_t *__restrict__ colormap, const uint8_t *__restrict__ src, uint8_t *__restrict__ dst,
                    size_t n, size_t stride) {
    __shared__ uint8_t cm[32 * 256];
    for (int i = threadIdx.x; i < 32 * 256; i += blockDim.x) cm[i] = colormap[i];
    __syncthreads();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t t = src[i];
#pragma unroll 4
        for (int r = 0; r < 32; r++) dst[(size_t)r * stride + i] = cm[r * 256 + t];
    }
}
}  // namespace

namespace {
// one CTA per texture: pre-lit copies in the layout tex_interleaved() selects
__global__ void __launch_bounds__(256)
b2d_prelight_tex_kernel(const uint8_t *__restrict__ colormap, const uint8_t *__restrict__ texels,
                        const TexRec *__restrict__ tex, int ntex, uint8_t *__restrict__ dst, size_t stride) {
    __shared__ uint8_t cm[32 * 256];
    for (int i = threadIdx.x; i < 32 * 256; i += blockDim.x) cm[i] = colormap[i];
    __syncthreads();
    for (int ti = blockIdx.x; ti < ntex; ti += gridDim.x) {
        const TexRec T = tex[ti];
        const bool inter = tex_interleaved(T);
        const uint32_t n = T.w * T.h;
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
            const uint32_t row = i / T.w, col = i - row * T.w;
            const uint32_t o = lit_index(inter, T.w, row, col);
            const uint32_t t = texels[T.texel_off + i];
            for (int r = 0; r < 32; r++) dst[(size_t)r * stride + T.texel_off + o] = cm[r * 256 + t];
            if (T.mask_off != 0xFFFFFFFFu) dst[(size_t)32 * stride + T.texel_off + o] = texels[T.mask_off + i];   // opacity
        }
    }
}
}  // namespace

namespace {
// one more pre-lit plane, of one COLORMAP row: flats (row-major) and textures (one CTA per texture, in the planes' layout)
__global__ void __launch_bounds__(256)
b2d_prelight_row_kernel(const uint8_t *__restrict__ row, const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, size_t n) {
    __shared__ uint8_t cm[256];
    cm[threadIdx.x] = row[threadIdx.x];
    __syncthreads();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = cm[src[i]];
}

__global__ void __launch_bounds__(256)
b2d_prelight_tex_row_kernel(const uint8_t *__restrict__ row, const uint8_t *__restrict__ texels, const TexRec *__restrict__ tex,
                            int ntex, uint8_t *__restrict__ dst) {
    __shared__ uint8_t cm[256];
    cm[threadIdx.x] = row[threadIdx.x];
    __syncthreads();
    for (int ti = blockIdx.x; ti < ntex; ti += gridDim.x) {
        const TexRec T = tex[ti];
        const bool inter = tex_interleaved(T);
        const uint32_t n = T.w * T.h;
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
            const uint32_t r = i / T.w, col = i - r * T.w;
            dst[T.texel_off + lit_index(inter, T.w, r, col)] = cm[texels[T.texel_off + i]];
        }
    }
}
}  // namespace

cudaError_t launch_prelight_row(const uint8_t *d_row, const uint8_t *d_src, uint8_t *d_dst, size_t n, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    int blocks = (int)((n + 255) / 256);
    if (blocks > device_sms() * 8) blocks = device_sms() * 8;
    b2d_prelight_row_kernel<<<blocks, 256, 0, stream>>>(d_row, d_src, d_dst, n);
    return cudaGetLastError();
}

cudaError_t launch_prelight_textures_row(const uint8_t *d_row, const uint8_t *d_texels, const TexRec *d_tex, int ntex,
                                         uint8_t *d_dst, cudaStream_t stream) {
    if (ntex <= 0) return cudaSuccess;
    const int cap = device_sms() * 8;
    b2d_prelight_tex_row_kernel<<<ntex < cap ? ntex : cap, 256, 0, stream>>>(d_row, d_texels, d_tex, ntex, d_dst);
    return cudaGetLastError();
}

cudaError_t launch_prelight_textures(const uint8_t *d_colormap, const uint8_t *d_texels, const TexRec *d_tex, int ntex,
                                     uint8_t *d_dst, size_t stride, cudaStream_t stream) {
    if (ntex <= 0) return cudaSuccess;
    const int cap = device_sms() * 8;
    b2d_prelight_tex_kernel<<<ntex < cap ? ntex : cap, 256, 0, stream>>>(d_colormap, d_texels, d_tex, ntex, d_dst, stride);
    return cudaGetLastError();
}

cudaError_t launch_prelight(const uint8_t *d_colormap, const uint8_t *d_src, uint8_t *d_dst, size_t n, size_t stride,
                            cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    int blocks = (int)((n + 255) / 256);
    if (blocks > device_sms() * 8) blocks = device_sms() * 8;
    b2d_prelight_kernel<<<blocks, 256, 0, stream>>>(d_colormap, d_src, d_dst, n, stride);
    return cudaGetLastError();
}

namespace {
// Every table set expansion (a batch's per-frame sets, a stale set of a worklist slot, a level's tic-0 sets): one thread
// per output record of every set of the launch, whatever its level -- the state rule of b2d_scene.hpp, the same functions
// scene_at_time runs on the host.  The sets number their records one after the other (StateSet::first, ascending): a
// thread finds its set by binary search.
__global__ void __launch_bounds__(256)
b2d_state_sets_kernel(const StateSrc *__restrict__ srcs, const StateSet *__restrict__ sets, const TableSet *__restrict__ out,
                      const uint32_t *__restrict__ states, int nsets, uint32_t records) {
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < records; g += gridDim.x * blockDim.x) {
        int lo = 0, hi = nsets - 1;          // the last set with first <= g
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (sets[mid].first <= g) lo = mid; else hi = mid - 1;
        }
        const StateSet S = sets[lo];
        const StateSrc &src = srcs[S.level];
        const TableSet o = out[lo];
        StateIn st = state_in(states + S.state, src.ndyn);
        st.extra = S.extralight;
        uint32_t i = g - S.first;
        if (i < src.ntex) { const_cast<TexRec *>(o.tex)[i] = tex_at(src, st, i); continue; }
        i -= src.ntex;
        if (i < src.nsectors) { const_cast<SectorRec *>(o.sectors)[i] = sector_at(src, st, i); continue; }
        i -= src.nsectors;
        if (i < src.nsegs) { const_cast<SegRec *>(o.segs)[i] = seg_at(src, st, i); continue; }
        i -= src.nsegs;
        if (i < src.nsprites) { const_cast<SpriteRec *>(o.sprites)[i] = sprite_at(src, st, i); continue; }
        i -= src.nsprites;
        const_cast<MidRec *>(o.mids)[i] = mid_at(src, st, i);
    }
}
}  // namespace

cudaError_t launch_state_sets(const StateSrc *d_srcs, const StateSet *d_sets, const TableSet *d_out, const uint32_t *d_states,
                              int nsets, uint32_t records, cudaStream_t stream) {
    if (nsets <= 0 || records == 0) return cudaSuccess;
    size_t blocks = ((size_t)records + 255) / 256;
    const size_t cap = (size_t)device_sms() * 16;
    if (blocks > cap) blocks = cap;
    b2d_state_sets_kernel<<<(int)blocks, 256, 0, stream>>>(d_srcs, d_sets, d_out, d_states, nsets, records);
    return cudaGetLastError();
}

cudaError_t launch_palette_levels(const uint32_t *d_palettes, const uint32_t *d_tables, const uint8_t *d_index, uint32_t *d_rgba,
                                  size_t n_frames, size_t npix, cudaStream_t stream) {
    if (n_frames == 0 || npix == 0) return cudaSuccess;
    // ~32 KB of a frame's index bytes per CTA (8 128-bit loads per thread): 64 CTAs per 1080p frame
    const size_t parts = (npix + 32767) / 32768;
    if (n_frames * parts > 0x7FFFFFFFull) return cudaErrorInvalidValue;
    b2d_palette_levels_kernel<<<(unsigned)(n_frames * parts), 256, 0, stream>>>(d_palettes, d_tables, d_index, d_rgba, npix, (int)parts);
    return cudaGetLastError();
}

using ResolveFn = void (*)(const uint32_t *, const uint32_t *, const uint8_t *, uint8_t *, int, int, int, bool);

template <int K>
static ResolveFn resolve_kernel_of(int format) {
    switch (format) {
    case kResolveRgba: return b2d_resolve_kernel<K, kResolveRgba>;
    case kResolveRgb: return b2d_resolve_kernel<K, kResolveRgb>;
    case kResolvePlanar: return b2d_resolve_kernel<K, kResolvePlanar>;
    case kResolveGray: return b2d_resolve_kernel<K, kResolveGray>;
    default: return nullptr;
    }
}

cudaError_t launch_resolve(const uint32_t *d_palettes, const uint32_t *d_tables, const uint8_t *d_index, void *d_out,
                           size_t n_frames, int W, int H, int factor, int format, cudaStream_t stream) {
    if (n_frames == 0) return cudaSuccess;
    ResolveFn fn = nullptr;
    switch (factor) {
    case 1: fn = resolve_kernel_of<1>(format); break;
    case 2: fn = resolve_kernel_of<2>(format); break;
    case 3: fn = resolve_kernel_of<3>(format); break;
    case 4: fn = resolve_kernel_of<4>(format); break;
    case 5: fn = resolve_kernel_of<5>(format); break;
    case 6: fn = resolve_kernel_of<6>(format); break;
    case 7: fn = resolve_kernel_of<7>(format); break;
    case 8: fn = resolve_kernel_of<8>(format); break;
    }
    if (!fn || W % factor || H % factor) return cudaErrorInvalidValue;
    // output pixels per vector item: 16 / gcd(factor, 16), as in the kernel
    const int P = factor == 2 || factor == 6 ? 8 : factor == 4 ? 4 : factor == 8 ? 2 : 16;
    const bool vec = W % (P * factor) == 0 && (reinterpret_cast<uintptr_t>(d_index) & 15) == 0;
    // ~32 KB of a frame's index bytes per CTA, as K3 per level
    const size_t parts = ((size_t)W * H + 32767) / 32768;
    if (n_frames * parts > 0x7FFFFFFFull) return cudaErrorInvalidValue;
    fn<<<(unsigned)(n_frames * parts), 256, 0, stream>>>(d_palettes, d_tables, d_index, static_cast<uint8_t *>(d_out), W, H,
                                                         (int)parts, vec);
    return cudaGetLastError();
}

cudaError_t launch_palette(const uint32_t *d_palette, const uint8_t *d_index, uint32_t *d_rgba,
                           size_t n_pixels, cudaStream_t stream) {
    if (n_pixels == 0) return cudaSuccess;
    size_t nvec = n_pixels / 16 + 1;
    int blocks = (int)((nvec + 255) / 256);
    const int cap = device_sms() * 16;
    if (blocks > cap) blocks = cap;
    b2d_palette_kernel<<<blocks, 256, 0, stream>>>(d_palette, d_index, d_rgba, n_pixels);
    return cudaGetLastError();
}

namespace {
constexpr int kAutomapTileW = 128, kAutomapTileH = 32;

// Kernel 5, the automap (C19): one CTA per (frame, 128 x 32 tile).  The tile is a u32 key per pixel in shared memory:
// every thread takes items of the frame's level in turn, transforms it, and draws its pixels inside the tile with
// atomicMax of ((item + 1) << 8 | colour), so the last item in draw order wins whatever the schedule; 0 is the
// background, colour 0.  The key's low byte is then written out: 16 bytes per thread, a whole 128-byte line per tile row,
// when the tile is full-width and rows start 16-byte aligned; byte by byte otherwise.
// kSeen, the seen variant (b2d_automap_seen_device, C20): each line is coloured by its frame's row of seen lines
// (`seen` + frame * words; nullptr: every line mapped) and B2D_AUTOMAP_ALLMAP.  `vw` is taken by value: by reference,
// the compiler schedules K5's item loop differently.
template <bool kSeen>
__device__ __forceinline__ void automap_tile(const AutomapLevel *__restrict__ levels, const uint32_t *__restrict__ frame_level,
                                             const Pose *__restrict__ poses, View vw, int32_t scale, int flags,
                                             uint8_t *__restrict__ out, int tiles_x, int tiles, bool vec,
                                             const uint32_t *__restrict__ seen, uint32_t words) {
    __shared__ uint32_t keys[kAutomapTileH * kAutomapTileW];
    const size_t frame = blockIdx.x / tiles;
    const int tile = blockIdx.x - (int)(frame * tiles);
    const int tx0 = (tile % tiles_x) * kAutomapTileW, ty0 = (tile / tiles_x) * kAutomapTileH;
    const int tx1 = min(tx0 + kAutomapTileW, vw.W), ty1 = min(ty0 + kAutomapTileH, vw.H);
    for (int k = threadIdx.x; k < kAutomapTileH * kAutomapTileW; k += blockDim.x) keys[k] = 0;
    const AutomapLevel L = levels[frame_level ? frame_level[frame] : 0];
    const AutomapFrame f = automap_frame(poses[frame], vw, scale, flags);
    const uint32_t *mapped = seen ? seen + frame * words : nullptr;
    __syncthreads();
    const int n = automap_items(L, flags);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        int64_t e[4];
        const uint32_t colour = kSeen ? automap_seen_item(f, L, mapped, flags, i, e) : automap_item(f, L, flags, i, e);
        if (!colour) continue;
        const uint32_t key = ((uint32_t)(i + 1) << 8) | colour;
        automap_line(e[0], e[1], e[2], e[3], tx0, ty0, tx1, ty1,
                     [&](int32_t x, int32_t y) { atomicMax(&keys[(y - ty0) * kAutomapTileW + (x - tx0)], key); });
    }
    __syncthreads();
    uint8_t *dst = out + frame * (size_t)vw.W * vw.H;
    if (vec && tx1 - tx0 == kAutomapTileW) {
        const int r = threadIdx.x >> 3, c = (threadIdx.x & 7) * 16;     // 8 threads per 128-byte row
        if (ty0 + r < ty1) {
            const uint32_t *k = &keys[r * kAutomapTileW + c];
            uint32_t w[4];
            for (int q = 0; q < 4; q++)
                w[q] = (k[4 * q] & 0xFF) | (k[4 * q + 1] & 0xFF) << 8 | (k[4 * q + 2] & 0xFF) << 16 | (k[4 * q + 3] & 0xFF) << 24;
            *reinterpret_cast<uint4 *>(dst + (size_t)(ty0 + r) * vw.W + tx0 + c) = make_uint4(w[0], w[1], w[2], w[3]);
        }
    } else {
        for (int k = threadIdx.x; k < kAutomapTileH * kAutomapTileW; k += blockDim.x) {
            const int x = tx0 + (k % kAutomapTileW), y = ty0 + k / kAutomapTileW;
            if (x < tx1 && y < ty1) dst[(size_t)y * vw.W + x] = (uint8_t)keys[k];
        }
    }
}

__global__ void __launch_bounds__(256)
b2d_automap_kernel(const AutomapLevel *__restrict__ levels, const uint32_t *__restrict__ frame_level, const Pose *__restrict__ poses,
                   View vw, int32_t scale, int flags, uint8_t *__restrict__ out, int tiles_x, int tiles, bool vec) {
    automap_tile<false>(levels, frame_level, poses, vw, scale, flags, out, tiles_x, tiles, vec, nullptr, 0);
}

// Kernel 5's seen variant: a kernel of its own, so that K5's code stays as it is.
__global__ void __launch_bounds__(256)
b2d_automap_seen_kernel(const AutomapLevel *__restrict__ levels, const uint32_t *__restrict__ frame_level,
                        const Pose *__restrict__ poses, View vw, int32_t scale, int flags, uint8_t *__restrict__ out,
                        int tiles_x, int tiles, bool vec, const uint32_t *__restrict__ seen, uint32_t words) {
    automap_tile<true>(levels, frame_level, poses, vw, scale, flags, out, tiles_x, tiles, vec, seen, words);
}
}  // namespace

size_t automap_tiles(const View &vw) {
    return (size_t)((vw.W + kAutomapTileW - 1) / kAutomapTileW) * (size_t)((vw.H + kAutomapTileH - 1) / kAutomapTileH);
}

cudaError_t launch_automap(const AutomapLevel *d_levels, const uint32_t *d_frame_level, const Pose *d_poses, size_t n_frames,
                           const View &vw, int32_t scale, int flags, bool seen_variant, const uint32_t *d_seen, uint32_t words,
                           uint8_t *d_out, cudaStream_t stream) {
    if (n_frames == 0) return cudaSuccess;
    const int tiles_x = (vw.W + kAutomapTileW - 1) / kAutomapTileW;
    const int tiles = (int)automap_tiles(vw);
    if (n_frames * (size_t)tiles > 0x7FFFFFFFull) return cudaErrorInvalidValue;
    const bool vec = vw.W % 16 == 0 && (reinterpret_cast<uintptr_t>(d_out) & 15) == 0;
    const unsigned blocks = (unsigned)(n_frames * tiles);
    if (seen_variant)
        b2d_automap_seen_kernel<<<blocks, 256, 0, stream>>>(d_levels, d_frame_level, d_poses, vw, scale, flags, d_out, tiles_x,
                                                            tiles, vec, d_seen, words);
    else
        b2d_automap_kernel<<<blocks, 256, 0, stream>>>(d_levels, d_frame_level, d_poses, vw, scale, flags, d_out, tiles_x, tiles,
                                                       vec);
    return cudaGetLastError();
}

}  // namespace b2d
