// Integer pixel-contract arithmetic shared by the CUDA kernels (DESIGN.md "Pixel contract").
//
// Every function is exact integer math so that the palette-index framebuffer is reproducible bit
// for bit.  The functions are __host__ __device__ so that tests/hostcheck can run the very same
// code on the CPU (one lane at a time) and compare it with the oracle before any GPU time is spent;
// the shipped library contains no CPU rendering path.
//
// Reference semantics restated here (cristicbz/rust-doom):
//   BSP side rule                      math/src/line.rs:41-43, wad/src/visitor.rs:1051-1057
//   wall texel floor-mod sampling      assets/shaders/static.frag:19-22
//   flat texel rule                    game/src/level.rs:537-549
//   light -> colormap row              assets/shaders/static.vert:41-43, static.frag:15-27
//   sky lookup                         assets/shaders/sky.vert:9-16, sky.frag:12-26
//   projection constants               game/src/player.rs:84-89, engine/src/projections.rs:93-101
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2D_HD __host__ __device__ __forceinline__
#else
#define B2D_HD inline
#endif

namespace b2d {

struct Pose { int32_t x, y, z; uint32_t angle; };     // == b2d_pose
struct View { int32_t W, H, F, FY2; };                // == b2d_view

// Per-frame constants produced by the BSP-walk kernel and consumed by the raster kernel.
struct FrameConst {
    Pose pose;
    int32_t cosq, sinq;        // Q30
    int32_t px8, py8;          // camera position, Q8
    int32_t count;             // worklist length
    int32_t status;            // 0 ok, else kStatus* bits
    int32_t set;               // per-frame states: the frame's TableSet (LevelTables::sets), else 0
    int32_t level;             // per-frame levels: the frame's level (LevelTables::scenes), else 0
    int32_t pad[4];
};
static_assert(sizeof(FrameConst) == 64, "FrameConst");

// Completeness status of a frame (FrameConst::status), OR-ed over every launch into the renderer's status flag
// (b2d_renderer_status).  Any bit set: the frame is incomplete.
constexpr int32_t kStatusStackOverflow = 1;   // BSP traversal stack overflow
constexpr int32_t kStatusWorklistFull = 2;    // more worklist entries than the per-frame stride
constexpr int32_t kStatusNoTermination = 4;   // BSP traversal budget exhausted (cyclic node graph)
constexpr int32_t kStatusMaskedFull = 8;      // deferred masked entries: strip cap or arena exhausted

// One worklist entry: a front-facing seg that may be visible, with its per-frame projection
// coefficients.  N(x) = Nc + Nx*x and D(x) = Dc + Dx*x are the numerator / denominator of the
// seg parameter s = N/D at screen column x; 1/depth is proportional to D.
struct SegFrame {
    int64_t Nc, Nx, Dc, Dx;
    int64_t Dmax;              // D clamp: depth >= 1 map unit
    uint32_t Rm;               // floor(2^62 / normalised(F*C))
    int16_t sh, e;             // normalisation shift of N,D; scale exponent
    int32_t seg;
    int16_t xlo, xhi;          // exact visible column interval
    int32_t flags;             // bit0: every column in [xlo,xhi] passes column_eval
    int32_t pad;
};
static_assert(sizeof(SegFrame) == 64, "SegFrame");

constexpr int32_t kSegFrameNoSkip = 1;

// ------------------------------------------------------------------------------------------------
B2D_HD int bitlen64(uint64_t v) {
#if defined(__CUDA_ARCH__)
    return 64 - __clzll((long long)v);
#else
    return v ? 64 - __builtin_clzll(v) : 0;
#endif
}
B2D_HD int64_t floordiv64(int64_t a, int64_t b) {      // b > 0
    int64_t q = a / b;
    return (a % b != 0 && a < 0) ? q - 1 : q;
}
B2D_HD int32_t floormod32(int32_t a, int32_t b) {      // b > 0
    int32_t r = a % b;
    return r < 0 ? r + b : r;
}
template <typename T> B2D_HD T clampv(T v, T lo, T hi) { return v < lo ? lo : (v > hi ? hi : v); }
B2D_HD uint32_t umulhi32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}

// sin/cos of a BAM angle, Q30, integer Taylor series on [0, pi/4] with octant folding.
B2D_HD void sincos_q30(uint32_t angle, int32_t &cosq, int32_t &sinq) {
    const int64_t one = (int64_t)1 << 30;
    uint32_t quad = angle >> 30;
    uint32_t r = angle & 0x3FFFFFFFu;
    bool swap = false;
    if (r > 0x20000000u) { r = 0x40000000u - r; swap = true; }
    int64_t x = ((int64_t)r * 1686629713LL) >> 30;
    int64_t x2 = (x * x) >> 30;
    int64_t t = one - x2 / 72;
    t = one - ((x2 * t) >> 30) / 42;
    t = one - ((x2 * t) >> 30) / 20;
    t = one - ((x2 * t) >> 30) / 6;
    int64_t s = (x * t) >> 30;
    t = one - x2 / 90;
    t = one - ((x2 * t) >> 30) / 56;
    t = one - ((x2 * t) >> 30) / 30;
    t = one - ((x2 * t) >> 30) / 12;
    int64_t c = one - ((x2 * t) >> 30) / 2;
    if (swap) { int64_t tmp = s; s = c; c = tmp; }
    int64_t cc, ss;
    if (quad == 0) { cc = c; ss = s; }
    else if (quad == 1) { cc = -s; ss = c; }
    else if (quad == 2) { cc = -c; ss = -s; }
    else { cc = s; ss = -c; }
    cosq = (int32_t)cc; sinq = (int32_t)ss;
}

B2D_HD void frame_setup(const Pose &p, FrameConst &f) {
    f.pose = p;
    sincos_q30(p.angle, f.cosq, f.sinq);
    f.px8 = p.x >> 8;
    f.py8 = p.y >> 8;
    f.count = 0;
    f.status = 0;
}

// world (map units) -> view space Q8: tx to the right, tz forward.
B2D_HD void to_view(const FrameConst &f, int32_t wx, int32_t wy, int32_t &tx, int32_t &tz) {
    int64_t dx = ((int64_t)wx << 8) - f.px8;
    int64_t dy = ((int64_t)wy << 8) - f.py8;
    tx = (int32_t)((dx * f.sinq - dy * f.cosq) >> 30);
    tz = (int32_t)((dx * f.cosq + dy * f.sinq) >> 30);
}

// BSP side: 1 = left child is on the camera's side (sd > 0), 0 = right child.
B2D_HD int node_side(const Pose &p, int32_t nx, int32_t ny, int32_t ndx, int32_t ndy) {
    int64_t sd = ((int64_t)p.y - ((int64_t)ny << 16)) * ndx - ((int64_t)p.x - ((int64_t)nx << 16)) * ndy;
    return sd > 0 ? 1 : 0;
}

// a + b*x >= c over integer x, intersected into [lo, hi]
B2D_HD void constrain(int64_t &lo, int64_t &hi, int64_t a, int64_t b, int64_t c) {
    if (b > 0) { int64_t v = -floordiv64(-(c - a), b); if (v > lo) lo = v; }
    else if (b < 0) { int64_t v = floordiv64(a - c, -b); if (v < hi) hi = v; }
    else if (a < c) { hi = lo - 1; }
}

// Largest focal length (F, FY2) a renderer accepts; b2d_view_init's largest is FY2 = 247 485 (2160 rows, fov just over
// 1 degree).  With F <= 2^18, M = F * C of seg_frame_setup fits in 63 bits while |C| <= (eye-to-vertex distance) x (seg
// length) stays below 2^45 in Q8 x Q8, i.e. 2^29 square map units (DESIGN.md "Pixel contract", arithmetic limits).
constexpr int32_t kViewFocalMax = 1 << 18;
// Widest view per unit of F a renderer accepts (W <= 256 F).  View space is Q8 (1/256 map unit); a screen-edge pixel spans
// about 2F / W^2 radians, so past this ratio the rounding of far vertices moves edges and texels by several pixels.
constexpr int32_t kViewWidthPerF = 256;

struct ColumnEval {
    uint32_t s24;      // seg parameter s in Q24
    int32_t scale;     // pixels per map unit, Q18, for the rows: row_scale() of the column's scale
    int32_t iscale;    // map units per pixel, Q20, clamped to [1, 2^23]
    int32_t z8;        // view depth in 1/8 map units, <= 65535
};

// The scale the rows are placed with (yrow, clip_rows): capped at 2^31 - 1 (8192 pixels per map unit).  A wall nearer than
// FY2 / 16384 map units is then placed as if at that depth, where the whole screen spans H / 16384 <= 0.14 map units
// vertically: only an eye within that distance of one of its edge heights can tell.  Texture step and light keep the
// full scale.
B2D_HD int32_t row_scale(int64_t scale) { return scale < 0x7FFFFFFF ? (int32_t)scale : 0x7FFFFFFF; }

// Per-frame projection setup of one seg from its view-space endpoints.  Returns false if the seg is
// back-facing / degenerate or covers no screen column.
B2D_HD bool seg_frame_setup(const View &vw, int32_t ax_, int32_t az_, int32_t bx_, int32_t bz_, SegFrame &sf,
                            bool want_noskip = true);

// map units per pixel (Q20, clamped to [1, 2^23]) and view depth in 1/8 map units (<= 65535) of a column drawn at
// `scale` pixels per map unit (Q18, >= 1)
B2D_HD void scale_depth(const View &vw, int64_t scale, int32_t &iscale, int32_t &z8) {
    iscale = (int32_t)clampv<int64_t>(((int64_t)1 << 38) / scale, 1, 1 << 23);
    const int64_t z = ((int64_t)iscale * vw.FY2) >> 18;
    z8 = z > 65535 ? 65535 : (int32_t)z;
}

// Column predicate + per-column projection values.  Exact: does not rely on xlo/xhi.
B2D_HD bool column_eval(const SegFrame &sf, const View &vw, int x, ColumnEval &out) {
    int64_t N = sf.Nc + sf.Nx * x, D = sf.Dc + sf.Dx * x;
    if (D <= 0 || N < 0 || N > D) return false;
    int64_t Dt = D >> sf.sh;
    if (Dt < 1) return false;
    uint64_t Nn = (uint64_t)(N >> sf.sh);
    out.s24 = (uint32_t)((Nn << 24) / (uint64_t)Dt);
    int64_t Dcl = D < sf.Dmax ? D : sf.Dmax;
    uint64_t Dn = (uint64_t)(Dcl >> sf.sh);
    if (Dn < 1) return false;
    uint64_t P = (Dn * (uint64_t)sf.Rm) >> 32;
    uint64_t prod = (uint64_t)vw.FY2 * P;
    const int64_t cap = (int64_t)vw.FY2 << 17;
    int e = sf.e;
    int64_t scale;
    if (e >= 0) scale = e > 63 ? 0 : (int64_t)(prod >> e);
    else scale = (-e) >= 20 ? cap : (int64_t)(prod << (-e));
    if (scale > cap) scale = cap;
    if (scale < 1) return false;
    out.scale = row_scale(scale);
    scale_depth(vw, scale, out.iscale, out.z8);
    return true;
}

B2D_HD bool seg_frame_setup(const View &vw, int32_t ax_, int32_t az_, int32_t bx_, int32_t bz_, SegFrame &sf,
                            bool want_noskip) {
    const int64_t ax = ax_, az = az_, bx = bx_, bz = bz_;
    const int64_t F = vw.F, W = vw.W;
    if (az_ <= 0 && bz_ <= 0) return false;       // wholly behind the camera plane: no column can see it
    int64_t dxs = bx - ax, dzs = bz - az;
    int64_t C = az * dxs - ax * dzs;
    if (C <= 0) return false;
    sf.Nx = 2 * az; sf.Nc = az * (1 - W) - ax * F;
    sf.Dx = -2 * dzs; sf.Dc = dxs * F - dzs * (1 - W);
    {   // division-free rejects: a linear function that is negative at both screen edges is negative on
        // the whole screen (exact; the interval solve below would come out empty)
        const int64_t xr = W - 1;
        const int64_t n0 = sf.Nc, n1 = sf.Nc + sf.Nx * xr, d0 = sf.Dc, d1 = sf.Dc + sf.Dx * xr;
        if ((n0 < 0 && n1 < 0) || (d0 < 1 && d1 < 1) || (d0 - n0 < 0 && d1 - n1 < 0)) return false;
    }
    int64_t lo = 0, hi = W - 1;
    constrain(lo, hi, sf.Dc, sf.Dx, 1);
    constrain(lo, hi, sf.Nc, sf.Nx, 0);
    constrain(lo, hi, sf.Dc - sf.Nc, sf.Dx - sf.Nx, 0);
    if (lo > hi) return false;
    sf.xlo = (int16_t)lo; sf.xhi = (int16_t)hi;
    int64_t Dbound = (dxs < 0 ? -dxs : dxs) * F + (dzs < 0 ? -dzs : dzs) * W;
    int sh = bitlen64((uint64_t)Dbound) - 31;
    if (sh < 0) sh = 0;
    int64_t M = F * C;
    int shm = bitlen64((uint64_t)M) - 31;
    uint64_t Mn = shm >= 0 ? ((uint64_t)M >> shm) : ((uint64_t)M << (-shm));
    uint64_t Rm = ((uint64_t)1 << 62) / Mn;
    if (Rm > 0xFFFFFFFFull) Rm = 0xFFFFFFFFull;
    sf.Rm = (uint32_t)Rm;
    sf.sh = (int16_t)sh;
    sf.e = (int16_t)(5 - sh + shm);
    sf.Dmax = M >> 8;
    // no-skip guarantee (only solid segs need it): column_eval's early-outs are monotone in D, so the
    // two endpoints decide for the whole interval
    sf.flags = 0;
    if (want_noskip) {
        ColumnEval ce;
        bool ok = column_eval(sf, vw, (int)lo, ce) && column_eval(sf, vw, (int)hi, ce);
        sf.flags = ok ? kSegFrameNoSkip : 0;
    }
    sf.pad = 0;
    return true;
}

// A seg closes every column it covers when it is one-sided or its back sector is shut.  It is solid for the walk (marks
// its columns in the solid-column mask) when it closes and passes column_eval on every column of [xlo, xhi].
B2D_HD bool seg_closes(bool two, int32_t otop, int32_t obot) { return !two || otop <= obot; }
B2D_HD bool seg_solid(bool closes, const SegFrame &sf) { return closes && (sf.flags & kSegFrameNoSkip); }

// colormap row from light byte b and depth z8: clamp(floor(64(255-b)/255 - 2880/(z+90)), 0, 31)
B2D_HD int light_row(int b, int32_t z8) {
    uint32_t Z = (uint32_t)z8 + 720u;
    int32_t num = (int32_t)(64u * (uint32_t)(255 - b) * Z) - 5875200;    // < 2^31
    if (num <= 0) return 0;
    uint32_t r = (uint32_t)num / (255u * Z);
    return r > 31u ? 31 : (int)r;
}

// first row whose centre lies at or below the projection of height h (map units): ceil(Y - 1/2)
B2D_HD int yrow(int32_t h, int32_t scale, int32_t pose_z, int32_t H) {
    int64_t hrel8 = ((int64_t)h << 8) - (int64_t)(pose_z >> 8);
    int64_t Y = ((int64_t)H << 25) - hrel8 * scale;
    int64_t r = (Y + ((int64_t)1 << 25) - 1) >> 26;
    return (int)clampv<int64_t>(r, 0, H);
}

// ---- one wall column inside the open window [ct, cb) of its screen column (DESIGN.md C6, C7) ----
// A ceiling is drawn only above the eye and a floor only below it; a sky plane either way.
B2D_HD bool plane_visible(bool ceiling, int32_t h, bool sky, int32_t pose_z) {
    const int64_t h16 = (int64_t)h << 16;
    return (ceiling ? h16 > pose_z : h16 < pose_z) || sky;
}
// y1 wall top, y2 end of the upper piece (one-sided: of the middle), y3 start of the lower piece, y4 start of the floor:
// ceiling [ct, y1), upper [y1, y2), opening [y2, y3), lower [y3, y4), floor [y4, cb)
struct WallRows { int y1, y2, y3, y4; };
B2D_HD WallRows wall_rows(int32_t ceil, int32_t floor, bool two, int32_t otop, int32_t obot, int32_t scale, int32_t pose_z,
                          int32_t H, int ct, int cb) {
    WallRows r;
    const int yfc = yrow(ceil, scale, pose_z, H), yff = yrow(floor, scale, pose_z, H);
    r.y1 = clampv(yfc, ct, cb);
    if (!two) {
        r.y2 = clampv(yff, r.y1, cb);
        r.y3 = r.y2; r.y4 = r.y2;
    } else {
        r.y2 = clampv(yrow(otop, scale, pose_z, H), r.y1, cb);
        r.y3 = clampv(yrow(obot, scale, pose_z, H), r.y2, cb);
        r.y4 = clampv(yff, r.y3, cb);
    }
    return r;
}
// Piece A is the upper piece of a two-sided seg (only below a higher front ceiling) or the middle of a one-sided one;
// piece B is the lower piece of a two-sided seg (only above a lower front floor).
B2D_HD bool wall_piece(bool upper, bool two, int32_t ceil, int32_t floor, int32_t otop, int32_t obot) {
    return upper ? (!two || otop < ceil) : (two && obot > floor);
}
// the window the column leaves open behind the seg: the opening of a two-sided seg, else none
B2D_HD void wall_window(bool two, const WallRows &r, int32_t H, int &ct, int &cb) {
    if (!two || r.y2 >= r.y3) { ct = H; cb = 0; }
    else { ct = r.y2; cb = r.y3; }
}
// texture column at seg parameter s24 (Q24) of a seg with offset uoff and length len_q12 (Q12), before the floor-mod
B2D_HD int32_t wall_column(int32_t uoff, int32_t len_q12, uint32_t s24) {
    return uoff + (int32_t)(((uint64_t)s24 * (uint32_t)len_q12) >> 36);
}
// clip a deferred window [ya, yb) to the rows of a masked piece (masked middle or sprite) between heights low and high
B2D_HD void clip_rows(int32_t high, int32_t low, int32_t scale, int32_t pose_z, int32_t H, int &ya, int &yb) {
    const int a = yrow(high, scale, pose_z, H), b = yrow(low, scale, pose_z, H);
    if (a > ya) ya = a;
    if (b < yb) yb = b;
}

B2D_HD uint32_t yslope_entry(int y, const View &vw) {
    int32_t r2 = 2 * y + 1 - vw.H;
    if (r2 < 0) r2 = -r2;
    if (r2 == 0) r2 = 1;
    // saturated: past 2^32 - 1 (FY2 > 65535, the centre rows only) plane_row's depth saturates as well for |h - eye| >= 1/2
    const uint64_t s = ((uint64_t)vw.FY2 << 16) / (uint32_t)r2;
    return s > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)s;
}

// |h*2^16 - eye_z| clamped to 2048 map units
B2D_HD uint32_t plane_habs(int32_t h, int32_t pose_z) {
    int64_t hrel = clampv<int64_t>(((int64_t)h << 16) - pose_z, -((int64_t)1 << 27), (int64_t)1 << 27);
    return (uint32_t)(hrel < 0 ? -hrel : hrel);
}
B2D_HD int32_t wall_hrel(int32_t h, int32_t pose_z) {
    return (int32_t)clampv<int64_t>(((int64_t)h << 16) - pose_z, -((int64_t)1 << 27), (int64_t)1 << 27);
}

// Texture mapping of a horizontal plane (DESIGN.md C8): the map position under pixel (x, y) is eye + z(y) * dir(x) with
// z the view depth of screen row y on the plane and dir(x) = forward + right * (2x+1-W)/F the direction of column x's ray
// (unit forward component).  Per column (once per frame): dir in Q18.  Per row and plane: z in Q8 and the light row.
// Per pixel: U = (pose.x << 10) + z * dirx, V likewise -- two 32-bit multiply-adds, Q26 modulo 64 texels by wrap-around.
struct PlaneDir { int32_t ax, ay; };                     // Q18
B2D_HD PlaneDir plane_dir(const FrameConst &f, const View &vw, int x, uint32_t invF) {
    const int64_t c2 = 2 * (int64_t)x + 1 - vw.W;
    // (cos*F + sin*c2) / F and (sin*F - cos*c2) / F, Q30 -> Q18 through invF = floor(2^32 / F): (n * invF) >> 40 as the
    // high word of n * (invF << 24), since n * invF passes 2^63 once |c2| / F is above about 32 (short, wide views)
    const int64_t nx = ((int64_t)f.cosq * vw.F + (int64_t)f.sinq * c2) >> 4;
    const int64_t ny = ((int64_t)f.sinq * vw.F - (int64_t)f.cosq * c2) >> 4;
    const int64_t m = (int64_t)invF << 24;
    PlaneDir d;
#if defined(__CUDA_ARCH__)
    d.ax = (int32_t)__mul64hi(nx, m);
    d.ay = (int32_t)__mul64hi(ny, m);
#else
    d.ax = (int32_t)(int64_t)(((__int128)nx * m) >> 64);
    d.ay = (int32_t)(int64_t)(((__int128)ny * m) >> 64);
#endif
    return d;
}
struct PlaneRow { uint32_t z8q; int32_t z8; };           // depth Q8 (for the texel), depth in 1/8 units (for the light row)
B2D_HD PlaneRow plane_row(uint32_t habs, uint32_t yslope) {
    PlaneRow pr;
    uint64_t zz = ((uint64_t)habs * yslope) >> 16;
    int32_t z16 = zz > 0x7FFFFFFFull ? 0x7FFFFFFF : (int32_t)zz;
    pr.z8q = (uint32_t)(z16 >> 8);
    int32_t z8 = z16 >> 13;
    pr.z8 = z8 > 65535 ? 65535 : z8;
    return pr;
}
B2D_HD uint32_t plane_u(int32_t pose_xy, uint32_t z8q, int32_t a) { return ((uint32_t)pose_xy << 10) + z8q * (uint32_t)a; }
B2D_HD uint32_t flat_index(uint32_t U, uint32_t V) { return ((U >> 26) << 6) | (V >> 26); }
// the same index on top of a plane/flat offset given in units of 64 bytes: ((cm6 + (U >> 26)) << 6) | (V >> 26)
B2D_HD uint32_t flat_offset(uint32_t cm6, uint32_t U, uint32_t V) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(V, cm6 + (U >> 26), 6);
#else
    return ((cm6 + (U >> 26)) << 6) | (V >> 26);
#endif
}

// wall texture row: t(y) = tbase + y*tstep (Q16); row index = floor-mod of t>>16 by the height,
// evaluated with the per-texture magic reciprocal hmagic = floor(2^32 / h) + 1 (mod 2^32): exact for 1 <= h <= 4096 and
// |t>>16| < 2^14, which every wall, masked middle and sprite column stays inside (tests/test_texture_sizes.py derives the
// bound).  For h = 1 the magic wraps to 1 and the quotient to 0; the final select maps that case (and, defensively, any
// t outside the domain) to a row inside the texture.
B2D_HD int32_t wall_tbase(int32_t tA, int32_t hA, int32_t pose_z, int32_t H, int32_t iscale) {
    int64_t t = ((int64_t)tA << 16) + wall_hrel(hA, pose_z) + (((int64_t)(1 - H) * iscale) >> 5);
    return (int32_t)t;
}
B2D_HD uint32_t wall_row(int32_t t, uint32_t h, uint32_t hmagic, uint32_t hbias) {
    uint32_t n = ((uint32_t)t + (hbias << 16)) >> 16;
    uint32_t q = umulhi32(n, hmagic);
    const uint32_t r = n - q * h;
    return r < h ? r : 0u;
}

// ---- pre-lit texel planes (product-side data layout; results are the same bytes as colormap[row][texel]) -------
// Layout of a texture inside a pre-lit plane.  Heights that are a multiple of 4 (every stock wall texture) are
// stored **4 rows interleaved**: texel (row, col) lives at ((row >> 2) * w + col) * 4 + (row & 3), so one aligned
// 32-bit word holds four vertically adjacent texels of a column and the 32 lanes of a warp (adjacent columns) read
// one 128-byte line.  A wall column that is magnified on screen -- the common case at 1080p -- then needs two word
// loads for eight rows instead of eight byte loads.  Other heights keep the blob's row-major layout.
B2D_HD bool tex_interleaved(uint32_t h, uint32_t texel_off) { return (h & 3u) == 0u && (texel_off & 3u) == 0u && h <= 4096u; }
B2D_HD uint32_t lit_index(bool inter, uint32_t w, uint32_t row, uint32_t col) {
    return inter ? ((row >> 2) * w + col) * 4u + (row & 3u) : row * w + col;
}
// Word path of a batch of rows t, t + tstep, ...: `acc` is t with its integer part replaced by (first row & 3);
// pixel k of the batch reads byte (acc + k * tstep) >> 16 of the 8 bytes {row quad r0 >> 2, next row quad}.
B2D_HD uint32_t wall_acc(uint32_t t, uint32_t r0) { return (t & 0xFFFFu) | ((r0 & 3u) << 16); }
B2D_HD uint32_t next_quad(uint32_t q0, uint32_t h) { return q0 + 1u == (h >> 2) ? 0u : q0 + 1u; }
// the byte PRMT selects for a selector below 8 (bytes 0-3 from lo, 4-7 from hi)
B2D_HD uint32_t pick_byte(uint32_t lo, uint32_t hi, uint32_t sel) {
#if defined(__CUDA_ARCH__)
    uint32_t d;                      // raw PRMT: sel < 8, so no sign-replicate bit and no need for __byte_perm's mask
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(lo), "r"(hi), "r"(sel));
    return d;
#else
    return ((sel & 4u) ? hi : lo) >> (8u * (sel & 3u)) & 0xFFu;
#endif
}

// ---- magnified wall columns: incremental row tracking -----------------------------------------------------------
// A column whose texture step is small enough that R consecutive screen rows (and the step to the next batch),
// starting anywhere inside a row quad, stay inside that quad and the next one (R * tstep <= 4 texture rows) needs no
// per-batch floor-mod: the state is the row quad q (0 .. h/4-1) and a Q29 accumulator whose top three bits are the
// byte index inside the 8-byte window {quad q, quad q+1} and whose low 29 bits are the fraction of the texture row.
// Row k of a batch reads byte (acc + k * (tstep << 13)) >> 29 of that window: one IMAD, one shift.  Same rows as
// wall_row(t0 + k*tstep) by construction: (t0 + k*tstep) >> 16 == (t0 >> 16) + (((t0 & 0xFFFF) + k*tstep) >> 16)
// while nothing wraps, and the byte index never exceeds 3 + 4 = 7.
constexpr uint32_t kWallFast8 = 32768u;    // 8 * tstep <= 4 * 65536
constexpr uint32_t kWallFast16 = 16384u;   // 16 * tstep <= 4 * 65536
B2D_HD uint32_t wall_acc29(uint32_t t, uint32_t r0) { return ((r0 & 3u) << 29) | ((t & 0xFFFFu) << 13); }
B2D_HD uint32_t wall_sel(uint32_t acc, uint32_t ts29, uint32_t k) { return (acc + k * ts29) >> 29; }
// after R rows: move the window by whole quads (at most one: the index is <= 7; nq >= 2), keep (row & 3 | fraction)
B2D_HD void wall_advance(uint32_t &acc, uint32_t &q, uint32_t ts29, uint32_t R, uint32_t nq) {
    acc += R * ts29;
    q += acc >> 31;
    if (q >= nq) q -= nq;
    acc &= 0x7FFFFFFFu;
}
// bit k set <=> row y + k lies in [ya, yb), k < R <= 16
B2D_HD uint32_t row_mask(int y, int ya, int yb, int R) {
    int lo = ya - y, hi = yb - y;
    if (lo < 0) lo = 0;
    if (hi > R) hi = R;
    if (hi <= lo) return 0u;
    return ((1u << hi) - 1u) & ~((1u << lo) - 1u);
}

// sky: column from yaw + screen x (one texture width per NDC unit, 8 widths per turn); row mirrored
// below the horizon.
B2D_HD uint32_t sky_u32(int x, const View &vw, uint32_t angle) {
    uint64_t num = ((uint64_t)(2 * x + 1)) << 32;
    return (uint32_t)(num / (uint32_t)vw.W) - (angle << 3);
}
B2D_HD int32_t sky_row(int y, int32_t H, int32_t skyh) {
    int32_t r = 2 * y + 1;
    if (r < H) return (r * skyh) / H;
    return floormod32(((2 * H - r) * skyh) / H, skyh);
}

// Conservative screen-column range of an axis-aligned map box (top, bottom, left, right).
// false => nothing inside the box can be visible.  Boxes that come within 32 map units of the
// camera plane are treated as covering the whole screen.
constexpr int32_t kBoxNearQ8 = 32 * 256;
B2D_HD bool box_range(const FrameConst &f, const View &vw, const int32_t box[4], int &lo, int &hi) {
    bool all_behind = true, any_near = false;
    int64_t mn = 0x7FFFFFFFFFFFFFFFLL, mx = -0x7FFFFFFFFFFFFFFFLL;
    for (int i = 0; i < 4; i++) {
        int32_t tx, tz;
        to_view(f, box[2 + (i & 1)], box[i >> 1], tx, tz);
        if (tz >= -256) all_behind = false;
        if (tz < kBoxNearQ8) { any_near = true; continue; }
        int64_t c = floordiv64((int64_t)tx * vw.F, tz);
        int64_t xc = floordiv64(c - 1 + vw.W, 2);
        if (xc < mn) mn = xc;
        if (xc > mx) mx = xc;
    }
    if (all_behind) return false;
    if (any_near) { lo = 0; hi = vw.W - 1; return true; }
    mn -= 2; mx += 2;
    if (mx < 0 || mn > vw.W - 1) return false;
    lo = (int)(mn < 0 ? 0 : mn);
    hi = (int)(mx > vw.W - 1 ? vw.W - 1 : mx);
    return true;
}

// ---- decoration sprites (billboards at constant view depth; visitor.rs:1062-1137, sprite.vert:40-42) ----
// light (sprite.frag:15-27): light = min(v, 2v - dist), dist = 1 - 1/(w+1), w = z/100
B2D_HD int light_row_sprite(int b, int32_t z8) {
    int32_t r1 = (32 * (255 - b)) / 255;
    uint32_t Z = (uint32_t)z8 + 800u;
    int32_t num = (int32_t)(64u * (uint32_t)(255 - b) * Z) - 6528000;
    int32_t r2 = num <= 0 ? 0 : (int32_t)((uint32_t)num / (255u * Z));
    int32_t r = r1 > r2 ? r1 : r2;
    return r > 31 ? 31 : r;
}

struct SpriteFrame {
    int64_t cx, cz;          // view-space centre, Q8
    int32_t lo, hi;          // exact covered column interval
    int32_t scale, iscale, z8;
};

// pixels per map unit (Q18, capped as in column_eval) of a sprite at view depth cz (Q8, >= 256); < 1: no size on screen
B2D_HD int64_t sprite_scale(const View &vw, int64_t cz) {
    const int64_t scale = ((int64_t)vw.FY2 << 25) / cz, cap = (int64_t)vw.FY2 << 17;
    return scale > cap ? cap : scale;
}

// Per-frame projection of a sprite of width w (map units) centred at world (x, y).  false = not on screen.
B2D_HD bool sprite_setup(const FrameConst &f, const View &vw, int32_t x, int32_t y, int32_t w, SpriteFrame &sp) {
    int32_t tx, tz;
    to_view(f, x, y, tx, tz);
    sp.cx = tx; sp.cz = tz;
    if (tz < 256) return false;                              // nearer than one map unit, or behind
    const int64_t F = vw.F, W = vw.W;
    const int64_t L = (sp.cx - (int64_t)w * 128) * F, R = (sp.cx + (int64_t)w * 128) * F;
    int64_t lo = 0, hi = W - 1;
    constrain(lo, hi, sp.cz * (1 - W) - L, 2 * sp.cz, 0);            // cz*c2 >= L
    constrain(lo, hi, R - 1 - sp.cz * (1 - W), -2 * sp.cz, 0);       // cz*c2 <= R-1
    if (lo > hi) return false;
    sp.lo = (int32_t)lo; sp.hi = (int32_t)hi;
    const int64_t scale = sprite_scale(vw, sp.cz);
    if (scale < 1) return false;
    sp.scale = row_scale(scale);
    scale_depth(vw, scale, sp.iscale, sp.z8);
    return true;
}

// A sprite travels through the worklist as a SegFrame: seg = -1 - sprite index, view-space centre (cx, cz) in (Nc, Nx),
// column interval in (xlo, xhi), every other field zero.
B2D_HD void sprite_entry(int sprite, const SpriteFrame &sp, SegFrame &sf) {
    sf.Nc = sp.cx; sf.Nx = sp.cz; sf.Dc = 0; sf.Dx = 0; sf.Dmax = 0; sf.Rm = 0; sf.sh = 0; sf.e = 0;
    sf.seg = -1 - sprite; sf.xlo = (int16_t)sp.lo; sf.xhi = (int16_t)sp.hi; sf.flags = 0; sf.pad = 0;
}
B2D_HD bool is_sprite_entry(const SegFrame &sf) { return sf.seg < 0; }
// sprite index of a sprite entry; sp.cx, sp.cz := its view-space centre
B2D_HD int entry_sprite(const SegFrame &sf, SpriteFrame &sp) {
    sp.cx = sf.Nc; sp.cz = sf.Nx;
    return -1 - sf.seg;
}

// Masked middles and sprites met by the raster's front-to-back pass are deferred to a back-to-front pass, at most
// strip_masked_cap() entries per 32-column strip and frame: the level's total, at least 8, at most kMaskedCapMax
// (more -> kStatusMaskedFull).
constexpr int kMaskedCapMax = 128;
B2D_HD int strip_masked_cap(int nmids, int nsprites) { return clampv(nmids + nsprites, 8, kMaskedCapMax); }

// texture column of screen column x (0..w-1)
B2D_HD int32_t sprite_column(const SpriteFrame &sp, const View &vw, int x, int32_t w) {
    const int64_t c2 = 2 * (int64_t)x + 1 - vw.W;
    const int64_t L = (sp.cx - (int64_t)w * 128) * vw.F;
    return (int32_t)clampv<int64_t>(floordiv64(sp.cz * c2 - L, 256 * (int64_t)vw.F), 0, w - 1);
}

// ---- automap (DESIGN.md C19) -------------------------------------------------------------------
// Flags (== B2D_AUTOMAP_*), the accepted scale range in pixels per map unit, Q16 (1/256 .. 64), and Doom's colours.
constexpr int kAutomapRotate = 1, kAutomapAllLines = 2, kAutomapThings = 4;
constexpr int32_t kAutomapScaleMin = 1 << 8, kAutomapScaleMax = 64 << 16;
constexpr uint32_t kAutomapArrowColour = 209, kAutomapThingColour = 112;
constexpr int32_t kAutomapArrowR = 8 * 16 * 65536 / 7;      // player_arrow's R: 8 * PLAYERRADIUS / 7, 16.16
constexpr int kAutomapArrowSegs = 7, kAutomapThingSegs = 3;
// The seen automap (b2d_automap_seen_device, C20): B2D_AUTOMAP_ALLMAP, the computer area map's grey (GRAYS + 3), and the
// device line table's don't-draw bit.
constexpr int kAutomapAllmap = 8;
constexpr uint32_t kAutomapAllmapColour = 99;
constexpr uint16_t kAutomapDontDraw = 1;

// One linedef of a level's automap table (b2d_automap_line): endpoints in map units, the colour drawn normally and under
// kAutomapAllLines (0: not drawn), and the linedef's index.  `dev_flags` is 0 in the scene's table; the renderer's device
// copy sets kAutomapDontDraw for an ML_DONTDRAW linedef (the seen automap's computer-area-map rule, C20).
struct AutomapLine {
    int32_t x0, y0, x1, y1;
    uint8_t colour, colour_all;
    uint16_t dev_flags;
    int32_t linedef;
};
static_assert(sizeof(AutomapLine) == 24, "AutomapLine");

// A level's automap items: its linedef table and the positions (x, y in map units) of its decoration things in blob order.
struct AutomapLevel {
    const AutomapLine *lines;
    const int32_t *things;
    int32_t nlines, nthings;
};

// A frame's transform: centre (pose x, y in 16.16), the map rotation by 90 deg - angle (used with kAutomapRotate) and the
// arrow's rotation (the pose angle, or 90 deg with kAutomapRotate), both Q30.
struct AutomapFrame {
    int64_t px, py;
    int32_t c, s, ac, as;
    int32_t scale, W, H;
    bool rot;
};
B2D_HD AutomapFrame automap_frame(const Pose &p, const View &vw, int32_t scale, int flags) {
    AutomapFrame f;
    f.px = p.x; f.py = p.y;
    f.rot = (flags & kAutomapRotate) != 0;
    sincos_q30(0x40000000u - p.angle, f.c, f.s);
    sincos_q30(f.rot ? 0x40000000u : p.angle, f.ac, f.as);
    f.scale = scale; f.W = vw.W; f.H = vw.H;
    return f;
}

// A 16.16 offset (dx, dy) from the frame's centre, rotated by (c, s) if `rot`, to Q8 screen coordinates (y down).
// |dx|, |dy| <= 2^32 + 2^20 and |c|, |s| <= 2^30 with min(|c|, |s|) <= 2^29.5 keep the rotation below 2^63; the rotated
// offset stays below 2^32.6 and, times scale <= 2^22, X and Y below 2^31 (C19).
B2D_HD void automap_screen(const AutomapFrame &f, int64_t dx, int64_t dy, bool rot, int32_t c, int32_t s, int64_t &X, int64_t &Y) {
    int64_t rx = dx, ry = dy;
    if (rot) {
        rx = (dx * c - dy * s) >> 30;
        ry = (dx * s + dy * c) >> 30;
    }
    X = ((int64_t)f.W << 7) + ((rx * f.scale) >> 24);
    Y = ((int64_t)f.H << 7) - ((ry * f.scale) >> 24);
}
// a map point in 16.16
B2D_HD void automap_map(const AutomapFrame &f, int64_t mx, int64_t my, int64_t &X, int64_t &Y) {
    automap_screen(f, mx - f.px, my - f.py, f.rot, f.c, f.s, X, Y);
}

// Items of a frame in draw order: the level's linedefs, the 7 segments of the player arrow, 3 segments per thing (with
// kAutomapThings).
B2D_HD int automap_items(const AutomapLevel &L, int flags) {
    return L.nlines + kAutomapArrowSegs + ((flags & kAutomapThings) ? kAutomapThingSegs * L.nthings : 0);
}
// Segment i (0..6) of player_arrow, (ax, 0) - (bx, by) in 16.16 offsets from the arrow's centre, pointing along +x.
B2D_HD void automap_arrow_seg(int i, int32_t &ax, int32_t &bx, int32_t &by) {
    constexpr int32_t R = kAutomapArrowR;
    ax = i == 0 ? -R + R / 8 : i <= 2 ? R : i <= 4 ? -R + R / 8 : -R + 3 * R / 8;
    bx = i == 0 ? R : i <= 2 ? R - R / 2 : i <= 4 ? -R - R / 8 : -R + R / 8;
    by = i == 0 ? 0 : (i & 1) ? R / 4 : -(R / 4);
}
// Item i's endpoints in Q8 screen coordinates (e[0], e[1]) - (e[2], e[3]) and its colour (0: not drawn).
B2D_HD uint32_t automap_item(const AutomapFrame &f, const AutomapLevel &L, int flags, int i, int64_t e[4]) {
    if (i < L.nlines) {
        const AutomapLine l = L.lines[i];
        const uint32_t colour = (flags & kAutomapAllLines) ? l.colour_all : l.colour;
        automap_map(f, (int64_t)l.x0 * 65536, (int64_t)l.y0 * 65536, e[0], e[1]);
        automap_map(f, (int64_t)l.x1 * 65536, (int64_t)l.y1 * 65536, e[2], e[3]);
        return colour;
    }
    i -= L.nlines;
    if (i < kAutomapArrowSegs) {          // player_arrow, in its own rotation about the centre
        int32_t ax, bx, by;
        automap_arrow_seg(i, ax, bx, by);
        automap_screen(f, ax, 0, true, f.ac, f.as, e[0], e[1]);
        automap_screen(f, bx, by, true, f.ac, f.as, e[2], e[3]);
        return kAutomapArrowColour;
    }
    i -= kAutomapArrowSegs;
    const int t = i / kAutomapThingSegs, k = i - t * kAutomapThingSegs;     // thintriangle_guy at size 16, angle 0
    const int64_t tx = (int64_t)L.things[2 * t] * 65536, ty = (int64_t)L.things[2 * t + 1] * 65536;
    const int32_t ax = k == 1 ? 1048576 : -524288, ay = k == 0 ? -734000 : k == 1 ? 0 : 734000;
    const int32_t bx = k == 0 ? 1048576 : -524288, by = k == 0 ? 0 : k == 1 ? 734000 : -734000;
    automap_map(f, tx + ax, ty + ay, e[0], e[1]);
    automap_map(f, tx + bx, ty + by, e[2], e[3]);
    return kAutomapThingColour;
}

// AM_drawWalls with mapped lines (C20): under kAutomapAllLines a line's all-lines colour, mapped or not; otherwise a mapped
// line's normal colour (0: not drawn); otherwise, under kAutomapAllmap, grey 99 unless the line is ML_DONTDRAW; else 0.
B2D_HD uint32_t automap_seen_colour(const AutomapLine &l, bool mapped, int flags) {
    if (flags & kAutomapAllLines) return l.colour_all;
    if (mapped) return l.colour;
    if ((flags & kAutomapAllmap) && !(l.dev_flags & kAutomapDontDraw)) return kAutomapAllmapColour;
    return 0;
}
// Item i as automap_item draws it, with the lines coloured by automap_seen_colour: `mapped` is the frame's row of seen
// lines (bit l & 31 of word l >> 5 for linedef l), nullptr for every line mapped.
B2D_HD uint32_t automap_seen_item(const AutomapFrame &f, const AutomapLevel &L, const uint32_t *mapped, int flags, int i,
                                  int64_t e[4]) {
    const uint32_t colour = automap_item(f, L, flags & ~kAutomapAllmap, i, e);
    if (i >= L.nlines) return colour;
    const AutomapLine &l = L.lines[i];
    const uint32_t ld = (uint32_t)l.linedef;
    return automap_seen_colour(l, mapped == nullptr || ((mapped[ld >> 5] >> (ld & 31)) & 1u), flags);
}

// ---- the automap at the frame's state, with other players' arrows (b2d_automap_states_device, C21) ----------------------
// The device line table's bit for a line whose colour can follow the frame's sector heights: two-sided, neither special 39
// nor ML_SECRET, with a dynamic sector on at least one side.  Its AutomapDynLine (same index as the line) holds the rest
// heights of its front [0] and back [1] sectors, from the SECTORS lump, and their dynamic slots (kAutomapNoSlot: none).
constexpr uint16_t kAutomapChangeable = 2;
constexpr uint32_t kAutomapNoSlot = 0xFFFFFFFFu;
constexpr uint32_t kAutomapFloorStep = 64, kAutomapCeilStep = 231, kAutomapPlain = 96;
struct AutomapDynLine {
    int32_t floor[2], ceil[2];
    uint32_t slot[2];
};
static_assert(sizeof(AutomapDynLine) == 24, "AutomapDynLine");
// Another player's arrow (b2d_automap_arrow): position in 16.16 map units, angle in BAM, colour 1..255.
struct AutomapArrow {
    int32_t x, y;
    uint32_t angle, colour;
};
static_assert(sizeof(AutomapArrow) == 16, "AutomapArrow");
// What a frame adds to C20's inputs: its sector offsets (floor, ceiling per dynamic slot; nullptr: at rest), its arrows,
// and its pose's angle (the arrows' rotation under kAutomapRotate).
struct AutomapStateFrame {
    const int32_t *off;
    const AutomapArrow *arrows;
    uint32_t n_arrows, pose_angle;
};

// A changeable line's colours at sector offsets `off`: C19's rule for a two-sided line that is neither a teleporter nor
// secret, with each sector's rest heights plus its slot's offsets (ML_DONTDRAW: not drawn normally).
B2D_HD void automap_state_colours(AutomapLine &l, const AutomapDynLine &d, const int32_t *off) {
    int32_t fl[2], ce[2];
    for (int k = 0; k < 2; k++) {
        const bool dyn = d.slot[k] != kAutomapNoSlot;
        fl[k] = d.floor[k] + (dyn ? off[2 * d.slot[k]] : 0);
        ce[k] = d.ceil[k] + (dyn ? off[2 * d.slot[k] + 1] : 0);
    }
    const uint32_t c = fl[0] != fl[1] ? kAutomapFloorStep : ce[0] != ce[1] ? kAutomapCeilStep : 0u;
    l.colour = (uint8_t)((l.dev_flags & kAutomapDontDraw) ? 0u : c);
    l.colour_all = (uint8_t)(c ? c : kAutomapPlain);
}

// Items of a frame in draw order: the level's linedefs, the player arrow, 7 segments per arrow of the frame, the things.
B2D_HD int automap_state_items(const AutomapLevel &L, const AutomapStateFrame &s, int flags) {
    return automap_items(L, flags) + kAutomapArrowSegs * (int)s.n_arrows;
}

// Segment k of arrow `a`: its centre is its position through the frame's map transform; its shape is turned once by
// sincos_q30 of the arrow's angle (north-up) or of angle + 90 deg - the pose's angle (kAutomapRotate), with the own
// arrow's formula, scaled as automap_screen scales and added to the centre.  An arrow at the pose draws the own arrow.
B2D_HD void automap_arrow(const AutomapFrame &f, const AutomapArrow &a, uint32_t pose_angle, int k, int64_t e[4]) {
    int32_t c, s, ax, bx, by;
    sincos_q30(f.rot ? a.angle + 0x40000000u - pose_angle : a.angle, c, s);
    automap_arrow_seg(k, ax, bx, by);
    int64_t X, Y;
    automap_map(f, a.x, a.y, X, Y);
    X -= (int64_t)f.W << 7;
    Y -= (int64_t)f.H << 7;
    automap_screen(f, ax, 0, true, c, s, e[0], e[1]);
    automap_screen(f, bx, by, true, c, s, e[2], e[3]);
    e[0] += X; e[1] += Y; e[2] += X; e[3] += Y;
}

// Item i as automap_seen_item draws it, with each changeable line coloured at the frame's offsets and the frame's arrows
// after the own arrow.  `dyn`: the level's AutomapDynLine table (read only for changeable lines).  With s.off nullptr and
// no arrows, automap_seen_item.
B2D_HD uint32_t automap_state_item(const AutomapFrame &f, const AutomapLevel &L, const AutomapDynLine *dyn,
                                   const AutomapStateFrame &s, const uint32_t *mapped, int flags, int i, int64_t e[4]) {
    const int own_end = L.nlines + kAutomapArrowSegs;
    if (i >= own_end) {
        const int j = i - own_end;
        if (j < kAutomapArrowSegs * (int)s.n_arrows) {
            const int a = j / kAutomapArrowSegs;
            automap_arrow(f, s.arrows[a], s.pose_angle, j - a * kAutomapArrowSegs, e);
            return s.arrows[a].colour;
        }
        i -= kAutomapArrowSegs * (int)s.n_arrows;      // a thing
    }
    const uint32_t colour = automap_item(f, L, flags & ~kAutomapAllmap, i, e);
    if (i >= L.nlines) return colour;
    AutomapLine l = L.lines[i];
    if (s.off && (l.dev_flags & kAutomapChangeable)) automap_state_colours(l, dyn[i], s.off);
    const uint32_t ld = (uint32_t)l.linedef;
    return automap_seen_colour(l, mapped == nullptr || ((mapped[ld >> 5] >> (ld & 31)) & 1u), flags);
}

// ---- the grid and the numbered marks (b2d_automap_marks_device, C22) ---------------------------------------------------
// B2D_AUTOMAP_GRID; the grid's colour (GRIDCOLORS: GRAYS + GRAYSRANGE / 2) and spacing (MAPBLOCKUNITS), and the map range
// its lines span and lie in.
constexpr int kAutomapGrid = 16;
constexpr uint32_t kAutomapGridColour = 104;
constexpr int64_t kAutomapGridStep = 128, kAutomapGridMin = -32768, kAutomapGridMax = 32767;
constexpr int kAutomapDigits = 10;
// A digit patch (AMMNUM0 .. AMMNUM9): w x h row-major texels, a texel with a non-zero high byte transparent, and its
// picture offsets.  px nullptr: the digit is missing and its marks are not drawn.
struct AutomapDigit {
    const uint16_t *px;
    int32_t w, h, left, top;
};
static_assert(sizeof(AutomapDigit) == 24, "AutomapDigit");
// A level's grid origin (the BLOCKMAP header's, map units) and its digits.
struct AutomapMarkLevel {
    int32_t ox, oy;
    AutomapDigit digit[kAutomapDigits];
};
// A mark (b2d_automap_mark): position in 16.16 map units, digit 0 .. 9.
struct AutomapMark {
    int32_t x, y;
    uint32_t number;
};
static_assert(sizeof(AutomapMark) == 12, "AutomapMark");

B2D_HD int64_t automap_floordiv(int64_t a, int64_t b) {      // b > 0
    const int64_t q = a / b;
    return q - ((a % b != 0 && a < 0) ? 1 : 0);
}
// The lattice of one line family: every j whose line o + 128 j (map units) lies in [-32768, 32767].
B2D_HD void automap_grid_lattice(int32_t o, int64_t &jlo, int64_t &jhi) {
    jlo = -automap_floordiv((int64_t)o - kAutomapGridMin, kAutomapGridStep);
    jhi = automap_floordiv(kAutomapGridMax - (int64_t)o, kAutomapGridStep);
}
// Grid line j of a family (vertical: constant map x = o + 128 j) from one end of the map range to the other, in Q8 screen
// coordinates through the frame's map transform.  |d| <= 2^32 keeps C19's bound.
B2D_HD void automap_grid_line(const AutomapFrame &f, int32_t o, bool vertical, int64_t j, int64_t e[4]) {
    const int64_t at = ((int64_t)o + kAutomapGridStep * j) * 65536, lo = kAutomapGridMin * 65536, hi = kAutomapGridMax * 65536;
    automap_map(f, vertical ? at : lo, vertical ? lo : at, e[0], e[1]);
    automap_map(f, vertical ? at : hi, vertical ? hi : at, e[2], e[3]);
}
// The lattice indices [jlo, jhi] (empty when jlo > jhi) of one family whose lines can draw a pixel of the rectangle
// [x0, x1) x [y0, y1).  Conservative: the rectangle, widened by 2 pixels on each side, is mapped back to map space by the
// transpose of the frame's rotation (north-up: none), and its corners bound the map offset along the family's normal.
// Rounding of the forward transform moves a line by a few Q8 units at most, and a drawn pixel's square meets the line.
B2D_HD void automap_grid_range(const AutomapFrame &f, int32_t o, bool vertical, int32_t x0, int32_t y0, int32_t x1, int32_t y1,
                               int64_t &jlo, int64_t &jhi) {
    constexpr int64_t M = 512;
    const int64_t u0 = (int64_t)x0 * 256 - M - ((int64_t)f.W << 7), u1 = (int64_t)x1 * 256 + M - ((int64_t)f.W << 7);
    const int64_t v0 = ((int64_t)f.H << 7) - (int64_t)y1 * 256 - M, v1 = ((int64_t)f.H << 7) - (int64_t)y0 * 256 + M;
    const int64_t c = f.rot ? f.c : (int64_t)1 << 30, s = f.rot ? f.s : 0;
    const int64_t a = vertical ? c : -s, b = vertical ? s : c;      // the offset along the normal is (a u + b v) / (64 scale)
    const int64_t au0 = a * u0, au1 = a * u1, bv0 = b * v0, bv1 = b * v1;
    const int64_t lo = (au0 < au1 ? au0 : au1) + (bv0 < bv1 ? bv0 : bv1), hi = (au0 < au1 ? au1 : au0) + (bv0 < bv1 ? bv1 : bv0);
    const int64_t div = 64 * (int64_t)f.scale, p = vertical ? f.px : f.py;
    const int64_t dlo = automap_floordiv(lo, div) - 1 + p - (int64_t)o * 65536;
    const int64_t dhi = -automap_floordiv(-hi, div) + 1 + p - (int64_t)o * 65536;
    int64_t llo, lhi;
    automap_grid_lattice(o, llo, lhi);
    jlo = -automap_floordiv(-dlo, kAutomapGridStep * 65536);
    jhi = automap_floordiv(dhi, kAutomapGridStep * 65536);
    if (jlo < llo) jlo = llo;
    if (jhi > lhi) jhi = lhi;
}

// The marks' magnification: Doom's patches are drawn for 200 lines.
B2D_HD int32_t automap_mark_k(int32_t H) { return H / 200 > 1 ? H / 200 : 1; }
// A mark's k w x k h rectangle: its point through the frame's map transform is pixel (X >> 8, Y >> 8), and the patch's
// top-left corner is that pixel minus k (left, top).  False when the digit is missing or the rectangle is not wholly
// inside the frame (Doom's fit test, at the patch's own size).
B2D_HD bool automap_mark_place(const AutomapFrame &f, const AutomapMark &m, const AutomapDigit &d, int32_t k, int32_t &left,
                               int32_t &top) {
    if (!d.px) return false;
    int64_t X, Y;
    automap_map(f, m.x, m.y, X, Y);
    const int64_t l = (X >> 8) - (int64_t)k * d.left, t = (Y >> 8) - (int64_t)k * d.top;
    if (l < 0 || t < 0 || l + (int64_t)k * d.w > f.W || t + (int64_t)k * d.h > f.H) return false;
    left = (int32_t)l;
    top = (int32_t)t;
    return true;
}
// The texel over pixel (x, y) of a mark placed at (left, top): its palette index in the low byte, transparent when the
// high byte is not 0.
B2D_HD uint32_t automap_mark_texel(const AutomapDigit &d, int32_t k, int32_t left, int32_t top, int32_t x, int32_t y) {
    return d.px[(size_t)((y - top) / k) * (size_t)d.w + (size_t)((x - left) / k)];
}

// The pixels of the line (X0, Y0) - (X1, Y1) (Q8, |X|, |Y| < 2^31) inside the pixel rectangle [x0, x1) x [y0, y1), each
// passed to plot(x, y) once.  Along the major axis (|dX| >= |dY|: X) every pixel whose centre lies in the endpoints'
// range, inclusive; its minor coordinate is the floor of the exact interpolation at that centre.  A range without a
// pixel centre draws the pixel holding (X0, Y0).  Pixels are independent, so the range is clamped to the rectangle, and
// the part of it whose minor coordinate falls inside is found by bisection (the minor coordinate is monotone).
template <typename Plot>
B2D_HD void automap_line(int64_t X0, int64_t Y0, int64_t X1, int64_t Y1, int32_t x0, int32_t y0, int32_t x1, int32_t y1,
                         Plot plot) {
    if ((X0 < X1 ? X1 : X0) >> 8 < x0 || (X0 < X1 ? X0 : X1) >> 8 >= x1 || (Y0 < Y1 ? Y1 : Y0) >> 8 < y0 ||
        (Y0 < Y1 ? Y0 : Y1) >> 8 >= y1)
        return;                                             // the bounding box of every pixel the line draws misses
    const bool xmaj = (X1 >= X0 ? X1 - X0 : X0 - X1) >= (Y1 >= Y0 ? Y1 - Y0 : Y0 - Y1);
    int64_t M0 = xmaj ? X0 : Y0, m0 = xmaj ? Y0 : X0, M1 = xmaj ? X1 : Y1, m1 = xmaj ? Y1 : X1;
    if (M1 < M0) {
        int64_t t = M0; M0 = M1; M1 = t;
        t = m0; m0 = m1; m1 = t;
    }
    int64_t lo = (M0 + 127) >> 8, hi = (M1 - 128) >> 8;    // pixels whose centre 256 i + 128 lies in [M0, M1]
    if (lo > hi) {
        const int64_t px = X0 >> 8, py = Y0 >> 8;
        if (px >= x0 && px < x1 && py >= y0 && py < y1) plot((int32_t)px, (int32_t)py);
        return;
    }
    const int32_t Mlo = xmaj ? x0 : y0, Mhi = xmaj ? x1 : y1, mlo = xmaj ? y0 : x0, mhi = xmaj ? y1 : x1;
    if (lo < Mlo) lo = Mlo;
    if (hi > Mhi - 1) hi = Mhi - 1;
    if (lo > hi) return;
    const uint64_t dM = (uint64_t)(M1 - M0);
    const bool up = m1 >= m0;
    const uint64_t dm = up ? (uint64_t)(m1 - m0) : (uint64_t)(m0 - m1);
    auto minor = [&](int64_t i) -> int64_t {               // the minor pixel at major pixel i
        if (dM == 0) return m0 >> 8;
        const uint64_t p = (uint64_t)(256 * i + 128 - M0) * dm;     // <= dM * dm < 2^64
        const uint64_t q = p / dM;
        return (up ? m0 + (int64_t)q : m0 - (int64_t)q - (q * dM != p ? 1 : 0)) >> 8;
    };
    int64_t a = lo, b = hi + 1;                             // first pixel not before [mlo, mhi)
    while (a < b) {
        const int64_t mid = a + ((b - a) >> 1);
        const int64_t j = minor(mid);
        if (up ? j < mlo : j >= mhi) a = mid + 1; else b = mid;
    }
    const int64_t first = a;
    b = hi + 1;                                             // first pixel past it
    while (a < b) {
        const int64_t mid = a + ((b - a) >> 1);
        const int64_t j = minor(mid);
        if (up ? j >= mhi : j < mlo) b = mid; else a = mid + 1;
    }
    for (int64_t i = first; i < a; i++) {
        const int64_t j = minor(i);
        if (xmaj) plot((int32_t)i, (int32_t)j); else plot((int32_t)j, (int32_t)i);
    }
}

// automap_line's rule in two steps, so that the lanes of a warp can share one long line's pixels (the marks variant's
// grid lines cross whole tiles): automap_line_span finds the major-axis pixels [first, last) the line draws inside the
// rectangle (returns 1), or the one pixel (px, py) of a line without a pixel centre in its range when it lies inside
// (returns 2), or nothing (0); automap_span_pixel gives the pixel at major index i.  The same pixels as automap_line.
struct AutomapSpan {
    int64_t M0, m0, first, last;
    uint64_t dM, dm;
    bool xmaj, up;
    int32_t px, py;
};
B2D_HD int64_t automap_span_minor(const AutomapSpan &s, int64_t i) {
    if (s.dM == 0) return s.m0 >> 8;
    const uint64_t p = (uint64_t)(256 * i + 128 - s.M0) * s.dm;
    const uint64_t q = p / s.dM;
    return (s.up ? s.m0 + (int64_t)q : s.m0 - (int64_t)q - (q * s.dM != p ? 1 : 0)) >> 8;
}
B2D_HD void automap_span_pixel(const AutomapSpan &s, int64_t i, int32_t &x, int32_t &y) {
    const int64_t j = automap_span_minor(s, i);
    x = (int32_t)(s.xmaj ? i : j);
    y = (int32_t)(s.xmaj ? j : i);
}
B2D_HD int automap_line_span(int64_t X0, int64_t Y0, int64_t X1, int64_t Y1, int32_t x0, int32_t y0, int32_t x1, int32_t y1,
                             AutomapSpan &s) {
    if ((X0 < X1 ? X1 : X0) >> 8 < x0 || (X0 < X1 ? X0 : X1) >> 8 >= x1 || (Y0 < Y1 ? Y1 : Y0) >> 8 < y0 ||
        (Y0 < Y1 ? Y0 : Y1) >> 8 >= y1)
        return 0;
    s.xmaj = (X1 >= X0 ? X1 - X0 : X0 - X1) >= (Y1 >= Y0 ? Y1 - Y0 : Y0 - Y1);
    int64_t M0 = s.xmaj ? X0 : Y0, m0 = s.xmaj ? Y0 : X0, M1 = s.xmaj ? X1 : Y1, m1 = s.xmaj ? Y1 : X1;
    if (M1 < M0) {
        int64_t t = M0; M0 = M1; M1 = t;
        t = m0; m0 = m1; m1 = t;
    }
    int64_t lo = (M0 + 127) >> 8, hi = (M1 - 128) >> 8;
    if (lo > hi) {
        s.px = (int32_t)(X0 >> 8);
        s.py = (int32_t)(Y0 >> 8);
        return (X0 >> 8) >= x0 && (X0 >> 8) < x1 && (Y0 >> 8) >= y0 && (Y0 >> 8) < y1 ? 2 : 0;
    }
    const int32_t Mlo = s.xmaj ? x0 : y0, Mhi = s.xmaj ? x1 : y1, mlo = s.xmaj ? y0 : x0, mhi = s.xmaj ? y1 : x1;
    if (lo < Mlo) lo = Mlo;
    if (hi > Mhi - 1) hi = Mhi - 1;
    if (lo > hi) return 0;
    s.M0 = M0;
    s.m0 = m0;
    s.dM = (uint64_t)(M1 - M0);
    s.up = m1 >= m0;
    s.dm = s.up ? (uint64_t)(m1 - m0) : (uint64_t)(m0 - m1);
    int64_t a = lo, b = hi + 1;                             // first pixel not before [mlo, mhi)
    while (a < b) {
        const int64_t mid = a + ((b - a) >> 1);
        const int64_t j = automap_span_minor(s, mid);
        if (s.up ? j < mlo : j >= mhi) a = mid + 1; else b = mid;
    }
    s.first = a;
    b = hi + 1;                                             // first pixel past it
    while (a < b) {
        const int64_t mid = a + ((b - a) >> 1);
        const int64_t j = automap_span_minor(s, mid);
        if (s.up ? j >= mhi : j < mlo) b = mid; else a = mid + 1;
    }
    s.last = a;
    return s.first < s.last ? 1 : 0;
}

}  // namespace b2d
