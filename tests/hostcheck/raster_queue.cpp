// TEST-ONLY: the raster kernel's CTA schedule with its draw queue (b2d_kernels.cu DrawQueue), executed on the CPU with the
// product's per-column rules, so that any queue size can be checked against the oracle without a GPU.  It builds on
// hostcheck.cpp (scene binding, pre-lit planes, the walk mirror and the texel probes) and is compiled on its own by
// tests/test_hostcheck_queue.py.  No product code calls it.
#include <functional>

#include "hostcheck.cpp"

namespace {
namespace queue_mirror {

struct Deferred { size_t k; std::vector<uint32_t> win; };
struct FrameRaster;

// One warp-wide draw of the raster kernel (a record of its CTA's draw queue, b2d_kernels.cu DrawQueue): a flat span (or,
// not visible, a void fill) with {plane height, flat, light}, or a wall piece with {texture, tA, hA} and per lane the
// texture column, iscale and light row; per lane the window [ya, yb) and the sky column of the owner's strip.
struct Draw {
    const FrameRaster *fr;
    int x0 = 0;
    bool wall = false, vis = false;
    int32_t a = 0, b = 0, c = 0;
    std::vector<int> ya, yb;
    std::vector<int32_t> ucol, iscale, row;
    std::vector<uint32_t> skycol;
    Draw(const FrameRaster *f, int x, int SW, bool w) : fr(f), x0(x), wall(w), ya(SW, 0), yb(SW, 0), ucol(SW, 0), iscale(SW, 1), row(SW, 0), skycol(SW, 0) {}
    bool any() const { for (size_t l = 0; l < ya.size(); l++) if (ya[l] < yb[l]) return true; return false; }
};

// the per-frame part of the raster: the draw routines and one strip's clip pass and masked pass
struct FrameRaster {
    const HostScene &sc;
    const View &vw;
    const FrameConst &fc;
    const std::vector<SegFrame> &wl;
    const std::vector<uint32_t> &yslope;
    uint32_t invF;
    uint8_t *fb;
    int W, H;

    void put(int x, int y, uint8_t v) const { fb[(size_t)y * W + x] = v; }
    void fill_void(int x, int ya, int yb) const { for (int y = ya; y < yb; y++) put(x, y, 0); }
    void draw_sky(int x, uint32_t skycol, int ya, int yb) const {
        if (sc.sky_tex < 0) { fill_void(x, ya, yb); return; }
        const TexRec &T = sc.tex[sc.sky_tex];
        const bool inter = tex_interleaved(T.h, T.texel_off);
        const uint8_t *px = sc.lit_texels + T.texel_off;                       // light row 0
        for (int y = ya; y < yb; y++) {
            int v = sky_row(y, H, (int32_t)T.h);
            put(x, y, (uint8_t)tex_read(px, T, lit_index(inter, T.w, (uint32_t)v, skycol), 1));
        }
    }
    void draw_plane(int x, uint32_t skycol, int ya, int yb, int32_t h, int32_t flat, int lightb, bool visible) const {
        if (ya >= yb) return;
        if (!visible) { fill_void(x, ya, yb); return; }
        if (flat == kFlatSky) { draw_sky(x, skycol, ya, yb); return; }
        if (flat < 0 || flat >= sc.nflats) { fill_void(x, ya, yb); return; }
        const uint8_t *px = sc.lit_flats;
        uint32_t habs = plane_habs(h, fc.pose.z);
        const PlaneDir dir = plane_dir(fc, vw, x, invF);
        for (int y = ya; y < yb; y++) {
            PlaneRow pr = plane_row(habs, yslope[(size_t)y]);
            const int lr = light_row(lightb, pr.z8);
            const uint32_t cm6 = (sc.lit_flat_stride >> 6) * (uint32_t)lr + 64u * (uint32_t)flat;
            const uint32_t off = flat_offset(cm6, plane_u(fc.pose.x, pr.z8q, dir.ax), plane_u(fc.pose.y, pr.z8q, dir.ay));
            const uint32_t own = (uint32_t)lr * sc.lit_flat_stride + 4096u * (uint32_t)flat;   // this flat in this light plane
            if (off - own >= 4096u) { g_probe.oob++; put(x, y, 0); continue; }
            put(x, y, px[off]);
        }
    }
    void draw_wall(int x, int ya, int yb, int32_t tex, int32_t tA, int32_t hA, int32_t ucol, int32_t iscale, int row) const {
        if (ya >= yb) return;
        if (tex < 0 || tex >= sc.ntex) { fill_void(x, ya, yb); return; }
        const TexRec &T = sc.tex[tex];
        const uint32_t col = (uint32_t)floormod32(ucol, (int32_t)T.w);
        const uint8_t *pl = sc.lit_texels + (size_t)row * sc.lit_texel_stride + T.texel_off;
        const uint32_t tstep = (uint32_t)(iscale >> 4);
        uint32_t t = (uint32_t)wall_tbase(tA, hA, fc.pose.z, H, iscale) + (uint32_t)ya * tstep;
        if (!tex_interleaved(T.h, T.texel_off)) {
            g_probe.path(kPathRowMajor, T.h);
            for (int y = ya; y < yb; y++, t += tstep)
                put(x, y, (uint8_t)tex_read(pl, T, wall_row((int32_t)t, T.h, T.hmagic, T.hbias) * T.w + col, 1));
            return;
        }
        if (T.h >= 8u && tstep <= kWallFast8) {
            // the incremental path of wall_fast_loop (the kernel takes it when every lane of the warp qualifies; here per
            // lane, alternating between the 16- and the 8-row form, and starting a few rows above ya the way a lane whose
            // neighbours start higher does)
            const int R = (tstep <= kWallFast16 && (x & 1) == 0) ? 16 : 8;
            g_probe.path(R == 16 ? kPathFast16 : kPathFast8, T.h);
            const int y0 = std::max(0, ya - (x % 5) * 3);
            const uint32_t t0 = (uint32_t)wall_tbase(tA, hA, fc.pose.z, H, iscale) + (uint32_t)y0 * tstep;
            const uint32_t r0 = wall_row((int32_t)t0, T.h, T.hmagic, T.hbias);
            uint32_t q = r0 >> 2, acc = wall_acc29(t0, r0);
            const uint32_t ts29 = tstep << 13, nq = T.h >> 2, w4f = 4u * T.w;
            for (int y = y0; y < yb; y += R) {
                const uint32_t q1 = q + 1u == nq ? 0u : q + 1u;
                const uint32_t w0 = tex_read(pl, T, 4u * col + (uint64_t)q * w4f, 4);
                const uint32_t w1 = tex_read(pl, T, 4u * col + (uint64_t)q1 * w4f, 4);
                const uint32_t m = row_mask(y, ya, yb, R);
                for (int k = 0; k < R; k++)
                    if ((m >> k) & 1u) put(x, y + k, (uint8_t)(pick_byte(w0, w1, wall_sel(acc, ts29, (uint32_t)k)) & 0xFFu));
                wall_advance(acc, q, ts29, (uint32_t)R, nq);
            }
            return;
        }
        // batches of 8 rows as in draw_wall_warp: two aligned words + byte pick when the 8 rows stay inside two
        // consecutive row quads, eight byte fetches otherwise (the kernel decides per warp, here per lane: both
        // forms must give the same bytes, which is what the comparison with the oracle checks)
        const uint32_t colb = 4u * col, w4 = 4u * T.w;
        uint32_t used = 0;
        for (int y = ya; y < yb; y += 8, t += 8u * tstep) {
            const uint32_t r0 = wall_row((int32_t)t, T.h, T.hmagic, T.hbias);
            const uint32_t acc = wall_acc(t, r0);
            uint32_t v[8];
            if (((acc + 7u * tstep) >> 16) < 8u) {
                used |= 1u << kPathWord8;
                const uint32_t q0 = r0 >> 2, q1 = next_quad(q0, T.h);
                const uint32_t w0 = tex_read(pl, T, q0 * w4 + colb, 4), w1 = tex_read(pl, T, q1 * w4 + colb, 4);
                for (uint32_t k = 0; k < 8; k++) v[k] = pick_byte(w0, w1, (acc + k * tstep) >> 16) & 0xFFu;
            } else {
                const uint32_t t4 = t + 4u * tstep;
                const uint32_t r4 = wall_row((int32_t)t4, T.h, T.hmagic, T.hbias);
                const uint32_t acc4 = wall_acc(t4, r4);
                if (((acc + 3u * tstep) >> 16) < 8u && ((acc4 + 3u * tstep) >> 16) < 8u) {   // two 4-row halves
                    used |= 1u << kPathSplit44;
                    const uint32_t q0 = r0 >> 2, q4 = r4 >> 2;
                    const uint32_t a0 = tex_read(pl, T, q0 * w4 + colb, 4), a1 = tex_read(pl, T, next_quad(q0, T.h) * w4 + colb, 4);
                    const uint32_t b0 = tex_read(pl, T, q4 * w4 + colb, 4), b1 = tex_read(pl, T, next_quad(q4, T.h) * w4 + colb, 4);
                    for (uint32_t k = 0; k < 4; k++) {
                        v[k] = pick_byte(a0, a1, (acc + k * tstep) >> 16) & 0xFFu;
                        v[k + 4] = pick_byte(b0, b1, (acc4 + k * tstep) >> 16) & 0xFFu;
                    }
                } else {
                    used |= 1u << kPathBytes;
                    for (uint32_t k = 0; k < 8; k++) {
                        const uint32_t rk = wall_row((int32_t)(t + k * tstep), T.h, T.hmagic, T.hbias);
                        v[k] = tex_read(pl, T, (rk >> 2) * w4 + colb + (rk & 3u), 1);
                    }
                }
            }
            for (int k = 0; k < 8 && y + k < yb; k++) put(x, y + k, (uint8_t)v[k]);
        }
        for (int p = kPathWord8; p <= kPathBytes; p++)
            if ((used >> p) & 1u) g_probe.path(p, T.h);
    }


    void run(const Draw &d) const {
        for (size_t l = 0; l < d.ya.size(); l++) {
            const int x = d.x0 + (int)l;
            if (x >= W) continue;
            if (d.wall) draw_wall(x, d.ya[l], d.yb[l], d.a, d.b, d.c, d.ucol[l], d.iscale[l], d.row[l]);
            else draw_plane(x, d.skycol[l], d.ya[l], d.yb[l], d.a, d.b, d.c, d.vis);
        }
    }

    // the front-to-back clip pass of one strip: every draw goes to `emit`, the deferred masked entries to `deferred`
    template <typename Emit>
    void clip_strip(int strip, int SW, Emit &&emit, std::vector<Deferred> &deferred) const {
        const int x0 = strip * SW;
        std::vector<Lane> lanes((size_t)SW);
        for (int l = 0; l < SW; l++) {
            int x = x0 + l;
            lanes[l].ct = 0; lanes[l].cb = x < W ? H : 0; lanes[l].skycol = 0;
            if (sc.sky_tex >= 0 && x < W) lanes[l].skycol = umulhi32(sky_u32(x, vw, fc.pose.angle), sc.tex[sc.sky_tex].w);
        }
        auto draw = [&](bool wall) {
            Draw d(this, x0, SW, wall);
            for (int l = 0; l < SW; l++) d.skycol[(size_t)l] = lanes[(size_t)l].skycol;
            return d;
        };
        const int masked_cap = strip_masked_cap(sc.nmids, sc.nsprites);
        for (size_t k = 0; k < wl.size(); k++) {
            const SegFrame &sf = wl[k];
            if (!(sf.xhi >= x0 && sf.xlo <= x0 + SW - 1)) continue;
            bool any_open = false;
            for (int l = 0; l < SW; l++) any_open |= lanes[l].ct < lanes[l].cb;
            if (!any_open) break;
            if (is_sprite_entry(sf)) {        // decoration sprite: defer with the windows open right now
                Deferred d{k, std::vector<uint32_t>((size_t)SW, 0u)};
                bool any = false;
                for (int l = 0; l < SW; l++) {
                    int x = x0 + l;
                    const Lane &ln = lanes[(size_t)l];
                    if (x < W && ln.ct < ln.cb && x >= sf.xlo && x <= sf.xhi) {
                        d.win[(size_t)l] = (uint32_t)ln.ct | ((uint32_t)ln.cb << 16);
                        any = true;
                    }
                }
                if (any && deferred.size() < (size_t)masked_cap) deferred.push_back(d);
                continue;
            }
            const SegRec &S = sc.segs[sf.seg];
            const SectorRec &SF = sc.sectors[S.front];
            const int32_t fcl = SF.ceil, ffl = SF.floor;
            const bool two = S.flags & kSegTwoSided;
            const bool ceil_vis = plane_visible(true, fcl, SF.ceil_flat == kFlatSky, fc.pose.z);
            const bool floor_vis = plane_visible(false, ffl, SF.floor_flat == kFlatSky, fc.pose.z);
            const bool has_a = wall_piece(true, two, fcl, ffl, S.otop, S.obot), has_b = wall_piece(false, two, fcl, ffl, S.otop, S.obot);
            Deferred dfr{k, std::vector<uint32_t>((size_t)SW, 0u)};
            bool any_deferred = false;
            // the kernel's draws of this entry, in its order: ceiling, floor, piece A, piece B
            Draw ceil = draw(false), floor = draw(false), wa = draw(true), wb = draw(true);
            ceil.vis = ceil_vis; ceil.a = fcl; ceil.b = SF.ceil_flat; ceil.c = SF.light;
            floor.vis = floor_vis; floor.a = ffl; floor.b = SF.floor_flat; floor.c = SF.light;
            wa.a = S.texA; wa.b = S.tA; wa.c = S.hA;
            wb.a = S.texB; wb.b = S.tB; wb.c = S.hB;
            for (int l = 0; l < SW; l++) {
                int x = x0 + l;
                Lane &ln = lanes[l];
                if (!(x < W && ln.ct < ln.cb && x >= sf.xlo && x <= sf.xhi)) continue;
                ColumnEval ce;
                if (!column_eval(sf, vw, x, ce)) continue;
                const int ct = ln.ct, cb = ln.cb;
                const int row = light_row(S.light, ce.z8);
                const int32_t ucol = wall_column(S.uoff, S.len_q12, ce.s24);
                const WallRows r = wall_rows(fcl, ffl, two, S.otop, S.obot, ce.scale, fc.pose.z, H, ct, cb);
                ceil.ya[l] = ct; ceil.yb[l] = r.y1;
                floor.ya[l] = r.y4; floor.yb[l] = cb;
                for (Draw *w : {&wa, &wb}) { w->ucol[l] = ucol; w->iscale[l] = ce.iscale; w->row[l] = row; }
                wa.ya[l] = r.y1; wa.yb[l] = r.y2;
                wb.ya[l] = r.y3; wb.yb[l] = r.y4;
                wall_window(two, r, H, ln.ct, ln.cb);
                if (two && S.mid >= 0 && r.y2 < r.y3) { dfr.win[(size_t)l] = (uint32_t)r.y2 | ((uint32_t)r.y3 << 16); any_deferred = true; }
            }
            emit(std::move(ceil));
            emit(std::move(floor));
            if (has_a) emit(std::move(wa));
            if (has_b) emit(std::move(wb));
            if (any_deferred && deferred.size() < (size_t)masked_cap) deferred.push_back(dfr);
        }
        Draw v = draw(false);              // whatever is still open is void
        for (int l = 0; l < SW; l++)
            if (x0 + l < W) { v.ya[(size_t)l] = lanes[(size_t)l].ct; v.yb[(size_t)l] = lanes[(size_t)l].cb; }
        emit(std::move(v));
    }

    // masked middle textures, back to front (mirrors masked_pass in b2d_kernels.cu)
    void masked(int strip, int SW, const std::vector<Deferred> &deferred) const {
        const int x0 = strip * SW;
        for (size_t e = deferred.size(); e-- > 0;) {
            const SegFrame &sf = wl[deferred[e].k];
            for (int l = 0; l < SW; l++) {
                uint32_t packed = deferred[e].win[(size_t)l];
                int ya = (int)(packed & 0xFFFFu), yb = (int)(packed >> 16), x = x0 + l;
                if (!(ya < yb)) continue;
                int32_t tex, tA, hA, ucol, iscale, row;
                if (is_sprite_entry(sf)) {
                    SpriteFrame sp;
                    const SpriteRec &P = sc.sprites[entry_sprite(sf, sp)];
                    if (P.tex < 0 || P.tex >= sc.ntex) continue;
                    const int32_t sw = (int32_t)sc.tex[P.tex].w, sh = (int32_t)sc.tex[P.tex].h;
                    const int64_t scale = sprite_scale(vw, sp.cz);
                    int32_t z8;
                    scale_depth(vw, scale, iscale, z8);
                    row = light_row_sprite(P.light, z8);
                    tex = P.tex; tA = 0; hA = P.low + sh;
                    clip_rows(P.low + sh, P.low, row_scale(scale), fc.pose.z, H, ya, yb);
                    ucol = sprite_column(sp, vw, x, sw);
                } else {
                    const SegRec &S = sc.segs[sf.seg];
                    if (S.mid < 0 || S.mid >= sc.nmids) continue;
                    const MidRec &M = sc.mids[S.mid];
                    ColumnEval ce;
                    if (!column_eval(sf, vw, x, ce)) continue;
                    tex = M.tex; tA = M.t_high; hA = M.high;
                    clip_rows(M.high, M.low, ce.scale, fc.pose.z, H, ya, yb);
                    ucol = wall_column(S.uoff, S.len_q12, ce.s24);
                    iscale = ce.iscale;
                    row = light_row(S.light, ce.z8);
                }
                if (tex < 0 || tex >= sc.ntex) continue;
                const TexRec &T = sc.tex[tex];
                uint32_t col = (uint32_t)floormod32(ucol, (int32_t)T.w);
                const bool inter = tex_interleaved(T.h, T.texel_off);
                const uint8_t *px = sc.lit_texels + (size_t)row * sc.lit_texel_stride + T.texel_off;
                const bool has_mask = T.mask_off != 0xFFFFFFFFu;
                const uint8_t *pm = sc.lit_texels + (size_t)32 * sc.lit_texel_stride + T.texel_off;   // opacity plane
                int32_t tbase = wall_tbase(tA, hA, fc.pose.z, H, iscale), tstep = iscale >> 4;
                if (ya < yb) g_probe.path(inter ? kPathMaskedInter : kPathMaskedRowMajor, T.h);
                for (int y = ya; y < yb; y++) {
                    const uint32_t r = wall_row(tbase + y * tstep, T.h, T.hmagic, T.hbias);
                    const uint32_t off = lit_index(inter, T.w, r, col);
                    if (has_mask && !tex_read(pm, T, off, 1)) continue;
                    put(x, y, (uint8_t)tex_read(px, T, off, 1));
                }
            }
        }
    }
};

// The raster kernel's schedule: CTAs of `warps` consecutive (frame, 32-column strip) warps over the whole batch (a CTA
// may straddle frames).  Each warp's clip pass appends its draws to the CTA's queue of `queue_words` per-lane words
// (32 per record, 96 for a wall piece; a header per 32 words) or, when a record does not fit, draws it at once; then the
// queue is drawn, then each warp's masked pass.
struct QueueStats { long long records = 0, overflow = 0, ctas = 0, ctas_overflow = 0; };

void raster_queued(const std::vector<FrameRaster> &frs, int warps, uint32_t queue_words, QueueStats &qs) {
    if (frs.empty()) return;
    const int SW = 32;
    const long long strips = (frs[0].W + SW - 1) / SW, total = (long long)frs.size() * strips;
    for (long long g0 = 0; g0 < total; g0 += warps) {
        std::vector<Draw> queue;
        uint32_t words = 0;
        long long over = 0;
        std::vector<std::vector<Deferred>> deferred((size_t)warps);
        for (int w = 0; w < warps && g0 + w < total; w++) {
            const FrameRaster &fr = frs[(size_t)((g0 + w) / strips)];
            fr.clip_strip((int)((g0 + w) % strips), SW, [&](Draw &&d) {
                if (!d.any()) return;
                qs.records++;
                const uint32_t need = d.wall ? 96u : 32u, off = words;
                words += need;
                if (off + need <= queue_words && queue.size() < queue_words / 32u) { queue.push_back(std::move(d)); return; }
                over++;
                fr.run(d);
            }, deferred[(size_t)w]);
        }
        for (const Draw &d : queue) d.fr->run(d);
        for (int w = 0; w < warps && g0 + w < total; w++)
            frs[(size_t)((g0 + w) / strips)].masked((int)((g0 + w) % strips), SW, deferred[(size_t)w]);
        qs.overflow += over;
        qs.ctas++;
        qs.ctas_overflow += over > 0;
    }
}

}  // namespace queue_mirror
}  // namespace

// Frames of `n` poses at level time `tics` through the kernel's CTA schedule: `warps` strips per CTA sharing a draw
// queue of `queue_words` per-lane words (0: every draw overflows and its owner draws it at once).  qstats[4] = records,
// records drawn by their owner because the queue was full, CTAs, CTAs with such a record.  fb may be nullptr
// (statistics only: the frames go to a ring of scratch frames).
extern "C" int hostcheck_render_queued(const uint8_t *blob, const View *vw, const Pose *poses, int n, uint8_t *fb, uint32_t tics,
                                       int warps, uint32_t queue_words, long long *qstats) {
    using namespace queue_mirror;
    if (warps < 1 || n < 0) return -1;
    HostScene sc = bind(blob);
    LitPlanes lit;
    build_lit(sc, lit);
    std::vector<TexRec> tex_t((size_t)sc.ntex);
    std::vector<SectorRec> sectors_t((size_t)sc.hdr[H_NSECTORS]);
    std::vector<SegRec> segs_t((size_t)sc.nsegs);
    std::vector<SpriteRec> sprites_t((size_t)sc.nsprites);
    std::vector<MidRec> mids_t((size_t)sc.hdr[H_NMIDS]);
    if (scene_is_timed(blob)) {
        scene_at_time(blob, tics, tex_t.data(), sectors_t.data(), segs_t.data(), sprites_t.data(), mids_t.data(), nullptr, nullptr);
        sc.tex = tex_t.data(); sc.sectors = sectors_t.data(); sc.segs = segs_t.data(); sc.sprites = sprites_t.data();
        sc.mids = mids_t.data();
    }
    std::vector<uint32_t> yslope((size_t)vw->H);
    for (int y = 0; y < vw->H; y++) yslope[(size_t)y] = yslope_entry(y, *vw);
    const uint32_t invF = (uint32_t)(4294967296ULL / (uint64_t)vw->F);
    const size_t npix = (size_t)vw->W * vw->H;
    const size_t ring = (size_t)warps + 2;     // a CTA's warps span at most warps + 1 frames
    std::vector<uint8_t> scratch(fb ? 0 : ring * npix);
    std::vector<FrameConst> fcs((size_t)n);
    std::vector<std::vector<SegFrame>> wls((size_t)n);
    std::vector<FrameRaster> frs;
    for (int i = 0; i < n; i++) {
        walk(sc, *vw, poses[i], fcs[(size_t)i], wls[(size_t)i]);
        uint8_t *f = fb ? fb + npix * (size_t)i : scratch.data() + npix * ((size_t)i % ring);
        if (fb) std::memset(f, 0xAB, npix);     // poisoned: the raster must write every pixel
        frs.push_back(FrameRaster{sc, *vw, fcs[(size_t)i], wls[(size_t)i], yslope, invF, f, vw->W, vw->H});
    }
    QueueStats qs;
    raster_queued(frs, warps, queue_words, qs);
    if (qstats) { qstats[0] = qs.records; qstats[1] = qs.overflow; qstats[2] = qs.ctas; qstats[3] = qs.ctas_overflow; }
    return 0;
}
