// TEST-ONLY: seen lines (DESIGN.md C20) with the product's rules on the CPU.  hostcheck_seen runs the raster kernel's strip
// clip loop (b2d_kernels.cu b2d_raster_kernel, kSeen) over the walk mirror's worklist, 32 lanes of a strip in lock step:
// when some lane of the strip owns a column of an entry's seg (in its interval, window open, column_eval passes), the
// seg's linedef is marked, and the windows are updated by wall_rows / wall_window.  hostcheck_automap_seen runs K5's tile
// algorithm with the seen variant's item rule (b2d_math.cuh automap_seen_item).  Builds on hostcheck.cpp; compiled on
// its own by tests/test_seen_lines.py.  No product code calls it.
#include "hostcheck.cpp"

// rows: n x words, OR-ed into; seg_line: the level's seg -> linedef table (-1: none); moves: the frame's sector moves
extern "C" int hostcheck_seen(const uint8_t *blob, const View *vw, const Pose *poses, int n, const int32_t *seg_line,
                              uint32_t words, uint32_t *rows, const SectorMove *moves, int n_moves) {
    HostScene sc = bind(blob);
    std::vector<TexRec> tex_t((size_t)sc.ntex);
    std::vector<SectorRec> sectors_t((size_t)sc.hdr[H_NSECTORS]);
    std::vector<SegRec> segs_t((size_t)sc.nsegs);
    std::vector<SpriteRec> sprites_t((size_t)sc.nsprites);
    std::vector<MidRec> mids_t((size_t)sc.hdr[H_NMIDS]);
    std::vector<int32_t> floor_off, ceil_off;
    if (n_moves > 0 && expand_moves(blob, moves, (size_t)n_moves, floor_off, ceil_off)) return -1;
    if (scene_is_timed(blob)) {
        scene_at_time(blob, 0, tex_t.data(), sectors_t.data(), segs_t.data(), sprites_t.data(), mids_t.data(),
                      n_moves > 0 ? floor_off.data() : nullptr, n_moves > 0 ? ceil_off.data() : nullptr);
        sc.tex = tex_t.data(); sc.sectors = sectors_t.data(); sc.segs = segs_t.data(); sc.sprites = sprites_t.data();
        sc.mids = mids_t.data();
    }
    const int W = vw->W, H = vw->H;
    for (int i = 0; i < n; i++) {
        FrameConst fc;
        std::vector<SegFrame> wl;
        walk(sc, *vw, poses[i], fc, wl);
        uint32_t *row = rows + (size_t)i * words;
        for (int x0 = 0; x0 < W; x0 += 32) {
            int ct[32], cb[32];
            for (int l = 0; l < 32; l++) { ct[l] = 0; cb[l] = x0 + l < W ? H : 0; }
            for (size_t k = 0; k < wl.size(); k++) {
                const SegFrame &sf = wl[k];
                if (!(sf.xhi >= x0 && sf.xlo <= x0 + 31)) continue;
                bool any_open = false;
                for (int l = 0; l < 32; l++) any_open |= ct[l] < cb[l];
                if (!any_open) break;
                if (is_sprite_entry(sf)) continue;
                const SegRec &S = sc.segs[sf.seg];
                const SectorRec &SF = sc.sectors[S.front];
                const bool two = S.flags & kSegTwoSided;
                bool owned = false;
                for (int l = 0; l < 32; l++) {
                    const int x = x0 + l;
                    if (!(x < W && ct[l] < cb[l] && x >= sf.xlo && x <= sf.xhi)) continue;
                    ColumnEval ce;
                    if (!column_eval(sf, *vw, x, ce)) continue;
                    owned = true;
                    const WallRows r = wall_rows(SF.ceil, SF.floor, two, S.otop, S.obot, ce.scale, fc.pose.z, H, ct[l], cb[l]);
                    wall_window(two, r, H, ct[l], cb[l]);
                }
                const int32_t ld = owned ? seg_line[sf.seg] : -1;
                if (ld >= 0) row[ld >> 5] |= 1u << (ld & 31);
            }
        }
    }
    return 0;
}

// K5's tiles with automap_seen_item: mapped = n x words rows, or nullptr (every line mapped)
extern "C" int hostcheck_automap_seen(const AutomapLine *lines, int nlines, const int32_t *things, int nthings, const View *vw,
                                      const Pose *poses, int n, int32_t scale, int flags, const uint32_t *mapped, uint32_t words,
                                      uint8_t *out) {
    constexpr int TW = 128, TH = 32;
    const AutomapLevel L{lines, things, nlines, nthings};
    std::vector<uint32_t> keys(TW * TH);
    for (int f = 0; f < n; f++) {
        const AutomapFrame fr = automap_frame(poses[f], *vw, scale, flags);
        const uint32_t *row = mapped ? mapped + (size_t)f * words : nullptr;
        uint8_t *dst = out + (size_t)f * vw->W * vw->H;
        for (int ty0 = 0; ty0 < vw->H; ty0 += TH)
            for (int tx0 = 0; tx0 < vw->W; tx0 += TW) {
                const int tx1 = std::min(tx0 + TW, vw->W), ty1 = std::min(ty0 + TH, vw->H);
                std::fill(keys.begin(), keys.end(), 0u);
                const int items = automap_items(L, flags);
                for (int i = 0; i < items; i++) {
                    int64_t e[4];
                    const uint32_t colour = automap_seen_item(fr, L, row, flags, i, e);
                    if (!colour) continue;
                    const uint32_t key = ((uint32_t)(i + 1) << 8) | colour;
                    bool outside = false;
                    automap_line(e[0], e[1], e[2], e[3], tx0, ty0, tx1, ty1, [&](int32_t x, int32_t y) {
                        if (x < tx0 || x >= tx1 || y < ty0 || y >= ty1) { outside = true; return; }
                        uint32_t &k = keys[(size_t)(y - ty0) * TW + (x - tx0)];
                        if (key > k) k = key;
                    });
                    if (outside) return -1;
                }
                for (int y = ty0; y < ty1; y++)
                    for (int x = tx0; x < tx1; x++) dst[(size_t)y * vw->W + x] = (uint8_t)keys[(size_t)(y - ty0) * TW + (x - tx0)];
            }
    }
    return 0;
}
