// TEST-ONLY: the marks automap kernel's algorithm (b2d_kernels.cu b2d_automap_marks_kernel, DESIGN.md C22) on the CPU,
// through the same B2D_HD rules (b2d_math.cuh automap_state_item, automap_grid_range, automap_grid_line,
// automap_mark_place, automap_mark_texel): K5's 128 x 32 tiles with C21's items, under B2D_AUTOMAP_GRID only the grid
// lines each tile's conservative range lets through, drawn with the exact line rule clamped to the tile, and each frame's
// marks over everything.  Compiled by tests/test_automap_marks.py into a temporary directory; not part of libb2d.so.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../rust-doom_b200/csrc/b2d_math.cuh"

using namespace b2d;

// As hostcheck_automap_states (tests/hostcheck/automap_states.cpp), plus the level's grid origin and digits (host
// texel pointers) and mark_ranges: 2 words per frame (first, n) into marks.  stats (nullable): [0] the grid lines the
// tiles drew, [1] the grid lines that would be drawn if every tile took the whole lattice.
extern "C" int hostcheck_automap_marks(const AutomapLine *lines, int nlines, const AutomapDynLine *dyn, const int32_t *things,
                                       int nthings, const View *vw, const Pose *poses, int n, int32_t scale, int flags,
                                       const uint32_t *mapped, uint32_t words, const int32_t *pool, const int32_t *off_at,
                                       const uint32_t *ranges, const AutomapArrow *arrows, int32_t ox, int32_t oy,
                                       const AutomapDigit *digits, const uint32_t *mark_ranges, const AutomapMark *marks,
                                       uint8_t *out, int64_t *stats) {
    constexpr int TW = 128, TH = 32;
    const AutomapLevel L{lines, things, nlines, nthings};
    std::vector<uint32_t> keys(TW * TH);
    bool outside = false;         // a pixel outside the tile would be a fault on the device
    for (int f = 0; f < n; f++) {
        const AutomapFrame fr = automap_frame(poses[f], *vw, scale, flags);
        const AutomapStateFrame sf{off_at[f] < 0 ? nullptr : pool + off_at[f], arrows + ranges[2 * f], ranges[2 * f + 1],
                                   poses[f].angle};
        const uint32_t *row = mapped ? mapped + (size_t)f * words : nullptr;
        uint8_t *dst = out + (size_t)f * vw->W * vw->H;
        for (int ty0 = 0; ty0 < vw->H; ty0 += TH)
            for (int tx0 = 0; tx0 < vw->W; tx0 += TW) {
                const int tx1 = std::min(tx0 + TW, vw->W), ty1 = std::min(ty0 + TH, vw->H);
                std::fill(keys.begin(), keys.end(), 0u);
                auto put = [&](int32_t x, int32_t y, uint32_t key) {
                    if (x < tx0 || x >= tx1 || y < ty0 || y >= ty1) { outside = true; return; }
                    uint32_t &k = keys[(size_t)(y - ty0) * TW + (x - tx0)];
                    if (key > k) k = key;
                };
                const int items = automap_state_items(L, sf, flags);
                for (int i = 0; i < items; i++) {
                    int64_t e[4];
                    const uint32_t colour = automap_state_item(fr, L, dyn, sf, row, flags, i, e);
                    if (!colour) continue;
                    const uint32_t key = ((uint32_t)(i + 1) << 8) | colour;
                    automap_line(e[0], e[1], e[2], e[3], tx0, ty0, tx1, ty1, [&](int32_t x, int32_t y) { put(x, y, key); });
                }
                if (flags & kAutomapGrid)
                    for (int v = 1; v >= 0; v--) {
                        const int32_t o = v ? ox : oy;
                        int64_t jlo, jhi, llo, lhi;
                        automap_grid_range(fr, o, v, tx0, ty0, tx1, ty1, jlo, jhi);
                        automap_grid_lattice(o, llo, lhi);
                        if (stats) stats[1] += lhi - llo + 1;
                        for (int64_t j = jlo; j <= jhi; j++) {
                            int64_t e[4];
                            automap_grid_line(fr, o, v, j, e);
                            for (int k = 0; k < 4; k++)
                                if (e[k] <= -(int64_t(1) << 31) || e[k] >= (int64_t(1) << 31)) return -2;     // C22's bound
                            if (stats) stats[0] += 1;
                            AutomapSpan sp;                 // as a warp draws it: the span, then each lane's pixels
                            const int kind = automap_line_span(e[0], e[1], e[2], e[3], tx0, ty0, tx1, ty1, sp);
                            if (kind == 2) put(sp.px, sp.py, kAutomapGridColour);
                            if (kind == 1)
                                for (int64_t i = sp.first; i < sp.last; i++) {
                                    int32_t x, y;
                                    automap_span_pixel(sp, i, x, y);
                                    put(x, y, kAutomapGridColour);
                                }
                        }
                    }
                const int32_t k = automap_mark_k(vw->H);
                for (uint32_t m = 0; m < (mark_ranges ? mark_ranges[2 * f + 1] : 0u); m++) {
                    const AutomapMark mk = marks[mark_ranges[2 * f] + m];
                    const AutomapDigit d = digits[mk.number];
                    int32_t left, top;
                    if (!automap_mark_place(fr, mk, d, k, left, top)) continue;
                    const int32_t x0 = std::max(left, tx0), x1 = std::min(left + k * d.w, tx1);
                    const int32_t y0 = std::max(top, ty0), y1 = std::min(top + k * d.h, ty1);
                    const uint32_t key = (uint32_t)(items + m + 1) << 8;
                    for (int32_t y = y0; y < y1; y++)
                        for (int32_t x = x0; x < x1; x++) {
                            const uint32_t t = automap_mark_texel(d, k, left, top, x, y);
                            if (!(t >> 8)) put(x, y, key | t);
                        }
                }
                if (outside) return -1;
                for (int y = ty0; y < ty1; y++)
                    for (int x = tx0; x < tx1; x++) dst[(size_t)y * vw->W + x] = (uint8_t)keys[(size_t)(y - ty0) * TW + (x - tx0)];
            }
    }
    return 0;
}

// automap_grid_range of one rectangle, for the range tests: out = (jlo, jhi)
extern "C" void hostcheck_grid_range(const View *vw, const Pose *pose, int32_t scale, int flags, int32_t o, int vertical, int32_t x0,
                                     int32_t y0, int32_t x1, int32_t y1, int64_t *out) {
    const AutomapFrame fr = automap_frame(*pose, *vw, scale, flags);
    automap_grid_range(fr, o, vertical != 0, x0, y0, x1, y1, out[0], out[1]);
}
