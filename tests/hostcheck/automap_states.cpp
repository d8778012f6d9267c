// TEST-ONLY: the state automap kernel's algorithm (b2d_kernels.cu b2d_automap_states_kernel, DESIGN.md C21) on the CPU,
// through the same B2D_HD rule (b2d_math.cuh automap_state_item): K5's 128 x 32 tiles with each frame's lines coloured at
// its sector offsets and by its row of seen lines, and its arrows after the own arrow.  Compiled by
// tests/test_automap_states.py into a temporary directory; not part of libb2d.so.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../rust-doom_b200/csrc/b2d_math.cuh"

using namespace b2d;

// lines: the device copy (dev_flags with kAutomapDontDraw / kAutomapChangeable); dyn: one record per line (nullptr: no
// changeable line); off_at[f]: frame f's offsets at pool + off_at[f] (-1: at rest); ranges: 2 words per frame (first, n)
// into arrows; mapped: n x words rows or nullptr.
extern "C" int hostcheck_automap_states(const AutomapLine *lines, int nlines, const AutomapDynLine *dyn, const int32_t *things,
                                        int nthings, const View *vw, const Pose *poses, int n, int32_t scale, int flags,
                                        const uint32_t *mapped, uint32_t words, const int32_t *pool, const int32_t *off_at,
                                        const uint32_t *ranges, const AutomapArrow *arrows, uint8_t *out) {
    constexpr int TW = 128, TH = 32;
    const AutomapLevel L{lines, things, nlines, nthings};
    std::vector<uint32_t> keys(TW * TH);
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
                const int items = automap_state_items(L, sf, flags);
                for (int i = 0; i < items; i++) {
                    int64_t e[4];
                    const uint32_t colour = automap_state_item(fr, L, dyn, sf, row, flags, i, e);
                    if (!colour) continue;
                    const uint32_t key = ((uint32_t)(i + 1) << 8) | colour;
                    bool outside = false;         // a pixel outside the tile would be a fault on the device
                    for (int k = 0; k < 4; k++)
                        if (e[k] <= -(int64_t(1) << 31) || e[k] >= (int64_t(1) << 31)) return -2;     // C21's bound
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

// automap_state_colours of one line: out = (colour, colour_all); the line's own colours when it is not changeable
extern "C" void hostcheck_state_colours(const AutomapLine *line, const AutomapDynLine *dyn, const int32_t *off, uint8_t *out) {
    AutomapLine l = *line;
    if (l.dev_flags & kAutomapChangeable) automap_state_colours(l, *dyn, off);
    out[0] = l.colour;
    out[1] = l.colour_all;
}
