// TEST-ONLY: the automap kernel's algorithm (b2d_kernels.cu b2d_automap_kernel) on the CPU, through the same B2D_HD rule
// (b2d_math.cuh automap_frame / automap_item / automap_line): each 128 x 32 tile keeps a key per pixel, every item is drawn
// into it clamped to the tile with max(key, (item + 1) << 8 | colour), and the key's low byte is the pixel.  Compiled by
// tests/test_automap.py into a temporary directory; not part of libb2d.so.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../rust-doom_b200/csrc/b2d_math.cuh"

using namespace b2d;

extern "C" int hostcheck_automap(const AutomapLine *lines, int nlines, const int32_t *things, int nthings, const View *vw,
                                 const Pose *poses, int n, int32_t scale, int flags, uint8_t *out) {
    constexpr int TW = 128, TH = 32;
    const AutomapLevel L{lines, things, nlines, nthings};
    std::vector<uint32_t> keys(TW * TH);
    for (int f = 0; f < n; f++) {
        const AutomapFrame fr = automap_frame(poses[f], *vw, scale, flags);
        uint8_t *dst = out + (size_t)f * vw->W * vw->H;
        for (int ty0 = 0; ty0 < vw->H; ty0 += TH)
            for (int tx0 = 0; tx0 < vw->W; tx0 += TW) {
                const int tx1 = tx0 + TW < vw->W ? tx0 + TW : vw->W, ty1 = ty0 + TH < vw->H ? ty0 + TH : vw->H;
                std::fill(keys.begin(), keys.end(), 0u);
                const int items = automap_items(L, flags);
                for (int i = 0; i < items; i++) {
                    int64_t e[4];
                    const uint32_t colour = automap_item(fr, L, flags, i, e);
                    if (!colour) continue;
                    const uint32_t key = ((uint32_t)(i + 1) << 8) | colour;
                    bool outside = false;         // a pixel outside the tile would be a fault on the device
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
