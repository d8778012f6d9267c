// TEST-ONLY: the raster kernel's band-major draw phase (b2d_kernels.cu kBandRows, kItemCap), executed on the CPU with the
// product's per-column rules, so that any band height and item-list capacity can be checked against the oracle without a
// GPU.  It builds on raster_queue.cpp (the CTA schedule with its draw queue) and is compiled on its own by
// tests/test_hostcheck_bands.py.  No product code calls it.
#include <algorithm>
#include <map>
#include <tuple>

#include "raster_queue.cpp"

namespace {
namespace band_mirror {

using queue_mirror::Deferred;
using queue_mirror::Draw;
using queue_mirror::FrameRaster;

// the record's warp extent [y0, y1): min ya and max yb over the lanes that own rows (queue_push's ext word)
void extent(const Draw &d, int &y0, int &y1) {
    y0 = 0x7FFFFFFF; y1 = 0;
    for (size_t l = 0; l < d.ya.size(); l++)
        if (d.ya[l] < d.yb[l]) { y0 = std::min(y0, d.ya[l]); y1 = std::max(y1, d.yb[l]); }
}

// the record with every lane's window clipped to [lo, hi)
Draw clipped(const Draw &d, int lo, int hi) {
    Draw c = d;
    for (size_t l = 0; l < c.ya.size(); l++) { c.ya[l] = std::max(c.ya[l], lo); c.yb[l] = std::min(c.yb[l], hi); }
    return c;
}

struct BandStats {
    long long rows = 0;                  // lock-step row iterations (warp max yb - warp min ya of every draw)
    long long ctas = 0, ctas_fallback = 0, ctas_masked = 0, items = 0, items_max = 0;
    double makespan = 0;                 // sum over CTAs of the list-scheduled makespan (row iterations)
    std::vector<int> open;               // per 128-byte frame line: row iterations between its first and last write
};

// The draw phase's model: the CTA's warps take work in pop order, each the moment it is free; a draw takes its
// lock-step rows and writes row y0 + k at its start + k.  A warp starts the draw phase after the draws it made itself
// during the clip pass (records the queue did not hold).  Lines: 128 bytes of one frame row (a 32-column strip lies in
// one); they are tracked per CTA.
struct Timeline {
    std::vector<long long> free;
    std::map<std::tuple<const FrameRaster *, int, int>, std::pair<long long, long long>> lines;
    explicit Timeline(int warps) : free((size_t)warps, 0) {}
    void draw(const Draw &d, size_t warp, BandStats &bs) {
        int y0, y1;
        extent(d, y0, y1);
        if (y0 >= y1) return;
        const long long s = free[warp];
        free[warp] += y1 - y0;
        bs.rows += y1 - y0;
        for (int y = y0; y < y1; y++) {
            bool any = false;
            for (size_t l = 0; l < d.ya.size(); l++) any |= y >= d.ya[l] && y < d.yb[l];
            if (!any) continue;
            auto key = std::make_tuple(d.fr, y, d.x0 >> 7);
            const long long t = s + (y - y0);
            auto it = lines.find(key);
            if (it == lines.end()) lines.emplace(key, std::make_pair(t, t));
            else { it->second.first = std::min(it->second.first, t); it->second.second = std::max(it->second.second, t); }
        }
    }
    size_t next() const { return (size_t)(std::min_element(free.begin(), free.end()) - free.begin()); }
};

// The raster kernel's schedule with a band-major draw phase: as raster_queue.cpp's raster_queued, but the queue is drawn
// as (band, record) items, band by band, each record clipped to the band (band_rows 0: the records whole, in record
// order).  A CTA whose items exceed item_cap draws its records whole, in record order, and so does a CTA with a deferred
// masked entry.
void raster_banded(const std::vector<FrameRaster> &frs, int warps, uint32_t queue_words, int band_rows, uint32_t item_cap,
                   queue_mirror::QueueStats &qs, BandStats &bs) {
    if (frs.empty()) return;
    const int SW = 32;
    const long long strips = (frs[0].W + SW - 1) / SW, total = (long long)frs.size() * strips;
    for (long long g0 = 0; g0 < total; g0 += warps) {
        std::vector<Draw> queue;
        uint32_t words = 0;
        long long over = 0;
        Timeline tl(warps);
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
                tl.draw(d, (size_t)w, bs);
                fr.run(d);
            }, deferred[(size_t)w]);
        }
        // the item list: (band, record) pairs in band order, records in queue order within a band
        std::vector<std::pair<int, size_t>> items;
        if (band_rows > 0) {
            int nb = 0;
            for (const Draw &d : queue) { int y0, y1; extent(d, y0, y1); nb = std::max(nb, (y1 - 1) / band_rows + 1); }
            for (int b = 0; b < nb; b++)
                for (size_t r = 0; r < queue.size(); r++) {
                    int y0, y1;
                    extent(queue[r], y0, y1);
                    if (y0 / band_rows <= b && b <= (y1 - 1) / band_rows) items.emplace_back(b, r);
                }
        }
        const long long nitems = (long long)(band_rows > 0 ? items.size() : queue.size());
        bool masked = false;
        for (const auto &d : deferred) masked |= !d.empty();
        const bool banded = band_rows > 0 && items.size() <= item_cap && !masked;
        if (!banded) {
            items.clear();
            for (size_t r = 0; r < queue.size(); r++) items.emplace_back(-1, r);
        }
        for (const auto &it : items) {
            const Draw &d = queue[it.second];
            const Draw c = it.first < 0 ? d : clipped(d, it.first * band_rows, (it.first + 1) * band_rows);
            tl.draw(c, tl.next(), bs);
            c.fr->run(c);
        }
        for (int w = 0; w < warps && g0 + w < total; w++)
            frs[(size_t)((g0 + w) / strips)].masked((int)((g0 + w) % strips), SW, deferred[(size_t)w]);
        qs.overflow += over;
        qs.ctas++;
        qs.ctas_overflow += over > 0;
        bs.ctas++;
        bs.ctas_fallback += band_rows > 0 && !banded && !masked;
        bs.ctas_masked += band_rows > 0 && masked;
        bs.items += nitems;
        bs.items_max = std::max(bs.items_max, nitems);
        bs.makespan += (double)*std::max_element(tl.free.begin(), tl.free.end());
        for (const auto &ln : tl.lines) bs.open.push_back((int)(ln.second.second - ln.second.first));
    }
}

}  // namespace band_mirror
}  // namespace

// Frames of `n` poses at level time `tics` through the kernel's CTA schedule with a band-major draw phase: `warps` strips
// per CTA sharing a draw queue of `queue_words` per-lane words, drawn in bands of `band_rows` rows (0: in record order)
// through an item list of `item_cap` items.  stats[9] = lock-step row iterations, CTAs, CTAs that fell back to record
// order because their items exceed the list, items (band_rows 0: records; counted before a fallback), items of the
// largest CTA, records drawn by their owner because the queue was full, the line-open time's mean and 90th percentile
// (row iterations, x1000), and CTAs in record order because they deferred masked entries; ms[1] = the
// mean modelled CTA makespan (row iterations).  fb may be nullptr (statistics only: the frames go to scratch frames).
extern "C" int hostcheck_render_banded(const uint8_t *blob, const View *vw, const Pose *poses, int n, uint8_t *fb, uint32_t tics,
                                       int warps, uint32_t queue_words, int band_rows, uint32_t item_cap, long long *stats,
                                       double *ms) {
    using namespace queue_mirror;
    if (warps < 1 || n < 0 || band_rows < 0) return -1;
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
    QueueStats qs;
    band_mirror::BandStats bs;
    // statistics only: a chunk of frames at a time, so that the scratch frames stay few (a multiple of `warps` frames
    // holds whole CTAs)
    const int chunk = fb ? std::max(n, 1) : 2 * warps;
    std::vector<uint8_t> scratch(fb ? 0 : (size_t)chunk * npix);
    for (int i0 = 0; i0 < n; i0 += chunk) {
        const int m = std::min(chunk, n - i0);
        std::vector<FrameConst> fcs((size_t)m);
        std::vector<std::vector<SegFrame>> wls((size_t)m);
        std::vector<FrameRaster> frs;
        for (int i = 0; i < m; i++) {
            walk(sc, *vw, poses[i0 + i], fcs[(size_t)i], wls[(size_t)i]);
            uint8_t *f = fb ? fb + npix * (size_t)(i0 + i) : scratch.data() + npix * (size_t)i;
            if (fb) std::memset(f, 0xAB, npix);     // poisoned: the raster must write every pixel
            frs.push_back(FrameRaster{sc, *vw, fcs[(size_t)i], wls[(size_t)i], yslope, invF, f, vw->W, vw->H});
        }
        band_mirror::raster_banded(frs, warps, queue_words, band_rows, item_cap, qs, bs);
    }
    if (stats) {
        std::vector<int> &o = bs.open;
        double mean = 0;
        for (int v : o) mean += v;
        mean = o.empty() ? 0 : mean / (double)o.size();
        long long p90 = 0;
        if (!o.empty()) {
            std::nth_element(o.begin(), o.begin() + (ptrdiff_t)(o.size() * 9 / 10), o.end());
            p90 = o[o.size() * 9 / 10];
        }
        stats[0] = bs.rows; stats[1] = bs.ctas; stats[2] = bs.ctas_fallback; stats[3] = bs.items; stats[4] = bs.items_max;
        stats[5] = qs.overflow; stats[6] = (long long)(mean * 1000.0); stats[7] = p90 * 1000; stats[8] = bs.ctas_masked;
    }
    if (ms) *ms = bs.ctas ? bs.makespan / (double)bs.ctas : 0.0;
    return 0;
}
