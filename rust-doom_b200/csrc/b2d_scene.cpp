// See b2d_scene.hpp for the reference citations.
#include "b2d_scene.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <string>

namespace b2d {

namespace {

// ---- sky table (assets/meta/doom.toml:29-68): first match wins, fallback = first entry ----------
bool match_episode(const std::string &s, char episode) {       // unanchored "E<d>M."
    for (size_t i = 0; i + 3 < s.size(); i++)
        if (s[i] == 'E' && s[i + 1] == episode && s[i + 2] == 'M') return true;
    return false;
}

int map_number(const std::string &s, size_t at) {               // two digits after "MAP", else -1
    if (at + 5 > s.size()) return -1;
    char a = s[at + 3], b = s[at + 4];
    if (a < '0' || a > '9' || b < '0' || b > '9') return -1;
    return (a - '0') * 10 + (b - '0');
}

Name sky_for(const Name &level_name) {
    std::string s = name_str(level_name);
    for (char e = '1'; e <= '4'; e++)
        if (match_episode(s, e)) return make_name((std::string("SKY") + e).c_str());
    auto any_map = [&](auto pred) {
        for (size_t i = 0; i + 5 <= s.size(); i++)
            if (s.compare(i, 3, "MAP") == 0) {
                int n = map_number(s, i);
                if (n >= 0 && pred(n)) return true;
            }
        return false;
    };
    if (any_map([](int n) { return n >= 1 && n <= 11; })) return make_name("SKY1");
    if (any_map([](int n) { return n >= 12 && n <= 20; })) return make_name("SKY2");
    if (any_map([](int n) { return (n >= 21 && n <= 29) || n == 32; })) return make_name("SKY3");
    return make_name("SKY1");
}

int32_t floormod(int32_t a, int32_t b) {
    int32_t r = a % b;
    return r < 0 ? r + b : r;
}

uint64_t isqrt64(uint64_t v) {
    if (v == 0) return 0;
    uint64_t r = (uint64_t)std::sqrt((double)v);
    while (r * r > v) r--;
    while ((r + 1) * (r + 1) <= v) r++;
    return r;
}

struct AnimGroup { bool is_flat; const char *frames[8]; };
const AnimGroup kAnimGroups[] = {
#include "b2d_anim_table.inc"
};

const AnimGroup *anim_group_of(const Name &n, bool is_flat) {
    const std::string s = name_str(n);
    for (const AnimGroup &g : kAnimGroups) {
        if (g.is_flat != is_flat) continue;
        for (int i = 0; i < 8 && g.frames[i]; i++)
            if (s == g.frames[i]) return &g;
    }
    return nullptr;
}

struct ThingMeta { int type; const char *sprite; char frame; bool hanging; };
const ThingMeta kThings[] = {
#include "b2d_thing_table.inc"
};

struct BlobWriter {
    std::vector<uint8_t> bytes;
    BlobWriter() : bytes(4 * H_COUNT, 0) {}
    uint32_t append(const void *p, size_t n) {
        // every offset and size in the header is 32-bit, and the device side indexes with 32-bit offsets: a level whose
        // textures would push the blob past 2 GiB (TEXTUREx entries are 22 bytes and can declare 4096x4096 images) is refused
        if (bytes.size() + n > (size_t)0x7FFFFFF0) throw WadError(kErrCorrupt, "compiled scene exceeds 2 GiB (texture data too large)");
        uint32_t off = (uint32_t)bytes.size();
        const uint8_t *b = static_cast<const uint8_t *>(p);
        bytes.insert(bytes.end(), b, b + n);
        while (bytes.size() % 16) bytes.push_back(0);
        return off;
    }
};

}  // namespace

uint8_t light_byte(int16_t light, int contrast) {
    volatile float level = (float)(int16_t)(light >> 3) / 31.0f;          // light.rs:113-115
    if (contrast) {
        volatile float c = contrast > 0 ? 2.0f / 31.0f : -2.0f / 31.0f;    // light.rs:82-91
        level = level + c;
        if (level > 1.0f) level = 1.0f; else if (level < 0.0f) level = 0.0f;
    }
    if (level > 1.0f) level = 1.0f; else if (level < 0.0f) level = 0.0f;   // lights.rs:26-29
    volatile float scaled = level * 255.0f;
    return (uint8_t)(int)scaled;
}

int sector_at(const Level &lv, double x, double y, int *subsector_out) {
    if (lv.nodes.empty()) return -1;
    unsigned child = (unsigned)lv.nodes.size() - 1;
    bool leaf = false;
    for (int guard = 0; guard < 4096 && !leaf; guard++) {
        const Node &n = lv.nodes[child];
        double sd = (y - (double)n.y) * (double)n.dx - (x - (double)n.x) * (double)n.dy;
        unsigned next = sd > 0.0 ? n.left : n.right;
        child = next & 0x7FFFu;
        leaf = (next & 0x8000u) != 0;
        if (!leaf && child >= lv.nodes.size()) return -1;
    }
    if (!leaf || child >= lv.subsectors.size()) return -1;
    const Subsector &ss = lv.subsectors[child];
    if (ss.num_segs == 0 || (size_t)ss.first_seg + ss.num_segs > lv.segs.size()) return -1;
    int side = lv.seg_sidedef(lv.segs[ss.first_seg]);
    if (side < 0) return -1;
    int sector = lv.sidedefs[(size_t)side].sector;
    if (sector >= (int)lv.sectors.size()) return -1;
    for (unsigned i = 0; i < ss.num_segs; i++) {
        const Seg &s = lv.segs[(size_t)ss.first_seg + i];
        if (s.v1 >= lv.vertices.size() || s.v2 >= lv.vertices.size()) continue;
        const Vertex &a = lv.vertices[s.v1], &b = lv.vertices[s.v2];
        double dx = (double)b.x - (double)a.x, dy = (double)b.y - (double)a.y;
        double len = std::hypot(dx, dy);
        if (len < 1e-14) continue;
        double sd = ((y - (double)a.y) * dx - (x - (double)a.x) * dy) / len;
        if (sd > 10.0) return -1;           // SEG_TOLERANCE 0.1 world units (visitor.rs:1159)
    }
    if (subsector_out) *subsector_out = (int)child;
    return sector;
}

std::vector<uint8_t> compile_scene(const Archive &wad, const TextureDirectory &td, int level_index,
                                   const std::vector<DynRec> &dynamic) {
    return compile_scene(Level::load(wad, level_index), td, dynamic);
}

std::vector<uint8_t> compile_scene(const Level &lv, const TextureDirectory &td, const std::vector<DynRec> &dynamic) {
    const int nverts = (int)lv.vertices.size(), nsegs = (int)lv.segs.size();
    const int nsect = (int)lv.sectors.size(), nss = (int)lv.subsectors.size(), nnodes = (int)lv.nodes.size();

    // sectors that may move and their height ranges, widened to contain the heights in the lumps (visitor.rs:232-245)
    std::vector<DynRec> dyn;
    std::vector<int> dyn_of((size_t)nsect, -1);
    for (const DynRec &d : dynamic) {
        if (d.sector < 0 || d.sector >= nsect || dyn_of[(size_t)d.sector] >= 0)
            throw WadError(kErrArg, "dynamic sector out of range or listed twice");
        const Sector &sc = lv.sectors[(size_t)d.sector];
        DynRec n{};
        n.sector = d.sector;
        n.floor_min = std::min({d.floor_min, d.floor_max, (int32_t)sc.floor});
        n.floor_max = std::max({d.floor_min, d.floor_max, (int32_t)sc.floor});
        n.ceil_min = std::min({d.ceil_min, d.ceil_max, (int32_t)sc.ceil});
        n.ceil_max = std::max({d.ceil_min, d.ceil_max, (int32_t)sc.ceil});
        dyn_of[(size_t)d.sector] = (int)dyn.size();
        dyn.push_back(n);
    }
    std::sort(dyn.begin(), dyn.end(), [](const DynRec &a, const DynRec &b) { return a.sector < b.sector; });
    for (size_t i = 0; i < dyn.size(); i++) dyn_of[(size_t)dyn[i].sector] = (int)i;
    auto floor_lo = [&](int s) { return dyn_of[(size_t)s] >= 0 ? dyn[(size_t)dyn_of[(size_t)s]].floor_min : (int32_t)lv.sectors[(size_t)s].floor; };
    auto floor_hi = [&](int s) { return dyn_of[(size_t)s] >= 0 ? dyn[(size_t)dyn_of[(size_t)s]].floor_max : (int32_t)lv.sectors[(size_t)s].floor; };
    auto ceil_lo = [&](int s) { return dyn_of[(size_t)s] >= 0 ? dyn[(size_t)dyn_of[(size_t)s]].ceil_min : (int32_t)lv.sectors[(size_t)s].ceil; };
    auto ceil_hi = [&](int s) { return dyn_of[(size_t)s] >= 0 ? dyn[(size_t)dyn_of[(size_t)s]].ceil_max : (int32_t)lv.sectors[(size_t)s].ceil; };
    std::vector<SegDynRec> segdyn((size_t)nsegs, SegDynRec{-1, 0});

    // ids are handed out in first-use order: sky, then segs (A before B), flats by sector order
    std::unordered_map<Name, int, NameHash> tex_ids, flat_ids;
    std::vector<const Image *> tex_list;
    std::vector<const uint8_t *> flat_list;
    // animation frame lists (static.vert:23-39, tex.rs:421-473): when a texture / flat of an animation group is
    // used, every existing frame of the group is loaded and the group's ids are appended to `anim_frames`
    std::vector<int32_t> anim_frames;
    struct AnimRef { int32_t first, n, k; };
    std::unordered_map<int, AnimRef> tex_anim;
    std::vector<std::vector<int32_t>> flat_groups;
    std::function<int32_t(const Name &, bool)> tex_id_impl = [&](const Name &n, bool follow) -> int32_t {
        if (is_untextured(n)) return kTexNone;
        auto it = tex_ids.find(n);
        if (it != tex_ids.end()) return it->second;
        const Image *img = td.texture(n);
        if (!img || img->w == 0 || img->h == 0) return kTexNone;       // visitor.rs:857-860
        int id = (int)tex_list.size();
        tex_ids[n] = id;
        tex_list.push_back(img);
        const AnimGroup *g = follow ? anim_group_of(n, false) : nullptr;
        if (g) {
            std::vector<int32_t> ids;
            for (int i = 0; i < 8 && g->frames[i]; i++) {
                int32_t f = tex_id_impl(make_name(g->frames[i]), false);
                if (f >= 0) ids.push_back(f);
            }
            if (ids.size() > 1) {
                const int32_t first = (int32_t)anim_frames.size();
                for (size_t k = 0; k < ids.size(); k++) {
                    anim_frames.push_back(ids[k]);
                    tex_anim[ids[k]] = AnimRef{first, (int32_t)ids.size(), (int32_t)k};
                }
            }
        }
        return id;
    };
    auto tex_id = [&](const Name &n) -> int32_t { return tex_id_impl(n, true); };
    std::function<int32_t(const Name &, bool)> flat_id_impl = [&](const Name &n, bool follow) -> int32_t {
        if (is_sky_flat(n)) return kFlatSky;
        auto it = flat_ids.find(n);
        if (it != flat_ids.end()) return it->second;
        const uint8_t *p = td.flat(n);
        if (!p) return kFlatMissing;
        int id = (int)flat_list.size();
        flat_ids[n] = id;
        flat_list.push_back(p);
        const AnimGroup *g = follow ? anim_group_of(n, true) : nullptr;
        if (g) {
            std::vector<int32_t> ids;
            for (int i = 0; i < 8 && g->frames[i]; i++) {
                int32_t f = flat_id_impl(make_name(g->frames[i]), false);
                if (f >= 0) ids.push_back(f);
            }
            if (ids.size() > 1) flat_groups.push_back(ids);
        }
        return id;
    };
    auto flat_id = [&](const Name &n) -> int32_t { return flat_id_impl(n, true); };

    const int32_t sky_tex = tex_id(sky_for(lv.name));

    static const int kEffectTypes[] = {1, 2, 4, 13, 3, 12, 8, 17};    // light.rs:127-134
    std::vector<SectorRec> sectors((size_t)nsect);
    std::vector<char> has_effect((size_t)nsect, 0);
    std::vector<LightRec> lights((size_t)nsect, LightRec{});
    int32_t min_h = 32767, max_h = -32768;
    for (int i = 0; i < nsect; i++) {
        const Sector &s = lv.sectors[(size_t)i];
        bool eff = false;
        for (int t : kEffectTypes)
            if (s.type == t) eff = (lv.sector_min_light(i) >> 3) != (s.light >> 3);
        has_effect[(size_t)i] = eff;
        LightRec &L = lights[(size_t)i];                                // light.rs:27-80 new_light
        L.level = (float)(int16_t)(s.light >> 3) / 31.0f;
        if (eff) {
            L.alt = (float)(int16_t)(lv.sector_min_light(i) >> 3) / 31.0f;
            const bool synced = s.type == 12 || s.type == 13 || s.type == 8;
            L.sync = synced ? 0.0f : (float)(((uint64_t)i * 1664525u + 1013904223u) & 0xFFFFu) / 15.0f;
            switch (s.type) {
                case 1: L.kind = kLightRandom; L.speed = 20.0f; L.duration = 0.06f; break;          // FLASH
                case 17: L.kind = kLightRandom; L.speed = 8.0f; L.duration = 0.5f; break;           // FLICKER
                case 3: case 12: L.kind = kLightAlternate; L.speed = 1.0f; L.duration = 0.85f; break;   // slow strobe
                case 2: case 4: case 13: L.kind = kLightAlternate; L.speed = 2.0f; L.duration = 0.7f; break;
                default: L.kind = kLightGlow; L.speed = 0.5f; L.duration = 0.0f; break;             // GLOW (8)
            }
        }
        SectorRec r{};
        r.floor = s.floor; r.ceil = s.ceil;
        r.floor_flat = flat_id(s.floor_tex);
        r.ceil_flat = flat_id(s.ceil_tex);
        r.light = eff ? light_byte_at(L, 0) : light_byte(s.light, 0);     // effects evaluated at tic 0
        sectors[(size_t)i] = r;
        if (s.floor < min_h) min_h = s.floor;
        if (s.ceil > max_h) max_h = s.ceil;
    }
    if (nsect == 0) { min_h = 0; max_h = 0; }
    min_h -= 512; max_h += 512;                                         // visitor.rs:1173-1182

    // subsector sector = front sector of its first seg (visitor.rs:636-643); that sector is the
    // `sector` every seg of the subsector is emitted with (visitor.rs:666).
    std::vector<SSectorRec> ssectors((size_t)nss);
    std::vector<int> seg_front((size_t)nsegs, -1);
    for (int i = 0; i < nss; i++) {
        const Subsector &ss = lv.subsectors[(size_t)i];
        SSectorRec r{};
        r.sector = -1;
        if (ss.num_segs > 0 && (int)ss.first_seg + (int)ss.num_segs <= nsegs) {
            r.first_seg = ss.first_seg; r.num_segs = ss.num_segs;
            int side = lv.seg_sidedef(lv.segs[ss.first_seg]);
            if (side >= 0 && lv.sidedefs[(size_t)side].sector < nsect) r.sector = lv.sidedefs[(size_t)side].sector;
            for (int k = 0; k < ss.num_segs; k++) seg_front[(size_t)ss.first_seg + (size_t)k] = r.sector;
        }
        ssectors[(size_t)i] = r;
    }

    std::vector<SegRec> segs((size_t)nsegs);
    std::vector<MidRec> mids;
    for (int i = 0; i < nsegs; i++) {
        const Seg &sg = lv.segs[(size_t)i];
        SegRec r{};
        r.flags = kSegInvalid; r.texA = r.texB = kTexNone; r.mid = -1;
        bool ok = sg.v1 < nverts && sg.v2 < nverts && sg.linedef < lv.linedefs.size();
        int side = ok ? lv.seg_sidedef(sg) : -1;
        int front = seg_front[(size_t)i];
        if (front < 0 && side >= 0 && lv.sidedefs[(size_t)side].sector < nsect)
            front = lv.sidedefs[(size_t)side].sector;
        if (!ok || side < 0 || front < 0) { segs[(size_t)i] = r; continue; }
        const Linedef &line = lv.linedefs[sg.linedef];
        const Sidedef &sd = lv.sidedefs[(size_t)side];
        const Sector &fs = lv.sectors[(size_t)front];
        const int32_t ff = fs.floor, fc = fs.ceil;
        const Vertex &a = lv.vertices[sg.v1], &b = lv.vertices[sg.v2];
        const int64_t dx = (int64_t)b.x - a.x, dy = (int64_t)b.y - a.y;
        const bool unpeg_upper = line.flags & 0x0008, unpeg_lower = line.flags & 0x0010;
        // world X = -wad_y/100, world Z = -wad_x/100: "v1[0]==v2[0]" <=> dy==0 => Brighten,
        // "v1[1]==v2[1]" <=> dx==0 => Darken (visitor.rs:887-901)
        int contrast = 0;
        if (!has_effect[(size_t)front]) contrast = dy == 0 ? 1 : (dx == 0 ? -1 : 0);
        int back = -1;
        int bside = lv.seg_back_sidedef(sg);
        if (bside >= 0 && lv.sidedefs[(size_t)bside].sector < nsect) back = lv.sidedefs[(size_t)bside].sector;

        // texture row at the piece's top edge, reduced modulo the texture height
        auto piece = [&](const Name &nm, int32_t &tex_out, int32_t &t_out, auto top_row) {
            tex_out = tex_id(nm);
            t_out = 0;
            if (tex_out < 0) return;
            int32_t th = tex_list[(size_t)tex_out]->h;
            t_out = floormod(top_row(th) + sd.yoff, th);
        };

        r.v1 = sg.v1; r.v2 = sg.v2; r.front = front; r.mid = -1;
        const int32_t scroll = line.special == 0x30 ? kSegScroll : 0;          // visitor.rs:922
        r.uoff = (int32_t)sg.offset + sd.xoff;                                   // visitor.rs:904
        r.len_q12 = (int32_t)isqrt64((uint64_t)(dx * dx + dy * dy) << 24);       // visitor.rs:905
        r.light = has_effect[(size_t)front] ? sectors[(size_t)front].light : light_byte(fs.light, contrast);
        if (back < 0) {
            // one-sided: full-height middle (visitor.rs:733-749); Peg::Bottom -> texture bottom at
            // the floor, Peg::Top -> texture top at the ceiling (visitor.rs:909-912)
            r.flags = scroll;
            if (unpeg_lower) piece(sd.middle, r.texA, r.tA, [&](int32_t th) { return th - (fc - ff); });
            else piece(sd.middle, r.texA, r.tA, [&](int32_t) { return 0; });
            r.hA = fc;
            r.otop = fc; r.obot = ff;
            segdyn[(size_t)i] = SegDynRec{-1, unpeg_lower ? kSegDynUnpegLower : 0};
        } else {
            const Sector &bs = lv.sectors[(size_t)back];
            const int32_t bf = bs.floor, bc = bs.ceil;
            const bool back_sky = is_sky_flat(bs.ceil_tex);
            r.flags = kSegTwoSided | scroll;
            segdyn[(size_t)i] = SegDynRec{back, (unpeg_lower ? kSegDynUnpegLower : 0) | (back_sky ? kSegDynBackSky : 0)};
            r.otop = fc;
            // next to a sector that may move, a piece that can come into existence is resolved as well (the
            // reference pre-extends the lower quad over the floor ranges, visitor.rs:772-790; the upper likewise here)
            if (ceil_lo(back) < ceil_hi(front) && !back_sky) {                   // visitor.rs:791-807 (= bc < fc when static)
                if (bc < fc) r.otop = bc;
                if (unpeg_upper) piece(sd.upper, r.texA, r.tA, [&](int32_t) { return 0; });
                else piece(sd.upper, r.texA, r.tA, [&](int32_t th) { return th - (fc - bc); });
            }
            r.hA = fc;
            r.obot = ff;
            const int32_t bf_hi = floor_hi(back), ff_lo = floor_lo(front);
            const bool lower = bf_hi > ff_lo;                                    // visitor.rs:772 (= bf > ff when static)
            if (lower) {
                if (bf > ff) r.obot = bf;
                if (unpeg_lower)             // quad height = back_range.1 - front_range.0 (visitor.rs:777-780, 913-917)
                    piece(sd.lower, r.texB, r.tB, [&](int32_t th) { return th - (bf_hi - ff_lo) + (fc - ff); });
                else piece(sd.lower, r.texB, r.tB, [&](int32_t) { return 0; });
            }
            r.hB = lower ? bf : r.obot;          // anchor of tB: the back floor (the piece moves with it)
            // masked middle (visitor.rs:808-836): spans max(floors)..min(ceilings); float pegs clamp the quad to
            // the texture height (visitor.rs:875-885); t at `high`: Top/Floats 0, Bottom texh-height (:909-919)
            const int32_t low0 = lower ? bf : ff, high0 = bc < fc ? bc : fc;
            int32_t mtex = low0 < high0 ? tex_id(sd.middle) : kTexNone;
            if (mtex >= 0) {
                const int32_t th = tex_list[(size_t)mtex]->h;
                enum { kTop, kBottom, kTopFloat, kBottomFloat } peg;
                if (unpeg_lower) peg = is_untextured(sd.upper) ? kTopFloat : kBottom;
                else peg = is_untextured(sd.lower) ? kBottomFloat : kTop;
                int32_t low = low0, high = high0;
                if (peg == kTopFloat) { low = low0 + sd.yoff; high = low0 + th + sd.yoff; }
                else if (peg == kBottomFloat) { low = high0 + sd.yoff - th; high = high0 + sd.yoff; }
                const int32_t t_high = peg == kBottom ? th - (high - low) : 0;
                MidRec m{};
                m.tex = mtex; m.t_high = floormod(t_high + sd.yoff, th); m.low = low; m.high = high;
                r.mid = (int32_t)mids.size();
                mids.push_back(m);
            }
        }
        segs[(size_t)i] = r;
    }

    // decoration things -> sprites, grouped by subsector (visitor.rs:1010-1026, 1062-1137)
    struct SpriteRow { int ss, thing; SpriteRec rec; };
    std::vector<SpriteRow> sprite_rows;
    for (size_t ti = 0; ti < lv.things.size(); ti++) {
        const Thing &t = lv.things[ti];
        if (t.type == 1 || t.type == 2 || t.type == 3 || t.type == 4 || t.type == 11 || t.type == 14) continue;
        int ssid = -1;
        int sec = sector_at(lv, (double)t.x, (double)t.y, &ssid);
        if (sec < 0 || ssid < 0 || ssid >= nss || ssectors[(size_t)ssid].sector != sec) continue;
        const ThingMeta *meta = nullptr;
        for (const ThingMeta &m : kThings)
            if (m.type == t.type) { meta = &m; break; }
        if (!meta) continue;
        int32_t tid = kTexNone;
        for (char rot : {'0', '1'}) {                      // <sprite><frame>0, then <sprite><frame>1
            std::string nm = std::string(meta->sprite) + meta->frame + rot;
            Name name;
            try { name = make_name(nm.c_str()); } catch (const WadError &) { break; }
            if (td.texture(name)) { tid = tex_id(name); break; }
        }
        if (tid < 0) continue;
        const Sector &sct = lv.sectors[(size_t)sec];
        const int32_t th = tex_list[(size_t)tid]->h;
        SpriteRow row{ssid, (int)ti, SpriteRec{}};
        row.rec.x = t.x; row.rec.y = t.y;
        row.rec.low = meta->hanging ? sct.ceil - th : sct.floor;
        row.rec.tex = tid;
        row.rec.light = sectors[(size_t)sec].light;
        row.rec.sector = sec;
        row.rec.hanging = meta->hanging ? 1 : 0;
        sprite_rows.push_back(row);
    }
    std::stable_sort(sprite_rows.begin(), sprite_rows.end(),
                     [](const SpriteRow &a, const SpriteRow &b) { return a.ss != b.ss ? a.ss < b.ss : a.thing < b.thing; });
    std::vector<SpriteRec> sprites;
    for (size_t k = 0; k < sprite_rows.size();) {
        size_t j = k;
        while (j < sprite_rows.size() && sprite_rows[j].ss == sprite_rows[k].ss) j++;
        if (j - k > 255)      // the count shares a word with the first index: refuse instead of dropping sprites silently
            throw WadError(kErrCorrupt, "more than 255 decoration things in one subsector");
        size_t cnt = j - k;
        ssectors[(size_t)sprite_rows[k].ss].sprites = (int32_t)(k | (cnt << 24));
        k = j;
    }
    for (const SpriteRow &r : sprite_rows) sprites.push_back(r.rec);

    std::vector<NodeRec> nodes((size_t)nnodes);
    auto child = [](uint16_t c) -> uint32_t { return (c & 0x8000u) ? ((c & 0x7FFFu) | kLeaf) : (c & 0x7FFFu); };
    // Child bounding boxes are recomputed from the segs each subtree actually holds (never trusted from the
    // file), so that bounding-box culling in the walk kernel stays conservative for inconsistent maps.
    // box = {top, bottom, left, right}; empty subtree -> {0,0,0,0}; cyclic reference -> whole range.
    struct Box { bool valid; int32_t b[4]; };
    const Box kFull{true, {32767, -32768, -32768, 32767}};
    auto unite = [](const Box &a, const Box &c) -> Box {
        if (!a.valid) return c;
        if (!c.valid) return a;
        Box r{true, {a.b[0] > c.b[0] ? a.b[0] : c.b[0], a.b[1] < c.b[1] ? a.b[1] : c.b[1],
                     a.b[2] < c.b[2] ? a.b[2] : c.b[2], a.b[3] > c.b[3] ? a.b[3] : c.b[3]}};
        return r;
    };
    auto leaf_box = [&](uint32_t ss_id) -> Box {
        Box box{false, {0, 0, 0, 0}};
        if (ss_id >= (uint32_t)nss) return box;
        const SSectorRec &ss = ssectors[ss_id];
        for (int k = ss.first_seg; k < ss.first_seg + ss.num_segs; k++) {
            const SegRec &sg = segs[(size_t)k];
            if (sg.flags & kSegInvalid) continue;
            for (int32_t v : {sg.v1, sg.v2}) {
                int32_t x = lv.vertices[(size_t)v].x, y = lv.vertices[(size_t)v].y;
                Box p{true, {y, y, x, x}};
                box = unite(box, p);
            }
        }
        return box;
    };
    std::vector<char> state((size_t)nnodes, 0);              // 0 unvisited, 1 on the stack, 2 done
    std::vector<Box> node_box((size_t)nnodes, Box{false, {0, 0, 0, 0}});
    std::vector<std::array<Box, 2>> child_box((size_t)nnodes, {Box{false, {0, 0, 0, 0}}, Box{false, {0, 0, 0, 0}}});
    if (nnodes > 0) {
        std::vector<int> stack{nnodes - 1};
        state[(size_t)nnodes - 1] = 1;
        while (!stack.empty()) {
            const int i = stack.back();
            const Node &n = lv.nodes[(size_t)i];
            int pending = -1;
            const uint16_t raw[2] = {n.right, n.left};
            for (int side = 0; side < 2 && pending < 0; side++) {
                uint32_t c = child(raw[side]);
                Box box{false, {0, 0, 0, 0}};
                if (c & kLeaf) box = leaf_box(c & 0x7FFFFFFFu);
                else if ((int)c >= nnodes) box = Box{false, {0, 0, 0, 0}};
                else if (state[c] == 2) box = node_box[c];
                else if (state[c] == 1) box = kFull;
                else { pending = (int)c; break; }
                child_box[(size_t)i][(size_t)side] = box;
            }
            if (pending >= 0) {
                state[(size_t)pending] = 1;
                stack.push_back(pending);
                continue;
            }
            node_box[(size_t)i] = unite(child_box[(size_t)i][0], child_box[(size_t)i][1]);
            state[(size_t)i] = 2;
            stack.pop_back();
        }
    }
    for (int i = 0; i < nnodes; i++) {
        const Node &n = lv.nodes[(size_t)i];
        NodeRec r{};
        r.x = n.x; r.y = n.y; r.dx = n.dx; r.dy = n.dy;
        if (state[(size_t)i] == 2) {
            const Box &rb = child_box[(size_t)i][0], &lb = child_box[(size_t)i][1];
            for (int k = 0; k < 4; k++) { r.rbox[k] = rb.valid ? rb.b[k] : 0; r.lbox[k] = lb.valid ? lb.b[k] : 0; }
        }
        r.child[0] = child(n.right);
        r.child[1] = child(n.left);
        nodes[(size_t)i] = r;
    }

    std::vector<int32_t> verts((size_t)nverts * 2);
    for (int i = 0; i < nverts; i++) { verts[2 * (size_t)i] = lv.vertices[(size_t)i].x; verts[2 * (size_t)i + 1] = lv.vertices[(size_t)i].y; }

    // textures: u8 row-major, transparent texels (high byte set) become 0
    std::vector<TexRec> texrec(tex_list.size());
    std::vector<uint8_t> texels;
    for (size_t i = 0; i < tex_list.size(); i++) {
        const Image &im = *tex_list[i];
        TexRec t{};
        t.texel_off = (uint32_t)texels.size();
        t.w = (uint32_t)im.w; t.h = (uint32_t)im.h;
        t.hmagic = (uint32_t)((((uint64_t)1 << 32) / (uint64_t)im.h + 1) & 0xFFFFFFFFu);
        t.hbias = (uint32_t)im.h * (uint32_t)((16384 + im.h - 1) / im.h);
        t.mask_off = 0xFFFFFFFFu;
        {
            auto an = tex_anim.find((int)i);
            if (an != tex_anim.end()) { t.anim_first = (uint32_t)an->second.first; t.anim_nk = (uint32_t)an->second.n | ((uint32_t)an->second.k << 16); }
        }
        bool holes = false;
        for (uint16_t v : im.px) { texels.push_back((v >> 8) ? 0 : (uint8_t)(v & 0xFF)); holes |= (v >> 8) != 0; }
        while (texels.size() % 16) texels.push_back(0);
        if (holes) {            // opacity plane (1 = opaque) right behind the texels
            t.mask_off = (uint32_t)texels.size();
            for (uint16_t v : im.px) texels.push_back((v >> 8) ? 0 : 1);
            while (texels.size() % 16) texels.push_back(0);
        }
        texrec[i] = t;
    }
    std::vector<uint8_t> flats(flat_list.size() * 4096);
    for (size_t i = 0; i < flat_list.size(); i++) std::memcpy(&flats[i * 4096], flat_list[i], 4096);
    std::vector<FlatAnimRec> flat_anim(flat_list.size(), FlatAnimRec{0, 0});
    for (const auto &ids : flat_groups) {
        const int32_t first = (int32_t)anim_frames.size();
        for (size_t k = 0; k < ids.size(); k++) {
            anim_frames.push_back(ids[k]);
            flat_anim[(size_t)ids[k]] = FlatAnimRec{first, (int32_t)ids.size() | ((int32_t)k << 16)};
        }
    }
    std::vector<uint8_t> colormap(34 * 256, 0);
    for (size_t k = 0; k < td.colormaps.size() && k < 34; k++) std::memcpy(&colormap[k * 256], td.colormaps[k].data(), 256);
    std::vector<uint32_t> palette(256, 0xFF000000u);
    if (!td.palettes.empty())
        for (int i = 0; i < 256; i++)
            palette[(size_t)i] = palette_word(&td.palettes[0][(size_t)i * 3]);

    // player-1 start (visitor.rs:1010-1026; game/src/level.rs:757-762; player.rs:88 camera_height)
    int32_t has_start = 0, sx = 0, sy = 0, sz = 0, sang = 0;
    for (const Thing &t : lv.things) {
        if (t.type != 1) continue;
        int sec = sector_at(lv, (double)t.x, (double)t.y);
        if (sec < 0) continue;
        float yaw = std::round((float)t.angle / 45.0f) * 45.0f;
        has_start = 1;
        sx = t.x - 32; sy = t.y;
        sz = lv.sectors[(size_t)sec].floor + 50 + 12;
        sang = (((int)yaw % 360) + 360) % 360;
        // no break: visit_marker overwrites start_pos on every player-1 start, so the LAST one wins
        // (game/src/level.rs:757-762) -- maps with voodoo dolls have several
    }

    BlobWriter w;
    uint32_t hdr[H_COUNT] = {0};
    hdr[H_MAGIC] = kSceneMagic; hdr[H_VERSION] = kSceneVersion;
    hdr[H_NVERTS] = (uint32_t)nverts; hdr[H_NNODES] = (uint32_t)nnodes; hdr[H_NSSECTORS] = (uint32_t)nss;
    hdr[H_NSEGS] = (uint32_t)nsegs; hdr[H_NSECTORS] = (uint32_t)nsect;
    hdr[H_NTEX] = (uint32_t)tex_list.size(); hdr[H_NFLATS] = (uint32_t)flat_list.size();
    hdr[H_OFF_VERTS] = w.append(verts.data(), verts.size() * 4);
    hdr[H_OFF_NODES] = w.append(nodes.data(), nodes.size() * sizeof(NodeRec));
    hdr[H_OFF_SSECTORS] = w.append(ssectors.data(), ssectors.size() * sizeof(SSectorRec));
    hdr[H_OFF_SEGS] = w.append(segs.data(), segs.size() * sizeof(SegRec));
    hdr[H_OFF_SECTORS] = w.append(sectors.data(), sectors.size() * sizeof(SectorRec));
    hdr[H_OFF_TEX] = w.append(texrec.data(), texrec.size() * sizeof(TexRec));
    hdr[H_OFF_MIDS] = w.append(mids.data(), mids.size() * sizeof(MidRec));
    hdr[H_NMIDS] = (uint32_t)mids.size();
    hdr[H_OFF_SPRITES] = w.append(sprites.data(), sprites.size() * sizeof(SpriteRec));
    hdr[H_NSPRITES] = (uint32_t)sprites.size();
    hdr[H_OFF_ANIM] = w.append(anim_frames.data(), anim_frames.size() * 4);
    hdr[H_NANIM] = (uint32_t)anim_frames.size();
    hdr[H_OFF_FLAT_ANIM] = w.append(flat_anim.data(), flat_anim.size() * sizeof(FlatAnimRec));
    hdr[H_OFF_LIGHTS] = w.append(lights.data(), lights.size() * sizeof(LightRec));
    hdr[H_OFF_TEXELS] = w.append(texels.data(), texels.size());
    hdr[H_TEXEL_BYTES] = (uint32_t)texels.size();
    hdr[H_OFF_FLATS] = w.append(flats.data(), flats.size());
    hdr[H_OFF_COLORMAP] = w.append(colormap.data(), colormap.size());
    hdr[H_OFF_PALETTE] = w.append(palette.data(), palette.size() * 4);
    hdr[H_OFF_SEGDYN] = w.append(segdyn.data(), segdyn.size() * sizeof(SegDynRec));
    hdr[H_OFF_DYN] = w.append(dyn.data(), dyn.size() * sizeof(DynRec));
    hdr[H_NDYN] = (uint32_t)dyn.size();
    hdr[H_TOTAL] = (uint32_t)w.bytes.size();
    hdr[H_ROOT] = nnodes > 0 ? (uint32_t)(nnodes - 1) : kLeaf;
    hdr[H_SKY_TEX] = (uint32_t)sky_tex;
    hdr[H_START_X] = (uint32_t)sx; hdr[H_START_Y] = (uint32_t)sy; hdr[H_START_Z] = (uint32_t)sz;
    hdr[H_START_ANGLE] = (uint32_t)sang; hdr[H_HAS_START] = (uint32_t)has_start;
    hdr[H_MIN_H] = (uint32_t)min_h; hdr[H_MAX_H] = (uint32_t)max_h;
    std::memcpy(w.bytes.data(), hdr, sizeof hdr);
    return std::move(w.bytes);
}

std::vector<AutomapLine> automap_lines(const Level &lv) {
    constexpr uint16_t kSecret = 0x20, kDontDraw = 0x80;         // ML_SECRET, ML_DONTDRAW
    constexpr uint8_t kWall = 176, kTeleport = 184, kFloorStep = 64, kCeilStep = 231, kPlain = 96;
    // the sector of sidedef `side`, or -1 when the sidedef or its sector does not exist
    auto side_sector = [&](int side) -> int {
        if (side < 0 || (size_t)side >= lv.sidedefs.size()) return -1;
        const int sec = lv.sidedefs[(size_t)side].sector;
        return (size_t)sec < lv.sectors.size() ? sec : -1;
    };
    std::vector<AutomapLine> out;
    for (size_t i = 0; i < lv.linedefs.size(); i++) {
        const Linedef &l = lv.linedefs[i];
        if (l.v1 >= lv.vertices.size() || l.v2 >= lv.vertices.size()) continue;
        const int front = side_sector(l.right), back = side_sector(l.left);
        uint8_t c = kWall, all = kWall;
        if (front >= 0 && back >= 0) {
            const Sector &F = lv.sectors[(size_t)front], &B = lv.sectors[(size_t)back];
            if (l.special == 39) c = kTeleport;
            else if (l.flags & kSecret) c = kWall;
            else if (F.floor != B.floor) c = kFloorStep;
            else if (F.ceil != B.ceil) c = kCeilStep;
            else c = 0;
            all = c ? c : kPlain;
        }
        AutomapLine r{};
        r.x0 = lv.vertices[l.v1].x; r.y0 = lv.vertices[l.v1].y;
        r.x1 = lv.vertices[l.v2].x; r.y1 = lv.vertices[l.v2].y;
        r.colour = (l.flags & kDontDraw) ? 0 : c;
        r.colour_all = all;
        r.linedef = (int32_t)i;
        out.push_back(r);
    }
    return out;
}

}  // namespace b2d
