// Scene compiler: raw level lumps + texture directory -> one flat "B2DS" blob that is uploaded to
// HBM as-is and indexed by the kernels (layout: DESIGN.md "Scene blob"; records below).
//
// What is pre-resolved here is the reference's geometry emitter, per seg instead of per triangle:
//   which wall pieces a seg has, their texture, pegging anchor and offsets   wad/src/visitor.rs:711-937
//   fake contrast and the static light byte   visitor.rs:887-901, wad/src/light.rs:27-115,
//                                              game/src/lights.rs:14-30
//   flats / sky flats per sector               visitor.rs:939-985
//   sky texture of the level                   wad/src/meta.rs:156-172, assets/meta/doom.toml:29-68
//   player-1 start                             visitor.rs:1010-1060, game/src/level.rs:757-762
#pragma once
#include <cmath>
#include <cstdint>
#include <vector>

#include "b2d_math.cuh"
#include "b2d_wad.hpp"

namespace b2d {

constexpr uint32_t kSceneMagic = 0x53443242u;   // "B2DS"
constexpr uint32_t kSceneVersion = 6;
constexpr uint32_t kLeaf = 0x80000000u;

enum HeaderField : int {
    H_MAGIC, H_VERSION, H_TOTAL, H_NVERTS, H_NNODES, H_NSSECTORS, H_NSEGS, H_NSECTORS, H_NTEX, H_NFLATS,
    H_OFF_VERTS, H_OFF_NODES, H_OFF_SSECTORS, H_OFF_SEGS, H_OFF_SECTORS, H_OFF_TEX, H_OFF_TEXELS,
    H_TEXEL_BYTES, H_OFF_FLATS, H_OFF_COLORMAP, H_OFF_PALETTE, H_ROOT, H_SKY_TEX, H_START_X, H_START_Y,
    H_START_Z, H_START_ANGLE, H_HAS_START, H_MIN_H, H_MAX_H, H_NMIDS, H_OFF_MIDS, H_NSPRITES, H_OFF_SPRITES,
    H_NANIM, H_OFF_ANIM, H_OFF_FLAT_ANIM, H_OFF_LIGHTS, H_NDYN, H_OFF_DYN, H_OFF_SEGDYN, H_COUNT = 64
};

// 64-byte records; all int32.
struct NodeRec { int32_t x, y, dx, dy, rbox[4], lbox[4]; uint32_t child[2]; int32_t pad[2]; };  // child[0]=right
struct SSectorRec { int32_t first_seg, num_segs, sector, sprites; };   // sprites = first | count << 24
// decoration thing: billboard of its sprite image's size, centred on (x,y), bottom edge at `low`
// (floor, or ceiling - height for hanging things; visitor.rs:1062-1137), lit by the sector light
struct SpriteRec { int32_t x, y, low, tex, light, sector, hanging, pad; };
struct SegRec {
    int32_t v1, v2, front, flags;
    int32_t uoff, len_q12;
    int32_t texA, tA, hA;      // upper (two-sided) or full-height middle (one-sided)
    int32_t texB, tB, hB;      // lower
    int32_t light, otop, obot, mid;   // mid: index into the mids section, -1 = no masked middle texture
};
// masked two-sided middle texture (visitor.rs:808-836,875-919): vertical extent [low, high) and the
// texture row at `high` (pegging and y offset folded in)
struct MidRec { int32_t tex, t_high, low, high, pad[4]; };
struct SectorRec { int32_t floor, ceil, floor_flat, ceil_flat, light, pad[3]; };
// mask_off = ~0u: opaque.  anim_nk = n | k << 16: frame k of an n-frame animation whose ids are anim[anim_first..+n)
struct TexRec { uint32_t texel_off, w, h, hmagic, hbias, mask_off, anim_first, anim_nk; };
struct FlatAnimRec { int32_t anim_first, anim_nk; };
// sector light effect (wad/src/light.rs:5-25): kind 0 none, 1 glow, 2 random, 3 alternate
struct LightRec { uint32_t kind; float level, alt, speed, duration, sync; uint32_t pad[2]; };
constexpr uint32_t kLightNone = 0, kLightGlow = 1, kLightRandom = 2, kLightAlternate = 3;
// what scene_at_state needs beyond the seg record: back sector (-1 = one-sided) and pegging / sky bits
struct SegDynRec { int32_t back, bits; };
constexpr int32_t kSegDynUnpegLower = 1, kSegDynBackSky = 2;
// a sector that may move, with the height ranges the host's LevelAnalysis found (visitor.rs:146-245)
struct DynRec { int32_t sector, floor_min, floor_max, ceil_min, ceil_max, pad[3]; };
// one state of a moving sector: offsets in map units relative to the heights in the level lumps
struct SectorMove { int32_t sector, floor_offset, ceil_offset; };
static_assert(sizeof(SegDynRec) == 8 && sizeof(DynRec) == 32 && sizeof(SectorMove) == 12, "record layout");
static_assert(sizeof(NodeRec) == 64 && sizeof(SegRec) == 64 && sizeof(SectorRec) == 32 &&
              sizeof(TexRec) == 32 && sizeof(SSectorRec) == 16 && sizeof(MidRec) == 32 &&
              sizeof(SpriteRec) == 32 && sizeof(LightRec) == 32, "record layout");

constexpr int32_t kSegTwoSided = 1, kSegScroll = 2, kSegInvalid = 0x80;   // scroll: special 0x30 (visitor.rs:922)
constexpr int32_t kFlatSky = -1, kFlatMissing = -2, kTexNone = -1;

// Level time (DESIGN.md C14; static.vert:23-39, visitor.rs:922).  `tics` counts 1/35 s.  Every frame name of an
// n-frame animation group is bound to the group's first frame (tex.rs:260, 302-306), so an animated image shows
// group frame (tics/8) mod n whichever frame name the map uses (frame 0 at tic 0: the tables are resolved at
// renderer creation too); walls of a scrolling line (special 0x30) advance their texture column by one texel per tic.  The kernels never see time: the three small tables that
// depend on it (texture records, sector flats, seg column offsets) are re-derived from the blob by the state rule below,
// on the host for a per-batch time and on the device for per-frame states.  Sector light effects (C15) ride on the same mechanism: the light bytes of
// effect sectors, their segs and their sprites are re-evaluated.  Outputs hold H_NTEX / H_NSECTORS / H_NSEGS /
// H_NSPRITES records.
// Light level of a sector at `tics` (game/src/lights.rs:26-66), float32 operation by operation (volatile keeps
// every intermediate a rounded float32: no x87 excess precision, no fused multiply-add).  The sine of the random
// effect's hash is the correctly rounded float32 sine: double-precision sine, rounded once (DESIGN.md C15).
// `extralight` (0..2, DESIGN.md C18): the player's extra light adds f32(2 e) / f32(31) to the level before the clamp.
inline uint8_t light_byte_at(const LightRec &L, uint32_t tics, uint32_t extralight = 0) {
    volatile float time = (float)tics / 35.0f;
    volatile float v = L.level;
    auto fract = [](float x) -> float { volatile float f = std::floor(x); volatile float r = x - f; return r; };
    if (L.kind == kLightGlow) {
        volatile float scale = L.level - L.alt;
        volatile float ts = time * L.speed;
        volatile float phase = ts / scale;
        volatile float d = 0.5f - fract(phase);
        volatile float a = std::fabs(d);
        volatile float a2 = a * 2.0f;
        volatile float a3 = a2 * scale;
        v = a3 + L.alt;
    } else if (L.kind == kLightRandom) {
        volatile float ts = time * L.speed;
        volatile float t = std::floor(ts);
        volatile float t1 = t / 1000.0f;
        volatile float s1 = L.sync + t1;
        volatile float s2 = s1 * 12.9898f;
        volatile float s3 = L.sync * 78.233f;
        volatile float arg = s2 + s3;
        volatile float sn = (float)std::sin((double)arg);
        volatile float n1 = sn * 43758.547f;
        volatile float n2 = 1.0f + n1;
        v = fract(n2) < L.duration ? L.alt : L.level;
    } else if (L.kind == kLightAlternate) {
        volatile float ts = time * L.speed;
        volatile float s3 = L.sync * 3.5435f;
        volatile float ph = ts + s3;
        v = fract(ph) < L.duration ? L.alt : L.level;
    }
    if (extralight) {
        volatile float x = (float)(2 * extralight) / 31.0f;
        v = v + x;
    }
    if (v < 0.0f) v = 0.0f; else if (v > 1.0f) v = 1.0f;
    volatile float scaled = v * 255.0f;
    return scaled >= 0.0f ? (uint8_t)(int)scaled : 0;
}

inline bool scene_is_timed(const uint8_t *blob) {
    const uint32_t *h = reinterpret_cast<const uint32_t *>(blob);
    if (h[H_NANIM] > 0 || h[H_NDYN] > 0) return true;      // sectors that may move: their tables are state too
    const LightRec *lights = reinterpret_cast<const LightRec *>(blob + h[H_OFF_LIGHTS]);
    for (uint32_t i = 0; i < h[H_NSECTORS]; i++)
        if (lights[i].kind != kLightNone) return true;
    const SegRec *segs = reinterpret_cast<const SegRec *>(blob + h[H_OFF_SEGS]);
    for (uint32_t i = 0; i < h[H_NSEGS]; i++)
        if (segs[i].flags & kSegScroll) return true;
    return false;
}

// ---- The state rule: one record of the state-dependent tables at one state -------------------------------------------
// The same functions run on the host (scene_at_time, for b2d_scene_tables_at) and on the device (b2d_state_sets_kernel,
// one thread per record, for every state a renderer draws: its own and per-frame states).
//
// A *compact state* holds only what the tables depend on, as 32-bit words (StateLayout::words of them):
//   [0]                  tics, reduced to what the level uses (state_tics): the animation step tics >> 3 if it animates,
//                        tics & 0xFFFFFF if it scrolls -- two tics that give the same tables give the same word
//   [1]                  1 if any declared sector is off its rest heights (the moving-sector pass runs), else 0
//   [2 .. 2 + 2*ndyn)    floor and ceiling offset of each declared dynamic sector, in DynRec order
//   then                 the light byte of each sector with a light effect, four to a word (light_byte_at on the host:
//                        it is the reference's float32 sequence with a correctly rounded sine)
// Equal compact states give byte-identical tables.
constexpr uint32_t kNoSlot = 0xFFFFu;

// The rest-state sections the rule reads, wherever they are (the blob on the host, their device copy).
struct StateSrc {
    const TexRec *tex;
    const SectorRec *sectors;
    const SegRec *segs;
    const SpriteRec *sprites;
    const MidRec *mids;
    const int32_t *anim;
    const FlatAnimRec *flat_anim;
    const SegDynRec *segdyn;
    const uint32_t *sector_slots;   // per sector: light slot (low 16 bits) | dynamic slot << 16; kNoSlot = none
    const int32_t *mid_seg;         // per masked middle: the seg that owns it (each has exactly one), -1 = none
    uint32_t ntex, nflats, nanim, nsectors, nsegs, nsprites, nmids, ndyn;
    // Extra light (C18; read only by a state with extra light): per sector its static light in steps of 1/31
    // (light >> 3, light_steps), then per seg its fake contrast (-1, 0, +1; 0 in front of a light effect)
    const int16_t *sector_steps;
    const int8_t *seg_contrast;
};

// One compact state as the per-record functions read it.
struct StateIn {
    uint32_t tics, moved;
    const int32_t *off;             // floor, ceiling offset per dynamic slot
    const uint8_t *light;           // light byte per light slot
    uint32_t extra;                 // the player's extra light, 0..2 (C18): the light bytes of the state already hold it
};

B2D_HD StateIn state_in(const uint32_t *words, uint32_t ndyn) {
    StateIn s;
    s.extra = 0;
    s.tics = words[0];
    s.moved = words[1];
    s.off = reinterpret_cast<const int32_t *>(words + 2);
    s.light = reinterpret_cast<const uint8_t *>(words + 2 + 2 * ndyn);
    return s;
}

B2D_HD int32_t anim_now(const StateSrc &s, uint32_t tics, int64_t first, uint32_t nk, int32_t self) {
    const uint32_t n = nk & 0xFFFFu;
    if (n < 2 || first < 0 || first + n > s.nanim) return self;
    return s.anim[first + (int64_t)((tics >> 3) % n)];
}
B2D_HD int32_t flat_now(const StateSrc &s, uint32_t tics, int32_t f) {
    if (f < 0 || (uint32_t)f >= s.nflats) return f;
    const int32_t j = anim_now(s, tics, s.flat_anim[f].anim_first, (uint32_t)s.flat_anim[f].anim_nk, f);
    return (j >= 0 && (uint32_t)j < s.nflats) ? j : f;
}
// light slot / offsets of sector f (f < nsectors)
B2D_HD bool has_light_slot(const StateSrc &s, uint32_t f) { return (s.sector_slots[f] & 0xFFFFu) != kNoSlot; }
B2D_HD int32_t light_of(const StateSrc &s, const StateIn &st, uint32_t f) { return st.light[s.sector_slots[f] & 0xFFFFu]; }
B2D_HD int32_t floor_off_of(const StateSrc &s, const StateIn &st, uint32_t f) {
    const uint32_t d = s.sector_slots[f] >> 16;
    return d == kNoSlot ? 0 : st.off[2 * d];
}
B2D_HD int32_t ceil_off_of(const StateSrc &s, const StateIn &st, uint32_t f) {
    const uint32_t d = s.sector_slots[f] >> 16;
    return d == kNoSlot ? 0 : st.off[2 * d + 1];
}

// The static light byte of `steps` (a sector's light >> 3, plus 2 per step of extra light) with fake contrast `contrast`:
// light_byte's float32 sequence (C12, C18), rounded operation by operation on the device as on the host.
B2D_HD uint8_t light_byte_steps(int32_t steps, int contrast) {
#ifdef __CUDA_ARCH__
    float level = __fdiv_rn((float)steps, 31.0f);
    if (contrast) {
        level = __fadd_rn(level, contrast > 0 ? 2.0f / 31.0f : -2.0f / 31.0f);
        level = level > 1.0f ? 1.0f : (level < 0.0f ? 0.0f : level);
    }
    level = level > 1.0f ? 1.0f : (level < 0.0f ? 0.0f : level);
    return (uint8_t)(int)__fmul_rn(level, 255.0f);
#else
    volatile float level = (float)steps / 31.0f;
    if (contrast) {
        volatile float c = contrast > 0 ? 2.0f / 31.0f : -2.0f / 31.0f;
        level = level + c;
        if (level > 1.0f) level = 1.0f; else if (level < 0.0f) level = 0.0f;
    }
    if (level > 1.0f) level = 1.0f; else if (level < 0.0f) level = 0.0f;
    volatile float scaled = level * 255.0f;
    return (uint8_t)(int)scaled;
#endif
}
// the static light byte of sector f (no light effect) raised by the state's extra light
B2D_HD int32_t extra_light_of(const StateSrc &s, const StateIn &st, uint32_t f, int contrast) {
    return light_byte_steps((int32_t)s.sector_steps[f] + 2 * (int32_t)st.extra, contrast);
}

// Level time (C14): every frame name of an animation group shows group frame (tics/8) mod n.
B2D_HD TexRec tex_at(const StateSrc &s, const StateIn &st, uint32_t i) {
    const int32_t j = anim_now(s, st.tics, (int32_t)s.tex[i].anim_first, s.tex[i].anim_nk, (int32_t)i);
    return (j >= 0 && (uint32_t)j < s.ntex) ? s.tex[j] : s.tex[i];
}

// The moving sectors (C16): the reference attaches every wall quad, flat and decoration to the floor or the ceiling object
// of a sector and translates it rigidly with that object (visitor.rs:733-836 object_id, 957-983, 1106-1121;
// game/src/level.rs:201-245): one-sided wall and masked middle texture -> own floor if the line is lower-unpegged, else own
// ceiling; upper piece -> back ceiling; lower piece -> back floor; decoration -> floor, or ceiling if it hangs.  The
// anchors of the pre-resolved pieces move accordingly and the opening of a two-sided seg follows the moved heights (what
// the depth test leaves visible of the reference's pre-extended quads).
B2D_HD SectorRec sector_at(const StateSrc &s, const StateIn &st, uint32_t i) {
    SectorRec r = s.sectors[i];
    r.floor_flat = flat_now(s, st.tics, r.floor_flat);
    r.ceil_flat = flat_now(s, st.tics, r.ceil_flat);
    if (has_light_slot(s, i)) r.light = light_of(s, st, i);
    else if (st.extra) r.light = extra_light_of(s, st, i, 0);
    if (st.moved) {
        r.floor += floor_off_of(s, st, i);
        r.ceil += ceil_off_of(s, st, i);
    }
    return r;
}

// Walls and sprites of a sector with a light effect carry the sector's light (no fake contrast, visitor.rs:889); walls of
// a scrolling line advance one texel column per tic.
B2D_HD SegRec seg_at(const StateSrc &s, const StateIn &st, uint32_t i) {
    SegRec S = s.segs[i];
    if (S.flags & kSegInvalid) return S;
    if (S.flags & kSegScroll) S.uoff = (int32_t)((uint32_t)S.uoff + (st.tics & 0xFFFFFFu));
    const uint32_t f = (uint32_t)S.front;
    if (f >= s.nsectors) return S;
    if (has_light_slot(s, f)) S.light = light_of(s, st, f);
    else if (st.extra) S.light = extra_light_of(s, st, f, s.seg_contrast[i]);
    if (!st.moved) return S;
    const SegDynRec D = s.segdyn[i];
    const int32_t fo = floor_off_of(s, st, f), co = ceil_off_of(s, st, f);
    const int32_t ff = s.sectors[f].floor + fo, fc = s.sectors[f].ceil + co;
    if (!(S.flags & kSegTwoSided)) {
        S.hA += (D.bits & kSegDynUnpegLower) ? fo : co;
        S.otop = fc;
        S.obot = ff;
        return S;
    }
    const uint32_t b = (uint32_t)D.back;
    if (b >= s.nsectors) return S;
    const int32_t bfo = floor_off_of(s, st, b), bco = ceil_off_of(s, st, b);
    S.hA += bco;
    S.hB += bfo;
    const int32_t bf = s.sectors[b].floor + bfo, bc = s.sectors[b].ceil + bco;
    S.otop = (bc < fc && !(D.bits & kSegDynBackSky)) ? bc : fc;
    S.obot = bf > ff ? bf : ff;
    return S;
}

B2D_HD SpriteRec sprite_at(const StateSrc &s, const StateIn &st, uint32_t i) {
    SpriteRec P = s.sprites[i];
    const uint32_t f = (uint32_t)P.sector;
    if (f >= s.nsectors) return P;
    if (has_light_slot(s, f)) P.light = light_of(s, st, f);
    else if (st.extra) P.light = extra_light_of(s, st, f, 0);
    if (st.moved) P.low += P.hanging ? ceil_off_of(s, st, f) : floor_off_of(s, st, f);
    return P;
}

// a masked middle moves with the object its (two-sided) seg's wall is attached to
B2D_HD MidRec mid_at(const StateSrc &s, const StateIn &st, uint32_t i) {
    MidRec M = s.mids[i];
    const int32_t si = s.mid_seg[i];
    if (!st.moved || si < 0) return M;
    const SegRec &S = s.segs[si];
    const uint32_t f = (uint32_t)S.front, b = (uint32_t)s.segdyn[si].back;
    if ((S.flags & kSegInvalid) || !(S.flags & kSegTwoSided) || f >= s.nsectors || b >= s.nsectors) return M;
    const int32_t own = (s.segdyn[si].bits & kSegDynUnpegLower) ? floor_off_of(s, st, f) : ceil_off_of(s, st, f);
    M.low += own;
    M.high += own;
    return M;
}

// What a scene's compact states look like, derived once from its blob.
struct StateLayout {
    std::vector<uint32_t> sector_slots;     // StateSrc::sector_slots
    std::vector<int32_t> mid_seg;           // StateSrc::mid_seg
    std::vector<uint32_t> light_sectors;    // sector of each light slot
    std::vector<uint32_t> dyn_sectors;      // sector of each dynamic slot (DynRec order)
    bool animates = false, scrolls = false;
    uint32_t words = 2;                     // 32-bit words per compact state
};

inline StateLayout state_layout(const uint8_t *blob) {
    const uint32_t *h = reinterpret_cast<const uint32_t *>(blob);
    const uint32_t nsect = h[H_NSECTORS];
    const LightRec *lights = reinterpret_cast<const LightRec *>(blob + h[H_OFF_LIGHTS]);
    const SegRec *segs = reinterpret_cast<const SegRec *>(blob + h[H_OFF_SEGS]);
    const DynRec *dyn = reinterpret_cast<const DynRec *>(blob + h[H_OFF_DYN]);
    StateLayout L;
    L.sector_slots.assign(nsect, kNoSlot | (kNoSlot << 16));
    for (uint32_t i = 0; i < nsect; i++)
        if (lights[i].kind != kLightNone) {
            L.sector_slots[i] = (L.sector_slots[i] & ~0xFFFFu) | (uint32_t)L.light_sectors.size();
            L.light_sectors.push_back(i);
        }
    for (uint32_t k = 0; k < h[H_NDYN]; k++) {
        const uint32_t s = (uint32_t)dyn[k].sector;
        if (s >= nsect || (L.sector_slots[s] >> 16) != kNoSlot) continue;
        L.sector_slots[s] = (L.sector_slots[s] & 0xFFFFu) | ((uint32_t)L.dyn_sectors.size() << 16);
        L.dyn_sectors.push_back(s);
    }
    if (L.light_sectors.size() >= kNoSlot || L.dyn_sectors.size() >= kNoSlot) throw std::length_error("too many light effect or dynamic sectors");
    L.mid_seg.assign(h[H_NMIDS], -1);
    for (uint32_t i = 0; i < h[H_NSEGS]; i++)
        if (segs[i].mid >= 0 && (uint32_t)segs[i].mid < h[H_NMIDS]) L.mid_seg[(size_t)segs[i].mid] = (int32_t)i;
    L.animates = h[H_NANIM] > 0;
    for (uint32_t i = 0; i < h[H_NSEGS] && !L.scrolls; i++) L.scrolls = (segs[i].flags & kSegScroll) != 0;
    L.words = 2 + 2 * (uint32_t)L.dyn_sectors.size() + ((uint32_t)L.light_sectors.size() + 3) / 4;
    return L;
}

inline uint32_t state_tics(const StateLayout &L, uint32_t tics) {
    if (L.animates && L.scrolls) return tics;
    if (L.animates) return tics & ~7u;
    if (L.scrolls) return tics & 0xFFFFFFu;
    return 0;
}

// The compact state of level time `tics` with `floor_off` / `ceil_off` (nullptr, or one offset per sector) into out[words];
// its light bytes with the player's `extralight` (C18).
inline void compact_state(const uint8_t *blob, const StateLayout &L, uint32_t tics, const int32_t *floor_off,
                          const int32_t *ceil_off, uint32_t *out, uint32_t extralight = 0) {
    const uint32_t *h = reinterpret_cast<const uint32_t *>(blob);
    const LightRec *lights = reinterpret_cast<const LightRec *>(blob + h[H_OFF_LIGHTS]);
    for (uint32_t w = 0; w < L.words; w++) out[w] = 0;
    out[0] = state_tics(L, tics);
    if (floor_off && ceil_off) {
        out[1] = 1;
        for (size_t d = 0; d < L.dyn_sectors.size(); d++) {
            out[2 + 2 * d] = (uint32_t)floor_off[L.dyn_sectors[d]];
            out[3 + 2 * d] = (uint32_t)ceil_off[L.dyn_sectors[d]];
        }
    }
    uint8_t *light = reinterpret_cast<uint8_t *>(out + 2 + 2 * L.dyn_sectors.size());
    for (size_t k = 0; k < L.light_sectors.size(); k++) light[k] = light_byte_at(lights[L.light_sectors[k]], tics, extralight);
}

// The side tables of StateSrc::sector_steps / seg_contrast, derived from the blob: a sector's lights record holds
// (light >> 3) / 31 whatever its effect, and a seg's contrast follows from its vertices as compile_scene derives it
// (visitor.rs:887-901: +1 for a wall along the map's x axis, -1 along its y axis, none in front of a light effect).
inline void light_steps(const uint8_t *blob, std::vector<int16_t> &sector_steps, std::vector<int8_t> &seg_contrast) {
    const uint32_t *h = reinterpret_cast<const uint32_t *>(blob);
    const LightRec *lights = reinterpret_cast<const LightRec *>(blob + h[H_OFF_LIGHTS]);
    const SegRec *segs = reinterpret_cast<const SegRec *>(blob + h[H_OFF_SEGS]);
    const int32_t *verts = reinterpret_cast<const int32_t *>(blob + h[H_OFF_VERTS]);
    sector_steps.assign(h[H_NSECTORS], 0);
    for (uint32_t i = 0; i < h[H_NSECTORS]; i++) sector_steps[i] = (int16_t)std::lrint((double)lights[i].level * 31.0);
    seg_contrast.assign(h[H_NSEGS], 0);
    for (uint32_t i = 0; i < h[H_NSEGS]; i++) {
        const SegRec &S = segs[i];
        if ((S.flags & kSegInvalid) || (uint32_t)S.front >= h[H_NSECTORS] || lights[S.front].kind != kLightNone) continue;
        if ((uint32_t)S.v1 >= h[H_NVERTS] || (uint32_t)S.v2 >= h[H_NVERTS]) continue;
        const int64_t dx = (int64_t)verts[2 * S.v2] - verts[2 * S.v1], dy = (int64_t)verts[2 * S.v2 + 1] - verts[2 * S.v1 + 1];
        seg_contrast[i] = dy == 0 ? 1 : (dx == 0 ? -1 : 0);
    }
}

inline StateSrc state_src(const uint8_t *blob, const StateLayout &L) {
    const uint32_t *h = reinterpret_cast<const uint32_t *>(blob);
    StateSrc s;
    s.tex = reinterpret_cast<const TexRec *>(blob + h[H_OFF_TEX]);
    s.sectors = reinterpret_cast<const SectorRec *>(blob + h[H_OFF_SECTORS]);
    s.segs = reinterpret_cast<const SegRec *>(blob + h[H_OFF_SEGS]);
    s.sprites = reinterpret_cast<const SpriteRec *>(blob + h[H_OFF_SPRITES]);
    s.mids = reinterpret_cast<const MidRec *>(blob + h[H_OFF_MIDS]);
    s.anim = reinterpret_cast<const int32_t *>(blob + h[H_OFF_ANIM]);
    s.flat_anim = reinterpret_cast<const FlatAnimRec *>(blob + h[H_OFF_FLAT_ANIM]);
    s.segdyn = reinterpret_cast<const SegDynRec *>(blob + h[H_OFF_SEGDYN]);
    s.sector_slots = L.sector_slots.data();
    s.mid_seg = L.mid_seg.data();
    s.ntex = h[H_NTEX]; s.nflats = h[H_NFLATS]; s.nanim = h[H_NANIM]; s.nsectors = h[H_NSECTORS];
    s.nsegs = h[H_NSEGS]; s.nsprites = h[H_NSPRITES]; s.nmids = h[H_NMIDS]; s.ndyn = (uint32_t)L.dyn_sectors.size();
    s.sector_steps = nullptr; s.seg_contrast = nullptr;     // the caller's, when it expands states with extra light
    return s;
}

// The state-dependent tables at level time `tics` with `floor_off` / `ceil_off` (nullptr, or one offset per sector, map
// units: the state of the moving sectors, DESIGN.md C16).  Outputs hold H_NTEX / H_NSECTORS / H_NSEGS / H_NSPRITES records,
// `mids_out` (nullable) H_NMIDS.  `layout`: state_layout(blob) if the caller keeps it (a renderer does), else derived here.
inline void scene_at_time(const uint8_t *blob, uint32_t tics, TexRec *tex_out, SectorRec *sectors_out, SegRec *segs_out,
                          SpriteRec *sprites_out, MidRec *mids_out = nullptr, const int32_t *floor_off = nullptr,
                          const int32_t *ceil_off = nullptr, const StateLayout *layout = nullptr) {
    StateLayout own;
    if (!layout) {
        own = state_layout(blob);
        layout = &own;
    }
    const StateLayout &L = *layout;
    const StateSrc s = state_src(blob, L);
    std::vector<uint32_t> words(L.words);
    compact_state(blob, L, tics, floor_off, ceil_off, words.data());
    const StateIn st = state_in(words.data(), s.ndyn);
    for (uint32_t i = 0; i < s.ntex; i++) tex_out[i] = tex_at(s, st, i);
    for (uint32_t i = 0; i < s.nsectors; i++) sectors_out[i] = sector_at(s, st, i);
    for (uint32_t i = 0; i < s.nsegs; i++) segs_out[i] = seg_at(s, st, i);
    for (uint32_t i = 0; i < s.nsprites; i++) sprites_out[i] = sprite_at(s, st, i);
    if (mids_out)
        for (uint32_t i = 0; i < s.nmids; i++) mids_out[i] = mid_at(s, st, i);
}

// Checks a list of sector moves against the scene's declared dynamic sectors and expands it to one floor and one ceiling
// offset per sector.  Returns nullptr, or the reason the list is rejected.
inline const char *expand_moves(const uint8_t *blob, const SectorMove *moves, size_t n, std::vector<int32_t> &floor_off,
                                std::vector<int32_t> &ceil_off) {
    const uint32_t *h = reinterpret_cast<const uint32_t *>(blob);
    const SectorRec *sectors = reinterpret_cast<const SectorRec *>(blob + h[H_OFF_SECTORS]);
    const DynRec *dyn = reinterpret_cast<const DynRec *>(blob + h[H_OFF_DYN]);
    floor_off.assign(h[H_NSECTORS], 0);
    ceil_off.assign(h[H_NSECTORS], 0);
    for (size_t k = 0; k < n; k++) {
        const DynRec *d = nullptr;
        for (uint32_t i = 0; i < h[H_NDYN]; i++)
            if (dyn[i].sector == moves[k].sector) { d = &dyn[i]; break; }
        if (!d) return "a moved sector was not declared dynamic when the scene was created";
        const int64_t f1 = (int64_t)sectors[d->sector].floor + moves[k].floor_offset;
        const int64_t c1 = (int64_t)sectors[d->sector].ceil + moves[k].ceil_offset;
        if (f1 < d->floor_min || f1 > d->floor_max || c1 < d->ceil_min || c1 > d->ceil_max || f1 > c1)
            return "a sector is moved outside its declared height range";
        floor_off[(size_t)d->sector] = moves[k].floor_offset;
        ceil_off[(size_t)d->sector] = moves[k].ceil_offset;
    }
    return nullptr;
}

// A PLAYPAL entry (R, G, B bytes) as the RGBA8 word the kernels read: R in the low byte, alpha 0xFF.
inline uint32_t palette_word(const uint8_t *c) {
    return (uint32_t)c[0] | ((uint32_t)c[1] << 8) | ((uint32_t)c[2] << 16) | 0xFF000000u;
}

std::vector<uint8_t> compile_scene(const Archive &wad, const TextureDirectory &tex, int level_index,
                                   const std::vector<DynRec> &dynamic = {});
std::vector<uint8_t> compile_scene(const Level &level, const TextureDirectory &tex, const std::vector<DynRec> &dynamic = {});

// LevelWalker::sector_at on the raw level (visitor.rs:1028-1060); -1 if outside.
int sector_at(const Level &level, double x, double y, int *subsector_out = nullptr);

// (light >> 3)/31 (+-2/31, clamped) * 255 truncated to u8, in the reference's float32 arithmetic.
uint8_t light_byte(int16_t light, int contrast);

// The level's automap table (DESIGN.md C19): a record per linedef whose vertices exist, in LINEDEFS order, coloured by
// Doom's AM_drawWalls rule at the level's rest heights with every line counted as mapped.
std::vector<AutomapLine> automap_lines(const Level &level);

}  // namespace b2d
