// `b2d` -- command line front end on the C ABI (include/b2d.h), mirroring rs_doom's flags
// (reference src/main.rs:17-80): -i/--iwad, -l/--level, -r/--resolution WxH, -f/--fov, and the sub-commands
// `list-levels` (main.rs:116-121) and `check` (main.rs:99-115).  Rendering options are ours: --poses N turns the
// camera N steps around the spawn point, --tics T sets the level time, --dump FILE writes the first frame and
// --stream FILE all frames as binary PPM.  This is the compiled-code host side of the boundary: it links
// libb2d.so and uses nothing but the header; every frame comes from the CUDA kernels (no CPU path).
// Multi-GPU (one process per GPU): --rank R --world N --id-file PATH --chunk C renders the pose list through
// b2d_render_sharded -- rank 0 writes the NCCL unique id to PATH, the others read it -- with the frame all-gather on, and
// prints one checksum line per rank over all gathered frames (every rank must print the same value).
// Level sets: --levels LIST (comma-separated level indices, or `all`) renders the look-around from every listed level's
// start, --poses per level, pose i at tic T + i (--tics T), through one b2d_renderer_create_levels renderer:
// b2d_render_levels_states in one process (--dump NAME writes NAME.L.ppm, the first frame of level L), and
// b2d_render_sharded_levels_states with --world.
// --supersample K (1..8) renders at K times the resolution with the same field of view and resolves every frame to
// --resolution RGB on the device (b2d_resolve_device, each frame through its own level's palette) for --dump and --stream;
// not with --world.  --palette P colours those frames through PLAYPAL palette P instead of palette 0
// (b2d_resolve_palettes_device; 1..8 Doom's damage flash, 9..12 the bonus flash, 13 the radiation suit), through the
// resolve at the --supersample factor (1 by default); not with --world.  --fixed-colormap R (-1..32) and --extralight E (0..2)
// light every frame of --levels as a player with those effects (b2d_*_levels_states_lights, DESIGN.md C18: 32 Doom's
// invulnerability, 1 its light-amplification visor, E its weapon flashes); not with --world.
// --automap SCALE (pixels per map unit, 0.2 is Doom's default) with --dump NAME.ppm also writes NAME.automap.ppm (with
// --levels NAME.automap.L.ppm): Doom's automap of the dumped pose (b2d_automap_device, DESIGN.md C19) through palette 0 of
// its level, resolved at the --supersample factor; --automap-flags rotate,all,things turns the map with the view, draws
// every line and draws the decoration things; seen draws only the lines the run's frames of that level saw (b2d_raster_device_seen,
// DESIGN.md C20), allmap adds the unseen ones in grey (the computer area map), others draws the arrows of the run's first
// four poses of that level in Doom's co-op colours 112, 96, 64, 176 (b2d_automap_states_device, C21), grid draws Doom's
// grid at the level's BLOCKMAP origin under the map (b2d_automap_marks_device, C22).  Not with --world.
#include <cmath>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <unistd.h>

#include "../../include/b2d.h"

namespace {

// "all" or comma-separated level indices into `out`; false on anything else
bool parse_levels(const std::string &text, int nlevels, std::vector<int> &out) {
    out.clear();
    if (text == "all") {
        for (int i = 0; i < nlevels; i++) out.push_back(i);
        return nlevels > 0;
    }
    size_t at = 0;
    while (at <= text.size()) {
        const size_t comma = std::min(text.find(',', at), text.size());
        const std::string item = text.substr(at, comma - at);
        char *end = nullptr;
        const long v = std::strtol(item.c_str(), &end, 10);
        if (item.empty() || *end || v < 0 || v >= nlevels) return false;
        out.push_back((int)v);
        at = comma + 1;
    }
    return !out.empty();
}

int fail(const char *what) {
    std::fprintf(stderr, "Fatal error: %s: %s\n", what, b2d_last_error());
    return 1;
}

void write_ppm(std::FILE *f, const uint32_t *rgba, int w, int h) {
    std::fprintf(f, "P6\n%d %d\n255\n", w, h);
    std::vector<uint8_t> row((size_t)w * 3);
    for (int y = 0; y < h; y++) {
        for (int x = 0; x < w; x++) {
            const uint32_t p = rgba[(size_t)y * w + x];
            row[3 * x] = (uint8_t)p; row[3 * x + 1] = (uint8_t)(p >> 8); row[3 * x + 2] = (uint8_t)(p >> 16);
        }
        std::fwrite(row.data(), 1, row.size(), f);
    }
}

void write_ppm_rgb(std::FILE *f, const uint8_t *rgb, int w, int h) {
    std::fprintf(f, "P6\n%d %d\n255\n", w, h);
    std::fwrite(rgb, 1, (size_t)w * h * 3, f);
}

// --supersample / --palette: render the n poses (levels: per-frame levels and states, else the renderer's own state) into
// device index frames at the renderer's view, resolve them by `factor` to RGB8 through palette `palette` of each frame's
// level and download them into `rgb` (n x (W/factor) x (H/factor) x 3)
int render_supersampled(b2d_renderer *r, int device, const b2d_view &view, const std::vector<b2d_pose> &poses, size_t max_batch,
                        const uint32_t *levels, const b2d_frame_state *states, const b2d_frame_light *lights, int factor,
                        int palette, std::vector<uint8_t> &rgb) {
    const size_t n = poses.size(), npix = (size_t)view.width * view.height;
    size_t frame_bytes = 0;
    if (b2d_resolve_frame_bytes(r, factor, B2D_RESOLVE_RGB8, &frame_bytes) != B2D_OK) return fail("resolve");
    void *d_poses = nullptr, *d_index = nullptr, *d_rgb = nullptr;
    struct Bufs {
        int device;
        void **p[3];
        ~Bufs() { for (void **q : p) if (*q) b2d_device_free(device, *q); }
    } owner{device, {&d_poses, &d_index, &d_rgb}};
    if (b2d_device_alloc(device, sizeof(b2d_pose) * n, &d_poses) != B2D_OK || b2d_device_alloc(device, npix * n, &d_index) != B2D_OK ||
        b2d_device_alloc(device, frame_bytes * n, &d_rgb) != B2D_OK)
        return fail("device memory");
    if (b2d_device_upload(device, d_poses, poses.data(), sizeof(b2d_pose) * n) != B2D_OK) return fail("upload");
    const b2d_pose *dp = static_cast<const b2d_pose *>(d_poses);
    uint8_t *di = static_cast<uint8_t *>(d_index);
    if (levels) {
        if (b2d_render_device_levels_states_lights(r, dp, levels, states, lights, n, nullptr, 0, di, nullptr, nullptr) != B2D_OK)
            return fail("render");
    } else {
        for (size_t i = 0; i < n; i += max_batch)
            if (b2d_render_device(r, dp + i, std::min(max_batch, n - i), di + npix * i, nullptr, nullptr) != B2D_OK) return fail("render");
    }
    const std::vector<uint32_t> palettes(n, (uint32_t)palette);
    if (b2d_resolve_palettes_device(r, di, levels, palettes.data(), n, factor, B2D_RESOLVE_RGB8, d_rgb, nullptr) != B2D_OK)
        return fail("resolve");
    int32_t bits = 0;
    if (b2d_renderer_status(r, &bits) != B2D_OK) return fail("status");
    if (bits) { std::fprintf(stderr, "Fatal error: frames incomplete (status %d)\n", bits); return 1; }
    rgb.resize(frame_bytes * n);
    if (b2d_device_download(device, rgb.data(), d_rgb, rgb.size()) != B2D_OK) return fail("download");
    return 0;
}

// --automap: the automaps of `poses` (levels: each pose's level, nullptr: level 0) at the renderer's view, coloured through
// palette 0 of each frame's level and resolved by `factor` to RGB8 (b2d_automap_device, b2d_resolve_device), frame k written
// to names[k]
// With `seen` (n rows of b2d_renderer_seen_words words) or B2D_AUTOMAP_ALLMAP, frame k draws the lines row k has mapped
// (b2d_automap_seen_device).  With `ranges` (one per frame) into `arrows`, frame k also draws those arrows
// (b2d_automap_states_device).  B2D_AUTOMAP_GRID draws the grid under the map (b2d_automap_marks_device).
int write_automaps(b2d_renderer *r, int device, const b2d_view &view, const std::vector<b2d_pose> &poses, const uint32_t *levels,
                   int32_t scale_q16, int flags, int factor, const std::vector<std::string> &names,
                   const std::vector<uint32_t> *seen = nullptr, const std::vector<b2d_arrow_range> *ranges = nullptr,
                   const std::vector<b2d_automap_arrow> *arrows = nullptr) {
    const size_t n = poses.size(), npix = (size_t)view.width * view.height;
    size_t frame_bytes = 0;
    if (b2d_resolve_frame_bytes(r, factor, B2D_RESOLVE_RGB8, &frame_bytes) != B2D_OK) return fail("resolve");
    void *d_poses = nullptr, *d_index = nullptr, *d_rgb = nullptr, *d_seen = nullptr;
    struct Bufs {
        int device;
        void **p[4];
        ~Bufs() { for (void **q : p) if (*q) b2d_device_free(device, *q); }
    } owner{device, {&d_poses, &d_index, &d_rgb, &d_seen}};
    if (b2d_device_alloc(device, sizeof(b2d_pose) * n, &d_poses) != B2D_OK || b2d_device_alloc(device, npix * n, &d_index) != B2D_OK ||
        b2d_device_alloc(device, frame_bytes * n, &d_rgb) != B2D_OK)
        return fail("device memory");
    if (b2d_device_upload(device, d_poses, poses.data(), sizeof(b2d_pose) * n) != B2D_OK) return fail("upload");
    if (seen) {
        if (b2d_device_alloc(device, seen->size() * sizeof(uint32_t), &d_seen) != B2D_OK) return fail("device memory");
        if (b2d_device_upload(device, d_seen, seen->data(), seen->size() * sizeof(uint32_t)) != B2D_OK) return fail("upload");
    }
    uint8_t *di = static_cast<uint8_t *>(d_index);
    const b2d_pose *dp = static_cast<const b2d_pose *>(d_poses);
    const uint32_t *ds = static_cast<const uint32_t *>(d_seen);
    const int rc = (flags & B2D_AUTOMAP_GRID)
                       ? b2d_automap_marks_device(r, dp, levels, nullptr, nullptr, 0, ranges ? ranges->data() : nullptr,
                                                  ranges ? arrows->data() : nullptr, ranges ? arrows->size() : 0, ds, n, scale_q16,
                                                  flags, di, nullptr, nullptr, nullptr, 0)
                   : ranges ? b2d_automap_states_device(r, dp, levels, nullptr, nullptr, 0, ranges->data(), arrows->data(), arrows->size(),
                                                      ds, n, scale_q16, flags, di, nullptr)
                   : seen || (flags & B2D_AUTOMAP_ALLMAP) ? b2d_automap_seen_device(r, dp, levels, ds, n, scale_q16, flags, di, nullptr)
                                                          : b2d_automap_device(r, dp, levels, n, scale_q16, flags, di, nullptr);
    if (rc != B2D_OK) return fail("automap");
    if (b2d_resolve_device(r, di, levels, n, factor, B2D_RESOLVE_RGB8, d_rgb, nullptr) != B2D_OK) return fail("resolve");
    std::vector<uint8_t> rgb(frame_bytes * n);
    if (b2d_device_download(device, rgb.data(), d_rgb, rgb.size()) != B2D_OK) return fail("download");
    for (size_t k = 0; k < n; k++) {
        std::FILE *f = std::fopen(names[k].c_str(), "wb");
        if (!f) { std::perror(names[k].c_str()); return 1; }
        write_ppm_rgb(f, rgb.data() + frame_bytes * k, view.width / factor, view.height / factor);
        std::fclose(f);
    }
    return 0;
}

// --automap-flags seen: the lines the run's frames saw (b2d_walk_device / b2d_walk_device_levels, then
// b2d_raster_device_seen in batches of max_batch), OR-ed per level into rows[level * words ..] of n_levels rows
int run_seen_rows(b2d_renderer *r, int device, const b2d_view &view, const std::vector<b2d_pose> &poses, const uint32_t *levels,
                  size_t n_levels, int max_batch, std::vector<uint32_t> &rows) {
    uint32_t words = 0;
    if (b2d_renderer_seen_words(r, &words) != B2D_OK) return fail("seen words");
    const size_t n = poses.size(), npix = (size_t)view.width * view.height, mb = (size_t)max_batch;
    void *d_poses = nullptr, *d_index = nullptr, *d_seen = nullptr;
    struct Bufs {
        int device;
        void **p[3];
        ~Bufs() { for (void **q : p) if (*q) b2d_device_free(device, *q); }
    } owner{device, {&d_poses, &d_index, &d_seen}};
    if (b2d_device_alloc(device, sizeof(b2d_pose) * n, &d_poses) != B2D_OK || b2d_device_alloc(device, npix * mb, &d_index) != B2D_OK ||
        b2d_device_alloc(device, sizeof(uint32_t) * words * mb, &d_seen) != B2D_OK)
        return fail("device memory");
    if (b2d_device_upload(device, d_poses, poses.data(), sizeof(b2d_pose) * n) != B2D_OK) return fail("upload");
    rows.assign(n_levels * words, 0u);
    std::vector<uint32_t> batch(words * mb);
    for (size_t i = 0; i < n; i += mb) {
        const size_t k = std::min(mb, n - i);
        std::fill(batch.begin(), batch.end(), 0u);
        if (b2d_device_upload(device, d_seen, batch.data(), batch.size() * sizeof(uint32_t)) != B2D_OK) return fail("upload");
        const b2d_pose *dp = static_cast<const b2d_pose *>(d_poses) + i;
        int64_t ticket = -1;
        const int rc = levels ? b2d_walk_device_levels(r, dp, levels + i, k, nullptr, &ticket) : b2d_walk_device(r, dp, k, nullptr, &ticket);
        if (rc != B2D_OK) return fail("walk");
        if (b2d_raster_device_seen(r, ticket, static_cast<uint8_t *>(d_index), static_cast<uint32_t *>(d_seen), nullptr) != B2D_OK)
            return fail("seen raster");
        if (b2d_device_download(device, batch.data(), d_seen, sizeof(uint32_t) * words * k) != B2D_OK) return fail("download");
        for (size_t f = 0; f < k; f++)
            for (uint32_t w = 0; w < words; w++) rows[(levels ? levels[i + f] : 0u) * words + w] |= batch[f * words + w];
    }
    return 0;
}

// --automap-flags others: for automap frame k, on level frame_levels[k], the arrows of the first four of the run's poses
// (levels: each one's level, nullptr: level 0) on that level, in Doom's co-op colours: green, grey, brown, red
void team_arrows(const std::vector<b2d_pose> &poses, const uint32_t *levels, const std::vector<uint32_t> &frame_levels,
                 std::vector<b2d_arrow_range> &ranges, std::vector<b2d_automap_arrow> &arrows) {
    static const uint32_t colours[4] = {112, 96, 64, 176};
    for (uint32_t level : frame_levels) {
        b2d_arrow_range g{(uint32_t)arrows.size(), 0};
        for (size_t i = 0; i < poses.size() && g.n < 4; i++)
            if ((levels ? levels[i] : 0u) == level) arrows.push_back({poses[i].x, poses[i].y, poses[i].angle, colours[g.n++]});
        ranges.push_back(g);
    }
}

// --automap on one level: the automap of the run's first pose, with `seen` of the lines all its poses saw and, with
// `others`, its first four poses' arrows
int write_run_automap(b2d_renderer *r, const b2d_view &view, const std::vector<b2d_pose> &poses, int max_batch, int32_t scale_q16,
                      int flags, bool seen, bool others, int factor, const std::string &name) {
    std::vector<uint32_t> rows;
    if (seen)
        if (int rc = run_seen_rows(r, 0, view, poses, nullptr, 1, max_batch, rows)) return rc;
    std::vector<b2d_arrow_range> ranges;
    std::vector<b2d_automap_arrow> arrows;
    if (others) team_arrows(poses, nullptr, {0u}, ranges, arrows);
    return write_automaps(r, 0, view, {poses[0]}, nullptr, scale_q16, flags, factor, {name}, seen ? &rows : nullptr,
                          others ? &ranges : nullptr, &arrows);
}

// the --dump name without its .ppm extension
std::string dump_stem(const std::string &dump) {
    return dump.size() > 4 && dump.compare(dump.size() - 4, 4, ".ppm") == 0 ? dump.substr(0, dump.size() - 4) : dump;
}

// b2d_render_sharded consumer: per-frame checksums of every gathered chunk into a device table (the table lives in device memory
// obtained through b2d_device_alloc: the CLI itself links no CUDA library)
struct ShardSink {
    uint32_t *d_sums;      // world x per, device
    size_t per, npix;
};
void on_chunk(void *user, int, size_t first, size_t cnt, const uint8_t *d_frames, int ranks, void *stream) {
    ShardSink *s = static_cast<ShardSink *>(user);
    for (int q = 0; q < ranks; q++)
        b2d_frame_checksums_device(d_frames + (size_t)q * cnt * s->npix, cnt, s->npix, s->d_sums + (size_t)q * s->per + first, stream);
}

// the communicator of an --id-file job: rank 0 writes the NCCL unique id to the file, the others read it
int make_comm(const std::string &id_file, int rank, int world, b2d_comm **comm) {
    uint8_t id[B2D_COMM_ID_BYTES];
    if (id_file.empty()) { std::fprintf(stderr, "--id-file PATH is required with --world\n"); return 2; }
    if (rank == 0) {
        if (b2d_comm_unique_id(id) != B2D_OK) return fail("unique id");
        const std::string tmp = id_file + ".tmp";
        std::FILE *f = std::fopen(tmp.c_str(), "wb");
        if (!f || std::fwrite(id, 1, sizeof id, f) != sizeof id) { std::perror(tmp.c_str()); return 1; }
        std::fclose(f);
        std::rename(tmp.c_str(), id_file.c_str());
    } else {
        std::FILE *f = nullptr;
        for (int tries = 0; tries < 600 && !(f = std::fopen(id_file.c_str(), "rb")); tries++) usleep(100000);
        if (!f || std::fread(id, 1, sizeof id, f) != sizeof id) { std::fprintf(stderr, "cannot read %s\n", id_file.c_str()); return 1; }
        std::fclose(f);
    }
    if (b2d_comm_create(id, rank, world, rank, comm) != B2D_OK) return fail("communicator");
    return 0;
}

// after a sharded render: the renderer's status, then one checksum line over every gathered frame; frees the sink's table
int report_sharded(b2d_renderer *r, ShardSink &sink, const b2d_sharded_stats &st, int rank, int world) {
    int32_t bits = 0;
    if (b2d_renderer_status(r, &bits) != B2D_OK) return fail("status");
    if (bits) { std::fprintf(stderr, "Fatal error: frames incomplete (status %d)\n", bits); return 1; }
    std::vector<uint32_t> sums(sink.per * (size_t)world);
    if (b2d_device_download(rank, sums.data(), sink.d_sums, sums.size() * sizeof(uint32_t)) != B2D_OK) return fail("download");
    uint32_t all = 0;
    for (size_t i = 0; i < sums.size(); i++) all = all * 31u + sums[i];
    std::printf("rank %d/%d: %lld frames gathered in %lld chunk(s), %.3f ms, checksum %08x, buffers %s\n", rank, world,
                (long long)st.frames_gathered, (long long)st.chunks, st.total_ms, all, st.registration);
    b2d_device_free(rank, sink.d_sums);
    return 0;
}

// --levels: the look-around of every level of `set` from its start, nposes per level, pose i at tic tics + i
int render_level_set(b2d_archive *arch, const std::vector<int> &set, int width, int height, double fov, int nposes, uint32_t tics,
                     const std::string &dump, const std::string &stream, int world, int rank, int chunk, const std::string &id_file,
                     int supersample, int palette, b2d_frame_light light, int32_t automap_scale, int automap_flags,
                     bool automap_seen, bool automap_others) {
    std::vector<b2d_scene *> scenes;
    struct Scenes {
        std::vector<b2d_scene *> &v;
        ~Scenes() { for (b2d_scene *s : v) b2d_scene_destroy(s); }
    } owner{scenes};
    const size_t per_level = (size_t)nposes, n = per_level * set.size();
    std::vector<b2d_pose> poses(n);
    std::vector<uint32_t> levels(n);
    std::vector<b2d_frame_state> states(n);
    for (size_t k = 0; k < set.size(); k++) {
        b2d_scene *sc = nullptr;
        if (b2d_scene_create(arch, set[k], &sc) != B2D_OK) return fail("level");
        scenes.push_back(sc);
        b2d_scene_info info;
        b2d_scene_info_get(sc, &info);
        if (!info.has_start) { std::fprintf(stderr, "Fatal error: level %d has no player-1 start\n", set[k]); return 1; }
        if (palette >= b2d_scene_num_palettes(sc)) {
            std::fprintf(stderr, "--palette takes a palette index below %d\n", b2d_scene_num_palettes(sc));
            return 2;
        }
        for (size_t i = 0; i < per_level; i++) {        // look around from the spawn point
            b2d_pose &p = poses[k * per_level + i];
            p = info.start;
            p.angle = info.start.angle + (uint32_t)(((uint64_t)i << 32) / (uint64_t)per_level);
            levels[k * per_level + i] = (uint32_t)k;
        }
    }
    for (size_t i = 0; i < n; i++) states[i] = b2d_frame_state{tics + (uint32_t)i, 0, 0};
    const std::vector<b2d_frame_light> light_v(n, light);
    const b2d_frame_light *lights = light.fixed_colormap != -1 || light.extralight != 0 ? light_v.data() : nullptr;
    b2d_view view;
    if (b2d_view_init(&view, width * supersample, height * supersample, fov) != B2D_OK) return fail("view");
    b2d_renderer *r = nullptr;
    if (b2d_renderer_create_levels(scenes.data(), scenes.size(), &view, world > 0 ? rank : 0, n < 64 ? (int)n : 64, &r) != B2D_OK)
        return fail("renderer");
    struct Renderer {
        b2d_renderer *r;
        ~Renderer() { b2d_renderer_destroy(r); }
    } rown{r};
    const size_t npix = (size_t)width * height;
    if (world > 0) {
        b2d_comm *comm = nullptr;
        if (int rc = make_comm(id_file, rank, world, &comm)) return rc;
        const size_t per = (n + (size_t)world - 1) / (size_t)world;
        ShardSink sink{nullptr, per, npix};
        if (b2d_device_alloc(rank, sizeof(uint32_t) * per * (size_t)world, reinterpret_cast<void **>(&sink.d_sums)) != B2D_OK) return fail("device memory");
        b2d_sharded_stats st;
        if (b2d_render_sharded_levels_states(r, comm, poses.data(), levels.data(), states.data(), n, nullptr, 0, (size_t)chunk,
                                             B2D_SHARD_RENDER_GATHER, on_chunk, &sink, &st) != B2D_OK)
            return fail("sharded render");
        const int rc = report_sharded(r, sink, st, rank, world);
        b2d_comm_destroy(comm);
        return rc;
    }
    std::vector<uint8_t> index, rgb;
    std::vector<uint32_t> rgba;
    const bool resolved = supersample > 1 || palette > 0;
    if (resolved) {
        if (int rc = render_supersampled(r, 0, view, poses, n < 64 ? n : 64, levels.data(), states.data(), lights, supersample, palette, rgb))
            return rc;
        std::printf("rendered %zu frame(s) %dx%d of %zu level(s), supersampled %dx, palette %d\n", n, width, height, set.size(),
                    supersample, palette);
    } else {
        index.resize(npix * n);
        rgba.resize(npix * n);
        if (b2d_render_levels_states_lights(r, poses.data(), levels.data(), states.data(), lights, n, nullptr, 0, index.data(),
                                            rgba.data()) != B2D_OK)
            return fail("render");
        std::printf("rendered %zu frame(s) %dx%d of %zu level(s)\n", n, width, height, set.size());
    }
    auto write_frame = [&](std::FILE *f, size_t i) {
        if (resolved) write_ppm_rgb(f, rgb.data() + npix * 3 * i, width, height);
        else write_ppm(f, rgba.data() + npix * i, width, height);
    };
    if (!dump.empty()) {
        const std::string stem = dump_stem(dump);
        for (size_t k = 0; k < set.size(); k++) {
            const std::string name = stem + "." + std::to_string(set[k]) + ".ppm";
            std::FILE *f = std::fopen(name.c_str(), "wb");
            if (!f) { std::perror(name.c_str()); return 1; }
            write_frame(f, k * per_level);
            std::fclose(f);
        }
        if (automap_scale) {
            std::vector<b2d_pose> firsts;
            std::vector<uint32_t> first_levels;
            std::vector<std::string> names;
            for (size_t k = 0; k < set.size(); k++) {
                firsts.push_back(poses[k * per_level]);
                first_levels.push_back((uint32_t)k);
                names.push_back(stem + ".automap." + std::to_string(set[k]) + ".ppm");
            }
            std::vector<uint32_t> seen;
            if (automap_seen) {
                if (int rc = run_seen_rows(r, 0, view, poses, levels.data(), set.size(), n < 64 ? (int)n : 64, seen)) return rc;
            }
            std::vector<b2d_arrow_range> ranges;
            std::vector<b2d_automap_arrow> arrows;
            if (automap_others) team_arrows(poses, levels.data(), first_levels, ranges, arrows);
            if (int rc = write_automaps(r, 0, view, firsts, first_levels.data(), automap_scale, automap_flags, supersample, names,
                                        automap_seen ? &seen : nullptr, automap_others ? &ranges : nullptr, &arrows))
                return rc;
        }
    }
    if (!stream.empty()) {
        std::FILE *f = std::fopen(stream.c_str(), "wb");
        if (!f) { std::perror(stream.c_str()); return 1; }
        for (size_t i = 0; i < n; i++) write_frame(f, i);
        std::fclose(f);
    }
    return 0;
}

}  // namespace

int main(int argc, char **argv) {
    std::string iwad, dump, stream, command, id_file, levels_arg;
    int level = 0, width = 1280, height = 720, nposes = 1, rank = 0, world = 0, chunk = 16, supersample = 1, palette = 0;
    int32_t automap_scale = 0;        // 0: no --automap
    int automap_flags = 0;
    bool automap_seen = false;        // --automap-flags seen: the automap shows the lines the run's frames saw
    bool automap_others = false;      // --automap-flags others: ... and the run's first four poses as players' arrows
    b2d_frame_light light{-1, 0};
    double fov = 65.0;
    unsigned long tics = 0;
    bool with_levels = false;
    for (int i = 1; i < argc; i++) {
        const std::string a = argv[i];
        auto next = [&](const char *name) -> const char * {
            if (i + 1 >= argc) { std::fprintf(stderr, "missing value for %s\n", name); std::exit(2); }
            return argv[++i];
        };
        if (a == "-i" || a == "--iwad") iwad = next("--iwad");
        else if (a == "-m" || a == "--metadata") next("--metadata");           // accepted; the sky table is built in
        else if (a == "-l" || a == "--level") level = std::atoi(next("--level"));
        else if (a == "--levels") { levels_arg = next("--levels"); with_levels = true; }
        else if (a == "-f" || a == "--fov") fov = std::atof(next("--fov"));
        else if (a == "-r" || a == "--resolution") {
            if (std::sscanf(next("--resolution"), "%dx%d", &width, &height) != 2) {
                std::fprintf(stderr, "resolution format is WIDTHxHEIGHT\n");
                return 2;
            }
        } else if (a == "--poses") nposes = std::atoi(next("--poses"));
        else if (a == "--tics") tics = std::strtoul(next("--tics"), nullptr, 10);
        else if (a == "--dump") dump = next("--dump");
        else if (a == "--stream") stream = next("--stream");
        else if (a == "--rank") rank = std::atoi(next("--rank"));
        else if (a == "--world") world = std::atoi(next("--world"));
        else if (a == "--chunk") chunk = std::atoi(next("--chunk"));
        else if (a == "--id-file") id_file = next("--id-file");
        else if (a == "--supersample") supersample = std::atoi(next("--supersample"));
        else if (a == "--palette") {
            const char *v = next("--palette");
            char *end = nullptr;
            const long p = std::strtol(v, &end, 10);
            if (!*v || *end || p < 0 || p > 0x7FFFFFFF) { std::fprintf(stderr, "--palette takes a palette index\n"); return 2; }
            palette = (int)p;
        }
        else if (a == "--fixed-colormap" || a == "--extralight") {
            const char *v = next(a.c_str());
            char *end = nullptr;
            const long x = std::strtol(v, &end, 10);
            const bool fixed = a == "--fixed-colormap";
            if (!*v || *end || (fixed ? x < -1 || x > 32 : x < 0 || x > 2)) {
                std::fprintf(stderr, fixed ? "--fixed-colormap takes a row in -1..32\n" : "--extralight takes a value in 0..2\n");
                return 2;
            }
            if (fixed) light.fixed_colormap = (int32_t)x;
            else light.extralight = (uint32_t)x;
        }
        else if (a == "--automap") {
            const char *v = next("--automap");
            char *end = nullptr;
            const double x = std::strtod(v, &end);
            if (!*v || *end || !(x >= 1.0 / 256 && x <= 64)) {
                std::fprintf(stderr, "--automap takes a scale in pixels per map unit, 1/256 .. 64\n");
                return 2;
            }
            automap_scale = (int32_t)std::lround(x * 65536);
        } else if (a == "--automap-flags") {
            std::string v = next("--automap-flags");
            size_t at = 0;
            while (at <= v.size()) {
                const size_t comma = std::min(v.find(',', at), v.size());
                const std::string name = v.substr(at, comma - at);
                if (name == "rotate") automap_flags |= B2D_AUTOMAP_ROTATE;
                else if (name == "all") automap_flags |= B2D_AUTOMAP_ALL_LINES;
                else if (name == "things") automap_flags |= B2D_AUTOMAP_THINGS;
                else if (name == "allmap") automap_flags |= B2D_AUTOMAP_ALLMAP;
                else if (name == "seen") automap_seen = true;
                else if (name == "others") automap_others = true;
                else if (name == "grid") automap_flags |= B2D_AUTOMAP_GRID;
                else if (!name.empty()) { std::fprintf(stderr, "--automap-flags takes rotate, all, things, allmap, seen, others, grid\n"); return 2; }
                at = comma + 1;
            }
        }
        else if (a == "list-levels" || a == "check") command = a;
        else { std::fprintf(stderr, "unknown argument %s\n", a.c_str()); return 2; }
    }
    if (iwad.empty()) { std::fprintf(stderr, "--iwad FILE is required\n"); return 2; }
    if (nposes < 1) nposes = 1;
    if (supersample < 1 || supersample > 8) { std::fprintf(stderr, "--supersample takes a factor in 1..8\n"); return 2; }
    if (supersample > 1 && world > 0) { std::fprintf(stderr, "--supersample does not combine with --world\n"); return 2; }
    if (palette > 0 && world > 0) { std::fprintf(stderr, "--palette does not combine with --world\n"); return 2; }
    const bool lit = light.fixed_colormap != -1 || light.extralight != 0;
    if (lit && world > 0) { std::fprintf(stderr, "--fixed-colormap and --extralight do not combine with --world\n"); return 2; }
    if (lit && !with_levels) { std::fprintf(stderr, "--fixed-colormap and --extralight take --levels\n"); return 2; }
    if (automap_scale && (dump.empty() || world > 0)) { std::fprintf(stderr, "--automap takes --dump and does not combine with --world\n"); return 2; }

    b2d_archive *arch = nullptr;
    if (b2d_archive_open(iwad.c_str(), &arch) != B2D_OK) return fail("open");
    const int nlevels = b2d_archive_num_levels(arch);
    if (command == "list-levels") {
        for (int i = 0; i < nlevels; i++) {
            char name[9] = {0};
            b2d_archive_level_name(arch, i, name);
            std::printf("%3d %8s\n", i, name);
        }
        b2d_archive_close(arch);
        return 0;
    }
    if (command == "check") {
        for (int i = 0; i < nlevels; i++) {
            char name[9] = {0};
            b2d_archive_level_name(arch, i, name);
            b2d_scene *sc = nullptr;
            if (b2d_scene_create(arch, i, &sc) != B2D_OK) { b2d_archive_close(arch); return fail(name); }
            b2d_scene_info info;
            b2d_scene_info_get(sc, &info);
            std::printf("Level %d (%s): %d segs, %d subsectors, %d sectors, %d textures: ok\n", i, name, info.n_segs,
                        info.n_ssectors, info.n_sectors, info.n_textures);
            b2d_scene_destroy(sc);
        }
        b2d_archive_close(arch);
        return 0;
    }

    if (with_levels) {
        std::vector<int> set;
        if (!parse_levels(levels_arg, nlevels, set)) {
            std::fprintf(stderr, "--levels takes `all` or comma-separated level indices below %d\n", nlevels);
            return 2;
        }
        const int rc = render_level_set(arch, set, width, height, fov, nposes, (uint32_t)tics, dump, stream, world, rank, chunk, id_file,
                                        supersample, palette, light, automap_scale, automap_flags, automap_seen,
                                        automap_others);
        b2d_archive_close(arch);
        return rc;
    }
    b2d_scene *sc = nullptr;
    if (b2d_scene_create(arch, level, &sc) != B2D_OK) { b2d_archive_close(arch); return fail("level"); }
    b2d_scene_info info;
    b2d_scene_info_get(sc, &info);
    if (!info.has_start) { std::fprintf(stderr, "Fatal error: the level has no player-1 start\n"); return 1; }
    if (palette >= b2d_scene_num_palettes(sc)) {
        std::fprintf(stderr, "--palette takes a palette index below %d\n", b2d_scene_num_palettes(sc));
        return 2;
    }
    b2d_view view;
    if (b2d_view_init(&view, width * supersample, height * supersample, fov) != B2D_OK) return fail("view");
    b2d_renderer *r = nullptr;
    if (b2d_renderer_create(sc, &view, world > 0 ? rank : 0, nposes < 64 ? nposes : 64, &r) != B2D_OK) return fail("renderer");
    if (b2d_renderer_set_time(r, (uint32_t)tics) != B2D_OK) return fail("time");

    std::vector<b2d_pose> poses((size_t)nposes, info.start);
    for (int i = 0; i < nposes; i++)          // look around from the spawn point
        poses[(size_t)i].angle = info.start.angle + (uint32_t)(((uint64_t)i << 32) / (uint64_t)nposes);
    const size_t npix = (size_t)width * height;
    if (supersample > 1 || palette > 0) {
        std::vector<uint8_t> rgb;
        if (int rc = render_supersampled(r, 0, view, poses, nposes < 64 ? nposes : 64, nullptr, nullptr, nullptr, supersample, palette, rgb))
            return rc;
        std::printf("rendered %d frame(s) %dx%d, supersampled %dx, palette %d\n", nposes, width, height, supersample, palette);
        if (!dump.empty()) {
            std::FILE *f = std::fopen(dump.c_str(), "wb");
            if (!f) { std::perror(dump.c_str()); return 1; }
            write_ppm_rgb(f, rgb.data(), width, height);
            std::fclose(f);
        }
        if (automap_scale && !dump.empty())
            if (int rc = write_run_automap(r, view, poses, nposes < 64 ? nposes : 64, automap_scale, automap_flags, automap_seen,
                                           automap_others, supersample, dump_stem(dump) + ".automap.ppm"))
                return rc;
        if (!stream.empty()) {
            std::FILE *f = std::fopen(stream.c_str(), "wb");
            if (!f) { std::perror(stream.c_str()); return 1; }
            for (int i = 0; i < nposes; i++) write_ppm_rgb(f, rgb.data() + npix * 3 * (size_t)i, width, height);
            std::fclose(f);
        }
        b2d_renderer_destroy(r);
        b2d_scene_destroy(sc);
        b2d_archive_close(arch);
        return 0;
    }
    if (world > 0) {
        // ---- sharded: every rank runs this with the same pose list
        b2d_comm *comm = nullptr;
        if (int rc = make_comm(id_file, rank, world, &comm)) return rc;
        const size_t per = ((size_t)nposes + (size_t)world - 1) / (size_t)world;
        ShardSink sink{nullptr, per, npix};
        if (b2d_device_alloc(rank, sizeof(uint32_t) * per * (size_t)world, reinterpret_cast<void **>(&sink.d_sums)) != B2D_OK) return fail("device memory");
        b2d_sharded_stats st;
        if (b2d_render_sharded(r, comm, poses.data(), (size_t)nposes, (size_t)chunk, B2D_SHARD_RENDER_GATHER, on_chunk, &sink, &st) != B2D_OK)
            return fail("sharded render");
        if (int rc = report_sharded(r, sink, st, rank, world)) return rc;
        b2d_comm_destroy(comm);
        b2d_renderer_destroy(r);
        b2d_scene_destroy(sc);
        b2d_archive_close(arch);
        return 0;
    }
    std::vector<uint8_t> index(npix * (size_t)nposes);
    std::vector<uint32_t> rgba(npix * (size_t)nposes);
    if (b2d_render(r, poses.data(), (size_t)nposes, index.data(), rgba.data()) != B2D_OK) return fail("render");
    std::printf("rendered %d frame(s) %dx%d\n", nposes, width, height);
    if (!dump.empty()) {
        std::FILE *f = std::fopen(dump.c_str(), "wb");
        if (!f) { std::perror(dump.c_str()); return 1; }
        write_ppm(f, rgba.data(), width, height);
        std::fclose(f);
    }
    if (automap_scale && !dump.empty())
        if (int rc = write_run_automap(r, view, poses, nposes < 64 ? nposes : 64, automap_scale, automap_flags, automap_seen,
                                       automap_others, 1, dump_stem(dump) + ".automap.ppm"))
            return rc;
    if (!stream.empty()) {
        std::FILE *f = std::fopen(stream.c_str(), "wb");
        if (!f) { std::perror(stream.c_str()); return 1; }
        for (int i = 0; i < nposes; i++) write_ppm(f, rgba.data() + npix * (size_t)i, width, height);
        std::fclose(f);
    }
    b2d_renderer_destroy(r);
    b2d_scene_destroy(sc);
    b2d_archive_close(arch);
    return 0;
}
