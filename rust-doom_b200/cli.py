"""`b2d` command line, mirroring rs_doom's flags (reference src/main.rs:17-80,89-124):

    python -m rust_doom_b200.cli --iwad doom1.wad --level 0 --resolution 1920x1080 [--fov 65]
                                 [--poses N] [--dump frame.ppm] [--device 0] [--supersample K] [--palette P]
    python -m rust_doom_b200.cli --iwad doom1.wad --levels 0,2,5 --poses N [--tics T] [--dump f.ppm] [--stream s.ppm]
                                 [--world W --rank R --id-file PATH [--chunk C]]
    python -m rust_doom_b200.cli --iwad doom1.wad list-levels
    python -m rust_doom_b200.cli --iwad doom1.wad check

`list-levels` prints "<index> <name>" per level (main.rs:116-121); `check` loads and compiles every level
(the reference's smoke test, main.rs:99-115 / game/src/game.rs:118-129) without needing a GPU.  Without
--iwad a synthetic IWAD is generated (no WAD ships with either project).  Unlike the reference, --fov is
honoured (its value is parsed but never read there: main.rs:131 vs game/src/game.rs:72).

--levels renders a level set through one renderer, as the compiled CLI does: the look-around from each listed level's
start, --poses per level, pose i at tic T + i.  --dump NAME.EXT writes NAME.L.EXT, the first frame of level L.  With
--world the poses are sharded over one process per GPU (b2d_render_sharded_levels_states; rank 0 writes the NCCL unique id
to --id-file, the others read it) and rank 0 colours every gathered frame with its own level's palette on the device
(b2d_palette_lut_levels_device) before it writes the --stream.

--supersample K (1..8) renders every frame at K times the resolution with the same field of view and resolves each K x K
block to one pixel of the --resolution frame on the device (b2d_resolve_device, C17: the half-up rounded mean of the
block's palette colours, each frame through its own level's palette): an anti-aliased --dump and --stream.  Not with
--world.

--automap SCALE with --dump NAME.EXT also writes NAME.automap.EXT (NAME.automap.L.EXT per level with --levels): Doom's
automap of the dumped pose at SCALE pixels per map unit (0.2 is Doom's default; b2d_automap_device, DESIGN.md C19),
coloured through palette 0 of its level and resolved at the --supersample factor; --automap-flags rotate,all,things turns
the map with the view, draws every line (IDDT) and draws the decoration things; seen draws only the lines the run's
frames of that level saw (Renderer.render_seen, DESIGN.md C20) and allmap adds the unseen ones in grey (the computer
area map); others draws the arrows of the run's first four poses of that level in Doom's co-op colours, the dumped pose's
own in green 112 and the next three in 96, 64 and 176 (b2d_automap_states_device, DESIGN.md C21); grid draws Doom's
grid at the level's BLOCKMAP origin under the map (b2d_automap_marks_device, DESIGN.md C22).  Not with --world.

--palette P colours the dumped and streamed frames through PLAYPAL palette P of each frame's level instead of palette 0
(b2d_resolve_palettes_device; in Doom 1..8 are the damage flash, 9..12 the bonus flash, 13 the radiation suit), through
the resolve at the --supersample factor (1 by default).  With --levels too; not with --world.

--fixed-colormap R and --extralight E light every frame of --levels as a player with those effects (DESIGN.md C18,
b2d_render_levels_states_lights): R = 32 is Doom's invulnerability (INVERSECOLORMAP), 1 its light-amplification visor;
E = 1 or 2 its weapon flashes.  Not with --world."""
from __future__ import annotations

import argparse
import os
import sys
import time

import numpy as np


def encode_ppm(rgb: np.ndarray) -> bytes:
    """Binary PPM (P6) of an (H, W, 3) uint8 image."""
    h, w, _ = rgb.shape
    return b"P6\n%d %d\n255\n" % (w, h) + np.ascontiguousarray(rgb).tobytes()


def encode_png(rgb: np.ndarray) -> bytes:
    """Minimal PNG (8-bit RGB, one IDAT, filter 0) of an (H, W, 3) uint8 image."""
    import struct
    import zlib
    h, w, _ = rgb.shape
    raw = np.zeros((h, 1 + 3 * w), dtype=np.uint8)
    raw[:, 1:] = np.ascontiguousarray(rgb).reshape(h, 3 * w)

    def chunk(tag: bytes, data: bytes) -> bytes:
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))
            + chunk(b"IDAT", zlib.compress(raw.tobytes(), 6)) + chunk(b"IEND", b""))


def rgba_to_rgb(rgba_frame: np.ndarray) -> np.ndarray:
    """(H, W) uint32 R | G<<8 | B<<16 | A<<24 (the library's RGBA8) -> (H, W, 3) uint8."""
    h, w = rgba_frame.shape
    return rgba_frame.view(np.uint8).reshape(h, w, 4)[:, :, :3]


def _main_sharded(b2d, scene, view, poses, args, w, h, world) -> int:
    """Under torchrun: every rank renders its contiguous block of the poses on its own GPU (no data-path
    collective); with --stream the finished index frames travel to rank 0 in pose order (parallel.
    write_frames_in_order), which applies the palette and writes the PPM stream."""
    import torch
    import torch.distributed as dist
    from rust_doom_b200 import parallel

    rank, local_rank = int(os.environ["RANK"]), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    try:
        s, e, per = parallel.shard_bounds(len(poses), rank, world)
        mine = poses[s:e]
        r = b2d.Renderer(scene, view, device=local_rank, max_batch=max(1, min(per, 256)))
        local = torch.empty((len(mine), h, w), dtype=torch.uint8, device="cuda")
        t0 = time.perf_counter()
        for c0 in range(0, len(mine), r.max_batch):
            c1 = min(len(mine), c0 + r.max_batch)
            dp = torch.from_numpy(mine[c0:c1].view(np.int32).reshape(-1, 4).copy()).cuda()
            r.render_device(dp.data_ptr(), c1 - c0, local[c0:c1].data_ptr())
        torch.cuda.synchronize()
        dist.barrier()
        if rank == 0:
            dt = time.perf_counter() - t0
            print("rendered %d frame(s) %dx%d on %d GPUs in %.2f ms" % (len(poses), w, h, world, dt * 1e3))
        if args.stream or args.dump:
            pal = scene.palette_rgb()
            out = open(args.stream, "wb") if (args.stream and rank == 0) else None

            def sink(frames, first):
                if out is not None:
                    for f in frames:
                        out.write(encode_ppm(pal[f]))
                if args.dump and first == 0:
                    with open(args.dump, "wb") as fh:
                        fh.write(encode_png(pal[frames[0]]) if args.dump.lower().endswith(".png") else encode_ppm(pal[frames[0]]))

            parallel.write_frames_in_order(local, len(poses), sink, chunk_frames=32)
            if out is not None:
                out.close()
        return 0
    finally:
        dist.destroy_process_group()


def parse_levels(text: str, n_levels: int):
    """--levels: `all` or comma-separated level indices below n_levels; ValueError otherwise"""
    if text == "all":
        return list(range(n_levels))
    out = [int(v) for v in text.split(",")]
    if not out or any(v < 0 or v >= n_levels for v in out):
        raise ValueError(text)
    return out


def level_set_job(b2d, scenes, per_level: int, tics: int):
    """(poses, levels, tics) of --levels: the look-around from each scene's start, per_level poses each, pose i at tics + i"""
    poses = np.concatenate([np.repeat(sc.start_pose, per_level) for sc in scenes])
    turn = (np.arange(per_level, dtype=np.uint64) << np.uint64(32)) // np.uint64(per_level)
    poses["angle"] = (poses["angle"].astype(np.uint64) + np.tile(turn, len(scenes))).astype(np.uint32)
    levels = np.repeat(np.arange(len(scenes), dtype=np.uint32), per_level)
    return poses, levels, (tics + np.arange(len(poses), dtype=np.int64)) & 0xFFFFFFFF


def _dump_name(dump: str, level: int) -> str:
    stem, ext = os.path.splitext(dump)
    return "%s.%d%s" % (stem, level, ext or ".ppm")


def _write_image(path: str, rgb: np.ndarray):
    with open(path, "wb") as f:
        f.write(encode_png(rgb) if path.lower().endswith(".png") else encode_ppm(rgb))


def _automap_name(dump: str, level=None) -> str:
    stem, ext = os.path.splitext(dump)
    return "%s.automap%s%s" % (stem, "" if level is None else ".%d" % level, ext or ".ppm")


# --automap-flags others: Doom's co-op player colours (green, grey, brown, red), the dumped pose's own first
OTHER_COLOURS = (112, 96, 64, 176)


def automap_flag_options(flags: str):
    """(the B2D_AUTOMAP_* names of --automap-flags, whether it names `seen`, whether it names `others`); unknown names
    raise ValueError"""
    names = [x.strip() for x in flags.split(",") if x.strip()]
    rest = ",".join(x for x in names if x not in ("seen", "others"))
    import rust_doom_b200 as b2d
    b2d.automap_flags(rest)
    return rest, "seen" in names, "others" in names


def automap_flag_names(flags: str):
    """(the B2D_AUTOMAP_* names of --automap-flags, whether it names `seen`); unknown names raise ValueError"""
    return automap_flag_options(flags)[:2]


def automap_rgb(r, poses: np.ndarray, levels, scale: float, flags: str, factor: int, run_poses=None, run_levels=None) -> np.ndarray:
    """(n, H, W, 3) uint8: the automaps of the poses (b2d_automap_device at the render size) through palette 0 of each
    frame's level, resolved by `factor` as the rendered frames are.  With `seen` in the flags, frame k draws the lines
    that the run's frames (run_poses, of levels run_levels) of its level saw (Renderer.render_seen, OR-ed per level).
    With `others`, frame k (the first of the run's poses of its level) also draws the arrows of the first four run poses
    of its level in OTHER_COLOURS, its own pose's in green (b2d_automap_states_device)."""
    import torch
    names, seen, others = automap_flag_options(flags)
    arrows = None
    if others:
        run_lv = np.zeros(len(run_poses), np.int64) if run_levels is None else np.asarray(run_levels)
        lv = np.zeros(len(poses), np.int64) if levels is None else np.asarray(levels)
        arrows = []
        for l in lv:
            mine = np.asarray(run_poses)[run_lv == l][:len(OTHER_COLOURS)]
            arrows.append([(int(p["x"]), int(p["y"]), int(p["angle"]), c) for p, c in zip(mine, OTHER_COLOURS)])
    rows = None
    if seen:
        kw = {} if run_levels is None else {"levels": list(run_levels)}
        per_frame = r.render_seen(np.ascontiguousarray(run_poses), **kw)[1].cpu().numpy().view(np.uint32)
        run_lv = np.zeros(len(per_frame), np.int64) if run_levels is None else np.asarray(run_levels)
        lv = np.zeros(len(poses), np.int64) if levels is None else np.asarray(levels)
        rows = np.stack([np.bitwise_or.reduce(per_frame[run_lv == l], axis=0) for l in lv])
        rows = torch.from_numpy(rows.view(np.int32).copy()).cuda(r.device)
    return r.resolve(r.automap(np.ascontiguousarray(poses), levels, scale, names, seen=rows, arrows=arrows), factor, "rgb",
                     levels).cpu().numpy()


def resolve_rgb(r, index: np.ndarray, factor: int, levels=None, palette: int = 0) -> np.ndarray:
    """(n, H, W, 3) uint8: the host index frames of renderer r resolved by `factor` on its device through palette `palette`
    of each frame's level (b2d_resolve_device, b2d_resolve_palettes_device)"""
    import torch
    dev = torch.device("cuda", r.device)
    palettes = [palette] * len(index) if palette else None
    with torch.cuda.device(dev):
        return r.resolve(torch.from_numpy(np.ascontiguousarray(index)).to(dev), factor, "rgb", levels, palettes).cpu().numpy()


def _palette_out_of_range(scenes, palette: int) -> bool:
    """--palette: P at or past a scene's palette count is a usage error, reported here"""
    n = min(sc.num_palettes for sc in scenes)
    if palette < n:
        return False
    print("--palette takes a palette index below %d" % n, file=sys.stderr)
    return True


def _comm_from_file(b2d, id_file: str, rank: int, world: int):
    if rank == 0:
        with open(id_file + ".tmp", "wb") as f:
            f.write(b2d.Comm.unique_id())
        os.replace(id_file + ".tmp", id_file)
    else:
        for _ in range(600):
            if os.path.exists(id_file):
                break
            time.sleep(0.1)
    with open(id_file, "rb") as f:
        uid = f.read()
    return b2d.Comm(uid, rank, world, rank)


def _main_levels(b2d, arch, set_, view, args, w, h) -> int:
    scenes = [b2d.Scene(arch, i) for i in set_]
    if any(sc.start_pose is None for sc in scenes):
        print("Fatal error: a level has no player-1 start", file=sys.stderr)
        return 1
    if _palette_out_of_range(scenes, args.palette):
        return 2
    per_level = max(args.poses, 1)
    poses, levels, tics = level_set_job(b2d, scenes, per_level, args.tics)
    n = len(poses)
    if not args.world:
        r = b2d.Renderer.from_levels(scenes, view, device=args.device, max_batch=min(n, 64))
        lights = [(args.fixed_colormap, args.extralight)] * n if (args.fixed_colormap, args.extralight) != (-1, 0) else None
        if args.supersample > 1 or args.palette:
            rgb = resolve_rgb(r, r.render_levels_states(poses, levels, tics, lights=lights), args.supersample, levels,
                              args.palette)
            print("rendered %d frame(s) %dx%d of %d level(s), supersampled %dx, palette %d" % (n, w, h, len(set_), args.supersample,
                                                                                             args.palette))
            frame = lambda i: rgb[i]    # noqa: E731
        else:
            rgba = r.render_levels_states(poses, levels, tics, rgba=True, lights=lights)[1]
            print("rendered %d frame(s) %dx%d of %d level(s)" % (n, w, h, len(set_)))
            frame = lambda i: rgba_to_rgb(rgba[i])    # noqa: E731
        if args.dump:
            for k, lvl in enumerate(set_):
                _write_image(_dump_name(args.dump, lvl), frame(k * per_level))
            if args.automap is not None:
                firsts = np.arange(len(set_)) * per_level
                am = automap_rgb(r, poses[firsts], list(range(len(set_))), args.automap, args.automap_flags, args.supersample,
                                 poses, levels)
                for k, lvl in enumerate(set_):
                    _write_image(_automap_name(args.dump, lvl), am[k])
        if args.stream:
            with open(args.stream, "wb") as f:
                for i in range(n):
                    f.write(encode_ppm(frame(i)))
        return 0
    import torch
    from rust_doom_b200 import _lib
    rank, world = args.rank, args.world
    torch.cuda.set_device(rank)
    r = b2d.Renderer.from_levels(scenes, view, device=rank, max_batch=min(n, 64))
    comm = _comm_from_file(b2d, args.id_file, rank, world)
    per = (n + world - 1) // world
    frame_bytes = len(encode_ppm(np.zeros((h, w, 3), np.uint8)))
    out = open(args.stream, "wb") if (args.stream and rank == 0) else None
    if out is not None:
        out.truncate(n * frame_bytes)
    firsts = {}

    def sink(k, first, cnt, ptr, ranks, stream):
        # every gathered frame through its own level's palette on the device, then to its place in the stream
        g = [q * per + first + j for q in range(ranks) for j in range(cnt)]
        rgba = torch.empty((len(g), h, w), dtype=torch.int32, device="cuda")
        r.palette_lut_levels_device(ptr, [levels[min(i, n - 1)] for i in g], len(g), rgba.data_ptr(), stream)
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            host = rgba.cpu().numpy().view(np.uint32)
        for i, frame in zip(g, host):
            if i < n:
                out.seek(i * frame_bytes)
                out.write(encode_ppm(rgba_to_rgb(frame)))
                if args.dump and i % per_level == 0:
                    firsts[int(levels[i])] = frame

    try:
        t0 = time.perf_counter()
        st = r.render_sharded_levels_states(comm, poses, levels, tics, None, args.chunk, _lib.SHARD_RENDER_GATHER,
                                            sink if out is not None else None)
        dt = time.perf_counter() - t0
        bits = r.status()
        if bits:
            print("Fatal error: frames incomplete (status %d)" % bits, file=sys.stderr)
            return 1
        print("rank %d/%d: %d frames gathered in %d chunk(s) of %d level(s), %.2f ms" % (rank, world, st["frames_gathered"],
                                                                                      st["chunks"], len(set_), dt * 1e3))
        for k, frame in firsts.items():
            _write_image(_dump_name(args.dump, set_[k]), rgba_to_rgb(frame))
        return 0
    finally:
        if out is not None:
            out.close()
        comm.close()


def main(argv=None) -> int:
    import rust_doom_b200 as b2d
    from rust_doom_b200 import poses as P
    from rust_doom_b200 import synthwad

    ap = argparse.ArgumentParser(prog="b2d")
    ap.add_argument("-i", "--iwad", default=None, help="initial WAD file (default: generated synthetic IWAD)")
    ap.add_argument("-m", "--metadata", default=None, help="accepted for compatibility; the sky table is built in")
    ap.add_argument("-r", "--resolution", default="1280x720")
    ap.add_argument("-l", "--level", type=int, default=0)
    ap.add_argument("-f", "--fov", type=float, default=65.0)
    ap.add_argument("--poses", type=int, default=1, help="1 = spawn pose, N>1 = N-pose fly-through")
    ap.add_argument("--dump", default=None, help="write the first frame (.png, otherwise binary PPM)")
    ap.add_argument("--stream", default=None,
                    help="write every frame, in order, as concatenated binary PPMs (e.g. ffmpeg -f image2pipe -i FILE)")
    ap.add_argument("--tics-per-frame", type=int, default=0,
                    help="advance the level time by this many tics (1/35 s) per frame: animated flats / walls, "
                         "scrolling walls, light effects")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--levels", default=None, help="render a level set: `all` or comma-separated level indices")
    ap.add_argument("--tics", type=int, default=0, help="with --levels: pose i at level time T + i")
    ap.add_argument("--world", type=int, default=0, help="with --levels: shard over this many processes, one per GPU")
    ap.add_argument("--rank", type=int, default=0)
    ap.add_argument("--id-file", default=None, help="with --world: the file rank 0 writes the NCCL unique id to")
    ap.add_argument("--chunk", type=int, default=16, help="with --world: frames per rank and chunk")
    ap.add_argument("--supersample", type=int, default=1,
                    help="render at K times the resolution (1..8) and resolve every K x K block to one output pixel")
    ap.add_argument("--palette", type=int, default=0,
                    help="colour the frames through PLAYPAL palette P (Doom: 1..8 damage, 9..12 bonus, 13 radiation suit)")
    ap.add_argument("--fixed-colormap", type=int, default=-1,
                    help="with --levels: light every frame through COLORMAP row R, -1..32 (32 invulnerability, 1 visor)")
    ap.add_argument("--extralight", type=int, default=0, help="with --levels: raise every light by E (0..2) weapon-flash steps")
    ap.add_argument("--automap", type=float, default=None, metavar="SCALE",
                    help="with --dump: also write NAME.automap.EXT (NAME.automap.L.EXT with --levels), Doom's automap of "
                         "the dumped pose at SCALE pixels per map unit (Doom's default: 0.2)")
    ap.add_argument("--automap-flags", default="", help="with --automap: comma-separated rotate, all, things, allmap (unseen lines in grey), "
                         "seen (only the lines the run's frames saw), others (the run's next three poses as team-mates' arrows), "
                         "grid (Doom's 128-unit grid)")
    ap.add_argument("command", nargs="?", choices=["check", "list-levels"], default=None)
    args = ap.parse_args(argv)

    try:
        w, h = (int(v) for v in args.resolution.lower().split("x"))
    except ValueError:
        print("resolution format is WIDTHxHEIGHT", file=sys.stderr)
        return 2
    ss = args.supersample
    if not 1 <= ss <= 8:
        print("--supersample takes a factor in 1..8", file=sys.stderr)
        return 2
    if ss > 1 and (args.world or int(os.environ.get("WORLD_SIZE", "1")) > 1):
        print("--supersample does not combine with sharded rendering (--world or torchrun)", file=sys.stderr)
        return 2
    if args.palette < 0:
        print("--palette takes a palette index", file=sys.stderr)
        return 2
    if args.palette and (args.world or int(os.environ.get("WORLD_SIZE", "1")) > 1):
        print("--palette does not combine with sharded rendering (--world or torchrun)", file=sys.stderr)
        return 2
    if not -1 <= args.fixed_colormap <= 32 or not 0 <= args.extralight <= 2:
        print("--fixed-colormap takes a row in -1..32 and --extralight a value in 0..2", file=sys.stderr)
        return 2
    if (args.fixed_colormap, args.extralight) != (-1, 0):
        if args.levels is None:
            print("--fixed-colormap and --extralight take --levels", file=sys.stderr)
            return 2
        if args.world or int(os.environ.get("WORLD_SIZE", "1")) > 1:
            print("--fixed-colormap and --extralight do not combine with sharded rendering (--world or torchrun)", file=sys.stderr)
            return 2
    if args.automap is not None:
        if not 1.0 / 256 <= args.automap <= 64:
            print("--automap takes a scale in pixels per map unit, 1/256 .. 64", file=sys.stderr)
            return 2
        try:
            automap_flag_names(args.automap_flags)
        except ValueError as e:
            print("--automap-flags: %s" % e, file=sys.stderr)
            return 2
        if not args.dump or args.world or int(os.environ.get("WORLD_SIZE", "1")) > 1:
            print("--automap takes --dump and does not combine with sharded rendering (--world or torchrun)", file=sys.stderr)
            return 2
    try:
        arch = b2d.Archive.open(args.iwad) if args.iwad else b2d.Archive.from_bytes(synthwad.build_iwad(1, synthwad.E1_MAPS[:3]))
        if args.command == "list-levels":
            for i, name in enumerate(arch.level_names()):
                print("%3d %8s" % (i, name))
            return 0
        if args.command == "check":
            for i, name in enumerate(arch.level_names()):
                sc = b2d.Scene(arch, i)
                print("Level %d (%s): %d segs, %d subsectors, %d sectors, %d textures: ok"
                      % (i, name, sc.info.n_segs, sc.info.n_ssectors, sc.info.n_sectors, sc.info.n_textures))
            return 0
        if args.levels is not None:
            try:
                set_ = parse_levels(args.levels, arch.num_levels())
            except ValueError:
                print("--levels takes `all` or comma-separated level indices below %d" % arch.num_levels(), file=sys.stderr)
                return 2
            if args.world and not args.id_file:
                print("--id-file PATH is required with --world", file=sys.stderr)
                return 2
            return _main_levels(b2d, arch, set_, b2d.make_view(ss * w, ss * h, args.fov), args, w, h)
        if args.world:
            print("--world takes --levels (a single level shards under torchrun)", file=sys.stderr)
            return 2
        scene = b2d.Scene(arch, args.level)
        if _palette_out_of_range([scene], args.palette):
            return 2
        view = b2d.make_view(ss * w, ss * h, args.fov)
        if args.poses <= 1:
            poses = scene.start_pose if scene.start_pose is not None else P.random_poses(scene, 1, 1)
        else:
            poses = P.flythrough_poses(scene, args.poses, 2)
        world = int(os.environ.get("WORLD_SIZE", "1"))
        if world > 1:
            return _main_sharded(b2d, scene, view, poses, args, w, h, world)
        r = b2d.Renderer(scene, view, device=args.device, max_batch=min(len(poses), 256))
        t0 = time.perf_counter()
        if ss > 1 or args.palette:
            index = np.empty((len(poses), ss * h, ss * w), dtype=np.uint8)
            if args.tics_per_frame > 0:
                for i in range(len(poses)):
                    r.set_time(i * args.tics_per_frame)
                    index[i] = r.render(poses[i:i + 1])[0]
            else:
                r.render(poses, out_index=index)
            rgb = resolve_rgb(r, index, ss, palette=args.palette)
            frame = lambda i: rgb[i]    # noqa: E731
        elif args.tics_per_frame > 0:          # time is a per-batch input: one batch per frame
            rgba = np.empty((len(poses), h, w), dtype=np.uint32)
            for i in range(len(poses)):
                r.set_time(i * args.tics_per_frame)
                rgba[i] = r.render(poses[i:i + 1], rgba=True)[1][0]
        else:
            rgba = r.render(poses, rgba=True)[1]
        if ss == 1 and not args.palette:
            frame = lambda i: rgba_to_rgb(rgba[i])    # noqa: E731
        dt = time.perf_counter() - t0
        print("rendered %d frame(s) %dx%d in %.2f ms (%.0f frames/s end to end)" % (len(poses), w, h, dt * 1e3, len(poses) / dt))
        if args.dump:
            rgb0 = frame(0)
            with open(args.dump, "wb") as f:
                f.write(encode_png(rgb0) if args.dump.lower().endswith(".png") else encode_ppm(rgb0))
            if args.automap is not None:
                _write_image(_automap_name(args.dump), automap_rgb(r, poses[:1], None, args.automap, args.automap_flags, ss, poses)[0])
        if args.stream:
            with open(args.stream, "wb") as f:
                for i in range(len(poses)):
                    f.write(encode_ppm(frame(i)))
        return 0
    except b2d.B2dError as e:
        print("Fatal error: %s" % e, file=sys.stderr)
        return 1


if __name__ == "__main__":
    sys.exit(main())
