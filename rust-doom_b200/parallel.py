"""Multi-GPU sharding of independent camera poses (SURVEY.md 8e).

Frames for distinct poses are independent and the scene (< a few MB) is replicated on every GPU, so the
path shards with NO data-path collective: pose i goes to rank i // ceil(n / world) (contiguous blocks).
The only exchange the north star names is an optional all-gather of finished frames (config 5); it is an
NVLink-bound step that is reported separately from render throughput and runs through
torch.distributed (NCCL on GPUs, gloo in the CPU tests), chunked so that the gathered buffer of a chunk
-- not of the whole job -- has to fit in HBM.
"""
from __future__ import annotations

from typing import Iterator, Tuple

import numpy as np


def shard_bounds(n: int, rank: int, world: int) -> Tuple[int, int, int]:
    """(start, end, per_rank) of this rank's contiguous block; the last blocks may be short/empty."""
    per = (n + world - 1) // world
    start = min(n, rank * per)
    end = min(n, start + per)
    return start, end, per


def shard_poses(poses: np.ndarray, rank: int, world: int) -> np.ndarray:
    s, e, _ = shard_bounds(len(poses), rank, world)
    return poses[s:e]


def gather_chunks(per_rank: int, chunk_frames: int) -> Iterator[Tuple[int, int]]:
    c0 = 0
    while c0 < per_rank:
        yield c0, min(per_rank, c0 + chunk_frames)
        c0 += chunk_frames


def sharded_schedule(n_total: int, world: int, chunk_frames: int, max_batch: int = 1 << 30):
    """The chunk plan of b2d_render_sharded (csrc/b2d_sharded.cu), restated: per = ceil(n_total / world) poses per rank
    (a short last block is padded by repeating the job's last pose), chunks of min(chunk_frames, max_batch, per) frames.
    Returns (per, [(first_local_pose, frames_per_rank), ...])."""
    per = (n_total + world - 1) // world
    chunk = min(chunk_frames or 256, max_batch, per) if per else 0
    plan = []
    first = 0
    while first < per:
        cnt = min(chunk, per - first)
        plan.append((first, cnt))
        first += cnt
    return per, plan


def padded_block(poses: np.ndarray, rank: int, world: int) -> np.ndarray:
    """Rank `rank`'s block of the job as b2d_render_sharded renders it: poses[rank*per + i], indices past the end
    clamped to the last pose."""
    return poses[padded_block_indices(len(poses), rank, world)]


def padded_block_indices(n_total: int, rank: int, world: int) -> np.ndarray:
    """Indices into the whole job of rank `rank`'s padded block (padded_block): rank*per + i, clamped to the last entry."""
    per = (n_total + world - 1) // world
    return np.minimum(rank * per + np.arange(per), n_total - 1)


def padded_block_levels_states(poses: np.ndarray, levels, tics, rank: int, world: int, moves_per_pose=None):
    """Rank `rank`'s block of a level-set job as b2d_render_sharded_levels_states renders it: (poses, levels, tics,
    moves_per_pose or None) of the job's entries rank*per + i, a short last block padded by repeating the last pose
    WITH its level, time and moves.  Chunk k of the block is sharded_schedule's chunk k, as for b2d_render_sharded."""
    idx = padded_block_indices(len(poses), rank, world)
    per_pose = None if moves_per_pose is None else list(moves_per_pose)
    moves = None if per_pose is None else [per_pose[i] for i in idx.tolist()]
    return poses[idx], np.asarray(levels)[idx], np.asarray(tics)[idx], moves


def sharded_gather_emulated(local_frames, n_total: int, chunk_frames: int, on_chunk, group=None):
    """CPU stand-in (gloo) for the exchange of b2d_render_sharded, chunk for chunk and in the same buffer layout: for
    every chunk, `on_chunk(k, first_local_pose, frames_per_rank, gathered)` with gathered[q, j] = frame j of rank q's
    slice.  `local_frames` is this rank's padded block [per, H, W] (torch uint8)."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    per, plan = sharded_schedule(n_total, world, chunk_frames)
    assert local_frames.shape[0] == per
    for k, (first, cnt) in enumerate(plan):
        send = local_frames[first:first + cnt].contiguous()
        lst = [torch.empty_like(send) for _ in range(world)]
        dist.all_gather(lst, send, group=group)
        on_chunk(k, first, cnt, torch.stack(lst))


def all_gather_frames(local, n_total: int, chunk_frames: int = 256, group=None, out=None):
    """All-gather per-rank frame blocks [per_rank_valid, H, W] (torch uint8) into global pose order.

    Returns a tensor [n_total, H, W] on every rank (or fills `out`).  Works chunk by chunk: each step moves
    `chunk_frames` frames per rank, i.e. world * chunk_frames frames of receive buffer.
    """
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    per = (n_total + world - 1) // world
    H, W = local.shape[1], local.shape[2]
    if out is None:
        out = torch.empty((n_total, H, W), dtype=local.dtype, device=local.device)
    use_into = dist.get_backend(group) == "nccl"
    for c0, c1 in gather_chunks(per, chunk_frames):
        cnt = c1 - c0
        send = torch.zeros((cnt, H, W), dtype=local.dtype, device=local.device)
        have = max(0, min(local.shape[0], c1) - c0)
        if have > 0:
            send[:have] = local[c0:c0 + have]
        if use_into:
            recv = torch.empty((world * cnt, H, W), dtype=local.dtype, device=local.device)
            dist.all_gather_into_tensor(recv, send, group=group)
            parts = recv.view(world, cnt, H, W)
        else:
            lst = [torch.empty_like(send) for _ in range(world)]
            dist.all_gather(lst, send, group=group)
            parts = torch.stack(lst)
        for r in range(world):
            g0 = r * per + c0
            g1 = min(n_total, r * per + c1)
            if g1 > g0:
                out[g0:g1] = parts[r, :g1 - g0]
    return out


def write_frames_in_order(local, n_total: int, write_fn, chunk_frames: int = 64, group=None) -> int:
    """Frame sink on the gather rank (SURVEY.md 8-f3): streams every rank's finished frames to rank 0 in global
    pose order, `chunk_frames` at a time, and hands them to `write_fn(frames_uint8_cpu_numpy, first_index)` there.

    `local` is this rank's contiguous block [valid, H, W] (torch uint8, any device).  Only a chunk is ever in
    flight, so the job size is not bounded by rank 0's memory.  Point-to-point transfers (NCCL on GPUs, gloo in the
    CPU tests); ranks other than 0 and the current sender just advance.  Returns the number of frames written
    (on rank 0; 0 elsewhere)."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    per = (n_total + world - 1) // world
    H, W = int(local.shape[1]), int(local.shape[2])
    written = 0
    for r in range(world):
        g0, g1 = min(n_total, r * per), min(n_total, (r + 1) * per)
        for c0 in range(g0, g1, chunk_frames):
            c1 = min(g1, c0 + chunk_frames)
            if rank == r:
                chunk = local[c0 - g0:c1 - g0].contiguous()
                if rank == 0:
                    write_fn(chunk.cpu().numpy(), c0)
                    written += c1 - c0
                else:
                    dist.send(chunk, dst=0, group=group)
            elif rank == 0:
                buf = torch.empty((c1 - c0, H, W), dtype=local.dtype, device=local.device)
                dist.recv(buf, src=r, group=group)
                write_fn(buf.cpu().numpy(), c0)
                written += c1 - c0
    return written
