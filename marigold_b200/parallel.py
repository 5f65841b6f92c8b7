"""Ensemble-member sharding across the GPUs of one box (one process per GPU, torch.distributed).

The reference is single-process (SURVEY.md §2.2); the only place members meet is the ensemble
(marigold/marigold_depth_pipeline.py:281-300). So: the job list is (image, member); rank r takes members
r, r+G, r+2G, ...; every rank encodes its image locally (cheaper than a broadcast) and reads ITS rows
of the pre-drawn noise tensor; one all-gather of the decoded per-member maps (NCCL over NVLink on
GPUs, gloo on CPU in the tests) precedes the ensemble, which then runs replicated and deterministic.
There is no collective inside the denoising loop of a sharded call.

A size group of ONE job (one image with ensemble_size 1) would leave every rank but one idle, so at native resolution it
runs row-split instead (row_split_rule): every rank runs the whole job, and every attention computes only its rank's
share of the query rows, joined by one in-place all-gather per attention (mgb_set_row_split). Every rank ends with the
same maps, bit-identical to the one-GPU call.
"""
from __future__ import annotations

import contextlib
from typing import List, Optional

import torch

try:
    import torch.distributed as dist
except Exception:  # noqa: BLE001
    dist = None


def world() -> tuple:
    if dist is not None and dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def member_indices(ensemble_size: int, rank: int, world_size: int) -> List[int]:
    """Round-robin ownership: member m belongs to rank m % G."""
    return list(range(rank, ensemble_size, world_size))


def slots_per_rank(ensemble_size: int, world_size: int) -> int:
    return (ensemble_size + world_size - 1) // world_size


def gather_members(local: torch.Tensor, ensemble_size: int, group=None) -> torch.Tensor:
    """local: [n_local, C, H, W] predictions of this rank's members (in member_indices order).
    Returns [ensemble_size, C, H, W] in global member order on every rank: ONE all_gather of
    ceil(E/G) padded slots per rank."""
    rank, G = world()
    if G == 1:
        assert local.shape[0] == ensemble_size
        return local
    S = slots_per_rank(ensemble_size, G)
    pad = torch.zeros((S,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    out = torch.empty((G * S,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, pad.contiguous(), group=group)
    # slot (r, s) holds member r + s*G
    out = out.reshape(G, S, *local.shape[1:])
    members = [out[m % G, m // G] for m in range(ensemble_size)]
    return torch.stack(members, dim=0)


def _collective_device(device: Optional[torch.device]) -> torch.device:
    """Where a small host value travels for a collective: the caller's device under NCCL, the host under gloo."""
    if device is not None and dist.get_backend() == "nccl":
        return torch.device(device)
    return torch.device("cpu")


# ---- lists of images (pipeline.py _infer_list) ----------------------------------------------------------------------
# A size group's jobs are (image, member) pairs in image-major order; job k belongs to rank k mod G (for a one-image list
# these are member_indices). In round r every rank runs its r-th batch of at most bs jobs, and one all-gather gives every
# rank the round's jobs [r G bs, (r + 1) G bs) in job order.

def agree_batch_sizes(sizes: List[int], device: Optional[torch.device] = None) -> List[int]:
    """The MIN over ranks of each size group's member batch, in one all-reduce: a rank's own choice depends on its free
    memory, and the rounds' gathers need one slot count on every rank."""
    rank, G = world()
    if G == 1 or not sizes:
        return [int(b) for b in sizes]
    t = torch.tensor([int(b) for b in sizes], dtype=torch.int64, device=_collective_device(device))
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    return [int(b) for b in t.tolist()]


def num_rounds(n_jobs: int, bs: int, world_size: int) -> int:
    """Rounds of G batches of bs slots that cover n_jobs jobs."""
    return -(-n_jobs // (world_size * bs))


def round_jobs(n_jobs: int, bs: int, rnd: int, rank: int, world_size: int):
    """(jobs, mine) of round `rnd`: every job index of the round in job order, and this rank's (every G-th from rank)."""
    jobs = list(range(rnd * world_size * bs, min((rnd + 1) * world_size * bs, n_jobs)))
    return jobs, jobs[rank::world_size]


def open_images(bs: int, ensemble_size: int, world_size: int, n_images: int) -> int:
    """The most images one round's G bs consecutive jobs can span, E jobs per image: the images a list call holds device
    tensors for at once."""
    return min(n_images, -(-(world_size * bs - 1) // ensemble_size) + 1)


def gather_round(local: torch.Tensor, bs: int, n_round_jobs: int, group=None) -> torch.Tensor:
    """local: [n_mine, C, H, W], this rank's jobs of the round in round_jobs order (n_mine <= bs). Returns the round's
    [n_round_jobs, C, H, W] in job order on every rank: ONE all_gather of bs padded slots per rank. Slot s of rank r holds
    the round's job s G + r."""
    rank, G = world()
    if G == 1:
        assert local.shape[0] == n_round_jobs
        return local
    pad = torch.zeros((bs,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    out = torch.empty((G * bs,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, pad, group=group)
    return out.reshape(G, bs, *local.shape[1:]).transpose(0, 1).reshape(G * bs, *local.shape[1:])[:n_round_jobs]


def barrier_max_ms(ms: float, device: Optional[torch.device] = None) -> float:
    """Max over ranks of a locally measured duration (multi-GPU numbers are max-over-ranks)."""
    rank, G = world()
    if G == 1:
        return ms
    t = torch.tensor([ms], dtype=torch.float64, device=device if device is not None else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


# ---- one job on every rank: the attentions' query rows split over the ranks ------------------------------------------
# Smallest level-0 latent (h / 8 * w / 8 tokens) that runs row-split: 768 x 768. From tools/row_split.py on one H100
# 80GB HBM3 (700 W power limit, 1980 MHz maximum SM clock; DESIGN.md section 7): the smallest of the measured sizes
# (768², 1920x1080, 12, 24 and 48 MP) at which one rank's share of a UNet step at G = 2 beats the captured one-GPU step
# by more than the all-gather time a model gives (bytes received over NVLink's 450 GB/s per direction, not measured). At
# 768² that was 7.25 ms + 0.06 ms (model) against 8.09 ms. Smaller sizes were not measured, and the model leaves out
# the latency of the step's 16 collectives, of the order of that margin.
ROW_SPLIT_MIN_TOKENS = 9_216


def row_split_chunk(T: int, world_size: int) -> int:
    """Query rows per rank of a T-row attention: whole 128-row blocks (csrc/net.h row_split_chunk)."""
    return -(-(-(-T // 128)) // world_size) * 128


def row_split_rows(T: int, rank: int, world_size: int) -> range:
    """The query rows rank `rank` computes: [r chunk, (r + 1) chunk) within [0, T), possibly empty."""
    chunk = row_split_chunk(T, world_size)
    return range(min(T, rank * chunk), min(T, (rank + 1) * chunk))


def row_split_rule(n_jobs: int, h: int, w: int, world_size: int, min_tokens: Optional[int] = None) -> bool:
    """Whether a size group of n_jobs (image, member) jobs at h x w pixels runs row-split on world_size ranks: one job,
    several ranks, and a level-0 latent of at least min_tokens (ROW_SPLIT_MIN_TOKENS) tokens."""
    if min_tokens is None:
        min_tokens = ROW_SPLIT_MIN_TOKENS
    return world_size > 1 and n_jobs == 1 and (h // 8) * (w // 8) >= min_tokens


def exchange_rows(buf: torch.Tensor, rank: int, world_size: int, group=None) -> None:
    """The row split's exchange: buf holds world_size equal chunks, chunk `rank` this rank's; fills the others in place.
    NCCL all-gathers in place on the device; gloo goes through a host copy. Runs on torch's current stream."""
    n = buf.numel() // world_size
    if dist.get_backend(group) == "nccl":
        dist.all_gather_into_tensor(buf, buf[rank * n:(rank + 1) * n], group=group)
        return
    host = buf.cpu()
    out = torch.empty_like(host)
    dist.all_gather_into_tensor(out, host[rank * n:(rank + 1) * n].clone(), group=group)
    buf.copy_(out)


@contextlib.contextmanager
def row_split(engine, on: bool = True):
    """Installs the row split on engine for this rank while the block runs, and clears it after."""
    if not on:
        yield
        return
    rank, G = world()
    engine.set_row_split(rank, G, exchange_rows)
    try:
        yield
    finally:
        engine.set_row_split()


def broadcast_from_first(tensors, device: Optional[torch.device] = None):
    """Rank 0's tensors on every rank (None entries stay None): a row-split job must run on the same noise everywhere."""
    rank, G = world()
    if G == 1:
        return list(tensors)
    out = []
    for t in tensors:
        if t is None:
            out.append(None)
            continue
        c = t.to(_collective_device(device)).contiguous()
        dist.broadcast(c, src=0)
        out.append(c.to(t.device))
    return out
