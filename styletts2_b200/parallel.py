"""Multi-GPU plan: utterances are independent (no cross-utterance op anywhere on the path:
InstanceNorm is per (b,c), attention is within an utterance, LSTMs are per sequence), so the batch
is split contiguously across ranks with replicated weights and NO collective on the data path
(SURVEY.md section 8e).  The only optional collective is a final gather of the waveforms."""
from __future__ import annotations

import os
from typing import Dict, List, Sequence, Tuple

import torch


def shard_range(batch: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous split of `batch` utterances; the first (batch % world) ranks get one extra."""
    base, rem = divmod(batch, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def plan_equal_length_batches(lengths: Sequence[int], world: int, max_batch: int) -> List[List[List[int]]]:
    """Serving-side plan for a queue of utterances with DIFFERENT token counts (SURVEY section 8 f3, host part): utterances
    are bucketed by token count (no token padding inside a batch), cut into batches of at most `max_batch`, and the
    batches are dealt to ranks longest-processing-time first (cost ~ tokens x utterances) so that every GPU finishes at
    about the same time.  Equal token counts do NOT imply equal predicted frame counts: Synthesizer.synthesize groups
    each batch by total duration after the duration kernel and runs one launch chain per distinct length (the text
    side -- PL-BERT, text encoder, sampler, duration predictor -- stays batched).  Deterministic (ties by first index).
    Returns plan[rank] = list of batches, each a list of utterance indices."""
    assert world >= 1 and max_batch >= 1
    buckets: Dict[int, List[int]] = {}
    for i, n in enumerate(lengths):
        buckets.setdefault(int(n), []).append(i)
    batches = []
    for n in sorted(buckets):
        idx = buckets[n]
        for k in range(0, len(idx), max_batch):
            batches.append((n * len(idx[k:k + max_batch]), idx[k:k + max_batch]))
    batches.sort(key=lambda b: (-b[0], b[1][0]))
    load = [0] * world
    plan: List[List[List[int]]] = [[] for _ in range(world)]
    for cost, idx in batches:
        r = min(range(world), key=lambda q: (load[q], q))
        plan[r].append(idx)
        load[r] += cost
    return plan


def plan_token_batches(lengths: Sequence[int], world: int, max_batch: int, max_rows: int) -> List[List[List[int]]]:
    """Serving-side plan for Synthesizer.synthesize(..., token_packing=True), whose text side runs on packed token rows and
    so takes any mix of token counts in one batch.  Utterances are sorted by token count (longest first, ties by index)
    and cut into batches of at most `max_batch` utterances and `max_rows` tokens in all; the batches are dealt to ranks
    longest first (cost = the batch's token sum), each to the least loaded rank (ties to the lower rank), so that rank
    loads end within one batch's cost of each other.  Deterministic.  Returns plan[rank] = list of batches, each a list of
    utterance indices."""
    assert world >= 1 and max_batch >= 1 and max_rows >= 1
    order = sorted(range(len(lengths)), key=lambda i: (-int(lengths[i]), i))
    batches: List[Tuple[int, List[int]]] = []
    cur: List[int] = []
    rows = 0
    for i in order:
        n = int(lengths[i])
        if n < 1 or n > max_rows:
            raise ValueError(f"utterance {i} has {n} tokens; a batch holds 1 .. max_rows={max_rows}")
        if cur and (len(cur) == max_batch or rows + n > max_rows):
            batches.append((rows, cur))
            cur, rows = [], 0
        cur.append(i)
        rows += n
    if cur:
        batches.append((rows, cur))
    batches.sort(key=lambda b: (-b[0], b[1][0]))
    load = [0] * world
    plan: List[List[List[int]]] = [[] for _ in range(world)]
    for cost, idx in batches:
        r = min(range(world), key=lambda q: (load[q], q))
        plan[r].append(idx)
        load[r] += cost
    return plan


def init_from_env(backend: str = "nccl"):
    """torchrun environment -> (rank, local_rank, world).  Single process if WORLD_SIZE is unset."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not torch.distributed.is_initialized():
        kw = {}
        if backend == "nccl" and torch.cuda.is_available():
            torch.cuda.set_device(local)
            kw["device_id"] = torch.device("cuda", local)     # bind the communicator to this rank's GPU (no device guessing)
        torch.distributed.init_process_group(backend=backend, **kw)
    return rank, local, world


def gather_waveforms(wav_local: torch.Tensor, world: int, dst: int = 0, batch: int = None):
    """Optional final collective: gather the shard waveforms [B_r, L] (fp32) on `dst` (NCCL over NVLink on GPUs, gloo in
    the CPU tests).  Shards may be UNEVEN (shard_range gives the first batch % world ranks one utterance more): every
    rank pads its shard to the largest one, `dist.gather` moves equal-sized buffers to `dst` only, and `dst` slices the
    padding off.  `batch` = global utterance count when the shards came from shard_range(batch, r, world); None = every
    rank holds wav_local.shape[0] utterances.  Returns the list of shards on dst, None elsewhere."""
    if world == 1:
        return [wav_local]
    dist = torch.distributed
    rank = dist.get_rank()
    sizes = [wav_local.shape[0]] * world if batch is None else [shard_range(batch, r, world)[1] - shard_range(batch, r, world)[0]
                                                                 for r in range(world)]
    assert sizes[rank] == wav_local.shape[0], (sizes, rank, tuple(wav_local.shape))
    big = max(sizes)
    send = wav_local.contiguous()
    if send.shape[0] < big:
        pad = torch.zeros((big - send.shape[0],) + tuple(send.shape[1:]), dtype=send.dtype, device=send.device)
        send = torch.cat([send, pad], 0)
    bufs = [torch.empty_like(send) for _ in range(world)] if rank == dst else None
    dist.gather(send, bufs, dst=dst)
    if rank != dst:
        return None
    return [b[:n] for b, n in zip(bufs, sizes)]
