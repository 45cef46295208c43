"""Multi-GPU plumbing of the sampling run (SURVEY.md 8e): utterances are independent, so a batch is cut into contiguous
per-rank shards, every rank runs its own sampler loop with no communication, and ONE all-gather of the final latents
reassembles the batch (reference semantics: `NaturalSpeech2.sample` over a batch, model.py:605-696).  One process per GPU;
`torch.distributed` (NCCL on GPUs, gloo in the CPU tests) is the only transport.

Lists of utterances of different lengths (``convert.convert_utterances(group=...)``) use the second half: whole ragged batches
per rank by cost (``plan_batches``), one status exchange and one ragged all-gather (``run_sharded``, ``gather_ragged``)."""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.distributed as dist

from .api import batch_plan


def shard_bounds(n_utterances: int, world_size: int, rank: int) -> Tuple[int, int]:
    """[begin, end) of this rank's contiguous shard; equal shards are required by the single all-gather (weak scaling:
    B per rank is fixed), so the utterance count must divide evenly."""
    if world_size < 1 or not (0 <= rank < world_size):
        raise ValueError(f"bad rank {rank} / world size {world_size}")
    if n_utterances % world_size:
        raise ValueError(f"{n_utterances} utterances do not split evenly over {world_size} ranks (pad the batch)")
    per = n_utterances // world_size
    return rank * per, (rank + 1) * per


def gather_latents(local: torch.Tensor, group: Optional[dist.ProcessGroup] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """All ranks' final latents `[B_local, C, T]` as one `[world * B_local, C, T]` tensor in rank order (one collective)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return local
    local = local.contiguous()
    if out is None:
        out = torch.empty((world * local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local, group=group)
    return out


def shard_features(world_size: int, rank: int, *tensors: torch.Tensor) -> Tuple[torch.Tensor, ...]:
    """This rank's utterances of the batch-first inputs of the device pipeline (`api.sample_from_features`: x_T [B, 100, T],
    c_padded [B, 256, T], refer_padded [B, 100, S], lengths [B], refer_lengths [B]): the condition encoders have no cross-sample op
    either (per-utterance masks, LayerNorm, attention), so the same contiguous cut applies and no collective is added."""
    if not tensors:
        return ()
    n = tensors[0].shape[0]
    if any(t.shape[0] != n for t in tensors):
        raise ValueError("all inputs must share the utterance (first) dimension")
    lo, hi = shard_bounds(n, world_size, rank)
    return tuple(t[lo:hi] for t in tensors)


# ------------------------------------------------------------------------------------------- ragged utterance lists (convert.py)
def sample_step_flops(T: int, S: int) -> int:
    """Algorithmic FLOPs of one denoiser sample-step of one row padded to T frames with an S-frame prompt (BASELINE.md §4)."""
    return 31818240 * T + 4352 * T * T + 7296 * S * T + 4456448 * S


def plan_batches(plans: Sequence[Dict[str, int]], prompt_lengths: Sequence[int], world: int, max_batch: int) -> List[List[List[int]]]:
    """Each rank's ragged batches of utterance indices, ``out[rank] = [batch, ...]``.

    The batches are ``api.batch_plan`` over the 24 kHz lengths ``plans[i]["n24"]`` (``convert.frame_plan``) with at most
    ``min(max_batch, ceil(n / world))`` rows, so that every rank has work when there are enough utterances.  Whole batches then
    go to ranks by LPT: the costliest batch first, to the least-loaded rank, the lowest rank on ties.  A batch costs
    rows x ``sample_step_flops(T_pad, S_pad)``: the ragged programs run their GEMMs over the padded rows, and the sampler is
    most of a conversion.  Only host lengths enter, so every rank computes the same plan on its own.  ``world == 1`` gives
    ``[batch_plan(n24, max_batch)]``."""
    if world < 1:
        raise ValueError(f"bad world size {world}")
    if max_batch < 1:
        raise ValueError("max_batch must be >= 1")
    if len(prompt_lengths) != len(plans):
        raise ValueError(f"{len(prompt_lengths)} prompt lengths for {len(plans)} utterances")
    n = len(plans)
    batches = batch_plan([p["n24"] for p in plans], min(max_batch, max(1, math.ceil(n / world))))
    if world == 1:
        return [batches]
    cost = [len(b) * sample_step_flops(max(plans[i]["T"] for i in b), max(int(prompt_lengths[i]) for i in b)) for b in batches]
    return assign_batches(batches, cost, world)


def assign_batches(batches: Sequence[List[int]], cost: Sequence[int], world: int) -> List[List[List[int]]]:
    """Whole batches to ranks by LPT, ``out[rank] = [batch, ...]``: the costliest batch first (input order on ties), to the
    least-loaded rank, the lowest rank on ties.  ``cost[k]`` is batch k's work in any unit the caller's workload scales with."""
    if world < 1:
        raise ValueError(f"bad world size {world}")
    if len(cost) != len(batches):
        raise ValueError(f"{len(cost)} costs for {len(batches)} batches")
    out: List[List[List[int]]] = [[] for _ in range(world)]
    load = [0] * world
    for k in sorted(range(len(batches)), key=lambda k: -cost[k]):
        r = min(range(world), key=lambda r: load[r])
        out[r].append(batches[k])
        load[r] += cost[k]
    return out


def _all_gather(t: torch.Tensor, group: Optional[dist.ProcessGroup], device: Optional[torch.device]) -> torch.Tensor:
    """Every rank's ``t`` flattened and concatenated in rank order, in one collective: through ``device`` memory on a NCCL group
    (the current CUDA device if None), through host memory on any other (gloo)."""
    if "nccl" in str(dist.get_backend(group)):
        dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
    else:
        dev = torch.device("cpu")
    t = t.reshape(-1).to(dev)
    out = t.new_empty(dist.get_world_size(group) * t.numel())
    dist.all_gather_into_tensor(out, t, group=group)
    return out


def _check_local(local: Sequence[torch.Tensor], plan, sizes, rank: int) -> List[Tuple[int, ...]]:
    """The result shapes of ``sizes``; raises ValueError unless ``local`` has one tensor of the planned size per row of rank's batches."""
    shapes = [(s,) if isinstance(s, int) else tuple(s) for s in sizes]
    mine = [shapes[i] for b in plan[rank] for i in b]
    if [t.numel() for t in local] != [math.prod(s) for s in mine]:
        raise ValueError(f"rank {rank}: results of {[tuple(t.shape) for t in local]} for the plan's {mine}")
    return shapes


def gather_ragged(local: Sequence[torch.Tensor], plan: Sequence[Sequence[Sequence[int]]], sizes: Sequence[Union[int, Sequence[int]]],
                  group: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None,
                  dtype: torch.dtype = torch.float32) -> List[torch.Tensor]:
    """Every utterance's tensor, in input order, on every rank.

    ``local`` holds this rank's results in plan order (its batches in turn, each batch's rows in turn); ``sizes[i]`` is the
    shape (or length) of utterance i's result, which every rank knows from the host plan, so no size is exchanged.  Each rank
    packs its results into one flat buffer padded to the largest rank's packed size; one ``all_gather_into_tensor`` follows,
    through ``device`` on a NCCL group and through host memory on a gloo group.  A rank with no batches joins with zeros.  The
    results are views of one buffer on ``device`` (the host on gloo with ``device`` None)."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if len(plan) != world:
        raise ValueError(f"a plan for {len(plan)} ranks in a group of {world}")
    shapes = _check_local(local, plan, sizes, rank)
    numel = [math.prod(s) for s in shapes]
    order = [[i for b in batches for i in b] for batches in plan]
    packed = [sum(numel[i] for i in o) for o in order]
    buf = torch.zeros(max(packed), dtype=dtype, device=device)
    off = 0
    for t, i in zip(local, order[rank]):
        buf[off:off + numel[i]] = t.reshape(-1)
        off += numel[i]
    flat = _all_gather(buf, group, device)
    if device is not None:
        flat = flat.to(device)
    out: List[Optional[torch.Tensor]] = [None] * len(shapes)
    for r, o in enumerate(order):
        off = r * max(packed)
        for i in o:
            out[i] = flat[off:off + numel[i]].view(shapes[i])
            off += numel[i]
    return out


def check_generator(gen: torch.Generator, group: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None) -> None:
    """Raises ValueError on every rank unless every rank's ``gen`` has the same seed and offset (one all-gather).  A CPU
    generator has no offset, so only its seed is compared."""
    seed = gen.initial_seed()
    key = torch.tensor([seed - (1 << 64) if seed >= 1 << 63 else seed, gen.get_offset() if gen.device.type == "cuda" else 0],
                       dtype=torch.int64)
    keys = _all_gather(key, group, device).view(-1, 2).cpu()
    if not bool((keys == keys[0]).all()):
        raise ValueError(f"the ranks' {gen.device.type} generators differ (seed, offset per rank: {keys.tolist()}): call "
                         "torch.manual_seed with the same seed on every rank")


def run_sharded(work: Callable[[List[int]], Sequence[torch.Tensor]], plan: Sequence[Sequence[Sequence[int]]],
                sizes: Sequence[Union[int, Sequence[int]]], group: Optional[dist.ProcessGroup] = None,
                device: Optional[torch.device] = None, dtype: torch.dtype = torch.float32) -> List[torch.Tensor]:
    """Runs ``work(batch)`` (one result per row) on each of this rank's batches of ``plan`` and returns ``gather_ragged`` of the
    results.  Before the gather the ranks exchange one status flag, so an exception on any rank (a NaN assertion of the sampler,
    out of memory, ...) raises a RuntimeError naming the failing ranks on every rank instead of leaving the others waiting in
    the gather."""
    rank = dist.get_rank(group)
    local: List[torch.Tensor] = []
    err: Optional[Exception] = None
    try:
        for idx in plan[rank]:
            local.extend(work(list(idx)))
        _check_local(local, plan, sizes, rank)
    except Exception as e:
        err = e
        local = []
    failed = _all_gather(torch.tensor([err is not None], dtype=torch.int32), group, device).nonzero().flatten().tolist()
    if failed:
        mine = f"; rank {rank} raised {type(err).__name__}: {err}" if err is not None else ""
        raise RuntimeError(f"sharded run failed on rank(s) {failed}{mine}") from err
    return gather_ragged(local, plan, sizes, group, device, dtype)
