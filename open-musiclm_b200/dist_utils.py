"""Host-side pieces of the data-parallel path (device-agnostic so that they can be exercised under gloo on CPU).

The hot path shards by batch: every rank runs the same step on its own sequences and the gradients are summed over
ranks (DDP mean: the 1/world factor is folded into the clip/AdamW kernel; trainer.py:154-155,439 of the reference).
The sum is an all-reduce of the flat fp32 gradient arena, cut into BUCKETS that follow the order in which the backward
pass finishes them — logit heads, then the layers from last to first, then everything that completes at the very end
(embeddings, start tokens, the rel-pos MLP, the small 1-D parameters) — so that each bucket's all-reduce runs on a
side stream underneath the rest of the backward pass (SURVEY 8e) and only the last one is exposed.
"""
from typing import Dict, List, Sequence, Tuple

import torch
import torch.distributed as dist

Slice = Tuple[int, int]


def world_info(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group), dist.get_rank(group)
    return 1, 0


def allreduce_sum_(flat: torch.Tensor, group=None) -> torch.Tensor:
    """In-place sum of the flat gradient arena over all ranks (no-op for a single process)."""
    world, _ = world_info(group)
    if world > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    return flat


def grad_prescale(group=None) -> float:
    """Factor that turns the all-reduced SUM into DistributedDataParallel's mean."""
    world, _ = world_info(group)
    return 1.0 / world


def rank_seed(seed: int, rank: int) -> int:
    """Per-rank seed of the dropout / forgetful-mask streams (weights use the SAME seed on every rank)."""
    return seed * 1000003 + rank * 7919 + 1


def plan_buckets(layout: Dict[str, int], sizes: Dict[str, int], total: int, depth: int,
                 min_elems: int = 4 << 20) -> List[Tuple[str, List[Slice]]]:
    """Cuts the gradient arena [0, total) into all-reduce buckets in backward-completion order.

    layout / sizes: arena offset and element count of every parameter (state_dict names).  Returns
    [(trigger, [(start, end), ...]), ...] where trigger names the point of the backward pass after which the bucket is
    complete: 'heads', 'layer<l>' (l = depth-1 .. 0) or 'tail'.  Every arena element (padding included: it is zero on
    all ranks) belongs to exactly one bucket.  Layer buckets smaller than min_elems are merged into the next one, so a
    shallow toy model reduces in one or two calls while a 24-layer model gets ~24 of ~40 MB each."""
    def span(names: Sequence[str]) -> Slice:
        lo = min(layout[n] for n in names)
        hi = max(layout[n] + sizes[n] for n in names)
        # parameters start on 64-element boundaries: take the padding behind the last one along, so that every slice
        # length is a multiple of 64 (and with it of any power-of-two world size: reduce-scatter needs equal parts)
        return lo, min(total, (hi + 63) // 64 * 64)

    mats = lambda l: [n for n in layout if n.startswith(f"transformer.layers.{l}.") and n.endswith("weight")]
    heads = [n for n in layout if n.startswith("logit_weights.")]
    claimed: List[Slice] = []
    out: List[Tuple[str, List[Slice]]] = []
    if heads:
        out.append(("heads", [span(heads)]))
        claimed.append(span(heads))
    pending: List[Slice] = []
    pend_elems = 0
    for l in reversed(range(depth)):
        s = span(mats(l))
        pending.append(s)
        pend_elems += s[1] - s[0]
        if pend_elems >= min_elems or l == 0:
            # adjacent layer spans are contiguous in the arena: merge them into one slice
            lo, hi = min(p[0] for p in pending), max(p[1] for p in pending)
            merged = [(lo, hi)] if hi - lo <= pend_elems + 64 * len(pending) else sorted(pending)
            out.append((f"layer{l}", merged))
            claimed.extend(merged)
            pending, pend_elems = [], 0
    # the tail: whatever is left, as maximal contiguous slices
    claimed.sort()
    tail, pos = [], 0
    for lo, hi in claimed:
        if lo > pos:
            tail.append((pos, lo))
        pos = max(pos, hi)
    if pos < total:
        tail.append((pos, total))
    out.append(("tail", tail))
    # sanity: exact cover of [0, total)
    cover = sorted(s for _, sl in out for s in sl)
    p = 0
    for lo, hi in cover:
        assert lo == p, f"bucket plan does not tile the arena at {p} (next slice starts at {lo})"
        p = hi
    assert p == total
    return out


def drop_frozen_buckets(plan: List[Tuple[str, List[Slice]]], trainable: Sequence[Slice]) -> List[Tuple[str, List[Slice]]]:
    """The buckets of `plan` that overlap at least one arena span [a, b) of a trainable parameter.  The others hold only
    frozen parameters and padding, whose gradient is zero on every rank: they are not communicated."""
    live = lambda sl: any(lo < b and a < hi for lo, hi in sl for a, b in trainable)
    return [(t, sl) for t, sl in plan if live(sl)]


def shard_of(lo: int, hi: int, world: int, rank: int) -> Slice:
    """The part of the arena slice [lo, hi) that `rank` owns after a reduce-scatter (equal parts, rank order)."""
    n = hi - lo
    assert n % world == 0, f"arena slice [{lo}, {hi}) is not divisible by the world size {world}"
    return lo + rank * (n // world), lo + (rank + 1) * (n // world)


def reduce_scatter_sum_(view: torch.Tensor, world: int, rank: int, group=None):
    """In place: afterwards view[shard of rank] holds the sum over ranks of that part (the rest of `view` is undefined).
    NCCL: one reduce-scatter (output = the rank's part of the input buffer, NCCL's in-place form).  Backends without
    reduce-scatter (gloo, CPU tests): an all-reduce of the whole view."""
    n = view.numel() // world
    if dist.get_backend(group) == "nccl":
        dist.reduce_scatter_tensor(view[rank * n:(rank + 1) * n], view, op=dist.ReduceOp.SUM, group=group)
    else:
        dist.all_reduce(view, op=dist.ReduceOp.SUM, group=group)


def all_gather_(view: torch.Tensor, world: int, rank: int, group=None):
    """In place: every rank's part of `view` (see shard_of) is distributed to all ranks."""
    n = view.numel() // world
    if dist.get_backend(group) == "nccl":
        dist.all_gather_into_tensor(view, view[rank * n:(rank + 1) * n], group=group)
    else:
        parts = [torch.empty(n, dtype=view.dtype, device=view.device) for _ in range(world)]
        dist.all_gather(parts, view[rank * n:(rank + 1) * n].clone(), group=group)
        for r, part in enumerate(parts):
            view[r * n:(r + 1) * n].copy_(part)


class BucketReducer:
    """Issues the per-bucket collectives.  `fire(trigger)` is called by the backward pass when the named point is
    reached; on CUDA the collective is enqueued on `side_stream` after an event recorded on the compute stream, and
    `join()` makes the compute stream wait for all of them (both work under CUDA-graph capture: fork / join).  On CPU
    (gloo tests) everything is synchronous.
    scatter=False: all-reduce (every rank ends with the full summed arena).
    scatter=True : reduce-scatter (rank r ends with the sum of ITS part of every slice, see shard_of): half the bytes on
                   the wire; the optimiser then updates that part only and all-gathers the parameters (trainer.py)."""

    def __init__(self, flat: torch.Tensor, plan, group=None, side_stream=None, scatter=False):
        self.flat, self.plan, self.group, self.side = flat, {t: sl for t, sl in plan}, group, side_stream
        self.order = [t for t, _ in plan]
        self.world, self.rank = world_info(group)
        self.scatter = scatter
        self.fired: List[str] = []

    def slices(self) -> List[Slice]:
        """Every arena slice of the plan (they tile the arena)."""
        return [s for t in self.order for s in self.plan[t]]

    def _reduce(self, v: torch.Tensor):
        if self.scatter:
            reduce_scatter_sum_(v, self.world, self.rank, self.group)
        else:
            dist.all_reduce(v, op=dist.ReduceOp.SUM, group=self.group)

    def begin(self):
        self.fired = []

    def fire(self, trigger: str):
        if trigger not in self.plan or self.world == 1:
            return
        self.fired.append(trigger)
        views = [self.flat[lo:hi] for lo, hi in self.plan[trigger]]
        if self.side is not None:
            self.side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self.side):
                for v in views:
                    self._reduce(v)
        else:
            for v in views:
                self._reduce(v)

    def join(self):
        # (triggers of buckets left out of the plan, see drop_frozen_buckets, are ignored by fire)
        if self.world > 1:
            assert self.fired == self.order, f"buckets fired {self.fired}, expected {self.order}"
            if self.side is not None:
                torch.cuda.current_stream().wait_stream(self.side)
