"""H100-native replacement of the SingleStageTrainer step loop (open_musiclm/trainer.py:415-452) on
top of the engine: per micro-batch  wrapper pre-processing -> forward -> cross entropy -> backward
(gradients accumulate in the flat fp32 arena), then ONE gradient all-reduce over NCCL, global-norm
clip, AdamW and the LinearLR warm-up — every arithmetic step a libomlm_b200 kernel.

Semantics kept from the reference:
  * TokenConditionedTransformerWrapper.forward(return_loss=True) in training mode: eos append, labels,
    key mask with zeroed conditioning ids, 15 % forgetful mask, FFN dropout (open_musiclm.py:328-410);
    loss = sum_{w_s>0} CE_s * n_s * w_s / sum_{w_s>0} n_s (open_musiclm.py:391-410).
  * loss / grad_accum_every per micro-batch (trainer.py:437-439); clip_grad_norm_(max_grad_norm);
    AdamW(lr, betas (0.9, 0.99), eps 1e-8, wd on ndim>=2 params only; Adam when wd == 0) (optimizer.py:3-34), which
    leaves the logit heads of sequences weighted 0 untouched (they have no gradient, open_musiclm.py:398);
    LinearLR(start_factor 1e-7, total_iters lr_warmup) when lr_warmup > 0 (optimizer.py:36-40).
  * DDP mean of gradients over ranks (trainer.py:154-155, 439) — here a single all-reduce(sum) of the
    arena after the last micro-batch, the 1/world factor folded into the clip/AdamW kernel
    (the reference all-reduces on every micro-batch; the reduced result is identical).
"""
import os
from typing import List, Optional, Sequence

import torch
import torch.distributed as dist

from . import lib
from .dist_utils import BucketReducer, all_gather_, allreduce_sum_, grad_prescale, rank_seed, shard_of, world_info
from .model import TokenConditionedTransformer


def frozen_parameter_names(names, ce_weights, requires_grad=None):
    """Parameters the reference never updates, because their `grad` stays None and torch's optimizers and
    clip_grad_norm_ skip such a parameter (no weight decay, no moment update, no part in the norm):
      * the logit head of a sequence weighted 0: the reference adds a sequence's cross entropy only when its weight
        is > 0 (open_musiclm.py:398);
      * every parameter the user froze: requires_grad (name -> bool, optional) is False."""
    rg = requires_grad if requires_grad is not None else {}
    return {n for n in names if (n.startswith("logit_weights.") and not ce_weights[int(n.split(".")[1])] > 0)
            or not rg.get(n, True)}


def live_ranges(n, frozen_spans):
    """[0, n) without the arena spans [a, b) of the frozen parameters, as sorted disjoint (a, b) ranges."""
    out, lo = [], 0
    for a, b in sorted(frozen_spans):
        if a > lo:
            out.append((lo, a))
        lo = max(lo, b)
    if lo < n:
        out.append((lo, n))
    return out


class LossHandle:
    """Host-side view of one step's loss (see HotPathTrainer.train_step_async)."""

    def __init__(self, host_scalar: torch.Tensor, event: "torch.cuda.Event"):
        self._host, self._event = host_scalar, event

    def value(self) -> float:
        self._event.synchronize()
        return float(self._host)


class HotPathTrainer:
    def __init__(self, transformer: TokenConditionedTransformer, *, cross_entropy_loss_weights: Optional[List[float]] = None,
                 lr=3e-4, lr_warmup=0, wd=0., max_grad_norm=0.5, grad_accum_every=1, mask_prob=0.15,
                 betas=(0.9, 0.99), eps=1e-8, pad_id=-1, seed=0, process_group=None, use_cuda_graph=True):
        self.transformer = transformer
        self.eng = transformer.engine
        eng = self.eng
        S = len(eng.seqs)
        self.ce_weights = list(cross_entropy_loss_weights) if cross_entropy_loss_weights is not None else [1.0] * S
        assert len(self.ce_weights) == S
        self.lr, self.lr_warmup, self.wd, self.max_grad_norm = lr, lr_warmup, wd, max_grad_norm
        self.grad_accum_every = grad_accum_every
        self.mask_prob = mask_prob
        self.betas, self.eps, self.pad_id = betas, eps, pad_id
        sizes = {n: p.numel() for n, p in transformer.named_parameters()}
        # read once, like the loss weights: the backward pass, the AdamW ranges, the gradient buckets and the captured
        # graphs are planned for this set (train_step raises if requires_grad changes afterwards)
        self._requires_grad = {n: p.requires_grad for n, p in transformer.named_parameters()}
        self.frozen = frozen_parameter_names(sizes, self.ce_weights, self._requires_grad)
        # the AdamW launches cover these arena ranges only: frozen parameters keep p, m and v bit for bit
        self.live = live_ranges(eng.n_params_arena, [(eng.layout[n], eng.layout[n] + sizes[n]) for n in self.frozen])
        self.steps = 0
        self.pg = process_group
        self.world, self.rank = world_info(process_group)
        eng.seed.fill_(rank_seed(seed, self.rank))     # per-rank random streams (dropout / forgetful mask)
        if self.world > 1:
            # replicas must start from the same weights (DDP broadcasts rank 0's at wrap time, trainer.py:154-155 via
            # accelerate.prepare): do not rely on every rank having seeded its initialisation identically
            dist.broadcast(eng.arena_p, src=dist.get_global_rank(process_group, 0) if process_group is not None else 0,
                           group=process_group)
            eng.refresh_packed(force=True)
        eng.adam_m = torch.zeros_like(eng.arena_p)
        eng.adam_v = torch.zeros_like(eng.arena_p)
        # PAGEABLE on purpose: cudaMemcpyAsync stages a pageable source before it returns, so the host may already write
        # the next step's values while earlier steps are still queued (a pinned buffer would be read late -> wrong step)
        self.hyper_host = torch.zeros(9, dtype=torch.float32)
        self.hyper = torch.zeros(9, dtype=torch.float32, device=eng.dev)
        self.loss_acc = torch.zeros(grad_accum_every, 2, device=eng.dev)     # per micro-batch: (weighted loss, rows counted)
        self.loss_buf = self.loss_acc[:, 0]
        self._mask_draws = 0
        self.use_cuda_graph = use_cuda_graph
        self._graphs = {}
        # data parallel: bucketed gradient all-reduce on a side stream underneath the backward pass (SURVEY 8e).  The
        # persistent GEMMs schedule their tiles statically, so during the overlapped backward they leave `nccl_ctas` SMs
        # to the NCCL kernels (NCCL_MAX_CTAS is set to the same number before the communicator is created, see bench.py)
        self.reducer = None
        self.shard_opt = False
        self.allreduce_mode = "none (single GPU)"
        if self.world > 1:
            # high priority: an all-reduce's CTAs are placed as soon as any SM frees up instead of after the compute kernels queued
            # behind it (OMLM_NCCL_PRIO=0: same priority as the compute stream)
            prio = -1 if os.environ.get("OMLM_NCCL_PRIO", "1") != "0" else 0
            # sharded update (opt-in, OMLM_SHARD_OPT=1): the buckets are reduce-SCATTERED (half the bytes under the backward
            # pass), every rank runs clip + AdamW on its 1/world of the arena only, then the parameters are all-gathered --
            # the same bytes on the wire as one all-reduce, but the optimiser pass shrinks by 1/world.  The all-gather of
            # the fp32 parameters is exposed at the end of the step; off by default (not measured on H100).
            plan = eng.grad_bucket_plan(frozen=self.frozen)
            self.shard_opt = os.environ.get("OMLM_SHARD_OPT", "0") == "1" and all((hi - lo) % self.world == 0 for _, sl in plan for lo, hi in sl)
            self.reducer = BucketReducer(eng.arena_g, plan, process_group, side_stream=torch.cuda.Stream(priority=prio), scatter=self.shard_opt)
            nccl_ctas = int(os.environ.get("NCCL_MAX_CTAS", "0") or 0)
            eng.bwd_max_ctas = max(1, lib.num_sms() - nccl_ctas) if nccl_ctas > 0 else 0
            self.allreduce_mode = (f"{len(self.reducer.order)} buckets in backward order on a side stream, overlapped with the backward pass"
                                   + ("; reduce-scatter + AdamW on 1/world of the arena + all-gather of the parameters" if self.shard_opt else "")
                                   + (f"; backward GEMMs on {eng.bwd_max_ctas} CTAs, NCCL on <= {nccl_ctas}" if nccl_ctas else ""))
        self.loss_out = torch.zeros((), device=eng.dev)
        self._loss_ring = None
        eng.arena_g.zero_()

    # -------------------------------------------------------------------------------------------
    def _micro_batch(self, token_ids: Sequence[torch.Tensor], train: bool, slot: int, backward: bool, reducer=None, det: bool = False):
        eng = self.eng
        dev = eng.dev
        ids = [t.reshape(t.shape[0], -1).to(dev, torch.int64, non_blocking=True) for t in token_ids]
        B = ids[0].shape[0]
        S = len(eng.seqs)
        # shapes are static per configuration: N is known before the plan kernel runs
        n_tok = [t.shape[1] + 1 - (1 if s == S - 1 else 0) for s, t in enumerate(ids)]
        pl = eng.plan(B, n_tok)
        if train:
            eng.seed += 1       # device-side: every micro-batch draws its own dropout / forgetful masks (also under graph replay)
        forget = None
        if train and self.mask_prob > 0:
            num_drop = min(int(pl.N * self.mask_prob), pl.N - 1)        # utils.py:53
            self._mask_draws += 1
            forget = lib.forgetful_mask(B, pl.N, num_drop, eng.seed, self._mask_draws, dev)
        _, src_row, key_mask, labels, _ = lib.token_plan(
            ids, [s.codebook_size for s in eng.seqs], [s.num_quantizers for s in eng.seqs], eng.emb_row_base,
            eng.start_row, append_eos=True, drop_last=True, mask_cond=True, pad_id=self.pad_id, forget_keep=forget,
            err_flag=eng.err_flag)
        ws = eng.workspace(pl, backward, det)
        weighted = {s for s in range(S) if self.ce_weights[s] > 0}
        drop = train and eng.drop_p > 0
        eng.forward_core(pl, ws, src_row, key_mask, backward, weighted, drop)
        # ---- loss (+ dlogits): labels of sequence s live in columns [lab_off, lab_off + len_s + 1)
        total_n = sum(B * pl.n_out[s] for s in weighted)
        lab_off = [0]
        for s in range(S):
            lab_off.append(lab_off[-1] + ids[s].shape[1] + 1)
        # the CE kernels add  w_s / total_n * (sum of row losses)  straight into this micro-batch's slot of loss_acc and read
        # their labels through the strided view (sequence b, position qi + q t) of the label plane: no torch op in between
        acc = self.loss_acc[slot]
        if slot == 0:
            self.loss_acc.zero_()
        for s in sorted(weighted):
            q = eng.seqs[s].num_quantizers
            for gi, (gs, qi, cnt, base) in enumerate(pl.groups):
                if gs != s:
                    continue
                scale = self.ce_weights[s] / total_n / self.grad_accum_every
                lib.cross_entropy(ws["logits"][gi], labels[0, lab_off[s] + qi:], eng.C[s], acc, grad_scale=scale,
                                  dlogits=ws["dlogits"][gi] if backward else None, rows=B * cnt, label_stride=q, rows_per_batch=cnt,
                                  batch_stride=labels.stride(0), loss_scale=self.ce_weights[s] / total_n,
                                  part=ws["det_part"] if det else None)
        loss = acc[0]
        if backward:
            eng.backward_core(pl, ws, src_row, key_mask, weighted, drop, on_ready=reducer.fire if reducer is not None else None, det=det,
                              frozen=self.frozen)
        return loss

    def _set_hyper(self):
        t = self.steps + 1
        fac = 1.0
        if self.lr_warmup > 0:
            fac = 1e-7 + (1.0 - 1e-7) * min(self.steps, self.lr_warmup) / self.lr_warmup
        b1, b2 = self.betas
        h = self.hyper_host
        h[0] = self.lr * fac; h[1] = b1; h[2] = b2; h[3] = self.eps; h[4] = self.wd
        h[5] = 1 - b1 ** t; h[6] = 1 - b2 ** t
        h[7] = self.max_grad_norm if self.max_grad_norm is not None else 0.0
        h[8] = grad_prescale(self.pg)
        self.hyper.copy_(h, non_blocking=True)

    def _fwd_bwd_body(self, micro_batches, det, overlap=True):
        """Device work of one optimiser step up to the reduced gradient arena (capturable in a CUDA graph).  With several
        ranks the last micro-batch's backward pass fires the bucketed all-reduces (the reference reduces on every
        micro-batch, trainer.py:439; the reduced sum is the same)."""
        red = self.reducer if overlap else None
        if red is not None:
            red.begin()
        for i, mb in enumerate(micro_batches):
            self._micro_batch(mb, True, i, True, reducer=red if i == len(micro_batches) - 1 else None, det=det)
        if red is not None:
            red.join()
        elif self.world > 1:
            allreduce_sum_(self.eng.arena_g, self.pg)

    def _update_body(self, det):
        """Clip + AdamW + re-pack on the reduced gradient arena (capturable in a CUDA graph).  det: the gradient norm is
        summed in a fixed order."""
        eng = self.eng
        eng.sumsq.zero_()
        if self.shard_opt:
            self._sharded_update(det)
        else:
            if self.max_grad_norm is not None:
                lib.grad_sumsq(eng.arena_g, eng.sumsq, prescale=grad_prescale(self.pg), part=eng.det_sumsq_part if det else None)
            self._adamw(0, eng.n_params_arena)
        eng.arena_g.zero_()
        eng.refresh_packed(force=True)
        self.loss_out.copy_(self.loss_buf.sum() / self.grad_accum_every)

    def _sharded_update(self, det):
        """After the reduce-scatter this rank holds the summed gradient of ITS part of every arena slice: global norm from
        the parts (one 8-byte all-reduce), AdamW on the parts, all-gather of the updated parameters."""
        eng, W, r = self.eng, self.world, self.rank
        parts = [shard_of(lo, hi, W, r) for lo, hi in self.reducer.slices()]
        if self.max_grad_norm is not None:
            for a, b in parts:
                lib.grad_sumsq(eng.arena_g[a:b], eng.sumsq, prescale=grad_prescale(self.pg), part=eng.det_sumsq_part if det else None)
            dist.all_reduce(eng.sumsq, op=dist.ReduceOp.SUM, group=self.pg)
        for a, b in parts:
            self._adamw(a, b)
        for lo, hi in self.reducer.slices():
            all_gather_(eng.arena_p[lo:hi], W, r, self.pg)

    def _adamw(self, lo, hi):
        """AdamW on the live parts of the arena range [lo, hi): one launch per part, decay below n_decay."""
        eng = self.eng
        for a, b in self.live:
            a, b = max(a, lo), min(b, hi)
            if a < b:
                lib.adamw_step(eng.arena_p[a:b], eng.arena_g[a:b], eng.adam_m[a:b], eng.adam_v[a:b], max(0, min(b - a, eng.n_decay - a)),
                               self.hyper, eng.sumsq)

    def _gather_optimizer_state(self):
        """Sharded update: every rank holds the Adam moments of its parts only -- make them complete everywhere (checkpoints)."""
        if self.shard_opt:
            for lo, hi in self.reducer.slices():
                all_gather_(self.eng.adam_m[lo:hi], self.world, self.rank, self.pg)
                all_gather_(self.eng.adam_v[lo:hi], self.world, self.rank, self.pg)

    def _step_body(self, micro_batches, det):
        self._fwd_bwd_body(micro_batches, det)
        self._update_body(det)

    def _capture(self, st, det):
        """One CUDA graph for the whole step.  With several ranks the NCCL all-reduces are captured too (fork / join on
        the side stream; thread-local capture mode keeps NCCL's watchdog thread out of it).  If that capture is refused,
        fall back to two graphs around ONE eager all-reduce of the arena (no overlap)."""
        torch.cuda.synchronize()
        if self.world > 1:
            dist.barrier(group=self.pg)
        try:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                self._step_body(st["static"], det)
            return ("one", g)
        except Exception as e:
            import warnings
            torch.cuda.synchronize()
            if self.world == 1:
                warnings.warn(f"CUDA graph capture of the training step failed ({e}); continuing with eager launches")
                return None
            warnings.warn(f"CUDA graph capture with NCCL failed ({e}); using two graphs around one eager all-reduce")
        try:
            self.allreduce_mode = "one eager all-reduce of the arena between two CUDA graphs (not overlapped)"
            ga, gb = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(ga):
                for i, mb in enumerate(st["static"]):
                    self._micro_batch(mb, True, i, True, det=det)
            with torch.cuda.graph(gb, pool=ga.pool()):
                self._update_body(det)
            return ("two", ga, gb)
        except Exception as e:
            import warnings
            warnings.warn(f"CUDA graph capture of the training step failed ({e}); continuing with eager launches")
            torch.cuda.synchronize()
            return None

    def _replay(self, graphs):
        if graphs[0] == "one":
            graphs[1].replay()
        else:
            graphs[1].replay()
            allreduce_sum_(self.eng.arena_g, self.pg)
            graphs[2].replay()

    def train_step(self, micro_batches: Sequence[Sequence[torch.Tensor]]):
        """One optimiser step over `grad_accum_every` micro-batches (each a tuple of token-id tensors in
        the stage's order, e.g. (clap, semantic, coarse); host or device).  Returns the mean loss as a device
        scalar.  After two eager steps per input shape the step is replayed from ONE CUDA graph (forward, backward, the
        bucketed NCCL all-reduces on their side stream, clip, AdamW, re-pack); inputs are copied into static device
        buffers, hyper-parameters live in device memory.
        With torch.use_deterministic_algorithms(True) the step runs the fixed-order kernel variants: the same inputs,
        build, world size and GPU model (SM count) give bit-identical losses, gradient norms, parameters and Adam
        moments, eagerly and under graph replay.  The mode is part of the graph key: toggling it re-captures.
        Parameters with requires_grad=False at construction are frozen as in the reference: no gradient (their arena_g
        range stays zero), no part in the clip norm, no AdamW update, no optimizer state in save(); the backward pass
        runs only the work the trainable parameters need.
        transformer.engine.check_errors() raises if a deterministic step could not keep its order (never expected; the
        attention backward gives up waiting for an accumulation turn after seconds instead of hanging)."""
        assert len(micro_batches) == self.grad_accum_every
        eng = self.eng
        changed = sorted(n for n, p in self.transformer.named_parameters() if p.requires_grad != self._requires_grad[n])
        if changed:
            raise RuntimeError(f"requires_grad changed after this HotPathTrainer was built (for {changed[:4]}"
                               f"{' ...' if len(changed) > 4 else ''}): the frozen set is read at construction; "
                               "construct a new HotPathTrainer")
        det = torch.are_deterministic_algorithms_enabled()
        self.transformer.train()
        eng.refresh_packed()        # no-op unless the parameters were written from outside (load_state_dict, manual edits):
        self._set_hyper()           # the captured graph re-packs only after its own optimiser update
        if not self.use_cuda_graph:
            self._step_body(micro_batches, det)
            self.steps += 1
            return self.loss_out
        key = (det, frozenset(self.frozen)) + tuple(tuple(t.shape) for mb in micro_batches for t in mb)
        st = self._graphs.pop(key, None)
        if st is not None:
            self._graphs[key] = st                   # most recently used
        if st is None:
            while len(self._graphs) >= 8:            # least recently used shape: drop its graph, static buffers and workspaces
                self._graphs.pop(next(iter(self._graphs)))
            st = self._graphs[key] = dict(count=0, graphs=None, static=[
                [torch.empty(tuple(t.shape), dtype=torch.int64, device=eng.dev) for t in mb] for mb in micro_batches])
        for mb, smb in zip(micro_batches, st["static"]):
            for t, sbuf in zip(mb, smb):
                sbuf.copy_(t, non_blocking=True)
        if st["graphs"] is not None:
            self._replay(st["graphs"])
        elif st["count"] < 2:
            self._step_body(st["static"], det)
            st["count"] += 1
        else:
            st["graphs"] = self._capture(st, det)
            # a captured graph addresses the engine's plan / workspace buffers directly: keep them alive with the graph
            # even if the engine's own shape cache evicts them
            st["keepalive"] = (dict(eng._plans), dict(eng._ws))
            if st["graphs"] is None:
                self.use_cuda_graph = False
                self._step_body(st["static"], det)
            else:
                self._replay(st["graphs"])
        self.steps += 1
        return self.loss_out

    def train_step_async(self, micro_batches: Sequence[Sequence[torch.Tensor]]) -> "LossHandle":
        """train_step() plus an asynchronous device->host copy of the step's loss into pinned memory.  The returned
        handle's value() blocks only on that copy, so a training loop can log step i's loss while step i+1 is already
        running on the GPU (the usual one-step logging lag) instead of draining the stream after every step.
        The pinned slots form a ring of 4: read a handle before 4 further steps have been issued."""
        loss = self.train_step(micro_batches)
        if self._loss_ring is None:
            self._loss_ring = [torch.zeros((), dtype=torch.float32).pin_memory() for _ in range(4)]
        slot = self._loss_ring[self.steps % len(self._loss_ring)]
        slot.copy_(loss, non_blocking=True)       # stream-ordered before the next step overwrites loss_out
        ev = torch.cuda.Event()
        ev.record()
        return LossHandle(slot, ev)

    @torch.no_grad()
    def eval_loss(self, token_ids: Sequence[torch.Tensor]):
        """Wrapper forward in eval mode (no forgetful mask, no dropout): the parity configuration."""
        self.transformer.eval()
        return self._micro_batch(token_ids, False, 0, False, det=torch.are_deterministic_algorithms_enabled())

    def grad_norm(self):
        return torch.sqrt(self.eng.sumsq).float()

    # ------------------------------------------------------------------------------------------- checkpoint FILES
    def _torch_optimizer(self):
        """The torch optimizer the reference's get_optimizer builds over the module's parameters (optimizer.py:10-34):
        with wd == 0 one Adam group in module order, else AdamW with ndim >= 2 decayed and the rest not — used only to
        read / write the reference's optimizer checkpoint format."""
        params = list(self.transformer.parameters())
        if self.wd == 0:
            return torch.optim.Adam(params, lr=self.lr, betas=tuple(self.betas), eps=self.eps), params
        wd_params = [p for p in params if p.ndim >= 2]
        no_wd = [p for p in params if p.ndim < 2]
        opt = torch.optim.AdamW([{"params": wd_params}, {"params": no_wd, "weight_decay": 0}], lr=self.lr, weight_decay=self.wd,
                                betas=tuple(self.betas), eps=self.eps)
        return opt, wd_params + no_wd

    def _lr_factor(self, steps):
        return 1.0 if self.lr_warmup <= 0 else 1e-7 + (1.0 - 1e-7) * min(steps, self.lr_warmup) / self.lr_warmup

    def save(self, model_path, optim_path, scheduler_path=None):
        """SingleStageTrainer.save (trainer.py:359-372): transformer state_dict, torch AdamW state_dict, LinearLR state_dict —
        files the reference's trainer (and scripts/train_utils.py) can load back."""
        eng = self.eng
        self._gather_optimizer_state()
        torch.save({k: v.detach().clone() for k, v in self.transformer.state_dict().items()}, model_path)
        opt, ordered = self._torch_optimizer()
        name_of = {id(p): n for n, p in self.transformer.named_parameters()}
        if self.steps > 0:
            for p in ordered:
                if name_of[id(p)] in self.frozen:
                    continue                # no gradient, so torch keeps no state for it either
                o = eng.layout[name_of[id(p)]]
                opt.state[p] = {"step": torch.tensor(float(self.steps)), "exp_avg": eng.adam_m[o:o + p.numel()].view(p.shape).clone(),
                                "exp_avg_sq": eng.adam_v[o:o + p.numel()].view(p.shape).clone()}
        sched = None
        if self.lr_warmup > 0:
            sched = torch.optim.lr_scheduler.LinearLR(opt, start_factor=1e-7, end_factor=1.0, total_iters=self.lr_warmup)
            lr_now = self.lr * self._lr_factor(self.steps)
            sched.last_epoch, sched._step_count = self.steps, self.steps + 1
            sched._last_lr = [lr_now for _ in opt.param_groups]
            for g in opt.param_groups:
                g["lr"] = lr_now
        torch.save(opt.state_dict(), optim_path)
        if sched is not None:
            assert scheduler_path is not None, "lr_warmup is used: a scheduler checkpoint path is needed"
            torch.save(sched.state_dict(), scheduler_path)

    def load(self, model_path, optim_path, scheduler_path=None, steps=0):
        """SingleStageTrainer.load (trainer.py:374-391): accepts the reference's own checkpoint files."""
        eng = self.eng
        self.transformer.load_state_dict(torch.load(model_path, map_location=eng.dev))
        opt, ordered = self._torch_optimizer()
        opt.load_state_dict(torch.load(optim_path, map_location=eng.dev))
        name_of = {id(p): n for n, p in self.transformer.named_parameters()}
        eng.adam_m.zero_(); eng.adam_v.zero_()
        opt_steps = 0
        for p in ordered:
            st = opt.state.get(p)
            if st:
                o = eng.layout[name_of[id(p)]]
                eng.adam_m[o:o + p.numel()].view(p.shape).copy_(st["exp_avg"])
                eng.adam_v[o:o + p.numel()].view(p.shape).copy_(st["exp_avg_sq"])
                opt_steps = max(opt_steps, int(float(st["step"])))
        self.steps = opt_steps
        if scheduler_path is not None and self.lr_warmup > 0:
            sd = torch.load(scheduler_path, map_location="cpu")
            self.steps = int(sd["last_epoch"])
        elif self.lr_warmup > 0:
            raise AssertionError("the config specifies lr warmup is used, but no scheduler checkpoint is given. try setting lr_warmup to 0.")
        eng.arena_g.zero_()
        eng.refresh_packed(force=True)
        return self.steps

    # ------------------------------------------------------------------------------------------- checkpointing
    def state_dict(self):
        """Optimiser / scheduler / RNG state needed to resume training exactly where it stopped (the reference's
        SingleStageTrainer.save keeps optim + scheduler state next to the model, trainer.py:359-391).
        Layout: torch.optim.AdamW-style — per-parameter 'exp_avg' / 'exp_avg_sq' keyed by the parameter's state_dict
        name plus the shared step count (the reference steps all parameters together), so it converts to a torch
        optimizer state by a dict comprehension."""
        eng = self.eng
        self._gather_optimizer_state()
        state = {}
        for n, p in self.transformer.named_parameters():
            o = eng.layout[n]
            state[n] = {"step": self.steps, "exp_avg": eng.adam_m[o:o + p.numel()].view(p.shape).clone(),
                        "exp_avg_sq": eng.adam_v[o:o + p.numel()].view(p.shape).clone()}
        return {"state": state, "steps": self.steps, "seed": int(eng.seed.item()), "mask_draws": self._mask_draws,
                "hparams": dict(lr=self.lr, lr_warmup=self.lr_warmup, wd=self.wd, betas=tuple(self.betas), eps=self.eps,
                                max_grad_norm=self.max_grad_norm, grad_accum_every=self.grad_accum_every)}

    def load_state_dict(self, sd):
        """Inverse of state_dict().  Also call after transformer.load_state_dict(): the packed 16-bit weights are
        refreshed here, so graphs captured earlier stay valid."""
        eng = self.eng
        for n, p in self.transformer.named_parameters():
            o = eng.layout[n]
            st = sd["state"][n]
            eng.adam_m[o:o + p.numel()].view(p.shape).copy_(st["exp_avg"])
            eng.adam_v[o:o + p.numel()].view(p.shape).copy_(st["exp_avg_sq"])
        self.steps = int(sd["steps"])
        eng.seed.fill_(int(sd["seed"]))
        self._mask_draws = int(sd["mask_draws"])
        eng.arena_g.zero_()
        eng.refresh_packed(force=True)
