"""KV-cache autoregressive generation for the H100 hot path, behind the reference's wrapper API.

`TokenConditionedTransformerWrapper.generate` has the signature and the sampling semantics of the reference
(open_musiclm/open_musiclm.py:253-326, utils.py:71-93): eos appended to the conditioning sequences, no key mask, eos
forbidden except at the last quantizer of a time step (when allowed), top-k filtering, Gumbel-argmax sampling,
everything after an eos masked with -1, output folded to [b, n, q].  The reference re-runs the whole prefix through
the transformer for every sampled token; here the prompt is run once (the regular wgmma forward, which also fills the
caches) and every further token costs one incremental step over
    per layer:  K/V cache [B, Nmax, 128] bf16  +  the last two pre-conv FFN rows [B, 2, 2Fp]  (CausalDSConv history)
with the weight-streaming kernels of csrc/decode.cu, replayed from one CUDA graph per quantizer index.
Up to 16 sequences per call run the SIMT kernels (skinny_gemm, attn_decode); 17 to 256 run the wgmma GEMM of
csrc/decode_gemm.cu, whose batch is the tensor cores' N operand, and attn_decode_mqa, which reads every cached row once
per sequence instead of once per head.  The choice follows from the batch size; it is not an option.

Seeded generation (`generate(seeds=...)`) takes the tensor-core path at every batch size, with the GEMM's K split fixed
independently of B (omlm_decode_gemm_invariant), and draws each sequence's noise from its own seed: the tokens of a
sequence are then a function of its own inputs and seed, not of the batch it runs in (DESIGN section 4).

Nucleus sampling (`generate(top_p=...)`) runs in the same captured step, through omlm_sample_nucleus; its semantics are
stated in `generate`'s docstring.

Prefixes of different lengths (`generate(pred_lengths=...)`) run the same step with one position per sequence
(DecodeSession.pos [B], the _ragged attention and gather entry points, omlm_decode_advance_pos in place of the
sampler's position bump); every row gets what it would get alone (DESIGN section 4).

Sampling arguments per row (temperature, filter_thres, top_p, max_time_steps given as one value per row) reach the
sampler as device arrays (DecodeSession.rows, omlm_sample_rows); rows that sample different numbers of tokens take the
per-row-position path above.  Every row again gets what it would get alone (DESIGN section 4).
"""
import math
import numbers
from typing import List, Optional, Sequence

import torch
from torch import nn

from . import lib
from .model import TokenConditionedTransformer

SKINNY_MAX_BATCH = 16      # up to here the SIMT kernels (skinny_gemm, attn_decode); above, the tensor-core path
MAX_BATCH = 256            # sequences per generate() call


class _Capture:
    """Receives the per-layer K/V rows and pre-conv FFN rows of the prompt from Engine.forward_core."""

    def __init__(self, sess):
        self.s = sess

    def after_kv(self, l, kvn):
        s = self.s
        s.cache[l][:, :s.n_prompt].copy_(kvn.view(s.B, s.n_prompt, 128))

    def after_u(self, l, u):
        s = self.s
        rows = u.view(s.B, s.n_prompt, -1)
        if s.ragged:                  # rows n_b - 2, n_b - 1 of each sequence's own prompt (zero before its first row)
            idx = s.prompt_len[:, None] + torch.arange(-2, 0, device=rows.device)
            hist = rows[torch.arange(s.B, device=rows.device)[:, None], idx.clamp_min(0)]
            s.conv[l].copy_(hist.masked_fill((idx < 0)[..., None], 0))
            return
        k = min(2, s.n_prompt)
        s.conv[l].zero_()
        s.conv[l][:, 2 - k:].copy_(rows[:, s.n_prompt - k:])


def seeds_tensor(seeds, B: int, device) -> torch.Tensor:
    """B per-sequence seeds (ints, taken modulo 2^64, or an int64 tensor read as raw 64-bit patterns) as an int64
    device tensor of those bit patterns."""
    if isinstance(seeds, torch.Tensor):
        if seeds.dtype != torch.int64:
            raise ValueError(f"open_musiclm_b200 generate: seeds must be an int64 tensor or a list of ints, not {seeds.dtype}")
        vals = seeds.reshape(-1).tolist()
    else:
        vals = [int(s) for s in seeds]
    if len(vals) != B:
        raise ValueError(f"open_musiclm_b200 generate: {len(vals)} seeds for {B} sequences")
    vals = [v & 0xFFFFFFFFFFFFFFFF for v in vals]
    return torch.tensor([v - (1 << 64) if v >= 1 << 63 else v for v in vals], dtype=torch.int64, device=device)


def check_top_p(top_p, where: str = "generate"):
    """The nucleus mass of a generate call: None or 1 (no nucleus filtering) -> None, a number in (0, 1) -> that float;
    anything else (NaN, a bool, a non-number, a value outside (0, 1]) raises ValueError."""
    if top_p is None:
        return None
    if isinstance(top_p, bool) or not isinstance(top_p, numbers.Real):
        raise ValueError(f"open_musiclm_b200 {where}: top_p must be None or a number in (0, 1], not {top_p!r}")
    p = float(top_p)
    if p == 1.0:
        return None
    if not 0.0 < p < 1.0:           # also rejects NaN
        raise ValueError(f"open_musiclm_b200 {where}: top_p must lie in (0, 1], got {top_p!r}")
    return p


def check_pred_lengths(pred_lengths, pred_token_ids, B: int):
    """generate's pred_lengths -> a list of B ints in [0, pred_token_ids.shape[1]], or None when it is None or every
    value equals pred_token_ids.shape[1] (nothing ragged: the shared-position path).  A wrong count, a value out of
    range, a non-integer or a bool, or pred_lengths without pred_token_ids raises ValueError."""
    if pred_lengths is None:
        return None
    where = "open_musiclm_b200 generate: pred_lengths"
    if pred_token_ids is None:
        raise ValueError(f"{where} needs pred_token_ids")
    if isinstance(pred_lengths, torch.Tensor):
        if pred_lengths.dtype != torch.int64 or pred_lengths.dim() != 1:
            raise ValueError(f"{where} must be a list of ints or an int64 tensor of shape [{B}], not a {pred_lengths.dtype} "
                             f"tensor of shape {list(pred_lengths.shape)}")
        vals = [int(v) for v in pred_lengths.tolist()]
    else:
        vals = list(pred_lengths)
        for v in vals:
            if isinstance(v, bool) or not isinstance(v, numbers.Integral):
                raise ValueError(f"{where} must hold ints, not {v!r}")
        vals = [int(v) for v in vals]
    if len(vals) != B:
        raise ValueError(f"{where} has {len(vals)} values for {B} sequences")
    n = pred_token_ids.shape[1]
    for b, v in enumerate(vals):
        if not 0 <= v <= n:
            raise ValueError(f"{where}[{b}] = {v} lies outside [0, {n}] (pred_token_ids has {n} time steps)")
    return None if all(v == n for v in vals) else vals


def _row_values(value, B: int, name: str, integer: bool):
    """value's per-row form (a list or tuple of B values, or a 1-D tensor of B values: int64 when integer, floating
    point otherwise) -> a list of B Python values; None for a single value (a 0-d tensor included)."""
    where = f"open_musiclm_b200 generate: {name}"
    if isinstance(value, torch.Tensor):
        if value.dim() == 0:
            return None
        if value.dim() != 1 or (value.dtype != torch.int64 if integer else not value.is_floating_point()):
            raise ValueError(f"{where} per row must be a 1-D {'int64' if integer else 'floating-point'} tensor of shape [{B}], not a "
                             f"{value.dtype} tensor of shape {list(value.shape)}")
        vals = value.tolist()
    elif isinstance(value, (list, tuple)):
        vals = list(value)
    else:
        return None
    if len(vals) != B:
        raise ValueError(f"{where} has {len(vals)} values for {B} sequences")
    return vals


def _collapse(vals):
    return vals[0] if all(v == vals[0] for v in vals) else vals


def check_sampling_rows(B: int, C: int, temperature, filter_thres, top_p, max_time_steps):
    """generate's temperature, filter_thres, top_p and max_time_steps, each one value or one value per row ->
    (temperature, top_k, top_p, max_time_steps): a single value each (top_k None: filter_thres is a single value, unchecked;
    top_p through check_top_p; temperature and max_time_steps as given), or a list of B checked values (floats, the
    top-k sizes max(int((1 - filter_thres) C), 1), floats or None, ints).  A list whose values are all equal collapses to that value.  A wrong count, a bool or a non-number,
    a temperature that is not finite and > 0, a filter_thres that is not finite or gives k > C, a bad top_p element or
    a max_time_steps element that is not a non-negative int raises ValueError naming the keyword."""
    def number(name, v, integer=False):
        if isinstance(v, bool) or not isinstance(v, numbers.Integral if integer else numbers.Real):
            raise ValueError(f"open_musiclm_b200 generate: {name} must hold {'ints' if integer else 'numbers'}, not {v!r}")
        return int(v) if integer else float(v)

    temps = _row_values(temperature, B, "temperature", False)
    if temps is not None:
        temps = [number("temperature", v) for v in temps]
        for b, t in enumerate(temps):
            if not (math.isfinite(t) and t > 0):
                raise ValueError(f"open_musiclm_b200 generate: temperature[{b}] = {t!r} is not a finite number > 0")
        temperature = _collapse(temps)
    thres = _row_values(filter_thres, B, "filter_thres", False)
    top_k = None
    if thres is not None:
        top_k = []
        for b, t in enumerate(number("filter_thres", v) for v in thres):
            k = max(int((1 - t) * C), 1) if math.isfinite(t) else None                           # utils.py:80
            if k is None or k > C:
                raise ValueError(f"open_musiclm_b200 generate: filter_thres[{b}] = {t!r} does not give a top-k size in [1, {C}]")
            top_k.append(k)
        top_k = _collapse(top_k)
    ps = _row_values(top_p, B, "top_p", False)
    top_p = check_top_p(top_p) if ps is None else _collapse([check_top_p(p) for p in ps])
    steps = _row_values(max_time_steps, B, "max_time_steps", True)
    if steps is not None:
        steps = [number("max_time_steps", v, integer=True) for v in steps]
        for b, n in enumerate(steps):
            if n < 0:
                raise ValueError(f"open_musiclm_b200 generate: max_time_steps[{b}] = {n} is negative")
        max_time_steps = _collapse(steps)
    return temperature, top_k, top_p, max_time_steps


class DecodeSession:
    """Caches and scratch of one generate() call: B sequences, a prompt of n_prompt positions, up to n_new new tokens.
    seeded: batch-invariant mode (tensor-core path with the B-independent GEMM split at every B, per-sequence seeds in
    self.seeds).  pred_start: position of the predicted sequence's start token in the prompt (_Plan.pos0[-1]); with
    absolute position embeddings the token at position pos is token pos - pred_start - 1 of that sequence.
    ragged (prompts of different lengths): (prompt_len, pos_init, pos_last), B ints each: sequence b's real prompt
    length, its first decode position and the last position it processes; self.pos is then one position per sequence
    and n_max the cache capacity.  Otherwise self.pos is one counter for the whole batch, starting at n_prompt.
    rows (sampling arguments per sequence): (top_k, temperature, top_p), B values each (top_p None: no nucleus);
    self.rows then holds them as device arrays, which every sample() reads instead of its scalar arguments.
    logprob: the sampler also writes each token's two log-probabilities into self.lp and self.slp (fp32 [B, n_new], in
    the allocation of self.tokens, right after it, as omlm_sample_logprob requires)."""

    def __init__(self, eng, B: int, n_prompt: int, n_new: int, seeded: bool = False, pred_start: int = 0, ragged=None,
                 n_max: Optional[int] = None, rows=None, logprob: bool = False):
        if B > MAX_BATCH:
            raise lib.OmlmError(f"open_musiclm_b200 generate: batch sizes above {MAX_BATCH} are not supported by the decode kernels")
        if seeded and eng.h > 16:
            raise lib.OmlmError(f"open_musiclm_b200 generate: seeded generation supports at most 16 heads ({eng.h} given)")
        self.eng, self.B, self.n_prompt, self.n_new, self.seeded = eng, B, n_prompt, n_new, seeded
        dev, bf, f32, a16 = eng.dev, torch.bfloat16, torch.float32, eng.a16
        d, HD, Fp, h, Hr = eng.d, eng.HD, eng.Fp, eng.h, eng.Hr
        self.n_max = n_prompt + n_new if n_max is None else n_max
        E = lambda *shape, dt=bf: torch.empty(*shape, device=dev, dtype=dt)
        self.cache = [E(B, self.n_max, 128) for _ in range(eng.L)]
        self.conv = [E(B, 2, 2 * Fp, dt=a16) for _ in range(eng.L)]
        self.x = [E(B, d, dt=f32) for _ in range(2)]
        self.q_raw, self.kv_raw, self.o = E(B, HD), E(B, 128), E(B, HD)
        self.u_new, self.h = E(B, 2 * Fp, dt=a16), E(B, Fp, dt=a16)
        self.rowsum = E(B, Fp // 128, 2, dt=f32)
        self.logits = E(B, max(eng.Cp), dt=f32)
        W = max(n_new, 1)
        self.logprob = logprob
        self.lp = self.slp = None
        if logprob:              # the samplers' layout: tokens [B, W] int64, then lp and slp [B, W] fp32 each
            self.tokens, self.lp, self.slp = lib.logprob_buffers(B, W, dev)
        else:
            self.tokens = torch.zeros(B, W, device=dev, dtype=torch.int64)
        self.next_row = torch.zeros(B, device=dev, dtype=torch.int32)
        self.counters = torch.zeros(2, device=dev, dtype=torch.int32)          # [sampled so far, block arrival counter]
        self.ragged = ragged is not None
        if self.ragged:          # per sequence: the position the next decode step processes, and the last one it will
            i32 = lambda v: torch.tensor(v, device=dev, dtype=torch.int32)
            self.prompt_len = torch.tensor(ragged[0], device=dev, dtype=torch.int64)
            self.pos, self.pos_last = i32(ragged[1]), i32(ragged[2])
        else:
            self.pos = torch.full((1,), n_prompt, device=dev, dtype=torch.int32)   # position the next decode step processes
        self.pos_offset = -(pred_start + 1)
        self.rows = None
        if rows is not None:     # filled here, before any graph capture; top_p_rows only when some row has a nucleus
            k, t, p = rows
            self.rows = dict(top_k_rows=torch.tensor(k, device=dev, dtype=torch.int32),
                             temperature_rows=torch.tensor(t, device=dev, dtype=f32),
                             top_p_rows=None if all(v is None for v in p) else
                             torch.tensor([1.0 if v is None else v for v in p], device=dev, dtype=f32))
        # bias table for every distance the generation can reach (it depends on i - j only)
        N = self.n_max
        self.rp = dict(rp_in=E(N, 1, dt=f32), rp_z=[E(N, Hr, dt=f32) for _ in range(3)], rp_a=[E(N, Hr, dt=f32) for _ in range(3)],
                       table=E(h, N, dt=f32), rp_a3=[E(N, 3 * eng.Hr8) for _ in range(2)])
        lib.arange_f32(self.rp["rp_in"])
        eng.refresh_packed()
        if eng.bias_type == "none":
            self.rp["table"].zero_()
        elif eng.bias_type == "t5":
            self.rp["ones"] = torch.ones(N, device=dev, dtype=f32)
        eng.build_bias_table(self.rp, N)
        self.table = self.rp["table"]
        self._graphs = {}
        # more than 16 sequences, or seeded mode: tensor-core GEMMs and the cache-sharing attention, with their scratch
        # allocated here so that graph capture allocates nothing
        self.batched = B > SKINNY_MAX_BATCH or seeded
        self.seeds = torch.zeros(B, device=dev, dtype=torch.int64) if seeded else None
        if self.batched:
            shapes = [(HD, d), (128, d), (d, HD), (2 * Fp, d), (d, Fp)] + [(cp, d) for cp in eng.Cp]
            self.ws = lib.DecodeWorkspace(dev, B, shapes, max_pos=self.n_max, heads=h, invariant=seeded)

    # ------------------------------------------------------------------------------------------ one incremental step
    def embed(self, x):
        """x = the input rows of the position self.pos: embedding row self.next_row, plus with absolute position
        embeddings the predicted sequence's row for its token self.pos - pred_start - 1 (open_musiclm.py:134-136)."""
        eng = self.eng
        if eng.abs_pos:
            lib.embed_gather_pos(eng.table, self.next_row, self.pos, self.pos_offset, eng.abs_row_base[-1], eng.max_abs_pos, x,
                                 ragged=self.ragged)
        else:
            lib.embed_gather(eng.table, self.next_row, x)

    def step(self, qi_next: int):
        """Processes the position self.pos (embedding row self.next_row) through all layers and leaves the logits of
        head qi_next in self.logits (one launch per operation)."""
        if self.batched:
            return self.step_batched(qi_next)
        eng, B = self.eng, self.B
        pv, d, HD, F, Fp, h = eng.pview, eng.d, eng.HD, eng.F, eng.Fp, eng.h
        xa, xm = self.x
        self.embed(xa)
        for l in range(eng.L):
            p, pk = f"transformer.layers.{l}.", eng.pk[l]
            lib.skinny_gemm(xa, pk["wq"], self.q_raw, prologue=2, gamma=pv[p + "0.norm.gamma"])
            lib.skinny_gemm(xa, pk["wkv_b"], self.kv_raw, prologue=1)
            lib.attn_decode(self.q_raw, self.kv_raw, pv[p + "0.q_scale"], pv[p + "0.k_scale"], self.cache[l], self.table, self.pos,
                            self.n_max, self.o, h, ragged=self.ragged)
            lib.skinny_gemm(self.o, pk["wo_b"], xm, addend=xa)
            lib.skinny_gemm(xm, pk["w1"], self.u_new, prologue=2, gamma=pv[p + eng.ffk["g1"]])
            lib.decode_conv_geglu(self.u_new, self.conv[l], pk["conv"], self.h, self.rowsum)
            lib.skinny_gemm(self.h, pk["w2"], xa, prologue=3, gamma=pk["gin"], rowsum=self.rowsum, n_real=F, addend=xm)
        S = len(eng.seqs) - 1
        lib.skinny_gemm(xa, eng.pk_logit[S][qi_next], self.logits[:, :eng.Cp[S]], prologue=2, gamma=pv["transformer.norm.gamma"])

    def step_batched(self, qi_next: int):
        """step for more than 16 sequences (or seeded mode): the same operations on the tensor-core GEMM and the
        cache-sharing attention (same rounding points; fp32 sums in another order).  Seeded mode fixes the GEMMs' K split
        independently of B; attn_decode_mqa's per-sequence CTAs already are."""
        eng, ws, inv = self.eng, self.ws, self.seeded
        pv, F, h = eng.pview, eng.F, eng.h
        xa, xm = self.x
        self.embed(xa)
        for l in range(eng.L):
            p, pk = f"transformer.layers.{l}.", eng.pk[l]
            lib.decode_gemm(xa, pk["wq"], self.q_raw, prologue=2, gamma=pv[p + "0.norm.gamma"], ws=ws, invariant=inv)
            lib.decode_gemm(xa, pk["wkv_b"], self.kv_raw, prologue=1, ws=ws, invariant=inv)
            lib.attn_decode_mqa(self.q_raw, self.kv_raw, pv[p + "0.q_scale"], pv[p + "0.k_scale"], self.cache[l], self.table, self.pos,
                                self.n_max, self.o, h, ws=ws, ragged=self.ragged)
            lib.decode_gemm(self.o, pk["wo_b"], xm, addend=xa, ws=ws, invariant=inv)
            lib.decode_gemm(xm, pk["w1"], self.u_new, prologue=2, gamma=pv[p + eng.ffk["g1"]], ws=ws, invariant=inv)
            lib.decode_conv_geglu(self.u_new, self.conv[l], pk["conv"], self.h, self.rowsum)
            lib.decode_gemm(self.h, pk["w2"], xa, prologue=3, gamma=pk["gin"], rowsum=self.rowsum, n_real=F, addend=xm, ws=ws, invariant=inv)
        S = len(eng.seqs) - 1
        lib.decode_gemm(xa, eng.pk_logit[S][qi_next], self.logits[:, :eng.Cp[S]], prologue=2, gamma=pv["transformer.norm.gamma"], ws=ws,
                        invariant=inv)

    def sample(self, qi: int, top_k: int, temperature: float, allow_eos: bool, uniform, seed, bump_pos: bool, top_p=None):
        eng = self.eng
        S = len(eng.seqs) - 1
        q, cb = eng.seqs[S].num_quantizers, eng.seqs[S].codebook_size
        row_offset = eng.emb_row_base[S] + (cb * qi if q > 1 else 0)
        pos = self.pos if bump_pos and not self.ragged else None
        if self.rows is not None:        # per-row arguments: top_k, temperature and top_p are not used
            lib.sample(self.logits, eng.C[S], 1, 1.0, allow_eos, uniform, seed, self.tokens, self.next_row, row_offset,
                       self.counters, pos, self.B, seeds=self.seeds, logprobs=self.lp, sample_logprobs=self.slp, **self.rows)
        else:
            lib.sample(self.logits, eng.C[S], top_k, temperature, allow_eos, uniform, seed, self.tokens, self.next_row, row_offset,
                       self.counters, pos, self.B, seeds=self.seeds, top_p=top_p, logprobs=self.lp, sample_logprobs=self.slp)
        if bump_pos and self.ragged:
            lib.decode_advance_pos(self.pos, self.pos_last)

    def step_and_sample(self, qi: int, qi_next: int, top_k, temperature, allow_eos_next, uniform, seed, use_graph=True, top_p=None):
        """decode step on the token sampled for quantizer slot qi, then sample the token of slot qi_next."""
        if self.rows is not None:        # the arrays' contents are read at replay; only the kernel choice is captured
            key = (qi, qi_next, "rows", bool(allow_eos_next), uniform is not None, self.seeded, self.rows["top_p_rows"] is not None,
                   self.logprob)
        else:
            key = (qi, qi_next, top_k, float(temperature), bool(allow_eos_next), uniform is not None, self.seeded, top_p, self.logprob)
        g = self._graphs.get(key)
        if g is None or not use_graph:
            body = lambda: (self.step(qi_next), self.sample(qi_next, top_k, temperature, allow_eos_next, uniform, seed, True, top_p))
            if not use_graph:
                body()
                return
            count = self._graphs.get(("warm",) + key, 0)
            if count < 1:                 # one eager run first (lazy cudaFuncSetAttribute calls are not capturable)
                body()
                self._graphs[("warm",) + key] = count + 1
                return
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                body()
            self._graphs[key] = g
        g.replay()


def prefix_labels(prompt, q: int, C: int):
    """int32 [B, n + q] labels of the predicted sequence's prompt tokens [B, n] for omlm_token_logprob, padded with -100
    (a label outside [0, C) is not scored): group qi's row t predicts flat token t q + qi, read through the strided view
    (offset qi, stride q, one row of n + q per sequence), so its last row (the next token) reads the padding."""
    B, n = prompt.shape
    lab = torch.full((B, n + q), -100, device=prompt.device, dtype=torch.int32)
    lab[:, :n] = torch.where((prompt >= 0) & (prompt < C), prompt, -100).to(torch.int32)
    return lab


def prefix_logprobs(eng, pl, ws, prompt, q: int, C: int):
    """[B, n] float32: the log-probability of every prompt token of the predicted sequence under the prefill's logits row
    for its position (the head groups ws["logits"][gi] of the last sequence; the row that predicts the next token is
    not scored)."""
    B, n = prompt.shape
    S = len(eng.seqs) - 1
    lab = prefix_labels(prompt, q, C)
    out = torch.zeros(B, n, device=prompt.device, dtype=torch.float32)
    for gi, (s, qi, cnt, base) in enumerate(pl.groups):
        m = len(range(qi, n, q))
        if s != S or m == 0:
            continue
        row = torch.empty(B * cnt, device=prompt.device, dtype=torch.float32)
        lib.token_logprob(ws["logits"][gi], lab.view(-1)[qi:], C, row, label_stride=q, rows_per_batch=cnt, batch_stride=n + q)
        out[:, qi::q] = row.view(B, cnt)[:, :m]
    return out


def assemble_logprobs(sampled, pre_lp, lp_new, slp_new, n_real, n_end):
    """The [B, W] logprobs and sample_logprobs of generate's flat output `sampled` (after the eos masking): row b's
    columns below n_real[b] are prefix tokens (pre_lp [B, >= their count], sample log p 0), columns n_real[b] ...
    n_end[b] - 1 its samples in order (lp_new, slp_new [B, n_new]; None when nothing was sampled), and every column
    that holds -1 is 0 in both.  n_real, n_end: int64 [B, 1]."""
    B, W = sampled.shape
    col = torch.arange(W, device=sampled.device)[None]
    lp = torch.zeros(B, W, device=sampled.device, dtype=torch.float32)
    w = min(W, pre_lp.shape[1])
    lp[:, :w] = pre_lp[:, :w]
    lp.masked_fill_(col >= n_real, 0.0)
    slp = torch.zeros_like(lp)
    if lp_new is not None:
        in_new = (col >= n_real) & (col < n_end)
        src = (col - n_real).clamp(0, lp_new.shape[1] - 1).expand(B, -1)
        lp = torch.where(in_new, lp_new.gather(1, src), lp)
        slp = torch.where(in_new, slp_new.gather(1, src), slp)
    gone = sampled == -1
    return lp.masked_fill(gone, 0.0), slp.masked_fill(gone, 0.0)


class TokenConditionedTransformerWrapper(nn.Module):
    """open_musiclm.py:219-411 on the H100 path: `generate` (KV-cache decode) and `forward` (loss / logits)."""

    def __init__(self, *, transformer: TokenConditionedTransformer, pad_id=-1, unique_consecutive=True,
                 cross_entropy_loss_weights: Optional[List[float]] = None, mask_prob=0.15):
        super().__init__()
        self.transformer = transformer
        self.token_sequences = transformer.token_sequences
        self.unique_consecutive = unique_consecutive
        self.pad_id = pad_id
        self.cross_entropy_loss_weights = cross_entropy_loss_weights if cross_entropy_loss_weights is not None else [1 for _ in self.token_sequences]
        self.eos_ids = transformer.eos_ids
        self.mask_prob = mask_prob
        assert len(self.token_sequences) == len(self.eos_ids) == len(self.cross_entropy_loss_weights)
        if any(s.unique_consecutive for s in self.token_sequences):
            raise NotImplementedError("open_musiclm_b200: unique_consecutive token sequences are not supported")
        self._trainer = None

    @property
    def device(self):
        return self.transformer.device

    @torch.no_grad()
    def generate(self, *, conditioning_token_ids: List[torch.Tensor], pred_token_ids: Optional[torch.Tensor] = None,
                 max_time_steps=512, filter_thres=0.9, temperature=1., include_eos_in_output=False,
                 append_eos_to_conditioning_tokens=True, allow_eos_in_output=False, uniform_noise: Optional[torch.Tensor] = None,
                 use_cuda_graph=True, trace_logits: Optional[list] = None, seeds=None, top_p=None, pred_lengths=None,
                 return_logprobs=False, **kwargs):
        """Same contract as open_musiclm.py:253-326.  uniform_noise (optional, [n_sampled, b, codebook+1] in (0, 1)):
        the uniform draws behind the Gumbel noise, one slice per sampled token in order — parity runs pass the stream
        torch's default CPU generator would have produced; by default the noise comes from a device Philox stream keyed
        by Engine.seed, which every unseeded call advances.
        seeds (optional): one unsigned 64-bit seed per sequence (a list of ints, or an int64 tensor read as raw bits).
        The tokens of sequence b, and the logits they were sampled from, are then a function only of the weights, that
        sequence's conditioning and prefix, seeds[b] and the sampling arguments: not of the batch size, the row, the other
        rows, CUDA-graph or eager execution, or earlier calls (on one GPU model and build; DESIGN section 4).  Engine.seed
        is left untouched.  seeds=torch.randint(2**62, (b,)) puts generation under torch.manual_seed.  Excludes
        uniform_noise.
        Absolute position embeddings (use_absolute_position_embeddings=True): every token gets the row of its own
        position within its own sequence, counted from 0, as in the reference's full forward; the row of a fed-back
        token depends only on that sequence's prefix length and step, so seeded generation stays independent of the
        batch.  As the reference's nn.Embedding lookup would, IndexError is raised (before anything runs, Engine.seed
        untouched) when a conditioning sequence with its eos holds more than max_absolute_position_embeddings tokens,
        or when prefix length + n_new - 1 exceeds it (the last sampled token is never fed back).
        top_p (optional, nucleus sampling, Holtzman et al. 2019): for one row, with eos forbidden as above and the top-k
        set K chosen as above (exactly k entries; among values equal to the k-th largest the lower index wins; -0.0
        equals +0.0), let p_c = softmax(l / temperature) over K, the distribution the Gumbel-argmax samples from.  The
        nucleus is N = {c in K : sum of p_j over j in K with l_j > l_c < top_p}: the smallest prefix of K, by value,
        whose mass reaches top_p, extended to include ties (equal values are all in N or all out; the most likely token
        is always in).  The token is the argmax over N of l_c / temperature + g_c, where g_c comes from exactly the
        uniform the sampler uses without top_p (uniform_noise, the Engine.seed stream, or the sequence's seed); classes
        outside N are skipped.  A NaN logit is never in N and adds no mass; a row with no finite logit in K samples as
        without top_p.  N depends only on the row, so seeded generation stays independent of the batch.  None or 1.0:
        no nucleus filtering, bit-identical to a call without top_p.  Any other value must lie in (0, 1); NaN, a bool or
        an out-of-range value raises ValueError before anything runs (Engine.seed untouched).
        pred_lengths (optional, prefixes of different lengths in one batch): one int per row (a list, or an int64 tensor
        of shape [b]); pred_lengths[r] is the number of leading time steps of pred_token_ids[r] that are real, a whole
        number in [0, pred_token_ids.shape[1]].  The steps after it are padding and are never read, whatever they hold
        (-1 included).  Row r is then generated exactly as a call with that row alone and its first pred_lengths[r]
        steps as pred_token_ids would generate it: (max_time_steps - pred_lengths[r]) * q sampled tokens after its own
        prefix, eos masking per row, the output [b, max(max_time_steps, max(pred_lengths)), q] (rows shorter than that,
        which only happens when a prefix is longer than max_time_steps, end in -1).  The decode loop runs as many steps
        as the row with the most tokens to sample; a row that has all its tokens keeps its position and its further
        samples are discarded.  Sample index t of a row is its own t-th sampled token: with seeds, row r's tokens
        depend only on its conditioning, its real prefix, seeds[r] and the sampling arguments, on both decode paths;
        uniform_noise is [max over rows of n_new, b, codebook+1], row r using its first n_new slices.  With absolute
        position embeddings the IndexError check above applies per row, to the rows that sample.  A wrong count, a value
        out of range, a non-integer or a bool, or pred_lengths without pred_token_ids raises ValueError before anything
        runs (Engine.seed untouched).  None, or every value equal to pred_token_ids.shape[1]: exactly the call without
        it.  trace_logits then holds every row's logits at every step; a row past its last token holds discarded values.
        Sampling arguments per row: temperature, filter_thres and top_p each take one value for every row (as above) or
        one per row, a list or tuple of b values or a 1-D floating-point tensor of shape [b] (top_p: None or 1 in a list,
        1.0 in a tensor, means no nucleus for that row); max_time_steps likewise, as ints or an int64 tensor.  Row r is
        then generated exactly as a call with that row alone would generate it with the scalars temperature=float(v[r]),
        filter_thres=float(v[r]), top_p=v[r], max_time_steps=int(v[r]), its own conditioning, real prefix and seed, and
        every other argument shared: n_new_r = max(0, (max_time_steps_r - len_r) q) sampled tokens, the t-th with
        sample index t, eos masking per row; the output is [b, W, q] with W = max over rows of max(max_time_steps_r,
        len_r), rows ending in -1 as with pred_lengths, and uniform_noise is [max_r n_new_r, b, codebook+1].  Rows that
        sample different numbers of tokens run the pred_lengths path (a row with all its tokens stops).  A wrong count,
        a bool or a non-number, a temperature that is not finite and > 0, a filter_thres that is not finite or whose top-k
        size exceeds codebook+1, a top_p element outside (0, 1] or a negative max_time_steps raises ValueError before
        anything runs (Engine.seed untouched).  A list of equal values is that single value, so with all four equal and
        no ragged pred_lengths the call is exactly the single-value call.
        return_logprobs (a bool): True returns (tokens, logprobs, sample_logprobs), three [b, n, q] tensors, the two new
        ones float32 on the device.  logprobs[b, i, j] is the model's log-probability of the token at [b, i, j] given
        everything before it: l_c - (m + log sum_j exp(l_j - m)) over the fp32 logits row the engine computed for that
        position (all codebook+1 classes, eos included, before eos masking, temperature, top-k and top-p): for a sampled
        token the row it was sampled from (the row trace_logits copies), for a prefix token the prefill's row at its
        position.  sample_logprobs[b, i, j] is the log-probability of a sampled token under the distribution it was drawn
        from, (l_c - m_S) / T - log sum_{j in S} exp((l_j - m_S) / T) with S the candidate set the sampler builds (eos rule,
        top-k set K, then the nucleus N with top_p; NaN entries never in S, -inf entries add no mass), the row's own k, T
        and top_p; the 24-bit uniforms' discretisation is not modelled.  Prefix tokens have sample_logprobs 0, and every
        position whose token is -1 has 0 in both.  The tokens are bit-identical to the call without return_logprobs.  With
        nothing to sample the prefill still runs, so generate(pred_token_ids=x, max_time_steps=x.shape[1],
        return_logprobs=True) scores the given sequence x teacher-forced (any codebook size).  Seeded rows' values depend
        only on that row, as its tokens do.
        trace_logits (tests): receives a copy of the [b, codebook+1] logits every token was sampled from."""
        if kwargs:
            raise NotImplementedError(f"open_musiclm_b200 generate: unsupported arguments {sorted(kwargs)}")
        if not isinstance(return_logprobs, bool):
            raise ValueError(f"open_musiclm_b200 generate: return_logprobs must be a bool, not {return_logprobs!r}")
        if seeds is not None and uniform_noise is not None:
            raise ValueError("open_musiclm_b200 generate: seeds and uniform_noise exclude each other")
        B = conditioning_token_ids[0].shape[0]
        info, eos = self.token_sequences[-1], self.eos_ids[-1]
        C = info.codebook_size + 1
        temperature, top_k, top_p, max_time_steps = check_sampling_rows(B, C, temperature, filter_thres, top_p, max_time_steps)
        lengths = check_pred_lengths(pred_lengths, pred_token_ids, B)                               # None: one length
        per_row = any(isinstance(v, list) for v in (temperature, top_k, top_p))     # sampled from per-row arrays
        m, eng = self.transformer, self.transformer.engine
        S = len(self.token_sequences)
        assert len(conditioning_token_ids) == S - 1
        q = info.num_quantizers
        init_step = pred_token_ids.shape[1] if pred_token_ids is not None else 0                    # :276
        steps_b = max_time_steps if isinstance(max_time_steps, list) else [max_time_steps] * B
        if isinstance(max_time_steps, list) or lengths is not None:
            n_new_b = [max(0, (t - n) * q) for t, n in zip(steps_b, lengths or [init_step] * B)]   # per row, :276
            if lengths is None and len(set(n_new_b)) > 1:
                lengths = [init_step] * B        # rows that sample different numbers of tokens: the per-row-position path
            n_new = max(n_new_b)
        else:
            n_new = max(0, (max_time_steps - init_step) * q)
        if eng.abs_pos and n_new > 0:
            # the reference looks up arange(len) in each sequence's nn.Embedding(max_absolute_position_embeddings)
            lim = eng.max_abs_pos
            for s, t in enumerate(conditioning_token_ids):
                n = t.numel() // B + (1 if append_eos_to_conditioning_tokens else 0)
                if n > lim:
                    raise IndexError(f"open_musiclm_b200 generate: conditioning sequence {s} has {n} tokens but "
                                     f"max_absolute_position_embeddings is {lim}")
            if lengths is None:
                n_pre = pred_token_ids.numel() // B if pred_token_ids is not None else 0
                if n_pre + n_new - 1 > lim:
                    raise IndexError(f"open_musiclm_b200 generate: the predicted sequence reaches {n_pre + n_new - 1} tokens "
                                     f"({n_pre} given + {n_new} sampled - 1) but max_absolute_position_embeddings is {lim}")
            else:
                for b, (n, k) in enumerate(zip(lengths, n_new_b)):          # only rows that sample feed tokens back
                    if k > 0 and n * q + k - 1 > lim:
                        raise IndexError(f"open_musiclm_b200 generate: the predicted sequence of row {b} reaches {n * q + k - 1} "
                                         f"tokens ({n * q} given + {k} sampled - 1) but max_absolute_position_embeddings is {lim}")
        was_training = m.training
        m.eval()
        dev = eng.dev
        cond = [t.to(dev, torch.int64).reshape(B, -1) for t in conditioning_token_ids]
        if append_eos_to_conditioning_tokens:                                                       # :288-290
            cond = [torch.cat([t, torch.full((B, 1), e, device=dev, dtype=torch.int64)], 1) for t, e in zip(cond, self.eos_ids)]
        if pred_token_ids is not None:
            assert pred_token_ids.shape[0] == B
            prefix = pred_token_ids.to(dev, torch.int64).reshape(B, -1)
        else:
            prefix = torch.empty(B, 0, device=dev, dtype=torch.int64)
        seed_vals = seeds_tensor(seeds, B, dev) if seeds is not None else None
        if lengths is not None:
            # the prompt: the prefixes cut to the longest real prefix of a row that samples (a row that samples nothing
            # takes part cut to it), right-padded with token 0.  The predicted sequence comes last, so causal attention
            # keeps every real position away from the padding and the prefill runs unchanged.
            n_real = torch.tensor(lengths, device=dev, dtype=torch.int64)[:, None] * q
            Lp = max([n for n, k in zip(lengths, n_new_b) if k > 0], default=0)
            if return_logprobs:              # every real prefix token needs its prefill row
                Lp = max(Lp, max(lengths))
            L_eff = [min(n, Lp) for n in lengths]
            prompt = prefix[:, :Lp * q].masked_fill(torch.arange(Lp * q, device=dev)[None] >= n_real.clamp(max=Lp * q), 0)
        else:
            prompt = prefix
        pre_lp = None
        if n_new > 0 or (return_logprobs and prompt.shape[1] > 0):
            ids = cond + [prompt]
            _, src_row, key_mask, _, n_tok = lib.token_plan(
                ids, [s.codebook_size for s in eng.seqs], [s.num_quantizers for s in eng.seqs], eng.emb_row_base, eng.start_row,
                append_eos=False, drop_last=False, mask_cond=False, want_labels=False, err_flag=eng.err_flag)
            pl = eng.plan(B, n_tok)
            sess = None
        if n_new > 0:
            if top_k is None:
                top_k = max(int((1 - filter_thres) * C), 1)                                          # utils.py:80
            rows = None
            if per_row:                          # every argument as B values (a single value repeated)
                rows = tuple(v if isinstance(v, list) else [v] * B for v in (top_k, temperature, top_p))
            if lengths is None:
                sess = DecodeSession(eng, B, pl.N, n_new, seeded=seed_vals is not None, pred_start=pl.pos0[-1], rows=rows,
                                     logprob=return_logprobs)
            else:
                # per row: real prompt length, last position the row processes (a row with all its tokens stays there),
                # first decode position; the cache holds the longest prompt and every row's new positions
                P = [pl.pos0[-1] + 1 + n * q for n in L_eff]
                pos_last = [p + max(k, 1) - 2 for p, k in zip(P, n_new_b)]
                sess = DecodeSession(eng, B, pl.N, n_new, seeded=seed_vals is not None, pred_start=pl.pos0[-1],
                                     ragged=(P, [min(p, e) for p, e in zip(P, pos_last)], pos_last),
                                     n_max=max([pl.N] + [p + k for p, k in zip(P, n_new_b)]), rows=rows, logprob=return_logprobs)
            if seed_vals is not None:
                sess.seeds.copy_(seed_vals)
        if n_new > 0 or (return_logprobs and prompt.shape[1] > 0):
            ws = eng.workspace(pl, False)
            eng.forward_core(pl, ws, src_row, key_mask, False, {S - 1}, False, capture=_Capture(sess) if sess is not None else None)
            if return_logprobs and prompt.shape[1] > 0:
                pre_lp = prefix_logprobs(eng, pl, ws, prompt, q, C)
        if n_new > 0:
            # logits of the prompt's last position: final sequence, position p_last = its token count, head p_last mod q
            # (per row: its own last real position; every prefix is whole time steps, so the head is the same)
            p_last = n_tok[-1]
            gi = next(i for i, (s, qi, cnt, base) in enumerate(pl.groups) if s == S - 1 and qi == p_last % q)
            cnt = pl.groups[gi][2]
            last = p_last // q if lengths is None else torch.tensor(L_eff, device=dev)
            rows = torch.arange(B, device=dev) * cnt + last
            sess.logits[:, :eng.Cp[S - 1]].copy_(ws["logits"][gi][rows])
            uni = None
            if uniform_noise is not None:
                uni = uniform_noise.to(dev, torch.float32).contiguous()
                assert uni.shape == (n_new, B, info.codebook_size + 1), uni.shape
            p0 = prompt.shape[1]                                     # flat index of the first sampled token
            allow = lambda p: bool(allow_eos_in_output and (p % q) == q - 1)                        # :311-313
            if trace_logits is not None:
                trace_logits.append(sess.logits[:, :C].clone())
            sess.sample(p0 % q, top_k, temperature, allow(p0), uni, eng.seed, bump_pos=False, top_p=top_p)
            for s in range(1, n_new):
                p = p0 + s
                if trace_logits is not None:      # eager, in two halves, so that the logits can be copied in between
                    sess.step(p % q)
                    trace_logits.append(sess.logits[:, :C].clone())
                    sess.sample(p % q, top_k, temperature, allow(p), uni, eng.seed, True, top_p=top_p)
                else:
                    sess.step_and_sample((p - 1) % q, p % q, top_k, temperature, allow(p), uni, eng.seed, use_graph=use_cuda_graph,
                                         top_p=top_p)
            if seed_vals is None:
                eng.seed += 1
            new = sess.tokens[:, :n_new]
        if lengths is None:
            sampled = torch.cat([prefix, new], 1) if n_new > 0 else prefix
            n_real = torch.full((B, 1), prefix.shape[1], device=dev, dtype=torch.int64)
            n_end = n_real + n_new
        else:
            # row b: its n_real[b] prefix tokens, then its n_new_b[b] samples, then -1 up to the widest row
            width = max(max(t, n) for t, n in zip(steps_b, lengths)) * q
            col = torch.arange(width, device=dev)[None]
            n_end = n_real + torch.tensor(n_new_b, device=dev, dtype=torch.int64)[:, None]
            sampled = torch.full((B, width), -1, device=dev, dtype=torch.int64)
            sampled[:, :min(width, prefix.shape[1])] = prefix[:, :width]
            sampled.masked_fill_(col >= n_real, -1)
            if n_new > 0:
                sampled = torch.where((col >= n_real) & (col < n_end), new.gather(1, (col - n_real).clamp(0, n_new - 1).expand(B, -1)),
                                      sampled)
        eos_mask = (sampled == eos).float()                                                         # utils.py:86-93
        if include_eos_in_output:
            eos_mask = torch.nn.functional.pad(eos_mask, (1, -1))
        sampled = sampled.masked_fill(eos_mask.cumsum(-1) > 0, -1)
        if was_training:
            m.train()
        if return_logprobs:
            if pre_lp is None:
                pre_lp = torch.zeros(B, prompt.shape[1], device=dev, dtype=torch.float32)
            lp, slp = assemble_logprobs(sampled, pre_lp, sess.lp[:, :n_new] if n_new > 0 else None,
                                        sess.slp[:, :n_new] if n_new > 0 else None, n_real, n_end)
            return sampled.view(B, -1, q), lp.view(B, -1, q), slp.view(B, -1, q)
        return sampled.view(B, -1, q)                                                               # :323-324

    def forward(self, *, all_token_ids: List[torch.Tensor], return_loss: bool = False, **kwargs):
        """open_musiclm.py:328-411.  return_loss=True: (loss, None, None) with the loss computed by the fused path
        (training mode: forgetful mask + dropout as in the reference); otherwise the list of logits."""
        m = self.transformer
        if return_loss:
            from .trainer import HotPathTrainer
            if self._trainer is None:
                self._trainer = HotPathTrainer(m, cross_entropy_loss_weights=self.cross_entropy_loss_weights, mask_prob=self.mask_prob,
                                               pad_id=self.pad_id, use_cuda_graph=False)
            return self._trainer._micro_batch(all_token_ids, m.training, 0, False,
                                             det=torch.are_deterministic_algorithms_enabled()), None, None
        dev = m.device
        ids = [t.to(dev, torch.int64).reshape(t.shape[0], -1) for t in all_token_ids]
        ids = [torch.cat([t, torch.full((t.shape[0], 1), e, device=dev, dtype=torch.int64)], 1) for t, e in zip(ids, self.eos_ids)]
        return m(all_token_ids=ids, **kwargs)
