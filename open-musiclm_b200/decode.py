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

Every call decodes per row: each sequence has its own position, last position and predicted-sequence offset
(DecodeSession.pos, pos_last, pos_offset, read by the _ragged attention and omlm_embed_gather_pos_rows, advanced by
omlm_decode_advance_pos) and its own sampling arguments (DecodeSession.top_k, temperature, top_p, read by
omlm_sample_rows).  So prefixes of different lengths (`generate(pred_lengths=...)`), sampling arguments given one per
row, and rows that sample different numbers of tokens need no path of their own, and every row gets what it would get
alone (DESIGN section 4).  A call is one flow: check (check_sampling_rows, check_pred_lengths), plan (plan_rows,
check_abs_positions), prompt, prefill, decode loop, assemble (assemble_output); GenerationSession runs the same pieces
for one row at a time.
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


class GraphCache:
    """Runs a body by key: eagerly the first time (lazy cudaFuncSetAttribute calls are not capturable), captured into a
    CUDA graph the second time and replayed from then on.  Disabled, every call runs the body eagerly."""

    def __init__(self, enabled: bool = True):
        self.enabled, self.graphs, self._warm = enabled, {}, set()

    def run(self, key, body):
        if not self.enabled:
            body()
            return
        g = self.graphs.get(key)
        if g is None:
            if key not in self._warm:
                body()
                self._warm.add(key)
                return
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                body()
            self.graphs[key] = g
        g.replay()


class _PromptCapture:
    """Receives the prompt's per-layer K/V rows and pre-conv FFN rows from Engine.forward_core into rows `rows` (a
    slice) of a DecodeSession: the K/V rows of all n prompt positions, and as conv history rows p - 2, p - 1 of each
    sequence's own prompt length p (prompt_len, a device array; zero before its first row)."""

    def __init__(self, dec, rows, n, prompt_len):
        self.dec, self.rows, self.n = dec, rows, n
        idx = prompt_len[:, None].long() + torch.arange(-2, 0, device=prompt_len.device)
        self.before = (idx < 0)[..., None]
        self.idx = (torch.arange(len(prompt_len), device=prompt_len.device)[:, None] * n + idx.clamp_min(0)).view(-1)

    def after_kv(self, l, kvn):
        self.dec.cache[l][self.rows, :self.n].copy_(kvn.view(-1, self.n, 128))

    def after_u(self, l, u):
        hist = u.view(-1, u.shape[-1])[self.idx].view(-1, 2, u.shape[-1])
        self.dec.conv[l][self.rows].copy_(hist.masked_fill(self.before, 0))


def seeds_tensor(seeds, B: int, device) -> torch.Tensor:
    """B per-sequence seeds (ints, taken modulo 2^64, or an int64 tensor read as raw 64-bit patterns) as an int64
    device tensor of those bit patterns, sent in a non-blocking copy as row_arrays sends its arrays."""
    if isinstance(seeds, torch.Tensor):
        if seeds.dtype != torch.int64:
            raise ValueError(f"open_musiclm_b200 generate: seeds must be an int64 tensor or a list of ints, not {seeds.dtype}")
        vals = seeds.reshape(-1).tolist()
    else:
        vals = [int(s) for s in seeds]
    if len(vals) != B:
        raise ValueError(f"open_musiclm_b200 generate: {len(vals)} seeds for {B} sequences")
    vals = [v & 0xFFFFFFFFFFFFFFFF for v in vals]
    return torch.tensor([v - (1 << 64) if v >= 1 << 63 else v for v in vals], dtype=torch.int64).to(device, non_blocking=True)


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


def check_pred_lengths(pred_lengths, pred_token_ids, B: int, caller: str = "generate"):
    """generate's pred_lengths -> a list of B ints in [0, pred_token_ids.shape[1]], or None when it is None or every
    value equals pred_token_ids.shape[1] (every prefix whole).  A wrong count, a value out of
    range, a non-integer or a bool, or pred_lengths without pred_token_ids raises ValueError (naming `caller`)."""
    if pred_lengths is None:
        return None
    where = f"open_musiclm_b200 {caller}: pred_lengths"
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


_FLOAT_ROWS = ("temperature", "top_p")


def row_arrays(dev, B: int, **values):
    """Per-row device state: each keyword one value or a list of B values -> a [B] device array, float32 for
    temperature and top_p and int32 otherwise (top_p: None or a list of Nones -> None; a None element -> 1.0).  All of
    them go up in one non-blocking copy, which CUDA stages from pageable memory before it returns, so that building the
    state never waits for the device.  (Pinned memory would not help: every graph capture empties PyTorch's pinned
    cache, and pinning anew costs more than the copy.)"""
    names, host = [], []
    for name, v in values.items():
        if name == "top_p" and (v is None or (isinstance(v, list) and all(p is None for p in v))):
            continue
        v = v if isinstance(v, list) else [v] * B
        dt = torch.float32 if name in _FLOAT_ROWS else torch.int32
        names.append((name, dt))
        host.append(torch.tensor([1.0 if x is None else x for x in v], dtype=dt).view(torch.int32))
    up = torch.stack(host).to(dev, non_blocking=True)
    out = {name: row.view(dt) for (name, dt), row in zip(names, up)}
    out.setdefault("top_p", None)
    return out


def bias_table(eng, N: int):
    """The relative position bias of every distance 0 ... N - 1 (it depends on i - j only), as the scratch dict
    Engine.build_bias_table fills: its "table" entry is [heads, N] float32 (zero with no bias)."""
    dev, f32 = eng.dev, torch.float32
    E = lambda *shape, dt=torch.bfloat16: torch.empty(*shape, device=dev, dtype=dt)
    rp = dict(rp_in=E(N, 1, dt=f32), rp_z=[E(N, eng.Hr, dt=f32) for _ in range(3)], rp_a=[E(N, eng.Hr, dt=f32) for _ in range(3)],
              table=E(eng.h, N, dt=f32), rp_a3=[E(N, 3 * eng.Hr8) for _ in range(2)])
    lib.arange_f32(rp["rp_in"])
    eng.refresh_packed()
    if eng.bias_type == "none":
        rp["table"].zero_()
    elif eng.bias_type == "t5":
        rp["ones"] = torch.ones(N, device=dev, dtype=f32)
    eng.build_bias_table(rp, N)
    return rp


class DecodeSession:
    """Caches and scratch of one decode: B sequences, caches of n_max positions, up to n_new new tokens per sequence.
    rows (row_arrays): the per-sequence state every step and sample reads, as device arrays [B]: pos (the position the
    next decode step processes), pos_last (the last position the sequence processes; the advance after each sample
    stops there), pos_offset (with absolute position embeddings the token at position p is token p + pos_offset of the
    predicted sequence), and the sampling arguments top_k, temperature and top_p (None: no row narrows to a nucleus).
    seeded: batch-invariant mode (tensor-core path with the B-independent GEMM split at every B, per-sequence seeds in
    self.seeds).  logprob: the sampler also writes each token's two log-probabilities into self.lp and self.slp (fp32
    [B, n_new], in the allocation of self.tokens, right after it, as omlm_sample_logprob requires).  use_graph: replay
    step_and_sample from one CUDA graph per key."""

    def __init__(self, eng, B: int, n_max: int, n_new: int, rows, seeded: bool = False, logprob: bool = False,
                 use_graph: bool = True):
        if B > MAX_BATCH:
            raise lib.OmlmError(f"open_musiclm_b200 generate: batch sizes above {MAX_BATCH} are not supported by the decode kernels")
        if seeded and eng.h > 16:
            raise lib.OmlmError(f"open_musiclm_b200 generate: seeded generation supports at most 16 heads ({eng.h} given)")
        self.eng, self.B, self.n_max, self.n_new, self.seeded = eng, B, n_max, n_new, seeded
        dev, bf, f32, a16 = eng.dev, torch.bfloat16, torch.float32, eng.a16
        d, HD, Fp, h = eng.d, eng.HD, eng.Fp, eng.h
        E = lambda *shape, dt=bf: torch.empty(*shape, device=dev, dtype=dt)
        self.cache = [E(B, n_max, 128) for _ in range(eng.L)]
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
        self.pos, self.pos_last, self.pos_offset = rows["pos"], rows["pos_last"], rows["pos_offset"]
        self.top_k, self.temperature, self.top_p = rows["top_k"], rows["temperature"], rows["top_p"]
        # bias table for every distance the generation can reach (it depends on i - j only)
        self.rp = bias_table(eng, n_max)
        self.table = self.rp["table"]
        self.graphs = GraphCache(use_graph)
        # more than 16 sequences, or seeded mode: tensor-core GEMMs and the cache-sharing attention, with their scratch
        # allocated here so that graph capture allocates nothing.  Both paths have the same rounding points (fp32 sums
        # in another order); seeded mode fixes the GEMMs' K split independently of B, and attn_decode_mqa's
        # per-sequence CTAs already are.
        self.batched = B > SKINNY_MAX_BATCH or seeded
        self.seeds = torch.zeros(B, device=dev, dtype=torch.int64) if seeded else None
        if self.batched:
            shapes = [(HD, d), (128, d), (d, HD), (2 * Fp, d), (d, Fp)] + [(cp, d) for cp in eng.Cp]
            ws = self.ws = lib.DecodeWorkspace(dev, B, shapes, max_pos=n_max, heads=h, invariant=seeded)
            self._gemm = lambda *a, **k: lib.decode_gemm(*a, ws=ws, invariant=seeded, **k)
            self._attn = lambda *a: lib.attn_decode_mqa(*a, ws=ws, ragged=True)
        else:
            self._gemm = lib.skinny_gemm
            self._attn = lambda *a: lib.attn_decode(*a, ragged=True)

    # ------------------------------------------------------------------------------------------ one incremental step
    def embed(self, x):
        """x = the input rows of the positions self.pos: embedding row self.next_row, plus with absolute position
        embeddings the predicted sequence's row for its token pos + pos_offset (open_musiclm.py:134-136)."""
        eng = self.eng
        if eng.abs_pos:
            lib.embed_gather_pos_rows(eng.table, self.next_row, self.pos, self.pos_offset, eng.abs_row_base[-1], eng.max_abs_pos, x)
        else:
            lib.embed_gather(eng.table, self.next_row, x)

    def step(self, qi_next: int):
        """Processes the positions self.pos (embedding rows self.next_row) through all layers and leaves the logits of
        head qi_next in self.logits (one launch per operation)."""
        eng, gemm = self.eng, self._gemm
        pv, F, h = eng.pview, eng.F, eng.h
        xa, xm = self.x
        self.embed(xa)
        for l in range(eng.L):
            p, pk = f"transformer.layers.{l}.", eng.pk[l]
            gemm(xa, pk["wq"], self.q_raw, prologue=2, gamma=pv[p + "0.norm.gamma"])
            gemm(xa, pk["wkv_b"], self.kv_raw, prologue=1)
            self._attn(self.q_raw, self.kv_raw, pv[p + "0.q_scale"], pv[p + "0.k_scale"], self.cache[l], self.table, self.pos,
                       self.n_max, self.o, h)
            gemm(self.o, pk["wo_b"], xm, addend=xa)
            gemm(xm, pk["w1"], self.u_new, prologue=2, gamma=pv[p + eng.ffk["g1"]])
            lib.decode_conv_geglu(self.u_new, self.conv[l], pk["conv"], self.h, self.rowsum)
            gemm(self.h, pk["w2"], xa, prologue=3, gamma=pk["gin"], rowsum=self.rowsum, n_real=F, addend=xm)
        S = len(eng.seqs) - 1
        gemm(xa, eng.pk_logit[S][qi_next], self.logits[:, :eng.Cp[S]], prologue=2, gamma=pv["transformer.norm.gamma"])

    def row_offset(self, qi: int) -> int:
        """Embedding row of token 0 of quantizer slot qi in the predicted sequence."""
        eng = self.eng
        S = len(eng.seqs) - 1
        return eng.emb_row_base[S] + (eng.seqs[S].codebook_size * qi if eng.seqs[S].num_quantizers > 1 else 0)

    def sample(self, qi: int, allow_eos: bool, uniform, seed, advance: bool = True):
        """Every sequence samples the token of quantizer slot qi with its own arguments; then (advance) every position
        moves on, up to its sequence's last."""
        eng = self.eng
        lib.sample(self.logits, eng.C[-1], 1, 1.0, allow_eos, uniform, seed, self.tokens, self.next_row, self.row_offset(qi),
                   self.counters, None, self.B, seeds=self.seeds, top_k_rows=self.top_k, temperature_rows=self.temperature,
                   top_p_rows=self.top_p, logprobs=self.lp, sample_logprobs=self.slp)
        if advance:
            lib.decode_advance_pos(self.pos, self.pos_last)

    def step_and_sample(self, qi: int, qi_next: int, allow_eos_next, uniform, seed):
        """decode step on the token sampled for quantizer slot qi, then sample the token of slot qi_next.  The arrays'
        contents are read at replay; only the kernel choice is captured."""
        self.graphs.run((qi, qi_next, bool(allow_eos_next), uniform is not None),
                        lambda: (self.step(qi_next), self.sample(qi_next, allow_eos_next, uniform, seed)))


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


def plan_rows(pred_token_ids, B: int, q: int, lengths, max_time_steps):
    """Per row of a generate call: (n_real, n_new), the number of real prefix tokens and the number of tokens to sample
    (open_musiclm.py:276).  lengths: check_pred_lengths' result (None: every prefix is whole); max_time_steps: one int
    or B ints, as check_sampling_rows returns it.  A prefix given flat as [b, n] on a stage with q > 1 is n tokens,
    and sampling continues at quantizer n mod q."""
    T = 0 if pred_token_ids is None else pred_token_ids.shape[1]
    per_step = math.prod(pred_token_ids.shape[2:]) if T else q          # prefix tokens per step of pred_token_ids.shape[1]
    if lengths is not None and per_step != q:
        raise ValueError(f"open_musiclm_b200 generate: pred_lengths needs pred_token_ids of whole time steps, [b, t, {q}]")
    lengths = lengths if lengths is not None else [T] * B
    steps = max_time_steps if isinstance(max_time_steps, list) else [max_time_steps] * B
    return [n * per_step for n in lengths], [max(0, (t - n) * q) for t, n in zip(steps, lengths)]


def check_abs_positions(where: str, lim: int, cond_lens, n_real, n_new):
    """The reference looks up arange(len) in each sequence's nn.Embedding(max_absolute_position_embeddings): IndexError
    when something is sampled and a conditioning sequence (with its eos) has more than lim tokens, or a row that
    samples feeds back a token past lim (its last sampled token is never fed back).  The message names the row when the
    rows differ."""
    if not any(n_new):
        return
    for s, n in enumerate(cond_lens):
        if n > lim:
            raise IndexError(f"{where}: conditioning sequence {s} has {n} tokens but max_absolute_position_embeddings is {lim}")
    row = len(set(zip(n_real, n_new))) > 1
    for b, (n, k) in enumerate(zip(n_real, n_new)):
        if k > 0 and n + k - 1 > lim:
            raise IndexError(f"{where}: the predicted sequence{f' of row {b}' if row else ''} reaches {n + k - 1} tokens "
                             f"({n} given + {k} sampled - 1) but max_absolute_position_embeddings is {lim}")


def prefill(wrapper, cond, prompt, append_eos: bool, dec=None, rows=slice(None), prompt_len=None):
    """Runs the prompt (conditioning sequences, eos appended when append_eos, then the predicted sequence's prompt
    tokens) through the regular forward once.  With a DecodeSession dec it also writes the prompt's caches into dec's
    rows `rows` (_PromptCapture) and the logits of each sequence's last real prompt position into dec.logits; that
    position is prompt_len - 1 (int device array [b]), and the last real prompt tokens of all sequences share a
    quantizer slot.  Returns (plan, workspace) for prefix_logprobs."""
    eng = wrapper.transformer.engine
    B, S, q = prompt.shape[0], len(eng.seqs), eng.seqs[-1].num_quantizers
    if append_eos:                                                                                   # open_musiclm.py:288-290
        cond = [torch.cat([t, torch.full((B, 1), e, device=eng.dev, dtype=torch.int64)], 1) for t, e in zip(cond, wrapper.eos_ids)]
    _, src_row, key_mask, _, n_tok = lib.token_plan(
        cond + [prompt], [s.codebook_size for s in eng.seqs], [s.num_quantizers for s in eng.seqs], eng.emb_row_base, eng.start_row,
        append_eos=False, drop_last=False, mask_cond=False, want_labels=False, err_flag=eng.err_flag)
    pl = eng.plan(B, n_tok)
    ws = eng.workspace(pl, False)
    capture = None if dec is None else _PromptCapture(dec, rows, pl.N, prompt_len)
    eng.forward_core(pl, ws, src_row, key_mask, False, {S - 1}, False, capture=capture)
    if dec is not None:
        # final sequence, head group of the next token's quantizer slot; in it, each sequence's row of its last token
        gi = next(i for i, (s, qi, cnt, base) in enumerate(pl.groups) if s == S - 1 and qi == n_tok[-1] % q)
        cnt = pl.groups[gi][2]
        last = torch.arange(B, device=eng.dev) * cnt + (prompt_len - pl.pos0[-1] - 1) // q
        dec.logits[rows, :eng.Cp[S - 1]].copy_(ws["logits"][gi][last])
    return pl, ws


def assemble_output(prefix, new, n_real, n_end, width: int, eos: int, include_eos: bool, q: int, logprobs=None):
    """generate's output [b, width / q, q]: row r holds its n_real[r] prefix tokens (prefix [b, >= that]), then its
    samples new[r, :n_end[r] - n_real[r]], then -1; everything after an eos is -1 (the eos too unless include_eos;
    utils.py:86-93).  n_real, n_end: ints or int tensors [b, 1].  logprobs: (pre_lp [b, >= the prefix tokens' count]
    or None for zeros, lp_new, slp_new [b, >= the samples' count]) -> (tokens, logprobs, sample_logprobs): prefix
    columns take pre_lp (sample log p 0), sampled columns lp_new and slp_new in order, and every -1 is 0 in both."""
    B, n_new = new.shape
    col = torch.arange(width, device=prefix.device)[None]
    in_new = (col >= n_real) & (col < n_end)
    src = (col - n_real).clamp(0, max(n_new - 1, 0)).expand(B, -1)
    sampled = torch.full((B, width), -1, device=prefix.device, dtype=torch.int64)
    sampled[:, :min(width, prefix.shape[1])] = prefix[:, :width]
    sampled.masked_fill_(col >= n_real, -1)
    if n_new > 0:
        sampled = torch.where(in_new, new.gather(1, src), sampled)
    eos_mask = (sampled == eos).float()
    if include_eos:
        eos_mask = torch.nn.functional.pad(eos_mask, (1, -1))
    sampled = sampled.masked_fill(eos_mask.cumsum(-1) > 0, -1)
    if logprobs is None:
        return sampled.view(B, -1, q)
    pre_lp, lp_new, slp_new = logprobs
    lp = torch.zeros(B, width, device=prefix.device, dtype=torch.float32)
    if pre_lp is not None:
        w = min(width, pre_lp.shape[1])
        lp[:, :w] = pre_lp[:, :w]
        lp.masked_fill_(col >= n_real, 0.0)
    slp = torch.zeros_like(lp)
    if n_new > 0:
        lp = torch.where(in_new, lp_new.gather(1, src), lp)
        slp = torch.where(in_new, slp_new.gather(1, src), slp)
    gone = sampled == -1
    return sampled.view(B, -1, q), lp.masked_fill(gone, 0.0).view(B, -1, q), slp.masked_fill(gone, 0.0).view(B, -1, q)


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
        lengths = check_pred_lengths(pred_lengths, pred_token_ids, B)
        m, eng = self.transformer, self.transformer.engine
        assert len(conditioning_token_ids) == len(self.token_sequences) - 1
        q = info.num_quantizers
        n_real, n_new = plan_rows(pred_token_ids, B, q, lengths, max_time_steps)
        N = max(n_new)                                               # decode steps: those of the row that samples most
        eos_len = 1 if append_eos_to_conditioning_tokens else 0
        if eng.abs_pos:
            check_abs_positions("open_musiclm_b200 generate", eng.max_abs_pos, [t.numel() // B + eos_len for t in conditioning_token_ids],
                                n_real, n_new)
        was_training = m.training
        m.eval()
        dev = eng.dev
        cond = [t.to(dev, torch.int64).reshape(B, -1) for t in conditioning_token_ids]
        if pred_token_ids is not None:
            assert pred_token_ids.shape[0] == B
            prefix = pred_token_ids.to(dev, torch.int64).reshape(B, -1)
        else:
            prefix = torch.empty(B, 0, device=dev, dtype=torch.int64)
        seed_vals = seeds_tensor(seeds, B, dev) if seeds is not None else None
        # the prompt: the prefixes cut to the longest real prefix of a row that samples (of every row, for the prefix
        # log-probabilities; a longer prefix takes part cut to it), right-padded with token 0.  The predicted sequence
        # comes last, so causal attention keeps every real position away from the padding.  Row r's prompt is P[r]
        # positions long: it processes P[r], P[r] + 1, ... up to its last position, where it stays.
        Lp = max([n for n, k in zip(n_real, n_new) if k > 0 or return_logprobs], default=0)
        pred_start = sum(t.shape[1] + eos_len + 1 for t in cond)
        P = [pred_start + 1 + min(n, Lp) for n in n_real]
        state = dict(prompt_len=P, n_real=n_real, n_end=[n + k for n, k in zip(n_real, n_new)])
        if N > 0:
            pos_last = [p + max(k, 1) - 2 for p, k in zip(P, n_new)]
            state.update(pos=[min(p, e) for p, e in zip(P, pos_last)], pos_last=pos_last, pos_offset=-(pred_start + 1),
                         top_k=max(int((1 - filter_thres) * C), 1) if top_k is None else top_k,                  # utils.py:80
                         temperature=temperature, top_p=top_p)
        rows = row_arrays(dev, B, **state)
        prompt = prefix[:, :Lp].masked_fill(torch.arange(Lp, device=dev)[None] >= rows["n_real"][:, None], 0)
        sess = None
        if N > 0:
            sess = DecodeSession(eng, B, max(P[b] + n_new[b] for b in range(B)), N, rows, seeded=seed_vals is not None,
                                 logprob=return_logprobs, use_graph=use_cuda_graph)
            if seed_vals is not None:
                sess.seeds.copy_(seed_vals)
        pre_lp = lp_new = slp_new = None
        if N > 0 or (return_logprobs and Lp > 0):
            pl, ws = prefill(self, cond, prompt, append_eos_to_conditioning_tokens, sess, prompt_len=rows["prompt_len"])
            assert pl.pos0[-1] == pred_start, (pl.pos0, pred_start)
            if return_logprobs and Lp > 0:
                pre_lp = prefix_logprobs(eng, pl, ws, prompt, q, C)
        new = prefix.new_empty(B, 0)
        if N > 0:
            uni = None
            if uniform_noise is not None:
                uni = uniform_noise.to(dev, torch.float32).contiguous()
                assert uni.shape == (N, B, info.codebook_size + 1), uni.shape
            allow = lambda p: bool(allow_eos_in_output and (p % q) == q - 1)                        # :311-313
            if trace_logits is not None:
                trace_logits.append(sess.logits[:, :C].clone())
            sess.sample(Lp % q, allow(Lp), uni, eng.seed, advance=False)
            for p in range(Lp + 1, Lp + N):                          # p: flat index of the sampled token
                if trace_logits is not None:      # eager, in two halves, so that the logits can be copied in between
                    sess.step(p % q)
                    trace_logits.append(sess.logits[:, :C].clone())
                    sess.sample(p % q, allow(p), uni, eng.seed)
                else:
                    sess.step_and_sample((p - 1) % q, p % q, allow(p), uni, eng.seed)
            if seed_vals is None:
                eng.seed += 1
            new, lp_new, slp_new = sess.tokens[:, :N], sess.lp, sess.slp
        if was_training:
            m.train()
        return assemble_output(prefix, new, rows["n_real"][:, None], rows["n_end"][:, None], max(state["n_end"]), eos,
                               include_eos_in_output, q, (pre_lp, lp_new, slp_new) if return_logprobs else None)

    @torch.no_grad()
    def score(self, *, conditioning_token_ids: List[torch.Tensor], pred_token_ids: torch.Tensor, pred_lengths=None,
              max_rows: int = 16384):
        """The model's log-probability of every given token, teacher-forced: [b, t, q] float32 on the device for
        pred_token_ids [b, t, q] ([b, t] when q = 1).  Value [r, i, j] is log softmax of the fp32 logits row at that
        token's position over all codebook+1 classes (no temperature, top-k or eos rule) at the token, exactly the value
        generate(conditioning_token_ids=<row r>, pred_token_ids=x[r:r+1, :len_r], max_time_steps=len_r,
        return_logprobs=True)[1] reports for that row alone, bit for bit.  pred_lengths: as in generate (len_r whole
        time steps of row r are real, the rest is never read); positions past a row's length hold 0.
        The rows' prompts are packed back to back without padding into forwards of at most max_rows rows each (a prompt
        longer than that runs alone), on the varlen kernels of Engine.forward_packed (score.py).  There is no decode
        state, so no row limit.  Eval semantics whatever the module's mode; no random draw, Engine.seed untouched.
        Every id must lie in its sequence's codebook [0, codebook_size); a wrong count or shape, an id outside it, a
        bad pred_lengths or a max_rows that is not an int >= 1 raises ValueError, and with absolute position
        embeddings a sequence longer than max_absolute_position_embeddings raises IndexError, before any device work."""
        from .score import score_batch
        return score_batch(self, conditioning_token_ids, pred_token_ids, pred_lengths, max_rows)

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
