"""Host-side engine of the hot path: owns the flat parameter arena, the packed bf16 compute weights and
the activation workspaces, and sequences the libomlm_b200 kernels for forward, backward and the
optimiser step.  PyTorch supplies device memory and streams only; every arithmetic op is a call into
the C ABI (open_musiclm_b200.lib).

HBM layout
  arena_p / arena_g / adam_m / adam_v : one fp32 buffer each, parameters ordered
        [embeddings | logit heads | layer matrices | rel-pos MLP matrices]   <- weight-decayed (ndim >= 2)
        [start tokens | gammas, scales, MLP biases]                          <- not decayed
        every nn.Parameter of the module is a view into arena_p (and its .grad into arena_g).
  packed weights (16-bit, refreshed after every parameter update):
        wq [h*64, d], wkv [128, d], wo [d, h*64], w1 [2*Fp, d] (value rows | gate rows, zero padded),
        w2 [d, Fp], logit heads [q, Cp, d];  conv taps fp32 [2*Fp, 3], inner gamma fp32 [Fp].
  activations: residual stream fp32 [M, d]; GEMM operands 16-bit; attention statistics fp32.

16-bit operand formats (csrc/common.cuh): wgmma runs fp16 and bf16 at the same rate, but both operands of one
wgmma must share the format.  The FORWARD GEMMs whose operands are bounded
by construction -- LayerNorm outputs (xn, xn2, hn, xf) against weights, and the FFN activations between them (u, h) --
run in fp16 (11-bit significand: 8x less operand rounding than bf16, which is what keeps the logits of deep models within
1e-2 of the fp32 reference).  Everything that touches an unbounded range stays bf16: every
BACKWARD GEMM (gradients), the K/V projection of the raw residual stream, attention and its output projection.  So
the weights are packed twice (fp16 for forward, bf16 for backward) and the saved LayerNorm outputs carry a bf16
duplicate for the weight-gradient GEMMs.  OMLM_ACT16=bf16 switches the whole path back to bf16 (diagnostics only).
"""
import math
import os
import weakref
from typing import List, Optional

import torch

from . import lib

CE_IGNORE = -100


def _round_up(x, m):
    return (x + m - 1) // m * m


class _Plan:
    """Static shape bookkeeping for one (batch, sequence lengths) configuration."""

    def __init__(self, eng: "Engine", B: int, n_tok: List[int], device):
        self.B = B
        self.n_tok = list(n_tok)
        S = len(n_tok)
        self.N = sum(n + 1 for n in n_tok)
        self.M = B * self.N
        self.pos0 = list(itertools_accumulate([0] + [n + 1 for n in n_tok[:-1]]))
        # logits positions per sequence (open_musiclm.py:149-156)
        self.n_out = [n_tok[s] if s < S - 1 else n_tok[s] + 1 for s in range(S)]
        # head groups: (s, qi) -> rows ordered (b, t), position p = qi + q*t
        self.groups = []
        dest = torch.full((B, self.N), -1, dtype=torch.int32)
        base = 0
        self.seq_row_index = []   # per sequence: [B, n_out] -> row in the permuted buffers
        for s in range(S):
            q = eng.seqs[s].num_quantizers
            idx = torch.empty(B, self.n_out[s], dtype=torch.int64)
            for qi in range(min(q, self.n_out[s])):
                cnt = (self.n_out[s] - qi + q - 1) // q
                rows = base + torch.arange(B)[:, None] * cnt + torch.arange(cnt)[None, :]
                pos = qi + q * torch.arange(cnt)
                dest[:, self.pos0[s] + pos] = rows.to(torch.int32)
                idx[:, pos] = rows
                self.groups.append((s, qi, cnt, base))
                base += B * cnt
            self.seq_row_index.append(idx.to(device))
        self.rows_total = base
        self.dest_row = dest.reshape(-1).to(device)
        # absolute position embeddings (open_musiclm.py:134-136): token t of sequence s also gets row t of its
        # position table; start tokens get none.  Static per shape, so it is built here once.
        self.src_row2 = None
        if eng.abs_pos:
            r2 = torch.full((B, self.N), -1, dtype=torch.int32)
            for s in range(S):
                if n_tok[s] > eng.max_abs_pos:
                    raise IndexError(f"sequence {s} has {n_tok[s]} tokens but max_absolute_position_embeddings is {eng.max_abs_pos}")
                r2[:, self.pos0[s] + 1:self.pos0[s] + 1 + n_tok[s]] = eng.abs_row_base[s] + torch.arange(n_tok[s], dtype=torch.int32)
            self.src_row2 = r2.reshape(-1).to(device)


class _BackwardPlan:
    """The backward work a set of frozen parameters (requires_grad=False, or logit heads without gradient) leaves.
    A layer runs its backward pass when it holds a trainable parameter, when a gradient has to reach a layer or a row
    table below it, or when the bias table is trained (its gradient sums every layer's dS).  Inside a layer each step
    runs only when a trainable parameter or the gradient flowing further down consumes what it produces."""

    def __init__(self, eng: "Engine", frozen):
        self.frozen = frozenset(frozen)
        tr = self.trains
        names = list(eng.layout)
        row_tables = [n for n in names if n.startswith(("embeddings.", "absolute_position_embeddings.", "start_tokens."))]
        # 'none' has no bias parameters: its table gradient is never needed
        self.dtable = any(tr(n) for n in names if n.startswith("transformer.rel_pos_bias."))
        self.rows = any(tr(n) for n in row_tables)
        self.rows_partial = self.rows and not all(tr(n) for n in row_tables)
        layer_tr = [self.dtable or any(tr(n) for n in names if n.startswith(f"transformer.layers.{l}.")) for l in range(eng.L)]
        below, acc = [], self.rows           # below[l]: a gradient must reach the input of layer l (l = L: the final norm)
        for l in range(eng.L + 1):
            below.append(acc)
            acc = acc or (l < eng.L and layer_tr[l])
        self.below = below
        self.run = [layer_tr[l] or below[l] for l in range(eng.L)]
        self.final_norm = below[eng.L] or tr("transformer.norm.gamma")
        fk = eng.ffk
        self.steps = []
        for l in range(eng.L):
            t = lambda k, l=l: k is not None and tr(f"transformer.layers.{l}.{k}")
            g_in = below[l]
            ln_a = g_in or t("0.norm.gamma")                                              # attention pre-norm backward
            qk = ln_a or any(t(k) for k in ("0.to_q.weight", "0.to_kv.weight", "0.q_scale", "0.k_scale"))
            attn = qk or self.dtable                                                      # attention backward
            mid = attn or g_in or t("0.to_out.0.weight")                                  # gradient at the mid residual
            ln_f = mid or t(fk["g1"])                                                     # feed-forward pre-norm backward
            ffn = ln_f or t(fk["w1"]) or t(fk["gin"]) or t(fk["conv"])                    # d_hn GEMM + ffn_mid_bwd
            self.steps.append(dict(g_in=g_in, ln_a=ln_a, qk=qk, attn=attn, mid=mid, ln_f=ln_f, ffn=ffn))

    def trains(self, name):
        return name not in self.frozen


def itertools_accumulate(xs):
    t = 0
    out = []
    for x in xs:
        t += x
        out.append(t)
    return out


class Engine:
    def __init__(self, module):
        lib.load()
        self.m = module
        dev = module.device
        if dev.type != "cuda":
            raise lib.OmlmError("open_musiclm_b200 needs a CUDA (sm_90a) device: move the module with .to('cuda') "
                                "before calling it - there is no CPU fallback")
        lib.device_check()
        self.dev = dev
        self.seqs = module.token_sequences
        self.d, self.L, self.h = module.dim, module.depth, module.heads
        self.HD = self.h * 64
        self.use_conv_ff = bool(getattr(module, "use_conv_ff", True))
        self.bias_type = getattr(module, "relative_position_bias_type", "continuous")
        self.abs_pos = module.absolute_position_embeddings is not None
        self.max_abs_pos = int(getattr(module, "max_absolute_position_embeddings", 0))
        # feed-forward flavour (transformer.py:140-161): state_dict suffixes of (pre-norm gamma, up, conv, inner gamma, down).
        # The plain FeedForward runs through the same fused kernels with the conv taps pinned to (0, 0, 1).
        self.ffk = (dict(g1="2.0.gamma", w1="2.1.weight", conv="2.2.ds_conv.weight", gin="2.4.gamma", w2="2.6.weight") if self.use_conv_ff
                    else dict(g1="2.0.gamma", w1="2.1.weight", conv=None, gin="2.3.gamma", w2="2.5.weight"))
        self.F = int(self.d * 2 * 4 / 3) if self.use_conv_ff else int(self.d * 4)
        self.Fp = _round_up(self.F, 128)           # interleaved GEGLU layout: groups of 128 channels
        self.Hr = self.d // 2                      # rel-pos MLP width
        self.Hr8 = _round_up(self.Hr, 8)           # width of one third of its bf16x3 split operands (16-byte aligned thirds)
        self.C = [s.codebook_size + 1 for s in self.seqs]
        self.Cp = [_round_up(c, 64) for c in self.C]
        self.drop_p = float(module.ff_dropout)
        self.alpha = float(module.grad_shrink_alpha)
        mode = os.environ.get("OMLM_ACT16", "fp16")
        if mode not in ("fp16", "bf16"):
            raise lib.OmlmError(f"OMLM_ACT16 must be 'fp16' or 'bf16', got {mode!r}")
        self.a16 = torch.float16 if mode == "fp16" else torch.bfloat16     # bounded forward operands (see module doc)
        self._build_arena()
        self._alloc_packed()
        self._packed_version = None
        self.bwd_max_ctas = 0      # > 0: CTA cap of the backward GEMMs (data parallel: leaves SMs to the overlapped NCCL kernels)
        self._plans = {}
        self._ws = {}
        self.seed = torch.zeros(1, dtype=torch.int64, device=dev)      # dropout / forgetful-mask seed (device resident)
        self.step_count = 0
        self.adam_m = None
        self.adam_v = None
        self.err_flag = torch.zeros(1, dtype=torch.int32, device=dev)  # latched by omlm_token_plan (token id out of range)
        self.loss_acc = torch.zeros(2, device=dev)
        self.sumsq = torch.zeros(1, device=dev, dtype=torch.float64)
        self.det_sumsq_part = None      # deterministic mode (see workspace()): per-CTA partials of grad_sumsq
        self.det_rows = None            #   and the row markers of the embedding scatter-add
        self._det_attn = weakref.WeakSet()   # every live attention-backward workspace (also those kept by captured graphs)
        self._bwd_plans = {}
        self._row_live = {}

    # ------------------------------------------------------------------------------------------ arena
    def _build_arena(self):
        named = [(n, p) for n, p in self.m.named_parameters()]
        is_row_table = lambda n: n.startswith("embeddings.") or n.startswith("absolute_position_embeddings.")
        emb = [(n, p) for n, p in named if is_row_table(n)]
        start = [(n, p) for n, p in named if n.startswith("start_tokens.")]
        decay = emb + [(n, p) for n, p in named if p.ndim >= 2 and not is_row_table(n)]
        nodecay = start + [(n, p) for n, p in named if p.ndim < 2 and not n.startswith("start_tokens.")]
        # every slice starts on a 64-element boundary; the row tables (which come first) and the start tokens are also
        # addressed as rows of one embedding "table", so they start on whole rows of d from it: lcm(64, d) apart
        row_align = math.lcm(64, self.d)
        off, layout = 0, {}
        for n, p in decay:
            layout[n] = off
            off = _round_up(off + p.numel(), row_align if is_row_table(n) else 64)
        self.n_decay = off
        emb_off = layout[emb[0][0]]
        off = emb_off + _round_up(off - emb_off, row_align)
        self.n_decay = off
        for n, p in nodecay:
            layout[n] = off
            off = _round_up(off + p.numel(), row_align if n.startswith("start_tokens.") else 64)
        self.n_params_arena = off
        self.layout = layout
        arena_p = torch.zeros(off, device=self.dev, dtype=torch.float32)
        arena_g = torch.zeros(off, device=self.dev, dtype=torch.float32)
        self.pview, self.gview = {}, {}
        for n, p in named:
            o = layout[n]
            v = arena_p[o:o + p.numel()].view(p.shape)
            v.copy_(p.data)
            p.data = v
            g = arena_g[o:o + p.numel()].view(p.shape)
            if p.requires_grad:          # a frozen parameter keeps grad None, as autograd leaves it
                p.grad = g
            self.pview[n], self.gview[n] = v, g
        self.arena_p, self.arena_g = arena_p, arena_g
        # embedding table = [embeddings.0 | embeddings.1 | ... ] rows of d floats; start tokens further down
        self.emb_off = emb_off
        self.emb_row_base, self.abs_row_base = [], []
        for n, p in emb:
            assert (layout[n] - emb_off) % self.d == 0
            (self.emb_row_base if n.startswith("embeddings.") else self.abs_row_base).append((layout[n] - emb_off) // self.d)
        assert all((layout[n] - emb_off) % self.d == 0 for n, _ in start)
        self.start_row = [(layout[n] - emb_off) // self.d for n, _ in start]
        self.table = arena_p[emb_off:]
        self.dtable_emb = arena_g[emb_off:]
        self._param_list = [p for _, p in named]

    def params_version(self):
        return sum(p._version for p in self._param_list)

    def _alloc_packed(self):
        dev, bf, a16 = self.dev, torch.bfloat16, self.a16
        d, HD, Fp = self.d, self.HD, self.Fp
        dual = a16 != bf        # forward operands in fp16, backward operands (suffix _b) in bf16; one buffer when equal
        self.pk = []
        for _ in range(self.L):
            pk = dict(
                wq=torch.empty(HD, d, device=dev, dtype=a16), w1=torch.empty(2 * Fp, d, device=dev, dtype=a16),
                w2=torch.empty(d, Fp, device=dev, dtype=a16),
                wkv_b=torch.empty(128, d, device=dev, dtype=bf), wo_b=torch.empty(d, HD, device=dev, dtype=bf),
                conv=torch.empty(2 * Fp, 3, device=dev), gin=torch.empty(Fp, device=dev))
            for k in ("wq", "w1", "w2"):
                pk[k + "_b"] = torch.empty_like(pk[k], dtype=bf) if dual else pk[k]
            self.pk.append(pk)
        if not self.use_conv_ff:
            for pk in self.pk:
                pk["conv"].zero_()
                pk["conv"][:, 2] = 1.0          # y[t] = u[t]: no depthwise conv in FeedForward (transformer.py:152-161)
        self.pk_logit = [torch.empty(s.num_quantizers, cp, d, device=dev, dtype=a16) for s, cp in zip(self.seqs, self.Cp)]
        self.pk_logit_b = [torch.empty_like(t, dtype=bf) if dual else t for t in self.pk_logit]
        self._pack_table = None
        self.pk_rp = [torch.empty(self.Hr, 3 * self.Hr8, device=dev, dtype=torch.bfloat16) for _ in range(2)]  # rel-pos MLP layers 1, 2: [hi|lo|hi]

    def refresh_packed(self, force=False):
        ver = self.params_version()
        if not force and ver == self._packed_version:
            return
        d, HD, F, Fp = self.d, self.HD, self.F, self.Fp
        pv = self.pview
        if self._pack_table is None:      # the job table is built once: arena views and packed buffers never move
            tab = lib.PackTable(self.dev)
            for l, pk in enumerate(self.pk):
                p = f"transformer.layers.{l}."
                fk = self.ffk
                dual = pk["wq"] is not pk["wq_b"]       # fp16 forward copy + bf16 backward copy from ONE read of the matrix
                tab.add(pv[p + "0.to_q.weight"], d, HD, d, pk["wq"], HD, d, dst2=pk["wq_b"] if dual else None)
                tab.add(pv[p + fk["w1"]], d, 2 * F, d, pk["w1"], 2 * Fp, d, split_dst=-1, split_src=F, dst2=pk["w1_b"] if dual else None)
                tab.add(pv[p + fk["w2"]], F, d, F, pk["w2"], d, Fp, dst2=pk["w2_b"] if dual else None)
                tab.add(pv[p + "0.to_kv.weight"], d, 128, d, pk["wkv_b"], 128, d)
                tab.add(pv[p + "0.to_out.0.weight"], HD, d, HD, pk["wo_b"], d, HD)
                if fk["conv"] is not None:
                    tab.add(pv[p + fk["conv"]], 3, 2 * F, 3, pk["conv"], 2 * Fp, 3, split_dst=-1, split_src=F)
                tab.add(pv[p + fk["gin"]], F, 1, F, pk["gin"], 1, Fp)
            for s, seq in enumerate(self.seqs):
                # [q, C, d] -> [q, Cp, d]: every head padded with zero rows
                dual = self.pk_logit[s] is not self.pk_logit_b[s]
                tab.add(pv[f"logit_weights.{s}"], d, seq.num_quantizers * self.C[s], d, self.pk_logit[s].view(-1, d),
                        seq.num_quantizers * self.Cp[s], d, split_dst=self.Cp[s], split_src=self.C[s],
                        dst2=self.pk_logit_b[s].view(-1, d) if dual else None)
            self._pack_table = tab
        self._pack_table.run()
        if self.bias_type == "continuous":
            for j in (1, 2):
                lib.split3_bf16(pv[f"transformer.rel_pos_bias.net.{j}.0.weight"], self.pk_rp[j - 1], weight_mode=True)
        self._packed_version = ver

    def grad_bucket_plan(self, min_elems=4 << 20, frozen=()):
        """All-reduce buckets of the gradient arena in backward-completion order (dist_utils.plan_buckets).  Buckets
        that hold no trainable parameter (only names in `frozen`, and padding) are left out: their gradient is zero on
        every rank and nothing reads it."""
        from .dist_utils import drop_frozen_buckets, plan_buckets
        sizes = {n: p.numel() for n, p in self.m.named_parameters()}
        plan = plan_buckets(self.layout, sizes, self.n_params_arena, self.L, min_elems)
        return drop_frozen_buckets(plan, [(self.layout[n], self.layout[n] + sizes[n]) for n in sizes if n not in frozen])

    def backward_plan(self, frozen=()) -> _BackwardPlan:
        key = frozenset(frozen)
        if key not in self._bwd_plans:
            self._bwd_plans[key] = _BackwardPlan(self, key)
        return self._bwd_plans[key]

    def _trainable_rows(self, bp: _BackwardPlan, src_row):
        """src_row with the rows of frozen row tables set to -1 (the scatter-add skips them), for a partly frozen set of
        embedding / absolute-position tables and start tokens."""
        live = self._row_live.get(bp.frozen)
        if live is None:
            live = torch.zeros(self.table.numel() // self.d, dtype=torch.bool)
            for n, p in self.m.named_parameters():
                if n.startswith(("embeddings.", "absolute_position_embeddings.", "start_tokens.")) and bp.trains(n):
                    r0 = (self.layout[n] - self.emb_off) // self.d
                    live[r0:r0 + p.numel() // self.d] = True
            live = self._row_live[bp.frozen] = live.to(self.dev)
        return torch.where(live[src_row.clamp(min=0).long()], src_row, torch.full_like(src_row, -1))

    def check_errors(self):
        """Raises if a token id outside an embedding table was seen since the last check (nn.Embedding's IndexError;
        asynchronous like the reference's device-side assert on CUDA: this call synchronises).  Also raises if, in
        deterministic mode, the attention backward's ordered accumulation gave up waiting for a turn: those steps summed
        in arrival order (correct up to rounding) and are not reproducible.  Both flags are cleared by the raise."""
        bits = int(self.err_flag.item())
        if bits:
            self.err_flag.zero_()
            bad = [s for s in range(len(self.seqs)) if bits >> s & 1]
            raise lib.OmlmError(f"token id out of range for the embedding table of sequence(s) {bad} "
                                f"(valid ids: 0..codebook_size, or the pad id at quantizer-0 positions)")
        late = [w for w in list(self._det_attn) if w.error()]
        if late:
            for w in late:
                w.clear_error()
            raise lib.OmlmError("deterministic mode: the attention backward timed out waiting for an accumulation turn; "
                                "the steps since the last check summed dQ / dK|dV in arrival order (correct up to rounding, "
                                "not reproducible)")

    # ------------------------------------------------------------------------------------------ plans / workspaces
    _MAX_SHAPES = 8       # plans / workspaces kept (least recently used shapes are dropped: their HBM returns to torch)

    def plan(self, B, n_tok) -> _Plan:
        key = (B, tuple(n_tok))
        pl = self._plans.pop(key, None)
        if pl is None:
            pl = _Plan(self, B, n_tok, self.dev)
        self._plans[key] = pl                       # (re-)inserted last = most recently used
        while len(self._plans) > self._MAX_SHAPES:
            self._plans.pop(next(iter(self._plans)))
        return pl

    # deterministic mode: bytes of split-K partials the weight-gradient GEMMs may use (the split count is capped to fit)
    DET_WGRAD_PART_BYTES = 64 << 20

    def workspace(self, pl: _Plan, train: bool, det: bool = False):
        """Activation buffers of one shape.  det (torch.are_deterministic_algorithms_enabled() when the step is issued):
        a separate set that also holds the scratch of the fixed-order kernel variants (add_det_scratch)."""
        key = (pl.B, tuple(pl.n_tok), train, det)
        if key in self._ws:
            ws = self._ws.pop(key)
            self._ws[key] = ws                      # most recently used
            return ws
        while len(self._ws) >= self._MAX_SHAPES:
            self._ws.pop(next(iter(self._ws)))
        dev, bf, f32, a16 = self.dev, torch.bfloat16, torch.float32, self.a16
        M, d, HD, Fp, h = pl.M, self.d, self.HD, self.Fp, self.h
        E = lambda *shape, dt=bf: torch.empty(*shape, device=dev, dtype=dt)
        nl = self.L if train else 1
        ws = dict(
            x=[E(M, d, dt=f32) for _ in range(2 * nl + 1)],       # residual stream snapshots: x_l, x_mid_l, ..., x_L
            xn=[E(M, d) for _ in range(nl)], xraw=[E(M, d) for _ in range(nl)], st_a=[E(M, 2, dt=f32) for _ in range(nl)],
            q_raw=[E(M, HD) for _ in range(nl)], kv_raw=[E(M, 128) for _ in range(nl)],
            qn=[E(M, HD) for _ in range(nl)], kvn=[E(M, 128) for _ in range(nl)],
            o=[E(M, HD) for _ in range(nl)], lse=[E(M * h, dt=f32) for _ in range(nl)],
            xn2=[E(M, d) for _ in range(nl)], st_f=[E(M, 2, dt=f32) for _ in range(nl)],
            u=[E(M, 2 * Fp, dt=a16) for _ in range(nl)], hn=[E(M, Fp) for _ in range(nl)], st_i=[E(M, 2, dt=f32) for _ in range(nl)],
            keep=[E(M, Fp // 8, dt=torch.uint8) for _ in range(nl)],   # FFN dropout keep mask, 1 bit per element
            xf=E(max(pl.rows_total, 1), d), st_o=E(M, 2, dt=f32), h=E(M, Fp, dt=a16), rowsum=E(M, Fp // 128, 2, dt=f32),
            logits=[E(max(pl.B * c, 1), self.Cp[s], dt=f32) for (s, qi, c, b0) in pl.groups],
            # rel-pos MLP
            rp_in=E(pl.N, 1, dt=f32), rp_z=[E(pl.N, self.Hr, dt=f32) for _ in range(3)],
            rp_a=[E(pl.N, self.Hr, dt=f32) for _ in range(3)], table=E(h, pl.N, dt=f32),
            rp_a3=[E(pl.N, 3 * self.Hr8) for _ in range(2)],
        )
        if a16 != bf:   # fp16 forward operands (transient: one buffer each); xn / xn2 / hn / xf above are then the bf16
            ws.update(xn16=E(M, d, dt=a16), xn2_16=E(M, d, dt=a16), hn16=E(M, Fp, dt=a16),   # duplicates kept for backward
                      xf16=E(max(pl.rows_total, 1), d, dt=a16))
        lib.arange_f32(ws["rp_in"])
        if self.bias_type == "none":
            ws["table"].zero_()                 # no bias is added (transformer.py:372-373): written once, never touched again
        elif self.bias_type == "t5":
            ws["ones"] = torch.ones(pl.N, device=dev, dtype=f32)
        if train:
            ws.update(
                dlogits=[E(max(pl.B * c, 1), self.Cp[s]) for (s, qi, c, b0) in pl.groups],
                dxf=E(max(pl.rows_total, 1), d), dx=[E(M, d, dt=f32) for _ in range(2)], dx_bf=E(M, d),
                dhn=E(M, Fp), rowstat=E(M, Fp // 128, 2, dt=f32), du=E(M, 2 * Fp), dxn=E(M, d), dxraw=E(M, d),
                d_o=E(M, HD), dqn=E(M, HD, dt=f32), dkvn=E(M, 128, dt=f32), dsum=E(M * h, dt=f32),
                dq_raw=E(M, HD), dkv_raw=E(M, 128), dtable=E(h, pl.N, dt=f32),
                rp_d0=E(pl.N, self.Hr, dt=f32), rp_d1=E(pl.N, self.Hr, dt=f32), rp_dz3=E(pl.N, 3 * self.Hr8),
            )
        if det:
            self.add_det_scratch(pl, ws, train)
        self._ws[key] = ws
        return ws

    def add_det_scratch(self, pl: _Plan, ws, train: bool):
        """Scratch of the deterministic kernel variants (include/omlm_b200.h, *_det): one fp32 buffer for the per-CTA
        partial sums (the kernels run one after another on the stream and share it), the attention backward's workspace,
        the split-K partials of the weight gradients, and, once per engine, the grad_sumsq partials and the embedding
        row markers.  Allocated only in deterministic mode, before any graph capture."""
        if "det_part" in ws and (ws.get("det_train") or not train):
            return
        dev, sms, d, B, N = self.dev, self._num_sms(), self.d, pl.B, pl.N
        rows_ce = max(pl.B * c for (_, _, c, _) in pl.groups)
        floats = max(2 * ((rows_ce + 7) // 8), 64)                              # cross-entropy (loss, rows) pairs
        if train:
            floats = max(floats, 4 * sms * max(d, 128),                         # layernorm_bwd dgamma rows
                         8 * sms * 128,                                         # qk_l2norm_bwd scale rows
                         B * ((N + 127) // 128) * 7 * self.F)                   # ffn_mid_bwd gamma / conv rows
            ws["det_attn"] = lib.AttnBwdDetWorkspace(dev, B, N, self.h)
            self._det_attn.add(ws["det_attn"])
            shapes = [(cp, d) for cp in self.Cp] + [(d, self.F), (2 * self.F, d), (d, self.HD), (self.HD, d), (128, d)]
            need = max(48 * m * _round_up(n, 4) * 4 for m, n in shapes)
            ws["det_wgrad"] = torch.empty(min(need, self.DET_WGRAD_PART_BYTES) // 4, device=dev, dtype=torch.float32)
            if self.det_sumsq_part is None:
                self.det_sumsq_part = torch.empty(4 * sms, device=dev, dtype=torch.float64)
            if self.det_rows is None:
                self.det_rows = lib.embed_row_markers(self.table.numel() // d, dev)
        ws["det_part"] = torch.empty(floats, device=dev, dtype=torch.float32)
        ws["det_train"] = train

    # ------------------------------------------------------------------------------------------ forward
    # tile / split-K choice: minimise  waves x (k-blocks per unit x tile cost + epilogue)  over the device's SMs
    _sms = None
    # cost of one k-block of a 128x256 tile in units of a 128x128 one: 256-wide tiles measured ~4 % more efficient per
    # flop than 128-wide ones at the cfg2 GEMM shapes (tools/bench_gemm.py; H100 SXM, 400 W power limit)
    KB_COST_256 = 2.0 / 1.04

    @classmethod
    def _num_sms(cls):
        if cls._sms is None:
            cls._sms = lib.num_sms()
        return cls._sms

    @classmethod
    def _tile_cost(cls, m, n, kb, bn, splits, epi):
        sms = cls._num_sms()
        tiles = ((m + 127) // 128) * ((n + bn - 1) // bn)
        waves = (tiles * splits + sms - 1) // sms
        per_kb = 1.0 if bn == 128 else cls.KB_COST_256
        return waves * (((kb + splits - 1) // splits) * per_kb + epi * (bn / 128.0))

    @classmethod
    def _bn_for(cls, m, n, k):
        kb = (k + 63) // 64
        if n <= 128:
            return 128
        return min((128, 256), key=lambda bn: cls._tile_cost(m, n, kb, bn, 1, 6.0))

    @staticmethod
    def _bn(N):
        return 256 if N % 256 == 0 or N >= 2048 else 128

    def build_bias_table(self, ws, N):
        """table[h, delta] for delta = i - j in [0, N) of the configured relative position bias (transformer.py:366-373)."""
        if self.bias_type == "continuous":
            self._relpos_table(ws, N)
        elif self.bias_type == "t5":
            # T5RelativePositionBias (transformer.py:69-117) is fed i - j and negates it, so every causally visible pair
            # falls into bucket 0: the table is the constant row 0 of the bucket embedding, one value per head
            w = self.pview["transformer.rel_pos_bias.relative_attention_bias.weight"]       # [32, h]
            lib.sgemm_small(w, (1, 1), ws["ones"], (1, 1), ws["table"], (ws["table"].stride(0), 1), self.h, N, 1)
        # 'none': the table stays zero

    def bias_table_backward(self, ws, N, det=False, bp: Optional[_BackwardPlan] = None):
        """Gradients of the bias parameters from ws['dtable']; bp: the frozen ones are skipped."""
        if self.bias_type == "continuous":
            self._relpos_backward(ws, N, det, bp if bp is not None else self.backward_plan())
        elif self.bias_type == "t5":
            gw = self.gview["transformer.rel_pos_bias.relative_attention_bias.weight"]      # bucket 0 collects every delta
            # (the table has a gradient only when this, the T5 path's one parameter, is trainable)
            lib.colsum(ws["dtable"], 1, ws["dtable"].stride(0), gw[0], N, self.h, accumulate=True)

    def _relpos_table(self, ws, N):
        """RelativePositionBias MLP on the causal distances 0..N-1 -> table[h, N] (transformer.py:55-67).
        The two Hr x Hr layers run on the wgmma GEMM with bf16x3-split operands (fp32-class accuracy: the
        table reaches |b| ~ 100 and dominates the logits); the rank-1 first layer and the h-wide last layer are SIMT."""
        pv, Hr, h = self.pview, self.Hr, self.h
        pre = "transformer.rel_pos_bias.net."
        lib.sgemm_small(ws["rp_in"], (1, 1), pv[pre + "0.0.weight"], (1, 1), ws["rp_a"][0], (Hr, 1), N, Hr, 1,
                        Z=ws["rp_z"][0], bias=pv[pre + "0.0.bias"], act=1)
        for j in (1, 2):
            lib.split3_bf16(ws["rp_a"][j - 1], ws["rp_a3"][j - 1])
            lib.gemm(ws["rp_a3"][j - 1], self.pk_rp[j - 1], ws["rp_z"][j], block_n=128)
            lib.bias_silu(ws["rp_z"][j], pv[f"{pre}{j}.0.bias"], ws["rp_a"][j])
        # no split-K here: atomics would make the table, and through bf16 rounding every logit, depend on CTA timing
        lib.sgemm_small(ws["rp_a"][2], (Hr, 1), pv[pre + "3.weight"], (1, Hr), ws["table"], (1, N), N, h, Hr, bias=pv[pre + "3.bias"])

    def forward_core(self, pl: _Plan, ws, src_row, key_mask, train: bool, groups_wanted=None, drop: bool = False, capture=None):
        """Runs embeddings -> depth x (attention, conv-FFN) -> final LN -> logit heads.  Activations stay in `ws`.
        capture (decode.py): receives each layer's K/V rows and pre-conv FFN rows (the generation caches of the prompt)."""
        self.refresh_packed()
        B, N, h, Fp = pl.B, pl.N, self.h, self.Fp
        pv = self.pview
        lib.embed_gather(self.table, src_row, ws["x"][0], pl.src_row2)
        self.build_bias_table(ws, N)
        x_last = self._layers(ws, pl.M, train, drop, capture,
                              lambda i, l: lib.attn_fwd_tc(ws["qn"][i], ws["kvn"][i], ws["table"], key_mask, ws["o"][i], ws["lse"][i], B, N, h),
                              lambda xn2, i, l, pk: lib.gemm_ffn_up(xn2, pk["w1"], pk["conv"], ws["u"][i], ws["h"], ws["rowsum"], N, Fp))
        f16 = self.a16 != torch.bfloat16
        dup = f16 and train
        xf = ws["xf16"] if f16 else ws["xf"]
        lib.layernorm_fwd(x_last, pv["transformer.norm.gamma"], xf, None, ws["st_o"], pl.dest_row, ycopy=ws["xf"] if dup else None)
        for gi, (s, qi, cnt, base) in enumerate(pl.groups):
            if groups_wanted is not None and s not in groups_wanted:
                continue
            rows = B * cnt
            lib.gemm(xf[base:base + rows], self.pk_logit[s][qi], ws["logits"][gi], block_n=128)

    def _layers(self, ws, M: int, train: bool, drop: bool, capture, attn, ffn_up):
        """The depth x (attention, conv-FFN) loop over the M rows of ws["x"][0]; attn(i, l) and ffn_up(xn2, i, l, pk) launch
        the two kernels that depend on how the rows form sequences (i: the workspace slot of layer l).  Returns the last residual stream."""
        d, h, HD, F, Fp = self.d, self.h, self.HD, self.F, self.Fp
        pv = self.pview
        x = ws["x"]
        drop_p = self.drop_p if drop else 0.0
        f16 = self.a16 != torch.bfloat16
        dup = f16 and train            # the backward pass needs bf16 duplicates of the fp16 forward operands
        for l in range(self.L):
            i = l if train else 0
            xa, xm, xo = (x[2 * l], x[2 * l + 1], x[2 * l + 2]) if train else (x[0], x[1], x[0])
            p, pk = f"transformer.layers.{l}.", self.pk[l]
            xn = ws["xn16"] if f16 else ws["xn"][i]
            lib.layernorm_fwd(xa, pv[p + "0.norm.gamma"], xn, ws["xraw"][i], ws["st_a"][i], ycopy=ws["xn"][i] if dup else None)
            lib.gemm(xn, pk["wq"], ws["q_raw"][i], block_n=self._bn_for(M, HD, d))
            lib.gemm(ws["xraw"][i], pk["wkv_b"], ws["kv_raw"][i], block_n=128)
            lib.qk_l2norm_fwd(ws["q_raw"][i], ws["kv_raw"][i], pv[p + "0.q_scale"], pv[p + "0.k_scale"], ws["qn"][i], ws["kvn"][i], h)
            if capture is not None:
                capture.after_kv(l, ws["kvn"][i])
            attn(i, l)
            lib.gemm(ws["o"][i], pk["wo_b"], xm, addend=xa, block_n=self._bn_for(M, d, HD))
            xn2 = ws["xn2_16"] if f16 else ws["xn2"][i]
            lib.layernorm_fwd(xm, pv[p + self.ffk["g1"]], xn2, None, ws["st_f"][i], ycopy=ws["xn2"][i] if dup else None)
            ffn_up(xn2, i, l, pk)                                                 # conv + GEGLU in the epilogue
            if capture is not None:
                capture.after_u(l, ws["u"][i])
            hn = ws["hn16"] if f16 else ws["hn"][i]
            lib.ffn_norm_fwd(ws["h"], ws["rowsum"], pk["gin"], hn, ws["st_i"][i], F, Fp, drop_p, self.seed, l,
                             keep_bits=ws["keep"][i] if drop_p > 0 else None, hn_copy=ws["hn"][i] if dup else None)
            lib.gemm(hn, pk["w2"], xo, addend=xm, block_n=self._bn_for(M, d, Fp))
        return x[2 * self.L] if train else x[0]

    # ------------------------------------------------------------------------------------------ packed prefill
    def packed_workspace(self, rows: int, head_rows: int):
        """Inference activations for packed forwards of up to `rows` rows (forward_packed runs on views of the first M),
        and up to `head_rows` rows of final-norm output and logits of the last sequence's heads."""
        dev, bf, f32, a16 = self.dev, torch.bfloat16, torch.float32, self.a16
        d, HD, Fp, h = self.d, self.HD, self.Fp, self.h
        E = lambda *shape, dt=bf: torch.empty(*shape, device=dev, dtype=dt)
        ws = dict(x=[E(rows, d, dt=f32) for _ in range(2)], xraw=[E(rows, d)], st_a=[E(rows, 2, dt=f32)], q_raw=[E(rows, HD)],
                  kv_raw=[E(rows, 128)], qn=[E(rows, HD)], kvn=[E(rows, 128)], o=[E(rows, HD)], lse=[E(rows, h, dt=f32)],
                  st_f=[E(rows, 2, dt=f32)], u=[E(rows, 2 * Fp, dt=a16)], st_i=[E(rows, 2, dt=f32)], h=E(rows, Fp, dt=a16),
                  rowsum=E(rows, Fp // 128, 2, dt=f32), st_o=E(rows, 2, dt=f32),
                  logits=E(head_rows, self.Cp[-1], dt=f32))
        if a16 != bf:
            ws.update(xn16=E(rows, d, dt=a16), xn2_16=E(rows, d, dt=a16), hn16=E(rows, Fp, dt=a16), xf16=E(head_rows, d, dt=a16))
        else:
            ws.update(xn=[E(rows, d)], xn2=[E(rows, d)], hn=[E(rows, Fp)], xf=E(head_rows, d))
        return ws

    def forward_packed(self, ws, pk_plan, table, capture=None, kv=None, hist=None):
        """Inference forward of sequences of their own lengths packed back to back without padding (pk_plan: M rows,
        src_row, src_row2, row_pos, seq_start, seq_len, the attention work list, dest_row and the head groups; see
        session.PackedPrefill) in a packed_workspace.  The layer loop is forward_core's, with the varlen attention and
        FFN-up kernels; table: a bias table at least as long as the longest sequence.  The final norm writes only the
        rows dest_row names, and head group (qi, base, cnt) leaves the logits of head qi of the last sequence for its
        cnt rows in ws["logits"][base:base + cnt].  Every row's values are those of forward_core on its sequence alone.

        Chunks (pk_plan also has q_off, kv_start, max_end and hist_idx): sequence b is positions q_off[b] ... of a longer
        prompt.  With kv, layer l's attention reads its keys from kv[l] (viewed [rows, 128]) at rows kv_start[b] ...,
        which capture.after_kv must have filled for positions 0 ... q_off[b] + seq_len[b] - 1; with hist, its FFN-up
        takes the conv history of a chunk's first row from hist[l] (rows 2c, 2c + 1 for hist_idx = c; needed when some
        q_off > 0).  Every row's values are then those of forward_core on its whole prompt."""
        self.refresh_packed()
        pp, M, Fp = pk_plan, pk_plan.M, self.Fp
        v = {k: [e[:M] for e in t] if isinstance(t, list) else t[:M] for k, t in ws.items() if k not in ("logits", "xf", "xf16")}
        lib.embed_gather(self.table, pp.src_row, v["x"][0], pp.src_row2)
        if kv is None:
            attn = lambda i, l: lib.attn_fwd_tc_varlen(v["qn"][i], v["kvn"][i], table, pp.work, pp.seq_start, pp.seq_len, pp.max_len,
                                                       v["o"][i], v["lse"][i], self.h)
        else:
            attn = lambda i, l: lib.attn_fwd_tc_chunk(v["qn"][i], kv[l].view(-1, 128), table, pp.work, pp.seq_start, pp.seq_len,
                                                      pp.q_off, pp.kv_start, pp.max_end, v["o"][i], v["lse"][i], self.h)
        if hist is None:
            ffn_up = lambda xn2, i, l, pk: lib.gemm_ffn_up_varlen(xn2, pk["w1"], pk["conv"], v["u"][i], v["h"], v["rowsum"], pp.row_pos, Fp)
        else:
            ffn_up = lambda xn2, i, l, pk: lib.gemm_ffn_up_chunk(xn2, pk["w1"], pk["conv"], v["u"][i], v["h"], v["rowsum"], pp.row_pos,
                                                                 hist[l], pp.hist_idx, Fp)
        x_last = self._layers(v, M, False, False, capture, attn, ffn_up)
        xf = ws["xf16"] if self.a16 != torch.bfloat16 else ws["xf"]
        lib.layernorm_fwd(x_last, self.pview["transformer.norm.gamma"], xf, None, v["st_o"], pp.dest_row)
        S = len(self.seqs) - 1
        for qi, base, cnt in pp.groups:
            lib.gemm(xf[base:base + cnt], self.pk_logit[S][qi], ws["logits"][base:base + cnt], block_n=128)

    # ------------------------------------------------------------------------------------------ backward
    def _wgrad(self, dy, x, gout, m, n, det_part=None, **kw):
        """gout[m, n] += dy[rows, m]^T x[rows, n]   (both operands MN-major, fp32 accumulate into the grad arena).
        det_part (deterministic mode): split-K partials go to this scratch and are summed in split order; the split
        count is capped so that they fit."""
        k = dy.shape[0]
        kb = (k + 63) // 64
        s_max = max(1, min(kb // 8, 48))
        if det_part is not None:
            rs, rv, nv = kw.get("row_split", 0), kw.get("row_valid", 0), kw.get("n_valid", 0) or n
            rows_out = (m + rs - 1) // rs * rv if rs > 0 else (2 * rv if rs < 0 else m)
            s_max = max(1, min(s_max, det_part.numel() // (rows_out * _round_up(nv, 4))))
        best = None
        for bn in (128, 256):
            for s in range(1, s_max + 1):
                c = self._tile_cost(m, n, kb, bn, s, 14.0 if s > 1 else 10.0)
                if best is None or c < best[0]:
                    best = (c, bn, s)
        _, bn, s = best
        if det_part is not None:
            lib.gemm_splitk_det(dy, x, gout, det_part, a_mn=True, b_mn=True, M=m, N=n, K=k, splits=s, block_n=bn,
                                max_ctas=self.bwd_max_ctas, **kw)
        elif s > 1:
            lib.gemm(dy, x, gout, a_mn=True, b_mn=True, M=m, N=n, K=k, splits=s, block_n=bn, max_ctas=self.bwd_max_ctas, **kw)
        else:
            lib.gemm(dy, x, gout, a_mn=True, b_mn=True, M=m, N=n, K=k, addend=gout, block_n=bn, max_ctas=self.bwd_max_ctas, **kw)

    def backward_core(self, pl: _Plan, ws, src_row, key_mask, groups_with_grad, drop: bool = False, on_ready=None, det: bool = False,
                      frozen=()):
        """Consumes ws['dlogits'] (bf16, permuted rows) and accumulates every parameter gradient into arena_g.
        on_ready(trigger): called when a group of gradients is final -- 'heads', 'layer<l>' (matrices of layer l), 'tail'
        (everything else) -- so that a data-parallel caller can start reducing it underneath the rest of the pass.
        det: the fixed-order kernel variants (ws must hold their scratch, see add_det_scratch): bit-identical gradients
        for identical inputs on the same GPU model.
        frozen: names of parameters that get no gradient.  Their arena_g ranges are not written, and only the work a
        trainable parameter needs runs (_BackwardPlan): no weight-gradient GEMM of a frozen matrix, no bias-table gradient
        when nothing trains the table, and nothing below the lowest layer a gradient still has to reach.  The gradients of
        the trainable parameters are those of the full pass (bit for bit in deterministic mode).  on_ready is still
        called at every point (the data-parallel plan leaves the fully frozen buckets out, grad_bucket_plan)."""
        ready = on_ready if on_ready is not None else (lambda trigger: None)
        bp = self.backward_plan(frozen)
        tr = bp.trains
        gw = lambda n: self.gview[n] if tr(n) else None        # parameter-gradient output, None when frozen
        part = ws["det_part"] if det else None
        wpart = ws["det_wgrad"] if det else None
        B, N, M, d, h, HD, F, Fp = pl.B, pl.N, pl.M, self.d, self.h, self.HD, self.F, self.Fp
        pv, gv = self.pview, self.gview
        x = ws["x"]
        drop_p = self.drop_p if drop else 0.0
        # ---- logit heads
        gset = frozenset(groups_with_grad)
        if bp.final_norm and ws.get("dxf_groups") != gset:   # rows of head groups without a gradient stay zero; the others are overwritten
            ws["dxf"].zero_()
            ws["dxf_groups"] = gset
        for gi, (s, qi, cnt, base) in enumerate(pl.groups):
            if s not in groups_with_grad:
                continue
            rows = B * cnt
            dl = ws["dlogits"][gi]
            if bp.final_norm:
                lib.gemm(dl, self.pk_logit_b[s][qi], ws["dxf"][base:base + rows], b_mn=True, M=rows, N=d, K=self.Cp[s], block_n=128, max_ctas=self.bwd_max_ctas)
            if tr(f"logit_weights.{s}"):
                self._wgrad(dl, ws["xf"][base:base + rows], gv[f"logit_weights.{s}"][qi], self.Cp[s], d, det_part=wpart, row_split=self.Cp[s],
                            row_valid=self.C[s])
        ready("heads")
        dxa, dxb = ws["dx"]
        if bp.final_norm:
            lib.layernorm_bwd(ws["dxf"], x[2 * self.L], ws["st_o"], pv["transformer.norm.gamma"], dxa, gw("transformer.norm.gamma"),
                              src_row=pl.dest_row, dx_bf16=ws["dx_bf"], part=part)
        dtable = ws["dtable"] if bp.dtable else None
        if dtable is not None:
            dtable.zero_()
        for l in reversed(range(self.L)):
            if not bp.run[l]:
                ready(f"layer{l}")
                continue
            st = bp.steps[l]
            p, pk = f"transformer.layers.{l}.", self.pk[l]
            xa, xm = x[2 * l], x[2 * l + 1]
            # ---- conv feed-forward
            # d_hn = dx W2 with the LayerNorm-backward row sums (against the saved hn) taken in the GEMM's epilogue
            fk = self.ffk
            keep = ws["keep"][l] if drop_p > 0 else None
            if st["ffn"]:
                if Fp % 256 == 0:
                    lib.gemm_rowstat(ws["dx_bf"], pk["w2_b"], ws["dhn"], ws["hn"][l], pk["gin"], ws["rowstat"], b_mn=True, M=M, N=Fp, K=d,
                                     keep_bits=keep, keep_scale=1.0 / (1.0 - drop_p) if drop_p > 0 else 1.0, max_ctas=self.bwd_max_ctas)
                    parts = Fp // 128
                else:
                    lib.gemm(ws["dx_bf"], pk["w2_b"], ws["dhn"], b_mn=True, M=M, N=Fp, K=d, block_n=self._bn_for(M, Fp, d), max_ctas=self.bwd_max_ctas)
                    parts = 0
                # (the tile kernel runs right behind the GEMM that wrote dhn, while dhn is still in L2; the weight gradient after it)
                lib.ffn_mid_bwd(ws["dhn"], ws["hn"][l], ws["u"][l], ws["st_i"][l], pk["conv"], pk["gin"], ws["rowstat"], ws["du"],
                                gw(p + fk["gin"]), gw(p + fk["conv"]) if fk["conv"] is not None else None, B, N, F, Fp, drop_p,
                                keep_bits=keep, rowstat_parts=parts, part=part)
            if tr(p + fk["w2"]):
                self._wgrad(ws["dx_bf"], ws["hn"][l], gv[p + fk["w2"]], d, Fp, det_part=wpart, n_valid=F)
            if st["ln_f"]:
                lib.gemm(ws["du"], pk["w1_b"], ws["dxn"], b_mn=True, M=M, N=d, K=2 * Fp, block_n=self._bn_for(M, d, 2 * Fp), max_ctas=self.bwd_max_ctas)
            if tr(p + fk["w1"]):
                self._wgrad(ws["du"], ws["xn2"][l], gv[p + fk["w1"]], 2 * Fp, d, det_part=wpart, row_split=-1, row_valid=F)
            if st["ln_f"]:
                lib.layernorm_bwd(ws["dxn"], xm, ws["st_f"][l], pv[p + fk["g1"]], dxb, gw(p + fk["g1"]), dres=dxa, dx_bf16=ws["dx_bf"], part=part)
            # ---- attention
            if st["attn"]:
                lib.gemm(ws["dx_bf"], pk["wo_b"], ws["d_o"], b_mn=True, M=M, N=HD, K=d, block_n=self._bn_for(M, HD, d), max_ctas=self.bwd_max_ctas)
            if tr(p + "0.to_out.0.weight"):
                self._wgrad(ws["dx_bf"], ws["o"][l], gv[p + "0.to_out.0.weight"], d, HD, det_part=wpart)
            if st["attn"]:
                lib.attn_bwd_tc(ws["qn"][l], ws["kvn"][l], ws["d_o"], ws["o"][l], ws["lse"][l], ws["table"], key_mask, ws["dsum"],
                                ws["dqn"], ws["dkvn"], dtable, B, N, h, det=ws["det_attn"] if det else None)
            if st["qk"]:
                lib.qk_l2norm_bwd(ws["dqn"], ws["dkvn"], ws["q_raw"][l], ws["kv_raw"][l], pv[p + "0.q_scale"], pv[p + "0.k_scale"],
                                  ws["dq_raw"], ws["dkv_raw"], gw(p + "0.q_scale"), gw(p + "0.k_scale"), h, part=part)
            if st["ln_a"]:
                lib.gemm(ws["dq_raw"], pk["wq_b"], ws["dxn"], b_mn=True, M=M, N=d, K=HD, block_n=self._bn_for(M, d, HD), max_ctas=self.bwd_max_ctas)
            if st["g_in"]:
                lib.gemm(ws["dkv_raw"], pk["wkv_b"], ws["dxraw"], b_mn=True, M=M, N=d, K=128, block_n=self._bn_for(M, d, 128), max_ctas=self.bwd_max_ctas)
            if tr(p + "0.to_q.weight"):
                self._wgrad(ws["dq_raw"], ws["xn"][l], gv[p + "0.to_q.weight"], HD, d, det_part=wpart)
            if tr(p + "0.to_kv.weight"):
                self._wgrad(ws["dkv_raw"], ws["xraw"][l], gv[p + "0.to_kv.weight"], 128, d, det_part=wpart)
            ready(f"layer{l}")
            if st["ln_a"]:
                lib.layernorm_bwd(ws["dxn"], xa, ws["st_a"][l], pv[p + "0.norm.gamma"], dxa, gw(p + "0.norm.gamma"),
                                  dres=dxb if st["g_in"] else None, draw=ws["dxraw"] if st["g_in"] else None, dx_bf16=ws["dx_bf"], part=part)
        # ---- embeddings + start tokens (grad_shrink: utils.py:60-61)
        if bp.rows:
            rows = self.det_rows if det else None
            src1, src2 = src_row, pl.src_row2
            if bp.rows_partial:
                src1 = self._trainable_rows(bp, src1)
                src2 = self._trainable_rows(bp, src2) if src2 is not None else None
            lib.embed_scatter_add(self.dtable_emb, src1, dxa, self.alpha, first=rows)
            if src2 is not None:
                lib.embed_scatter_add(self.dtable_emb, src2, dxa, self.alpha, first=rows)
        if dtable is not None:
            self.bias_table_backward(ws, N, det, bp)
        ready("tail")

    def _relpos_backward(self, ws, N, det, bp: _BackwardPlan):
        pv, gv, Hr, T, h = self.pview, self.gview, self.Hr, self.Hr8, self.h
        pre = "transformer.rel_pos_bias.net."
        tr = bp.trains
        dT = ws["dtable"]                                   # [h, N]: dY[n, hh] = dT[hh, n]
        a3 = ws["rp_a"][2]
        if tr(pre + "3.weight"):
            lib.sgemm_small(dT, (N, 1), a3, (Hr, 1), gv[pre + "3.weight"], (Hr, 1), h, Hr, N, accumulate=True, det=det)   # dW4 = dY^T a3
        if tr(pre + "3.bias"):
            lib.colsum(dT, 1, N, gv[pre + "3.bias"], N, h, accumulate=True)
        # the MLP's gradient flows down only as far as its lowest trainable layer (j = 2, 1, 0)
        lowest = min([j for j in (0, 1, 2) if tr(f"{pre}{j}.0.weight") or tr(f"{pre}{j}.0.bias")], default=3)
        d_cur, d_nxt = ws["rp_d0"], ws["rp_d1"]
        if lowest < 3:
            lib.sgemm_small(dT, (1, N), pv[pre + "3.weight"], (Hr, 1), d_cur, (Hr, 1), N, Hr, h)                  # da3 = dY W4
        for j in (2, 1, 0):
            if j < lowest:
                break
            lib.silu_bwd(d_cur, ws["rp_z"][j], d_cur)                                                              # dz_j (fp32, in place)
            if tr(f"{pre}{j}.0.bias"):
                lib.colsum(d_cur, Hr, 1, gv[f"{pre}{j}.0.bias"], N, Hr, accumulate=True)
            if j > 0:
                # bf16x3 products, as in the forward pass (x y ~ x_hi y_hi + x_hi y_lo + x_lo y_hi: fp32-class): these
                # gradients are sums of cancelling terms, so a plain bf16 operand rounding shows up amplified
                lib.split3_bf16(d_cur, ws["rp_dz3"])                                                               # [hi | hi | lo]
                dz_hi, dz_lo = ws["rp_dz3"][:, :Hr], ws["rp_dz3"][:, 2 * T:2 * T + Hr]                             # thirds start at 0, T, 2T
                a_hi, a_lo = ws["rp_a3"][j - 1][:, :Hr], ws["rp_a3"][j - 1][:, 2 * T:2 * T + Hr]                   # forward split of a_{j-1}
                w_hi, w_lo = self.pk_rp[j - 1][:, :Hr], self.pk_rp[j - 1][:, T:T + Hr]                             # [hi | lo | hi]
                gw = gv[f"{pre}{j}.0.weight"]
                if tr(f"{pre}{j}.0.weight"):
                    for dz, a in ((dz_hi, a_hi), (dz_hi, a_lo), (dz_lo, a_hi)):                                     # dW_j += dz^T a
                        lib.gemm(dz, a, gw, a_mn=True, b_mn=True, M=Hr, N=Hr, K=N, addend=gw, block_n=128)
                if j == lowest:
                    break
                lib.gemm(dz_hi, w_hi, d_nxt, b_mn=True, M=N, N=Hr, K=Hr, block_n=128)                               # da = dz W
                lib.gemm(dz_hi, w_lo, d_nxt, b_mn=True, M=N, N=Hr, K=Hr, addend=d_nxt, block_n=128)
                lib.gemm(dz_lo, w_hi, d_nxt, b_mn=True, M=N, N=Hr, K=Hr, addend=d_nxt, block_n=128)
                d_cur, d_nxt = d_nxt, d_cur
            elif tr(f"{pre}0.0.weight"):
                lib.sgemm_small(d_cur, (1, Hr), ws["rp_in"], (1, 1), gv[f"{pre}0.0.weight"], (1, 1), Hr, 1, N, accumulate=True, det=det)

    # ------------------------------------------------------------------------------------------ reference-API path
    def api_forward(self, all_token_ids, self_attn_mask, only_final):
        ids = [t.reshape(t.shape[0], -1).to(self.dev, torch.int64).contiguous() for t in all_token_ids]
        assert len(ids) == len(self.seqs)
        B = ids[0].shape[0]
        mask_in = None
        if self_attn_mask is not None:
            mask_in = self_attn_mask.to(self.dev).to(torch.uint8).contiguous()
        _, src_row, key_mask, _, n_tok = lib.token_plan(
            ids, [s.codebook_size for s in self.seqs], [s.num_quantizers for s in self.seqs], self.emb_row_base,
            self.start_row, append_eos=False, drop_last=False, mask_cond=False, mask_in=mask_in, want_labels=False,
            err_flag=self.err_flag)
        pl = self.plan(B, n_tok)
        # requires_grad is read at every call, as autograd reads it: frozen parameters get no gradient (grad stays None)
        named = list(self.m.named_parameters())
        frozen = frozenset(n for n, p in named if not p.requires_grad)
        for n, p in named:
            if n in frozen and p.grad is self.gview[n]:
                p.grad = None           # the arena view handed out before the parameter was frozen, never written by autograd
        need_grad = torch.is_grad_enabled() and len(frozen) < len(named)
        wanted = {len(self.seqs) - 1} if only_final else set(range(len(self.seqs)))
        drop = self.m.training and self.drop_p > 0
        if drop:
            self.seed += 1
        outs = _ApiFunction.apply(self, pl, src_row, key_mask, need_grad, wanted, drop, torch.are_deterministic_algorithms_enabled(),
                                  frozen, *self._param_list)
        res, k = [], 0
        for s in range(len(self.seqs)):
            if s in wanted:
                res.append(outs[k]); k += 1
            else:
                res.append(None)
        return res

    def gather_logits(self, pl, ws, s):
        """Permuted group buffers -> [B, n_out, C] fp32 (re-layout only)."""
        parts = [ws["logits"][gi][:, :self.C[s]] for gi, g in enumerate(pl.groups) if g[0] == s]
        allrows = torch.cat(parts, 0)
        first = min(g[3] for g in pl.groups if g[0] == s)
        return allrows[(pl.seq_row_index[s] - first).reshape(-1)].view(pl.B, pl.n_out[s], self.C[s])

    def scatter_dlogits(self, pl, ws, s, grad):
        """[B, n_out, C] fp32 gradient -> permuted bf16 dlogits buffers (re-layout + cast only)."""
        first = min(g[3] for g in pl.groups if g[0] == s)
        total = sum(pl.B * g[2] for g in pl.groups if g[0] == s)
        buf = torch.zeros(total, self.Cp[s], device=self.dev, dtype=torch.bfloat16)
        buf[(pl.seq_row_index[s] - first).reshape(-1), :self.C[s]] = grad.reshape(-1, self.C[s]).to(torch.bfloat16)
        off = 0
        for gi, g in enumerate(pl.groups):
            if g[0] == s:
                n = pl.B * g[2]
                ws["dlogits"][gi].copy_(buf[off:off + n]); off += n


class _ApiFunction(torch.autograd.Function):
    """One autograd node for the whole TokenConditionedTransformer.forward: libomlm_b200 forward in
    forward(), libomlm_b200 backward in backward(); gradients are returned per parameter."""

    @staticmethod
    def forward(ctx, eng: Engine, pl, src_row, key_mask, need_grad, wanted, drop, det, frozen, *params):
        ws = eng.workspace(pl, need_grad, det)
        eng.forward_core(pl, ws, src_row, key_mask, need_grad, wanted, drop)
        ctx.eng, ctx.pl, ctx.src_row, ctx.key_mask, ctx.wanted, ctx.drop = eng, pl, src_row, key_mask, sorted(wanted), drop
        ctx.need_grad, ctx.frozen = need_grad, frozen
        # the saved activations live in the shape's workspace, not in the graph: a second forward of the same shape before
        # this call's backward would overwrite them -- remember which forward owns the workspace and check in backward
        ws["generation"] = ws.get("generation", 0) + 1
        ctx.ws, ctx.generation = ws, ws["generation"]
        outs = tuple(eng.gather_logits(pl, ws, s) for s in sorted(wanted))
        return outs

    @staticmethod
    def backward(ctx, *grads):
        eng, pl = ctx.eng, ctx.pl
        if not ctx.need_grad:
            raise RuntimeError("forward ran without gradient bookkeeping")
        ws = ctx.ws
        if ws.get("generation") != ctx.generation:
            raise RuntimeError("open_musiclm_b200: the activations of this forward pass were overwritten by a later forward of the "
                               "same shape (one workspace per shape): call backward() before the next forward, or use "
                               "HotPathTrainer for gradient accumulation")
        with_grad = set()
        for s, g in zip(ctx.wanted, grads):
            if g is not None:
                eng.scatter_dlogits(pl, ws, s, g)
                with_grad.add(s)
        # the switch is read again here: a backward issued in deterministic mode runs the fixed-order kernels
        det = torch.are_deterministic_algorithms_enabled()
        if det:
            eng.add_det_scratch(pl, ws, True)
        # gradients are produced in a scratch copy of the arena so that autograd can accumulate them itself
        saved = eng.arena_g.clone()
        eng.arena_g.zero_()
        eng.backward_core(pl, ws, ctx.src_row, ctx.key_mask, with_grad, ctx.drop, det=det, frozen=ctx.frozen)
        fresh = eng.arena_g.clone()
        eng.arena_g.copy_(saved)
        outs = []
        for n, p in eng.m.named_parameters():
            o = eng.layout[n]
            outs.append(None if n in ctx.frozen else fresh[o:o + p.numel()].view(p.shape))
        return (None, None, None, None, None, None, None, None, None, *outs)
