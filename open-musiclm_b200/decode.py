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
"""
import os
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
        k = min(2, s.n_prompt)
        s.conv[l].zero_()
        s.conv[l][:, 2 - k:].copy_(rows[:, s.n_prompt - k:])


class DecodeSession:
    """Caches and scratch of one generate() call: B sequences, a prompt of n_prompt positions, up to n_new new tokens."""

    def __init__(self, eng, B: int, n_prompt: int, n_new: int):
        if eng.abs_pos:
            raise NotImplementedError("open_musiclm_b200 generate: absolute position embeddings are not supported by the decode path")
        if B > MAX_BATCH:
            raise lib.OmlmError(f"open_musiclm_b200 generate: batch sizes above {MAX_BATCH} are not supported by the decode kernels")
        if B > SKINNY_MAX_BATCH and os.environ.get("OMLM_DECODE_FUSED", "0") == "1":
            raise lib.OmlmError(f"open_musiclm_b200 generate: the fused decode step (OMLM_DECODE_FUSED=1) supports at most "
                                f"{SKINNY_MAX_BATCH} sequences (got {B})")
        self.eng, self.B, self.n_prompt, self.n_new = eng, B, n_prompt, n_new
        dev, bf, f32, a16 = eng.dev, torch.bfloat16, torch.float32, eng.a16
        d, HD, Fp, h, Hr = eng.d, eng.HD, eng.Fp, eng.h, eng.Hr
        self.n_max = n_prompt + n_new
        E = lambda *shape, dt=bf: torch.empty(*shape, device=dev, dtype=dt)
        self.cache = [E(B, self.n_max, 128) for _ in range(eng.L)]
        self.conv = [E(B, 2, 2 * Fp, dt=a16) for _ in range(eng.L)]
        self.x = [E(B, d, dt=f32) for _ in range(2)]
        self.q_raw, self.kv_raw, self.o = E(B, HD), E(B, 128), E(B, HD)
        self.u_new, self.h = E(B, 2 * Fp, dt=a16), E(B, Fp, dt=a16)
        self.rowsum = E(B, Fp // 128, 2, dt=f32)
        self.logits = E(B, max(eng.Cp), dt=f32)
        self.tokens = torch.zeros(B, max(n_new, 1), device=dev, dtype=torch.int64)
        self.next_row = torch.zeros(B, device=dev, dtype=torch.int32)
        self.counters = torch.zeros(2, device=dev, dtype=torch.int32)          # [sampled so far, block arrival counter]
        self.pos = torch.full((1,), n_prompt, device=dev, dtype=torch.int32)   # position the next decode step processes
        # bias table for every distance the generation can reach (it depends on i - j only)
        N = self.n_max
        self.rp = dict(rp_in=E(N, 1, dt=f32), rp_z=[E(N, Hr, dt=f32) for _ in range(3)], rp_a=[E(N, Hr, dt=f32) for _ in range(3)],
                       table=E(h, N, dt=f32), rp_a3=[E(N, 3 * Hr) for _ in range(2)])
        lib.arange_f32(self.rp["rp_in"])
        eng.refresh_packed()
        if eng.bias_type == "none":
            self.rp["table"].zero_()
        elif eng.bias_type == "t5":
            self.rp["ones"] = torch.ones(N, device=dev, dtype=f32)
        eng.build_bias_table(self.rp, N)
        self.table = self.rp["table"]
        self._graphs = {}
        # OMLM_DECODE_FUSED=1: the whole step as ONE persistent kernel (csrc/decode_fused.cu; bit-identical to the per-op
        # sequence in step_ops).  Off by default: on the 10 s three-stage generation it is slower than the graph-replayed
        # per-op launches (5.41 s vs 4.10 s on an H100 SXM at a 400 W power limit, tools/time_generate.py) -- its 31
        # stages are each bound by a single-warp prologue (LayerNorm statistics, row-sum tree) and a grid barrier.
        self.fused = os.environ.get("OMLM_DECODE_FUSED", "0") == "1"
        # more than 16 sequences: tensor-core GEMMs and the cache-sharing attention, with their scratch allocated here so
        # that graph capture allocates nothing
        self.batched = B > SKINNY_MAX_BATCH
        if self.batched:
            shapes = [(HD, d), (128, d), (d, HD), (2 * Fp, d), (d, Fp)] + [(cp, d) for cp in eng.Cp]
            self.ws = lib.DecodeWorkspace(dev, B, shapes, max_pos=self.n_max, heads=h)
        if self.fused:
            pv = eng.pview
            layers = []
            for l in range(eng.L):
                p, pk = f"transformer.layers.{l}.", eng.pk[l]
                layers.append(dict(wq=pk["wq"], wkv=pk["wkv_b"], wo=pk["wo_b"], w1=pk["w1"], w2=pk["w2"], conv=pk["conv"], gin=pk["gin"],
                                   g_attn=pv[p + "0.norm.gamma"], g_ff=pv[p + eng.ffk["g1"]], q_scale=pv[p + "0.q_scale"],
                                   k_scale=pv[p + "0.k_scale"], cache=self.cache[l], conv_state=self.conv[l]))
            self.layer_table, self._keep = lib.decode_layer_table(layers, dev)
            self.hf32 = E(B, Fp, dt=f32)
            self.barrier = torch.zeros(1, device=dev, dtype=torch.int32)
            self.err_flag = torch.zeros(1, device=dev, dtype=torch.int32)

    # ------------------------------------------------------------------------------------------ one incremental step
    def step(self, qi_next: int):
        """Processes the position self.pos (embedding row self.next_row) through all layers and leaves the logits of
        head qi_next in self.logits."""
        if not self.fused:
            return self.step_ops(qi_next)
        eng = self.eng
        S = len(eng.seqs) - 1
        lib.decode_step(self.layer_table, eng.L, self.B, eng.d, eng.h, eng.F, eng.Fp, self.n_max, eng.a16 == torch.float16, eng.table,
                        self.next_row, self.table, self.pos, self.x[0], self.x[1], self.q_raw, self.kv_raw, self.o, self.h, self.hf32,
                        eng.pk_logit[S][qi_next], eng.pview["transformer.norm.gamma"], self.logits, self.barrier, self.err_flag)

    def check(self):
        """Raises if a grid-wide barrier of the fused step timed out (synchronises)."""
        if self.fused and int(self.err_flag.item()):
            raise lib.OmlmError("open_musiclm_b200 generate: the fused decode step timed out at a grid barrier")

    def step_ops(self, qi_next: int):
        """The same step as separate launches (one per operation)."""
        if self.batched:
            return self.step_batched(qi_next)
        eng, B = self.eng, self.B
        pv, d, HD, F, Fp, h = eng.pview, eng.d, eng.HD, eng.F, eng.Fp, eng.h
        xa, xm = self.x
        lib.embed_gather(eng.table, self.next_row, xa)
        for l in range(eng.L):
            p, pk = f"transformer.layers.{l}.", eng.pk[l]
            lib.skinny_gemm(xa, pk["wq"], self.q_raw, prologue=2, gamma=pv[p + "0.norm.gamma"])
            lib.skinny_gemm(xa, pk["wkv_b"], self.kv_raw, prologue=1)
            lib.attn_decode(self.q_raw, self.kv_raw, pv[p + "0.q_scale"], pv[p + "0.k_scale"], self.cache[l], self.table, self.pos,
                            self.n_max, self.o, h)
            lib.skinny_gemm(self.o, pk["wo_b"], xm, addend=xa)
            lib.skinny_gemm(xm, pk["w1"], self.u_new, prologue=2, gamma=pv[p + eng.ffk["g1"]])
            lib.decode_conv_geglu(self.u_new, self.conv[l], pk["conv"], self.h, self.rowsum)
            lib.skinny_gemm(self.h, pk["w2"], xa, prologue=3, gamma=pk["gin"], rowsum=self.rowsum, n_real=F, addend=xm)
        S = len(eng.seqs) - 1
        lib.skinny_gemm(xa, eng.pk_logit[S][qi_next], self.logits[:, :eng.Cp[S]], prologue=2, gamma=pv["transformer.norm.gamma"])

    def step_batched(self, qi_next: int):
        """step_ops for more than 16 sequences: the same operations on the tensor-core GEMM and the cache-sharing
        attention (same rounding points; fp32 sums in another order)."""
        eng, ws = self.eng, self.ws
        pv, F, h = eng.pview, eng.F, eng.h
        xa, xm = self.x
        lib.embed_gather(eng.table, self.next_row, xa)
        for l in range(eng.L):
            p, pk = f"transformer.layers.{l}.", eng.pk[l]
            lib.decode_gemm(xa, pk["wq"], self.q_raw, prologue=2, gamma=pv[p + "0.norm.gamma"], ws=ws)
            lib.decode_gemm(xa, pk["wkv_b"], self.kv_raw, prologue=1, ws=ws)
            lib.attn_decode_mqa(self.q_raw, self.kv_raw, pv[p + "0.q_scale"], pv[p + "0.k_scale"], self.cache[l], self.table, self.pos,
                                self.n_max, self.o, h, ws=ws)
            lib.decode_gemm(self.o, pk["wo_b"], xm, addend=xa, ws=ws)
            lib.decode_gemm(xm, pk["w1"], self.u_new, prologue=2, gamma=pv[p + eng.ffk["g1"]], ws=ws)
            lib.decode_conv_geglu(self.u_new, self.conv[l], pk["conv"], self.h, self.rowsum)
            lib.decode_gemm(self.h, pk["w2"], xa, prologue=3, gamma=pk["gin"], rowsum=self.rowsum, n_real=F, addend=xm, ws=ws)
        S = len(eng.seqs) - 1
        lib.decode_gemm(xa, eng.pk_logit[S][qi_next], self.logits[:, :eng.Cp[S]], prologue=2, gamma=pv["transformer.norm.gamma"], ws=ws)

    def sample(self, qi: int, top_k: int, temperature: float, allow_eos: bool, uniform, seed, bump_pos: bool):
        eng = self.eng
        S = len(eng.seqs) - 1
        q, cb = eng.seqs[S].num_quantizers, eng.seqs[S].codebook_size
        row_offset = eng.emb_row_base[S] + (cb * qi if q > 1 else 0)
        lib.sample(self.logits, eng.C[S], top_k, temperature, allow_eos, uniform, seed, self.tokens, self.next_row, row_offset,
                   self.counters, self.pos if bump_pos else None, self.B)

    def step_and_sample(self, qi: int, qi_next: int, top_k, temperature, allow_eos_next, uniform, seed, use_graph=True):
        """decode step on the token sampled for quantizer slot qi, then sample the token of slot qi_next."""
        key = (qi, qi_next, top_k, float(temperature), bool(allow_eos_next), uniform is not None)
        g = self._graphs.get(key)
        if g is None or not use_graph:
            body = lambda: (self.step(qi_next), self.sample(qi_next, top_k, temperature, allow_eos_next, uniform, seed, True))
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
                 use_cuda_graph=True, trace_logits: Optional[list] = None, **kwargs):
        """Same contract as open_musiclm.py:253-326.  uniform_noise (optional, [n_sampled, b, codebook+1] in (0, 1)):
        the uniform draws behind the Gumbel noise, one slice per sampled token in order — parity runs pass the stream
        torch's default CPU generator would have produced; by default the noise comes from a device Philox stream.
        trace_logits (tests): receives a copy of the [b, codebook+1] logits every token was sampled from."""
        if kwargs:
            raise NotImplementedError(f"open_musiclm_b200 generate: unsupported arguments {sorted(kwargs)}")
        m, eng = self.transformer, self.transformer.engine
        was_training = m.training
        m.eval()
        dev = eng.dev
        S = len(self.token_sequences)
        assert len(conditioning_token_ids) == S - 1
        B = conditioning_token_ids[0].shape[0]
        info, eos = self.token_sequences[-1], self.eos_ids[-1]
        q = info.num_quantizers
        cond = [t.to(dev, torch.int64).reshape(B, -1) for t in conditioning_token_ids]
        if append_eos_to_conditioning_tokens:                                                       # :288-290
            cond = [torch.cat([t, torch.full((B, 1), e, device=dev, dtype=torch.int64)], 1) for t, e in zip(cond, self.eos_ids)]
        if pred_token_ids is not None:
            assert pred_token_ids.shape[0] == B
            init_step = pred_token_ids.shape[1]                                                     # :276
            prefix = pred_token_ids.to(dev, torch.int64).reshape(B, -1)
        else:
            init_step = 0
            prefix = torch.empty(B, 0, device=dev, dtype=torch.int64)
        n_new = max(0, (max_time_steps - init_step) * q)
        if n_new > 0:
            ids = cond + [prefix]
            _, src_row, key_mask, _, n_tok = lib.token_plan(
                ids, [s.codebook_size for s in eng.seqs], [s.num_quantizers for s in eng.seqs], eng.emb_row_base, eng.start_row,
                append_eos=False, drop_last=False, mask_cond=False, want_labels=False, err_flag=eng.err_flag)
            pl = eng.plan(B, n_tok)
            sess = DecodeSession(eng, B, pl.N, n_new)
            ws = eng.workspace(pl, False)
            eng.forward_core(pl, ws, src_row, key_mask, False, {S - 1}, False, capture=_Capture(sess))
            # logits of the prompt's last position: final sequence, position p_last = its token count, head p_last mod q
            p_last = n_tok[-1]
            gi = next(i for i, (s, qi, cnt, base) in enumerate(pl.groups) if s == S - 1 and qi == p_last % q)
            cnt = pl.groups[gi][2]
            rows = torch.arange(B, device=dev) * cnt + p_last // q
            sess.logits[:, :eng.Cp[S - 1]].copy_(ws["logits"][gi][rows])
            top_k = max(int((1 - filter_thres) * (info.codebook_size + 1)), 1)                      # utils.py:80
            uni = None
            if uniform_noise is not None:
                uni = uniform_noise.to(dev, torch.float32).contiguous()
                assert uni.shape == (n_new, B, info.codebook_size + 1), uni.shape
            p0 = prefix.shape[1]                                     # flat index of the first sampled token
            allow = lambda p: bool(allow_eos_in_output and (p % q) == q - 1)                        # :311-313
            C = info.codebook_size + 1
            if trace_logits is not None:
                trace_logits.append(sess.logits[:, :C].clone())
            sess.sample(p0 % q, top_k, temperature, allow(p0), uni, eng.seed, bump_pos=False)
            for s in range(1, n_new):
                p = p0 + s
                if trace_logits is not None:      # eager, in two halves, so that the logits can be copied in between
                    sess.step(p % q)
                    trace_logits.append(sess.logits[:, :C].clone())
                    sess.sample(p % q, top_k, temperature, allow(p), uni, eng.seed, True)
                else:
                    sess.step_and_sample((p - 1) % q, p % q, top_k, temperature, allow(p), uni, eng.seed, use_graph=use_cuda_graph)
            eng.seed += 1
            sampled = torch.cat([prefix, sess.tokens[:, :n_new]], 1)
            sess.check()
        else:
            sampled = prefix
        eos_mask = (sampled == eos).float()                                                         # utils.py:86-93
        if include_eos_in_output:
            eos_mask = torch.nn.functional.pad(eos_mask, (1, -1))
        sampled = sampled.masked_fill(eos_mask.cumsum(-1) > 0, -1)
        if was_training:
            m.train()
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
            return self._trainer._micro_batch(all_token_ids, m.training, 0, False), None, None
        dev = m.device
        ids = [t.to(dev, torch.int64).reshape(t.shape[0], -1) for t in all_token_ids]
        ids = [torch.cat([t, torch.full((t.shape[0], 1), e, device=dev, dtype=torch.int64)], 1) for t, e in zip(ids, self.eos_ids)]
        return m(all_token_ids=ids, **kwargs)
