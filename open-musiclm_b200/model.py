"""Drop-in boundary: `TokenConditionedTransformer` and the `create_*_transformer` factories with the
reference's signatures, attributes and state_dict keys/shapes, whose compute runs entirely in
libomlm_b200 (hand-written sm_90a CUDA behind a C ABI) — no torch ops on the hot path, no fallback.

Mirrors open_musiclm/open_musiclm.py:23-215, 414-472 (API) and open_musiclm/transformer.py
(parameter structure).  The module tree below carries parameters only; it exists so that
`state_dict()` / `load_state_dict(strict=True)` / `parameters()` / DDP wrapping behave exactly as
with the reference module.  All parameters are views into ONE flat fp32 arena (see engine.py).
"""
import itertools
import math
from dataclasses import dataclass
from typing import List, Optional

import torch
from torch import nn

from .engine import Engine


@dataclass
class TokenSequenceInfo:
    """open_musiclm.py:23-30."""
    codebook_size: int
    num_quantizers: int
    unique_consecutive: bool


class _Weight(nn.Module):
    def __init__(self, weight, bias=None):
        super().__init__()
        self.weight = nn.Parameter(weight)
        if bias is not None:
            self.bias = nn.Parameter(bias)


class _LayerNorm(nn.Module):
    """transformer.py:24-31: learnable gamma, beta is a zero buffer."""
    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(dim))
        self.register_buffer("beta", torch.zeros(dim))


class _DSConv(nn.Module):
    def __init__(self, weight):
        super().__init__()
        self.ds_conv = _Weight(weight)


class _Attention(nn.Module):
    """Parameter structure of transformer.py:166-212 (self-attention instance)."""
    def __init__(self, dim, heads, dim_head=64):
        super().__init__()
        inner = heads * dim_head
        self.norm = _LayerNorm(dim)
        self.to_q = _Weight(nn.Linear(dim, inner, bias=False).weight.detach())
        self.to_kv = _Weight(nn.Linear(dim, dim_head * 2, bias=False).weight.detach())
        self.q_scale = nn.Parameter(torch.ones(dim_head))
        self.k_scale = nn.Parameter(torch.ones(dim_head))
        self.to_out = nn.ModuleList([_Weight(nn.Linear(inner, dim, bias=False).weight.detach()), nn.Identity()])


def _feed_forward(dim):
    """Parameter structure of the plain FeedForward, transformer.py:152-161 (GEGLU at index 2, Dropout at 4)."""
    inner = int(dim * 4)
    return nn.ModuleList([
        _LayerNorm(dim),
        _Weight(nn.Linear(dim, inner * 2, bias=False).weight.detach()),
        nn.Identity(),
        _LayerNorm(inner),
        nn.Identity(),
        _Weight(nn.Linear(inner, dim, bias=False).weight.detach()),
    ])


def _conv_feed_forward(dim):
    """Parameter structure of ConvFeedForward, transformer.py:140-150 (indices 3 and 5 hold no parameters)."""
    inner = int(dim * 2 * 4 / 3)
    return nn.ModuleList([
        _LayerNorm(dim),
        _Weight(nn.Linear(dim, inner * 2, bias=False).weight.detach()),
        _DSConv(nn.Conv1d(inner * 2, inner * 2, 3, bias=False, groups=inner * 2).weight.detach()),
        nn.Identity(),
        _LayerNorm(inner),
        nn.Identity(),
        _Weight(nn.Linear(inner, dim, bias=False).weight.detach()),
    ])


class _RelPosBias(nn.Module):
    """RelativePositionBias, transformer.py:36-53."""
    def __init__(self, dim, heads, layers=3):
        super().__init__()
        def lin(i, o):
            l = nn.Linear(i, o)
            return _Weight(l.weight.detach(), l.bias.detach())
        net = [nn.ModuleList([lin(1, dim)])]
        for _ in range(layers - 1):
            net.append(nn.ModuleList([lin(dim, dim)]))
        net.append(lin(dim, heads))
        self.net = nn.ModuleList(net)


class _T5RelPosBias(nn.Module):
    """T5RelativePositionBias, transformer.py:69-84: an Embedding(32 buckets, heads)."""
    def __init__(self, heads, num_buckets=32):
        super().__init__()
        self.relative_attention_bias = _Weight(nn.Embedding(num_buckets, heads).weight.detach())


class _Transformer(nn.Module):
    """Parameter structure of Transformer, transformer.py:338-383 (creation order = reference RNG order)."""
    def __init__(self, dim, depth, heads, use_conv_ff=True, relative_position_bias_type="continuous"):
        super().__init__()
        self.layers = nn.ModuleList([])
        if relative_position_bias_type == "continuous":
            self.rel_pos_bias = _RelPosBias(dim // 2, heads)
        elif relative_position_bias_type == "t5":
            self.rel_pos_bias = _T5RelPosBias(heads)
        elif relative_position_bias_type == "none":
            self.rel_pos_bias = None
        else:
            raise ValueError(f"invalid relative position bias type: {relative_position_bias_type}")
        for _ in range(depth):
            self.layers.append(nn.ModuleList([_Attention(dim, heads), None, _conv_feed_forward(dim) if use_conv_ff else _feed_forward(dim)]))
        self.norm = _LayerNorm(dim)


class TokenConditionedTransformer(nn.Module):
    """Same constructor / forward / forward_with_cond_scale contract as open_musiclm.py:33-215."""

    def __init__(self, *, token_sequences: List[TokenSequenceInfo], dim, depth, heads=8, attn_dropout=0.,
                 ff_dropout=0.1, has_condition=False, cond_as_self_attn_prefix=False, cond_drop_prob=0.5,
                 grad_shrink_alpha=0.1, use_absolute_position_embeddings=False,
                 max_absolute_position_embeddings=262, **kwargs):
        super().__init__()
        # configurations the H100 path does not implement fail loudly (no silent fallback)
        unsupported = []
        if has_condition or cond_as_self_attn_prefix:
            unsupported.append("has_condition / cond_as_self_attn_prefix (dead in every shipped config)")
        if kwargs.get("non_causal_prefix_size", 0) != 0:
            unsupported.append("non_causal_prefix_size>0")
        if kwargs.get("relative_position_bias_type", "continuous") not in ("continuous", "t5", "none"):
            raise ValueError(f"invalid relative position bias type: {kwargs.get('relative_position_bias_type')}")
        if kwargs.get("use_memory_efficient_attention", False):
            unsupported.append("use_memory_efficient_attention=True (xformers)")
        if attn_dropout != 0.:
            unsupported.append("attn_dropout != 0")
        if len(token_sequences) > 4:
            unsupported.append("more than 4 token sequences")
        if unsupported:
            raise NotImplementedError("open_musiclm_b200: unsupported configuration: " + "; ".join(unsupported))

        self.token_sequences = token_sequences
        self.has_condition = has_condition
        self.cond_drop_prob = cond_drop_prob
        self.use_absolute_position_embeddings = use_absolute_position_embeddings
        self.dim, self.depth, self.heads = dim, depth, heads
        self.ff_dropout = ff_dropout
        self.grad_shrink_alpha = grad_shrink_alpha
        self.use_conv_ff = bool(kwargs.get("use_conv_ff", True))
        self.relative_position_bias_type = kwargs.get("relative_position_bias_type", "continuous")
        self.max_absolute_position_embeddings = max_absolute_position_embeddings

        self.start_tokens = nn.ParameterList()
        self.logit_weights = nn.ParameterList()
        self.embeddings = nn.ModuleList()
        self.absolute_position_embeddings = nn.ModuleList() if use_absolute_position_embeddings else None
        self.eos_ids = []
        for seq in token_sequences:   # same RNG consumption order as open_musiclm.py:72-82
            self.start_tokens.append(nn.Parameter(torch.randn(dim)))
            self.eos_ids.append(seq.codebook_size)
            cb = seq.codebook_size + 1
            self.embeddings.append(_Weight(nn.Embedding(cb * seq.num_quantizers, dim).weight.detach()))
            self.logit_weights.append(nn.Parameter(torch.randn(seq.num_quantizers, cb, dim)))
            if use_absolute_position_embeddings:
                self.absolute_position_embeddings.append(_Weight(nn.Embedding(max_absolute_position_embeddings, dim).weight.detach()))
        self.transformer = _Transformer(dim, depth, heads, self.use_conv_ff, self.relative_position_bias_type)
        self._engine = None

    # ------------------------------------------------------------------ plumbing
    @property
    def device(self):
        return next(self.parameters()).device

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self._engine = None          # parameters were re-materialised: rebuild the arena lazily
        return out

    @property
    def engine(self) -> Engine:
        if self._engine is None:
            self._engine = Engine(self)
        return self._engine

    # ------------------------------------------------------------------ reference API
    def forward(self, *, all_token_ids: List[torch.Tensor], self_attn_mask=None, cond_drop_prob=None,
                return_only_final_seq_logits=False):
        """open_musiclm.py:100-190.  Returns a list with one [b, n_i, codebook+1] fp32 logits tensor per
        sequence (None for skipped sequences).  Differentiable w.r.t. the parameters (one autograd node)."""
        return self.engine.api_forward(all_token_ids, self_attn_mask, return_only_final_seq_logits)

    def forward_with_cond_scale(self, *args, cond_scale=3, **kwargs):
        """open_musiclm.py:192-215: without text conditioning this is forward()."""
        kwargs.pop("cond_drop_prob", None)
        return self.forward(*args, cond_drop_prob=0., **kwargs)


def create_semantic_transformer(dim=1024, depth=6, clap_codebook_size=1024, semantic_codebook_size=1024,
                                num_clap_quantizers=12, **kwargs):
    """open_musiclm.py:414-428."""
    clap = TokenSequenceInfo(clap_codebook_size, num_clap_quantizers, False)
    sem = TokenSequenceInfo(semantic_codebook_size, 1, False)
    return TokenConditionedTransformer(token_sequences=[clap, sem], dim=dim, depth=depth, **kwargs)


def create_coarse_transformer(dim=512, depth=6, clap_codebook_size=1024, semantic_codebook_size=1024,
                              acoustic_codebook_size=1024, num_clap_quantizers=12, num_coarse_quantizers=4, **kwargs):
    """open_musiclm.py:432-450."""
    clap = TokenSequenceInfo(clap_codebook_size, num_clap_quantizers, False)
    sem = TokenSequenceInfo(semantic_codebook_size, 1, False)
    coarse = TokenSequenceInfo(acoustic_codebook_size, num_coarse_quantizers, False)
    return TokenConditionedTransformer(token_sequences=[clap, sem, coarse], dim=dim, depth=depth, **kwargs)


def create_fine_transformer(dim=512, depth=6, clap_codebook_size=1024, acoustic_codebook_size=1024,
                            num_clap_quantizers=12, num_coarse_quantizers=4, num_fine_quantizers=8, **kwargs):
    """open_musiclm.py:454-472."""
    clap = TokenSequenceInfo(clap_codebook_size, num_clap_quantizers, False)
    coarse = TokenSequenceInfo(acoustic_codebook_size, num_coarse_quantizers, False)
    fine = TokenSequenceInfo(acoustic_codebook_size, num_fine_quantizers, False)
    return TokenConditionedTransformer(token_sequences=[clap, coarse, fine], dim=dim, depth=depth, **kwargs)
