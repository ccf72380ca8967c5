"""Float64 statements of the two token log-probabilities of KV-cache generation, with their derived fp32 bounds.

model_logprob: log softmax of the raw logits row (all C classes, eos included) at the token.
sample_logprob: the log-probability of the token under the distribution the sampler drew it from: softmax(l / T) over
the candidate set S (eos rule, top-k set K with its tie rule, then the nucleus N when top_p < 1; NaN never in S).
The bounds follow the kernel's arithmetic (csrc/decode.cu, sample_kernel<..., kLogprob>): each term is expf of an fp32
argument (rounded once for l - m, twice for (l - m) / T; expf within 2 ulp), the terms are summed in double, and the
result is rounded to fp32 once.  To first order a term exp(a) carries a relative error of r |a| u + 4 u (u = 2^-24,
r the argument's roundings), so log of the sum is off by at most sum e (r |a| u + 4 u) / sum e."""
import math

import numpy as np
import torch

from test_sampling_nucleus_cpu import nucleus_by_sort, prepare, top_k_set

U = 2.0 ** -24


def candidate_set(logits, k, T, allow_eos, top_p):
    """bool [B, C]: S as the sampler builds it."""
    x = prepare(logits, allow_eos)
    if top_p is None:
        return top_k_set(x, k) & ~torch.isnan(x)
    return nucleus_by_sort(logits, k, T, allow_eos, top_p) & ~torch.isnan(x)


def _lse_bound(a, w, r):
    """log-sum-exp error bound of the terms exp(a) with weights w (0 outside the set), r roundings in each argument."""
    w = w & torch.isfinite(a)                   # -inf terms are exact zeros
    e = torch.where(w, torch.exp(a), torch.zeros_like(a))
    sa = torch.where(w, a.abs(), torch.zeros_like(a))
    return (e * (r * sa * U + 4 * U)).sum(1) / e.sum(1)


def model_logprob(logits, token):
    """(value, bound) [B] float64 of log softmax(logits[b])[token[b]] over the raw row."""
    x = logits.double().cpu()
    tok = token.cpu().long()[:, None]
    m = torch.where(torch.isnan(x), torch.full_like(x, -math.inf), x).max(1, keepdim=True).values
    a = x - m
    lse = torch.log(torch.exp(a).sum(1))
    val = a.gather(1, tok)[:, 0] - lse
    bound = _lse_bound(a, torch.ones_like(x, dtype=torch.bool), 1) + U * val.abs() + 1e-12
    return val, bound


def sample_logprob(logits, token, k, T, allow_eos, top_p):
    """(value, bound) [B] float64 of log softmax((l - m_S) / T over S)[token]; T and top_p rounded to fp32 as the C ABI
    takes them."""
    T = float(np.float32(T))
    x = prepare(logits, allow_eos)
    S = candidate_set(logits, k, T, allow_eos, top_p)
    tok = token.cpu().long()[:, None]
    m = torch.where(S, x, torch.full_like(x, -math.inf)).max(1, keepdim=True).values
    a = torch.where(S, (x - m) / T, torch.full_like(x, -math.inf))
    lse = torch.log(torch.exp(a).sum(1))
    at = a.gather(1, tok)[:, 0]
    val = at - lse
    bound = _lse_bound(torch.where(S, a, torch.zeros_like(a)), S, 2) + 2 * U * at.abs() + U * val.abs() + 1e-12
    return val, bound
