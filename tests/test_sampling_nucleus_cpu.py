"""Nucleus (top-p) sampling without a GPU: the float64 reference the kernel is tested against (nucleus_reference,
used by tests/test_sampling_nucleus_gpu.py), checked here against a sort-and-cumsum statement of the same rule, the
top_p argument checks, and MusicLM.generate_tokens handing every window's generate call its stage's top_p."""
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))

import open_musiclm_b200 as O  # noqa: E402
from open_musiclm_b200.decode import check_top_p  # noqa: E402


# ------------------------------------------------------------------------------------------------ float64 reference
def top_k_set(x, k):
    """bool [B, C]: exactly k kept per row; among equal values the lower index first (x already has -0.0 -> +0.0 and
    eos -> -inf applied).  NaN sorts above +inf, as it does in the kernel's key order."""
    key = torch.where(torch.isnan(x), torch.full_like(x, math.inf), x)
    rank_nan = torch.isnan(x).double()
    # stable descending sort by value, then by "is NaN" (NaN before +inf): lower index first among equals
    o1 = torch.sort(key, dim=1, descending=True, stable=True).indices
    o2 = torch.sort(rank_nan.gather(1, o1), dim=1, descending=True, stable=True).indices
    order = o1.gather(1, o2)
    return torch.zeros_like(x, dtype=torch.bool).scatter_(1, order[:, :k], True)


def prepare(logits, allow_eos):
    """float64 copy with -0.0 -> +0.0 and eos (class C - 1) -> -inf unless allowed."""
    x = logits.double().cpu() + 0.0
    if not allow_eos:
        x[:, -1] = -math.inf
    return x


def nucleus_reference(logits, uniform, k, T, allow_eos, top_p):
    """float64 nucleus sampling of [B, C] logits under [B, C] uniforms (top_p rounded to float32, as the C ABI takes it;
    None: no nucleus filtering).  For each row: K = top-k set; p = softmax(l / T) over K's non-NaN entries; above[c] =
    sum of p_j over j in K with l_j > l_c, from the mass of each distinct value (inf outside K and for NaN);
    N = {c : above[c] < top_p}; token = argmax over N of l / T - log(-log(u + 1e-20) + 1e-20).  A row whose maximum over K
    is not finite samples over K.  Returns a namespace: token, kept (K), nuc (N), above, score, top_p."""
    x = prepare(logits, allow_eos)
    B, C = x.shape
    kept = top_k_set(x, k)
    ok = kept & ~torch.isnan(x)
    mx = torch.where(ok, x, torch.full_like(x, -math.inf)).max(1, keepdim=True).values
    finite = torch.isfinite(mx[:, 0])
    p = torch.where(ok & finite[:, None], torch.exp((x - torch.where(finite[:, None], mx, torch.zeros_like(mx))) / T),
                    torch.zeros_like(x))
    p = p / p.sum(1, keepdim=True).clamp_min(1e-300)
    above = torch.full_like(x, math.inf)
    for b in range(B):
        if not finite[b]:
            continue
        cls = ok[b].nonzero()[:, 0]
        vals, inv = torch.unique(x[b, cls], sorted=True, return_inverse=True)          # ascending distinct values
        mass = torch.zeros(len(vals), dtype=torch.float64).index_add_(0, inv, p[b, cls])
        strictly_above = mass.flip(0).cumsum(0).flip(0) - mass                         # sum over larger values
        above[b, cls] = strictly_above[inv]
    tp = None if top_p is None else float(np.float32(top_p))
    if tp is None:
        nuc = kept.clone()
    else:
        nuc = torch.where(finite[:, None], above < tp, kept)
    nuc &= ~torch.isnan(x)
    g = -torch.log(-torch.log(uniform.double().cpu() + 1e-20) + 1e-20)
    score = torch.where(nuc, x / T + g, torch.full_like(x, -math.inf))
    token = torch.where(nuc.any(1), score.argmax(1), torch.full((B,), -1, dtype=torch.int64))
    return SimpleNamespace(token=token, kept=kept, nuc=nuc, above=above, score=score, top_p=tp)


def nucleus_by_sort(logits, k, T, allow_eos, top_p):
    """The same rule as the smallest prefix: sort K by value (descending), take the shortest prefix whose cumulative p
    reaches top_p, then add every entry equal in value to the prefix's last one."""
    x = prepare(logits, allow_eos)
    kept = top_k_set(x, k)
    tp = float(np.float32(top_p))
    out = torch.zeros_like(kept)
    for b in range(x.shape[0]):
        cls = (kept[b] & ~torch.isnan(x[b])).nonzero()[:, 0]
        v = x[b, cls]
        if len(cls) == 0 or not torch.isfinite(v.max()):
            out[b, cls] = True
            continue
        p = torch.softmax(v / T, 0)
        order = torch.argsort(v, descending=True, stable=True)
        csum = torch.cumsum(p[order], 0)
        reach = int((csum >= tp).nonzero()[0, 0]) if bool((csum >= tp).any()) else len(order) - 1
        last = v[order[reach]]
        out[b, cls[v >= last]] = True
    return out


def edge_logits(B, C, g, scale=3.0):
    """[B, C] float32 rows of several kinds, by row index mod 6: normal (flat, peaked), small integers (large tie groups
    straddling the nucleus boundary), +-0.0 mixed with a few ones, a third -inf, two equal maxima and one NaN."""
    x = torch.randn(B, C, generator=g) * scale
    for r in range(B):
        kind = r % 6
        if kind == 1:
            x[r] = torch.randn(C, generator=g) * 0.3
        elif kind == 2:
            x[r] = torch.randint(0, 4, (C,), generator=g).float()
        elif kind == 3:
            x[r] = torch.where(torch.rand(C, generator=g) < 0.5, torch.tensor(0.0), torch.tensor(-0.0))
            x[r, torch.randperm(C, generator=g)[:max(1, C // 50)]] = 1.0
        elif kind == 4:
            x[r, torch.randperm(C, generator=g)[:C // 3]] = -math.inf
            x[r, 0] = 2.0
        elif kind == 5:
            i = torch.randperm(C, generator=g)[:3]
            x[r, i[0]] = x[r, i[1]] = float(x[r].max()) + 1.0
            if C > 2:
                x[r, i[2]] = math.nan
    return x


# ------------------------------------------------------------------------------------------------ reference self-check
@pytest.mark.parametrize("C", [2, 3, 64, 1025])
def test_reference_nucleus_equals_the_sorted_prefix(C):
    g = torch.Generator().manual_seed(C)
    for k in sorted({1, 2, max(C // 10, 1), C // 2 or 1, C}):
        for top_p in (1e-7, 0.05, 0.3, 0.5, 0.9, 0.999999):
            for T, allow in ((0.4, False), (1.0, True), (2.0, False)):
                x = edge_logits(12, C, g)
                u = torch.rand(12, C, generator=g)
                ref = nucleus_reference(x, u, k, T, allow, top_p)
                srt = nucleus_by_sort(x, k, T, allow, top_p)
                # both are float64 sums in different orders: they may disagree only where the mass sits at top_p
                diff = ref.nuc != srt
                assert not bool((diff & ((ref.above - ref.top_p).abs() > 1e-12)).any()), (C, k, top_p, T, allow)
                assert bool((ref.nuc <= ref.kept).all())
                # the most likely non-NaN entry of K is always in N, and ties are all in or all out
                xr = prepare(x, allow)
                for b in range(12):
                    cls = (ref.kept[b] & ~torch.isnan(xr[b])).nonzero()[:, 0]
                    if len(cls) == 0:
                        continue
                    top = xr[b, cls].max()
                    assert bool(ref.nuc[b, cls[xr[b, cls] == top]].all())
                    for v in torch.unique(xr[b, cls]):
                        grp = ref.nuc[b, cls[xr[b, cls] == v]]
                        assert bool(grp.all()) or not bool(grp.any())
                has = ref.token >= 0                      # -1: K holds NaN logits only
                assert bool(ref.nuc[has].gather(1, ref.token[has][:, None]).all())


def test_reference_limits():
    """top_p near 0 keeps the maximum (and its ties) only; near 1 keeps all of K with non-negligible mass; None keeps K."""
    x = torch.tensor([[3.0, 1.0, 3.0, 0.0, -math.inf, 2.0, 0.5, 9.0]])     # class 7 (eos) is forbidden below
    u = torch.full((1, 8), 0.5)
    r = nucleus_reference(x, u, 8, 1.0, False, 1e-7)
    assert r.nuc[0].tolist() == [True, False, True, False, False, False, False, False]
    r = nucleus_reference(x, u, 8, 1.0, False, 0.999999)
    assert r.nuc[0].tolist() == [True, True, True, True, False, True, True, False]
    r = nucleus_reference(x, u, 5, 1.0, False, None)
    assert r.nuc[0].tolist() == r.kept[0].tolist() == [True, True, True, False, False, True, True, False]
    allinf = torch.full((1, 4), -math.inf)
    r = nucleus_reference(allinf, torch.full((1, 4), 0.5), 2, 1.0, True, 0.5)
    assert r.nuc[0].tolist() == [True, True, False, False] and int(r.token[0]) == 0


# ------------------------------------------------------------------------------------------------ argument checks
def test_check_top_p():
    assert check_top_p(None) is None and check_top_p(1.0) is None and check_top_p(1) is None
    assert check_top_p(0.9) == 0.9 and check_top_p(np.float32(0.5)) == 0.5 and check_top_p(1e-7) == 1e-7
    for bad in (math.nan, True, False, 0, 0.0, -0.1, 1.5, math.inf, "0.9", [0.9]):
        with pytest.raises(ValueError, match="top_p"):
            check_top_p(bad)


# ------------------------------------------------------------------------------------------------ MusicLM plumbing
class RecordingWrapper:
    """generate() of a stage wrapper that records the top_p it is handed (None when the keyword is absent)."""

    def __init__(self, q, codebook, log, name):
        self.q, self.cb, self.log, self.name = q, codebook, log, name
        self.token_sequences = [SimpleNamespace(codebook_size=codebook, num_quantizers=q)] * 3
        self.device = torch.device("cpu")

    def generate(self, *, conditioning_token_ids, pred_token_ids=None, max_time_steps, **kw):
        self.log.append((self.name, kw.get("top_p")))
        B = conditioning_token_ids[0].shape[0]
        init = 0 if pred_token_ids is None else pred_token_ids.shape[1]
        new = torch.randint(0, self.cb, (B, max_time_steps - init, self.q), generator=torch.Generator().manual_seed(len(self.log)))
        return new if pred_token_ids is None else torch.cat([pred_token_ids, new], 1)


def _mlm(log):
    return O.MusicLM(stages=(O.SemanticStage(semantic_transformer=None, wrapper=RecordingWrapper(1, 64, log, "semantic")),
                             O.CoarseStage(coarse_transformer=None, wrapper=RecordingWrapper(3, 64, log, "coarse")),
                             O.FineStage(fine_transformer=None, wrapper=RecordingWrapper(5, 64, log, "fine"))))


ARGS = dict(output_seconds=3, semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5,
            semantic_steps_per_second=6, acoustic_steps_per_second=8)


@pytest.mark.parametrize("top_p,expect", [
    (0.9, dict(semantic=0.9, coarse=0.9, fine=0.9)),
    ((0.95, 0.9, 0.8), dict(semantic=0.95, coarse=0.9, fine=0.8)),
    ([None, 0.5, 1.0], dict(semantic=None, coarse=0.5, fine=None)),
    (None, dict(semantic=None, coarse=None, fine=None)),
])
def test_every_window_gets_its_stages_top_p(top_p, expect):
    log = []
    clap = torch.randint(0, 64, (2, 4), generator=torch.Generator().manual_seed(1))
    _mlm(log).generate_tokens(clap_token_ids=clap, top_p=top_p, **ARGS)
    names = [n for n, _ in log]
    assert names.count("semantic") >= 2 and names.count("coarse") >= 2 and names.count("fine") >= 2, names
    for name, got in log:
        assert got == expect[name], (name, got)


@pytest.mark.parametrize("top_p", [(0.9, 0.8), (0.9, 0.8, 0.7, 0.6), (0.9, 0.9, math.nan), (0.9, True, 0.9), 0.0, 1.5, -1.0,
                                   math.nan, True, "0.9"])
def test_bad_top_p_raises_before_any_window(top_p):
    log = []
    with pytest.raises(ValueError, match="top_p"):
        _mlm(log).generate_tokens(clap_token_ids=torch.zeros(2, 4, dtype=torch.int64), top_p=top_p, **ARGS)
    assert log == []
