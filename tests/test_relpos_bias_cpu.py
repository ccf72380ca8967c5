"""The float64 relative-position-bias reference (tests/relpos_reference.py) against the oracle restatement and against a
direct transcription of the reference's RelativePositionBias.forward; its componentwise scales against fp32 evaluations.
No GPU needed."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(__file__))
import relpos_reference as RP  # noqa: E402
from oracle import restatement as R  # noqa: E402

U32 = 2.0 ** -24         # fp32 unit roundoff


def state(dim, heads, bias_type="continuous", seed=0):
    return R.init_state(R.semantic_cfg(dim=dim, depth=1, heads=heads, codebook=16, n_clap_q=2, rel_pos_bias_type=bias_type), seed)


def transcription(params, n):
    """transformer.py:55-67 as written: the MLP over the 2n - 1 distances -n+1 .. n-1, gathered to [h, i, j] by
    rel_pos = i - j + n - 1.  float64."""
    pos = torch.arange(n)
    rel_pos = pos[:, None] - pos[None, :] + (n - 1)
    x = torch.arange(-n + 1, n, dtype=torch.float64)[:, None]
    for j in range(3):
        x = F.silu(x @ params[f"net.{j}.0.weight"].t() + params[f"net.{j}.0.bias"])
    x = x @ params["net.3.weight"].t() + params["net.3.bias"]
    return x[rel_pos].permute(2, 0, 1)


@pytest.mark.parametrize("dim,heads,n", [(64, 8, 2), (72, 3, 3), (72, 3, 130), (192, 16, 130), (1024, 8, 130)])
def test_reference_matches_the_reference_forward_on_the_causal_side(dim, heads, n):
    p = RP.params_of(state(dim, heads))
    full = transcription(p, n)
    tab = RP.table(p, n)
    i, j = torch.tril_indices(n, n)                        # i >= j: the entries the causal mask leaves
    want = full[:, i, j]
    got = tab[:, i - j]
    S = RP.magnitude(p, n)["table"][:, i - j]
    assert bool(((got - want).abs() <= 1e-13 * S).all()), float(((got - want).abs() / S).max())


@pytest.mark.parametrize("bias_type", ["continuous", "t5", "none"])
@pytest.mark.parametrize("dim,heads,n", [(64, 8, 1), (72, 3, 65), (1024, 16, 2048)])
def test_reference_matches_the_restatement(bias_type, dim, heads, n):
    sd = state(dim, heads, bias_type)
    want = R.rel_pos_table(sd, n, bias_type, heads)                       # fp32
    got = RP.bias_table(sd, n, bias_type, heads)                          # float64
    assert got.shape == want.shape == (heads, n) and got.dtype == torch.float64
    if bias_type != "continuous":
        assert torch.equal(got, want.double())
        return
    # fp32 evaluation: a few rounding units of the componentwise scale per layer
    S = RP.magnitude(RP.params_of(sd), n)["table"]
    ratio = float(((got - want.double()).abs() / (64 * U32 * S)).max())
    assert ratio <= 1.0, ratio


@pytest.mark.parametrize("dim,heads,n", [(64, 8, 129), (72, 3, 65), (192, 16, 300)])
@pytest.mark.parametrize("zero_sum", [False, True])
def test_gradient_scales_bound_fp32_autograd(dim, heads, n, zero_sum):
    """The gradient scales of magnitude() bound the error of an fp32 autograd of the same MLP to a few rounding units,
    so the GPU test's 2^-12 S bound has headroom for the bf16x3 products and nothing else."""
    sd = state(dim, heads)
    p = RP.params_of(sd)
    g = torch.Generator().manual_seed(3)
    dT = torch.randn(heads, n, generator=g)
    if zero_sum:
        dT = dT - dT.mean(1, keepdim=True)
    ref = RP.grads(p, n, dT)
    S = RP.magnitude(p, n, dT)
    leaves = {k: sd[RP.PREFIX + k].clone().requires_grad_(True) for k in RP.KEYS}
    R.rel_pos_table({RP.PREFIX + k: v for k, v in leaves.items()}, n).backward(dT)
    for k in RP.KEYS:
        ratio = float(((leaves[k].grad.double() - ref[k]).abs() / (64 * U32 * S[k])).max())
        assert ratio <= 1.0, (k, ratio)
    if zero_sum:
        # softmax is invariant to a per-head constant: the bias of the last layer gets no gradient (up to the fp32
        # rounding of the centred dT)
        assert bool((ref["net.3.bias"].abs() <= 4 * U32 * S["net.3.bias"]).all())


def test_magnitude_bounds_the_values_it_scales():
    p = RP.params_of(state(72, 3))
    n = 200
    dT = torch.randn(3, n, generator=torch.Generator().manual_seed(1))
    zs, acts, tab = RP.layers(p, n)
    S = RP.magnitude(p, n, dT)
    assert bool((tab.abs() <= S["table"]).all())
    for j in range(3):
        assert bool((zs[j].abs() <= S["z"][j]).all()) and bool((acts[j].abs() <= S["a"][j]).all())
    ref = RP.grads(p, n, dT)
    for k in RP.KEYS:
        assert bool((ref[k].abs() <= S[k] * (1 + 1e-12)).all()), k
    assert math.isclose(float(S["net.3.bias"].sum()), float(dT.double().abs().sum()), rel_tol=1e-12)
