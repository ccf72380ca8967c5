"""tests/ffn_reference.py on the CPU: the float64 reference against the oracle's ConvFeedForward / FeedForward, its
gradients against finite differences, its error scales against the values and first-order perturbations they bound,
and its layout helpers against the packing the engine does (csrc/optim.cu, split_dst = -1) and the keep-bit order
ffn_norm_fwd writes."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import ffn_reference as FR  # noqa: E402


def _params(d, F, use_conv, seed, zero_gamma=()):
    g = torch.Generator().manual_seed(seed)
    W1 = (torch.rand(2 * F, d, generator=g, dtype=torch.float64) * 2 - 1) / d ** 0.5
    cw = (torch.rand(2 * F, 3, generator=g, dtype=torch.float64) * 2 - 1) / 3 ** 0.5 if use_conv else None
    gam = 1 + 0.5 * torch.randn(F, generator=g, dtype=torch.float64)
    gam[list(zero_gamma)] = 0.0
    return W1, cw, gam


@pytest.mark.parametrize("use_conv", [True, False])
def test_per_sequence_references_equal_the_whole_batch(use_conv, monkeypatch):
    """The rows test_ffn_reference_gpu compares a large form on: each sequence's forward, magnitude and du alone equal
    those rows of the whole-batch reference, and dgamma / dconv_w and their scales accumulated over chunks of whole
    sequences equal the whole-batch sums."""
    import test_ffn_reference_gpu as TF
    d, F, B, N, p = 16, 20, 5, 9, 0.25
    W1, cw, gam = _params(d, F, use_conv, 11)
    g = torch.Generator().manual_seed(12)
    xn = torch.randn(B * N, d, generator=g, dtype=torch.float64)
    keep = torch.rand(B * N, F, generator=g) > p
    dh = torch.randn(B * N, F, generator=g, dtype=torch.float64)
    u = xn @ W1.t()
    whole = FR.forward(xn, W1, cw, gam, N, keep, p)
    whole_g = FR.grads(u, cw, gam, dh, N, keep, p)
    whole_S = FR.magnitude(None, None, cw, gam, N, keep, p, u=u, dhn=dh)
    for rows in TF.row_groups(N, [0, 2, B - 1], device="cpu"):
        part = FR.forward(xn[rows], W1, cw, gam, N, keep[rows], p)
        for k in ("u", "h", "s1", "s2", "mean", "rstd", "hn"):
            assert torch.allclose(part[k], whole[k][rows], rtol=1e-12, atol=1e-12), k
        assert torch.allclose(FR.grads(u[rows], cw, gam, dh[rows], N, keep[rows], p)["du"], whole_g["du"][rows], rtol=1e-10, atol=1e-12)
    assert TF.check_seqs(4, 1024) is None and TF.check_seqs(16, 1024) == [0, 8, 15] and TF.check_seqs(8, 2048) == [0, 4, 7]
    monkeypatch.setattr(TF, "REF_ROWS", 2 * N)          # chunks of two sequences, the last one alone
    c = dict(F=F, N=N, B=B, cw=cw, gam=gam)
    ref, S = TF.weight_grad_refs(c, u, dh, keep, p)
    for k in ("dgamma", "dconv_w") if use_conv else ("dgamma",):
        assert torch.allclose(ref[k], whole_g[k], rtol=1e-10, atol=1e-12), k
        assert torch.allclose(S[k], whole_S[k], rtol=1e-10, atol=1e-12), k


@pytest.mark.parametrize("use_conv", [True, False])
@pytest.mark.parametrize("with_drop", [False, True])
def test_forward_matches_oracle(use_conv, with_drop):
    """forward() followed by the down projection is oracle/restatement.conv_feed_forward, in float64."""
    from oracle import restatement as R
    d, B, N = 24, 3, 7
    cfg = R.Cfg(seqs=[], dim=d, depth=1, heads=1, use_conv_ff=use_conv, ff_dropout=0.3)
    F = cfg.ff_inner
    W1, cw, gam = _params(d, F, use_conv, 1)
    g = torch.Generator().manual_seed(2)
    k_g1, k_w1, k_conv, k_gin, k_w2 = cfg.ff_keys
    sd = {k_g1: 1 + 0.1 * torch.randn(d, generator=g, dtype=torch.float64), k_w1: W1, k_gin: gam,
          k_w2: torch.randn(d, F, generator=g, dtype=torch.float64) / F ** 0.5}
    if use_conv:
        sd[k_conv] = cw[:, None, :]
    x = torch.randn(B, N, d, generator=g, dtype=torch.float64)
    keep = torch.rand(B, N, F, generator=g) > 0.3 if with_drop else None
    want = R.conv_feed_forward(cfg, sd, "", x, keep)
    xn = R.layer_norm(x, sd[k_g1]).reshape(B * N, d)
    r = FR.forward(xn, W1, cw, gam, N, None if keep is None else keep.reshape(B * N, F), cfg.ff_dropout)
    got = r["hn"] @ sd[k_w2].t()
    assert torch.allclose(got.reshape(B, N, d), want, rtol=1e-12, atol=1e-12)
    # the stage entry points reproduce the chain when fed its own intermediates
    again = FR.forward(None, None, cw, gam, N, None if keep is None else keep.reshape(B * N, F), cfg.ff_dropout,
                       u=r["u"], h=r["h"], stats=(r["mean"], r["rstd"]))
    assert torch.allclose(again["hn"], r["hn"], rtol=1e-13, atol=1e-13)
    assert torch.allclose(r["s1"] / F, r["mean"], rtol=1e-12, atol=1e-14)


def test_forward_resets_the_conv_history_per_sequence():
    """Sequences are independent: the batch of B sequences equals B separate calls."""
    W1, cw, gam = _params(16, 40, True, 3)
    xn = torch.randn(4 * 5, 16, dtype=torch.float64, generator=torch.Generator().manual_seed(4))
    whole = FR.forward(xn, W1, cw, gam, 5)["hn"]
    parts = torch.cat([FR.forward(xn[5 * b:5 * b + 5], W1, cw, gam, 5)["hn"] for b in range(4)])
    assert torch.equal(whole, parts)


@pytest.mark.parametrize("use_conv", [True, False])
def test_forward_gradcheck(use_conv):
    B, N, F = 2, 4, 5
    g = torch.Generator().manual_seed(5)
    u = torch.randn(B * N, 2 * F, generator=g, dtype=torch.float64, requires_grad=True)
    _, cw, gam = _params(8, F, use_conv, 6, zero_gamma=(1,))
    gam.requires_grad_(True)
    keep = torch.rand(B * N, F, generator=g) > 0.3
    if use_conv:
        cw.requires_grad_(True)
        fn = lambda u_, w_, g_: FR.forward(None, None, w_, g_, N, keep, 0.3, u=u_)["hn"]
        assert torch.autograd.gradcheck(fn, (u, cw, gam))
    else:
        fn = lambda u_, g_: FR.forward(None, None, None, g_, N, keep, 0.3, u=u_)["hn"]
        assert torch.autograd.gradcheck(fn, (u, gam))


@pytest.mark.parametrize("use_conv", [True, False])
def test_grads_against_finite_differences(use_conv):
    """grads() against central differences of sum(hn dhn), with dropout and gamma = 0 at two channels: those channels
    keep a non-zero du (dh = rstd (-m1 - hhat m2)) and conv-tap gradient."""
    B, N, F = 2, 5, 6
    g = torch.Generator().manual_seed(7)
    u = torch.randn(B * N, 2 * F, generator=g, dtype=torch.float64)
    _, cw, gam = _params(8, F, use_conv, 8, zero_gamma=(0, 4))
    keep = torch.rand(B * N, F, generator=g) > 0.2
    dhn = torch.randn(B * N, F, generator=g, dtype=torch.float64)
    res = FR.grads(u, cw, gam, dhn, N, keep, 0.2)
    loss = lambda u_, w_, g_: float((FR.forward(None, None, w_, g_, N, keep, 0.2, u=u_)["hn"] * dhn).sum())
    eps = 1e-6

    def fd(j):
        """central differences with respect to argument j of loss(u, cw, gam)"""
        args = [u, cw, gam]
        out = torch.zeros_like(args[j])
        for i in range(out.numel()):
            ap, am = list(args), list(args)
            ap[j], am[j] = args[j].clone(), args[j].clone()
            ap[j].view(-1)[i] += eps
            am[j].view(-1)[i] -= eps
            out.view(-1)[i] = (loss(*ap) - loss(*am)) / (2 * eps)
        return out

    assert torch.allclose(res["du"], fd(0), rtol=1e-6, atol=1e-7)
    assert torch.allclose(res["dgamma"], fd(2), rtol=1e-6, atol=1e-7)
    if use_conv:
        assert torch.allclose(res["dconv_w"], fd(1), rtol=1e-6, atol=1e-7)
        assert bool((res["dconv_w"][[0, 4, F, F + 4]].abs() > 0).all())
    else:
        assert res["dconv_w"] is None
    assert bool((res["du"][:, [0, 4, F, F + 4]].abs().sum(0) > 0).all())


@pytest.mark.parametrize("use_conv", [True, False])
def test_magnitude_bounds_values_and_first_order_errors(use_conv):
    """|x| <= S_x for every scaled tensor, and a perturbation of u (resp. h) by e S componentwise moves h (resp. hn) by at
    most e S_h (resp. e S_hn), to first order."""
    B, N, F, d = 3, 9, 20, 16
    W1, cw, gam = _params(d, F, use_conv, 9, zero_gamma=(3,))
    g = torch.Generator().manual_seed(10)
    xn = torch.randn(B * N, d, generator=g, dtype=torch.float64)
    keep = torch.rand(B * N, F, generator=g) > 0.25
    dhn = torch.randn(B * N, F, generator=g, dtype=torch.float64)
    r = FR.forward(xn, W1, cw, gam, N, keep, 0.25)
    S = FR.magnitude(xn, W1, cw, gam, N, keep, 0.25)
    for k in ("u", "y", "h", "hn"):
        assert bool((r[k].abs() <= S[k] * (1 + 1e-12)).all()), k
    assert bool((r["s1"].abs() <= S["s1"]).all()) and bool((r["mean"].abs() <= S["mean"]).all())
    e = 1e-7
    for trial in range(4):
        sgn = torch.randint(0, 2, r["u"].shape, generator=g).double() * 2 - 1
        r2 = FR.forward(None, None, cw, gam, N, keep, 0.25, u=r["u"] + e * sgn * S["u"])
        assert bool(((r2["h"] - r["h"]).abs() <= e * S["h"] * 1.001 + 1e-15).all())
        sh = torch.randint(0, 2, r["h"].shape, generator=g).double() * 2 - 1
        r3 = FR.forward(None, None, cw, gam, N, keep, 0.25, u=r["u"], h=r["h"] + e * sh * S["h"])
        assert bool(((r3["hn"] - r["hn"]).abs() <= e * S["hn"] * 1.001 + 1e-15).all())
        assert bool(((r3["rstd"] - r["rstd"]).abs() <= e * S["rstd"] * 1.001 + 1e-15).all())
    Sb = FR.magnitude(None, None, cw, gam, N, keep, 0.25, u=r["u"], dhn=dhn)
    res = FR.grads(r["u"], cw, gam, dhn, N, keep, 0.25)
    for k in ("du", "dgamma") + (("dconv_w",) if use_conv else ()):
        assert bool((res[k].abs() <= Sb[k] * (1 + 1e-12)).all()), k


# ------------------------------------------------------------------------------------------------ layouts
def _pack_rows_numpy(src, rows_p, split_src):
    """csrc/optim.cu's pack with split_dst < 0: destination row r of the interleaved order reads source row
    (w >> 7) split_src + ch, w = r & 255, ch = (r >> 8) 128 + (w & 127), live iff ch < split_src."""
    out = np.zeros((rows_p,) + src.shape[1:], src.dtype)
    for r in range(rows_p):
        w = r & 255
        ch = ((r >> 8) << 7) + (w & 127)
        if ch < split_src:
            out[r] = src[(w >> 7) * split_src + ch]
    return out


@pytest.mark.parametrize("F", [1, 127, 128, 129, 170, 192, 341])
def test_interleaved_layout_matches_the_engine_packing(F):
    Fp = FR.padded(F)
    src = np.arange(2 * F * 3, dtype=np.float64).reshape(2 * F, 3) + 1       # every row distinct and non-zero
    packed = _pack_rows_numpy(src, 2 * Fp, F)
    t = torch.from_numpy(src)
    assert np.array_equal(FR.to_kernel(t.t(), F).t().numpy(), packed)
    assert torch.equal(FR.from_kernel(torch.from_numpy(packed).t(), F).t(), t)
    cols = FR.ileave_cols(F)
    assert len(set(cols.tolist())) == 2 * F and int(cols.max()) < 2 * Fp
    # value channel c and gate channel c sit 128 columns apart, in the same 256-column tile
    assert torch.equal(cols[F:] - cols[:F], torch.full((F,), 128))
    assert torch.equal(cols[:F] // 256, torch.arange(F) // 128)


@pytest.mark.parametrize("F,Fp", [(1, 128), (129, 256), (192, 256), (5120, 5120)])
def test_keep_bits_round_trip_in_the_kernel_bit_order(F, Fp):
    g = torch.Generator().manual_seed(F)
    keep = torch.rand(5, F, generator=g) > 0.5
    bits = FR.pack_keep(keep, Fp)
    assert bits.shape == (5, Fp // 8) and bits.dtype == torch.uint8
    assert torch.equal(FR.unpack_keep(bits, F), keep)
    # ffn_norm_fwd: byte `chunk` holds channels 8 chunk + i at bit i
    k = np.zeros((5, Fp), bool)
    k[:, :F] = keep.numpy()
    want = np.zeros((5, Fp // 8), np.uint8)
    for chunk in range(Fp // 8):
        for i in range(8):
            want[:, chunk] |= (k[:, 8 * chunk + i].astype(np.uint8) << i)
    assert np.array_equal(bits.numpy(), want)
