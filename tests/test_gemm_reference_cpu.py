"""Pins tests/gemm_reference.py without a GPU: the layout semantics against explicit loops, the decode prologues against
the oracle's LayerNorm and torch's, and the componentwise bounds against an fp32 replica of the kernels' accumulation
that rounds at the same points -- in k16 steps, 64-wide blocks and splits, in several orders, rounding to nearest and
truncating.  The replica must stay within the bound everywhere and reach a stated fraction of it (a bound that is never
approached would let a subtly wrong kernel pass)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as nnf

import gemm_reference as G


def _bf(shape, gen, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(shape, generator=gen) * scale).to(dtype)


# ------------------------------------------------------------------------------------------------ layouts
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
def test_majors_and_n_valid_against_loops(a_mn, b_mn):
    g = torch.Generator().manual_seed(1)
    M, N, K, nv = 5, 7, 9, 6
    A, B = _bf((M, K), g), _bf((N, K), g)
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    X = torch.randn(M, N, generator=g)
    c, ab, written = G.gemm_ref(a, b, a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K, alpha=1 / 3, addend=X, n_valid=nv)
    assert c.shape == (M, nv) and bool(written.all())
    for m in range(M):
        for n in range(nv):
            s = sum(float(A[m, k]) * float(B[n, k]) for k in range(K))
            sa = sum(abs(float(A[m, k]) * float(B[n, k])) for k in range(K))
            assert abs(float(c[m, n]) - (s / 3 + float(X[m, n]))) < 1e-12
            assert abs(float(ab[m, n]) - sa / 3) < 1e-12


def test_in_place_addend_is_the_previous_contents():
    """An addend that is the output itself (the in-place weight gradient): C = A B^T + the output before the call."""
    g = torch.Generator().manual_seed(2)
    A, B = _bf((4, 8), g), _bf((6, 8), g)
    out = torch.randn(4, 6, generator=g)
    c, _, _ = G.gemm_ref(A, B, M=4, N=6, K=8, addend=out)
    c2, _, _ = G.gemm_ref(A, B, M=4, N=6, K=8, out0=out)
    ref = A.double() @ B.double().t() + out.double()
    assert torch.equal(c, c2) and torch.allclose(c, ref, rtol=0, atol=1e-12)


@pytest.mark.parametrize("M,row_split,row_valid", [(64, 64, 61), (128, 64, 61), (100, 64, 61), (192, 192, 129)])
def test_row_split_remap_against_loop(M, row_split, row_valid):
    g = torch.Generator().manual_seed(M + row_valid)
    K, N = 16, 8
    dy, x = _bf((K, M), g), _bf((K, N), g)
    c, _, written = G.gemm_ref(dy, x, a_mn=True, b_mn=True, M=M, N=N, K=K, row_split=row_split, row_valid=row_valid)
    full = dy.double().t() @ x.double()
    halves = (M + row_split - 1) // row_split
    assert c.shape[0] == halves * row_valid
    for h in range(halves):
        for r in range(row_valid):
            src, dst = h * row_split + r, h * row_valid + r
            if src < M:
                assert bool(written[dst]) and torch.equal(c[dst], full[src])
            else:
                assert not bool(written[dst]) and bool((c[dst] == 0).all())


@pytest.mark.parametrize("F", [1, 127, 128, 200, 383])
def test_geglu_remap_against_loop(F):
    g = torch.Generator().manual_seed(F)
    Fp = (F + 127) // 128 * 128
    M, K, N = 2 * Fp, 8, 4
    dy, x = _bf((K, M), g), _bf((K, N), g)
    c, _, written = G.gemm_ref(dy, x, a_mn=True, b_mn=True, M=M, N=N, K=K, row_split=-1, row_valid=F)
    full = dy.double().t() @ x.double()
    assert c.shape[0] == 2 * F and bool(written.all())
    for ch in range(F):
        grp, cc = divmod(ch, 128)
        assert torch.equal(c[ch], full[grp * 256 + cc])            # value row
        assert torch.equal(c[F + ch], full[grp * 256 + 128 + cc])  # gate row
    assert torch.equal(G.ileave_cols(F), G.remap_sources(M, -1, F))


def test_split_clamp_matches_the_host():
    """gemm16_impl: splits <= k-blocks, then as many splits as the per-split share needs."""
    assert G.gemm_splits(72, 5) == (2, 4)        # 2 k-blocks: 2 splits of one block
    assert G.gemm_splits(520, 3) == (3, 12)      # 9 blocks: 3 per split
    assert G.gemm_splits(520, 4) == (3, 12)      # 9 blocks, 3 per split -> only 3 splits
    assert G.gemm_splits(4104, 1) == (1, 4 * 65)


# ------------------------------------------------------------------------------------------------ decode prologues
def test_prologue_2_is_the_oracles_layernorm():
    from oracle import restatement as R
    g = torch.Generator().manual_seed(3)
    x = torch.randn(5, 200, generator=g) * 2 + 0.3
    x[1] = 0.5 + torch.randn(200, generator=g) * 1e-2          # var ~ 1e-4: eps matters
    gam = 1 + 0.1 * torch.randn(200, generator=g)
    y, e = G.decode_operand(x, 2, torch.bfloat16, gamma_=gam)
    assert torch.allclose(y, R.layer_norm(x.double(), gam.double()).double(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(y, nnf.layer_norm(x.double(), (200,), gam.double(), None, 1e-5), rtol=1e-12, atol=1e-12)
    other = nnf.layer_norm(x.double(), (200,), gam.double(), None, 1e-6)
    assert float(((other - y).abs() / e)[1].max()) > 100, "eps 1e-6 must be far outside the bound on the small-variance row"


def test_prologue_3_takes_its_statistics_from_the_row_sums():
    g = torch.Generator().manual_seed(4)
    B, K, F = 3, 384, 300
    h = torch.zeros(B, K)
    h[:, :F] = torch.randn(B, F, generator=g) * 3 + 1
    h16 = h.bfloat16()
    gam = 1 + 0.1 * torch.randn(K, generator=g)
    gam[F:] = 0
    rs = torch.stack([h.view(B, -1, 128).sum(-1), (h ** 2).view(B, -1, 128).sum(-1)], -1)
    y, e = G.decode_operand(h16, 3, torch.bfloat16, gamma_=gam, rowsum=rs, n_real=F)
    hd = h[:, :F].double()          # statistics of the unrounded h over the F real channels (the row sums are fp32 sums of it)
    mean, var = hd.mean(-1, keepdim=True), hd.var(-1, unbiased=False, keepdim=True)
    ref = (h16[:, :F].double() - mean) / torch.sqrt(var + 1e-5) * gam[:F].double()
    assert torch.allclose(y[:, :F], ref, rtol=1e-5, atol=1e-5)
    assert bool((y[:, F:] == 0).all())
    mean_k = rs[..., 0].sum(-1, keepdim=True).double() / K                                   # dividing by K, not n_real
    wrong = (h16.double() - mean_k) * gam.double() / torch.sqrt(rs[..., 1].sum(-1, keepdim=True).double() / K - mean_k ** 2 + 1e-5)
    assert float(((wrong - y).abs() / e)[:, :F].max()) > 100


def test_fp16_rounding_saturates():
    y = torch.tensor([[7e4, -1e6, 1.0]], dtype=torch.float64)
    assert G.round16(y, torch.float16).tolist() == [[65504.0, -65504.0, 1.0]]


# ------------------------------------------------------------------------------------------------ the bound vs an fp32 replica
def _chop(x):
    """Round float64 values toward zero to fp32's 24 significant bits."""
    m, e = np.frexp(x)
    return np.ldexp(np.trunc(m * 2.0 ** 24) / 2.0 ** 24, e)


def _rn(x):
    return x.astype(np.float32).astype(np.float64)


def _step(acc, terms, mode):
    """One k16 step: acc + the products `terms` [..., 16] under one of the replica's accumulation modes."""
    if mode == "rn_seq":
        for j in range(terms.shape[-1]):
            acc = _rn(acc + terms[..., j])
    elif mode == "rn_rev":
        for j in reversed(range(terms.shape[-1])):
            acc = _rn(acc + terms[..., j])
    elif mode == "rn_tree":
        t = terms
        while t.shape[-1] > 1:
            t = _rn(t[..., 0::2] + t[..., 1::2])
        acc = _rn(acc + t[..., 0])
    elif mode == "chop_seq":
        for j in range(terms.shape[-1]):
            acc = _chop(acc + terms[..., j])
    elif mode == "chop_align":      # align to the largest exponent, truncate, add exactly, truncate the sum
        allt = np.concatenate([acc[..., None], terms], -1)
        mx = np.abs(allt).max(-1, keepdims=True)
        q = np.ldexp(1.0, (np.floor(np.log2(np.where(mx > 0, mx, 1.0))) - 23).astype(int))
        acc = _chop((np.trunc(allt / q) * q).sum(-1))
    return acc


def _replica(A, B, K, splits, mode, chunk, split_order, out0=None, alpha=1.0, addend=None):
    """fp32 replica of one omlm_gemm16 / gemm_splitk_det output (float64 arrays holding fp32 values)."""
    P = A[:, None, :] * B[None, :, :]                   # exact products [M, N, K]
    kb = (K + 63) // 64
    s, _ = G.gemm_splits(K, splits)
    per = (kb + s - 1) // s
    parts = []
    for sp in range(s):
        acc = np.zeros(P.shape[:2])
        k0, k1 = sp * per * 64, min(K, (sp + 1) * per * 64)
        if chunk == 64:      # each 64-wide block summed by itself, then added
            for b0 in range(k0, k1, 64):
                blk = np.zeros(P.shape[:2])
                for t0 in range(b0, min(b0 + 64, k1), 16):
                    blk = _step(blk, P[..., t0:t0 + 16], mode)
                acc = _rn(acc + blk) if mode.startswith("rn") else _chop(acc + blk)
        else:
            for t0 in range(k0, k1, 16):
                acc = _step(acc, P[..., t0:t0 + 16], mode)
        parts.append(acc)
    rnd = _rn if mode.startswith("rn") else _chop
    if out0 is not None:
        v = out0.copy()
        for sp in (range(s) if split_order == "fwd" else reversed(range(s))):
            v = rnd(v + parts[sp])
        return v
    v = _rn(parts[0] * alpha)
    if addend is not None:
        v = rnd(v + addend)
    return v


MODES = ["rn_seq", "rn_rev", "rn_tree", "chop_seq", "chop_align"]


@pytest.mark.parametrize("positive", [False, True], ids=["signed", "positive"])
@pytest.mark.parametrize("K,splits", [(72, 1), (520, 1), (1032, 1), (520, 3), (1032, 20)])
def test_bound_holds_for_the_fp32_replica_and_is_reached(K, splits, positive):
    g = torch.Generator().manual_seed(K + splits)
    M, N = 12, 10
    A, B = _bf((M, K), g), _bf((N, K), g, 0.5)
    if positive:
        A, B = A.abs(), B.abs()
    X = torch.randn(M, N, generator=g) * 4
    if positive:
        X = X.abs()
    An, Bn, Xn = A.double().numpy(), B.double().numpy(), X.double().numpy()
    accumulate = splits > 1
    alpha = 1.0 if accumulate or positive else 1 / 3        # same-signed products alone: the accumulation's share of the bound
    addend = None if accumulate or positive else X
    c64, ab, _ = G.gemm_ref(A, B, M=M, N=N, K=K, alpha=alpha, addend=addend, out0=X if accumulate else None)
    gacc = G.gamma_gemm(K, splits)
    s, _ = G.gemm_splits(K, splits)
    worst = {}
    for out_dtype in (torch.float32, torch.bfloat16):
        if accumulate and out_dtype != torch.float32:
            continue
        if accumulate:
            bnd = G.bound(c64, ab, gamma_acc=gacc, out_dtype=out_dtype, out0=X, gamma_split=G.gamma(s))
        else:
            bnd = G.bound(c64, ab, gamma_acc=gacc, out_dtype=out_dtype, addend=addend, alpha=alpha)
        for mode in MODES:
            for chunk in (16, 64):
                for order in ("fwd", "rev"):
                    if accumulate:
                        r = _replica(An, Bn, K, splits, mode, chunk, order, out0=Xn)
                    else:
                        r = _replica(An, Bn, K, splits, mode, chunk, order, alpha=np.float32(alpha),
                                     addend=None if addend is None else Xn)
                    got = torch.from_numpy(r).to(out_dtype)
                    ratio = G.check(got, c64, bnd, f"{mode}/{chunk}/{order}/{out_dtype}")
                    key = (out_dtype, mode.startswith("chop"))
                    worst[key] = max(worst.get(key, 0.0), ratio)
    # not vacuous: truncating accumulation of same-signed products reaches 1/64 of the fp32 bound at every K here and
    # 1/20 from K = 520 on (the bound allows 18 ulp of the running sum per k16 step, counts the zero-filled k tail and
    # holds for a sum that is largest from the first step on; a bf16 store's rounding reaches 0.45 of its bound
    if positive:
        assert worst[(torch.float32, True)] >= (0.05 if K >= 520 and not accumulate else 1 / 64), worst
    if not accumulate:
        assert worst[(torch.bfloat16, False)] >= 0.45, worst


def test_prologue_bound_holds_for_an_fp32_replica_and_is_reached():
    """The prologue's fp32 statistics and products (the kernels' 32 lane sums, then the warp sum), rounding to nearest
    and truncating, against decode_operand's bound; a small-variance row included."""
    g = torch.Generator().manual_seed(7)
    B, K = 6, 1024
    x = (torch.randn(B, K, generator=g) * 2 + 0.3)
    x[2] = 3.0 + torch.randn(K, generator=g) * 1e-2
    x[3] = x[3].abs() + 1.0
    gam = 1 + 0.1 * torch.randn(K, generator=g)
    y, e = G.decode_operand(x, 2, torch.float16, gamma_=gam)
    xn, gn = x.double().numpy(), gam.double().numpy()
    ratios = {}
    for name, rnd in (("rn", _rn), ("chop", _chop)):
        lanes = xn.reshape(B, K // 32, 32)
        s = np.zeros((B, 32))
        for t in range(K // 32):
            s = rnd(s + lanes[:, t])
        tot = s[:, 0]
        for j in range(1, 32):
            tot = rnd(tot + s[:, j])
        mean = rnd(tot / K)[:, None]
        d = rnd(xn - mean)
        dl = d.reshape(B, K // 32, 32)
        q = np.zeros((B, 32))
        for t in range(K // 32):
            q = rnd(q + rnd(dl[:, t] * dl[:, t]))
        qt = q[:, 0]
        for j in range(1, 32):
            qt = rnd(qt + q[:, j])
        rstd = rnd(1.0 / np.sqrt(rnd(rnd(qt / K) + np.float32(1e-5))))[:, None]
        y32 = torch.from_numpy(rnd(rnd(d * rstd) * gn))
        ratios[name] = float(((y32 - y).abs() / e).max())
        G.check(y32.half(), y, G.operand_bound(y, e, torch.float16), f"prologue 2 operand ({name})")
    assert max(ratios.values()) <= 1.0, ratios
    assert ratios["chop"] >= 0.1, ratios
