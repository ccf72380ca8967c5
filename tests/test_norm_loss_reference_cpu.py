"""tests/norm_loss_reference.py on the CPU: the float64 restatements against torch and the oracle, their gradients
against finite differences, and the error bounds against fp32 replicas of the kernels' arithmetic.  Each replica
follows its kernel's order of operations in torch float32; it must stay within the bound and reach a stated fraction
of it (so that the bound is not vacuous), and each listed mutation of a replica must exceed the bound."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(__file__))
import norm_loss_reference as R  # noqa: E402

F32, F64, BF16, F16 = torch.float32, torch.float64, torch.bfloat16, torch.float16


def fma32(a, b, c):
    """fp32 fma: the exact a b + c (float64 holds the product of two floats exactly) rounded once."""
    return (a.double() * b.double() + c.double()).float()


def store(y, dtype, rz=False):
    """y rounded to dtype as the kernels store it (nearest, fp16 saturating), or toward zero (bf16, a mutation)."""
    if rz:
        assert dtype == BF16
        return (y.float().view(torch.int32) & -65536).view(F32).to(BF16)
    if dtype == F16:
        y = y.clamp(-R.FP16_MAX, R.FP16_MAX)
    return y.to(dtype)


def butterfly(s):
    """The 5-level xor butterfly over the last dimension (32 lanes)."""
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., lane ^ o]
    return s[..., 0]


def lanes(x, D):
    """[M, NCHUNK, 32, 4] view of rows x [M, D] zero-padded to NCHUNK * 128 columns, and the column-valid mask."""
    nc = R.ln_nchunk(D)
    xp = torch.zeros(x.shape[0], nc * 128, dtype=x.dtype)
    xp[:, :D] = x
    valid = torch.zeros(nc * 128, dtype=torch.bool)
    valid[:D] = True
    return xp.view(-1, nc, 32, 4), valid.view(nc, 32, 4)


# ------------------------------------------------------------------------------------------------ fp32 replicas
def ln_fwd_replica(x, g, D, y_dtype, mut=None):
    v, valid = lanes(x, D)
    gv, _ = lanes(g[None], D)
    s = torch.zeros(x.shape[0], 32)
    for c in range(v.shape[1]):
        s = s + (((v[:, c, :, 0] + v[:, c, :, 1]) + v[:, c, :, 2]) + v[:, c, :, 3])
    mean = butterfly(s) / D
    sq = torch.zeros(x.shape[0], 32)
    for c in range(v.shape[1]):
        a = (v[:, c] - mean[:, None, None]) * valid[c]
        sq = sq + (((a[..., 0] * a[..., 0] + a[..., 1] * a[..., 1]) + a[..., 2] * a[..., 2]) + a[..., 3] * a[..., 3])
    var = butterfly(sq) / (D - 1 if mut == "var_d1" else D)
    eps = 1e-6 if mut == "eps6" else 1e-5
    rstd = 1.0 / (torch.sqrt(var) + eps) if mut == "eps_out" else torch.rsqrt(var + eps)
    y = ((x - mean[:, None]) * rstd[:, None]) * g
    return store(y, y_dtype, rz=mut == "rz"), mean, rstd


def ln_bwd_replica(dy, x, stats, g, D, dres=None, draw=None, mut=None):
    mean, rstd = stats[:, 0:1], stats[:, 1:2]
    nmr = -mean * rstd
    xh = fma32(x, rstd.expand_as(x), nmr.expand_as(x))
    gg = g * dy.float()
    gv, valid = lanes(gg, D)
    hv, _ = lanes(xh, D)
    s1 = torch.zeros(x.shape[0], 32, 2)
    s2 = torch.zeros(x.shape[0], 32, 2)
    for c in range(gv.shape[1]):
        gA, gB, hA, hB = gv[:, c, :, 0:2], gv[:, c, :, 2:4], hv[:, c, :, 0:2], hv[:, c, :, 2:4]
        s1 = s1 + (gA + gB)
        s2 = fma32(gA, hA, fma32(gB, hB, s2))
    s1 = butterfly(s1[..., 0] + s1[..., 1])[:, None] / D
    s2 = butterfly(s2[..., 0] + s2[..., 1])[:, None] / D
    if mut == "no_s1":
        s1 = torch.zeros_like(s1)
    if mut == "no_s2":
        s2 = torch.zeros_like(s2)
    ns1r, ns2r = -s1 * rstd, -s2 * rstd
    dx = fma32(xh, ns2r.expand_as(x), fma32(gg, rstd.expand_as(x), ns1r.expand_as(x)))
    if dres is not None:
        dx = dx + dres
    if draw is not None:
        dx = dx + draw.float()
    dg = torch.zeros(D)
    for r in range(x.shape[0]):
        dg = fma32(dy[r].float(), xh[r], dg)
    return dx, dg


def qk_replica(v, s, dy=None, mut=None):
    """One 64-vector per row of v [n, 64] (bf16 values): the forward y, and with dy the backward dx and dy xh."""
    f = v.float().view(-1, 8, 8)
    ss = torch.zeros(f.shape[0], 8)
    for i in range(8):
        ss = fma32(f[:, :, i], f[:, :, i], ss)
    lane = torch.arange(8)
    for o in (1, 2, 4):
        ss = ss + ss[:, lane ^ o]
    ss = ss[:, :1]
    nrm = torch.sqrt(ss)
    inv = torch.rsqrt(ss + 1e-12) if mut == "rsqrt_eps" else 1.0 / torch.clamp_min(nrm, 1e-12)
    f = f.view(-1, 64)
    if dy is None:
        return store((f * inv) * s, BF16)
    xh = f * inv
    sg = dy * s
    dot = torch.zeros(f.shape[0], 8)
    xh8, sg8 = xh.view(-1, 8, 8), sg.view(-1, 8, 8)
    for i in range(8):
        dot = fma32(xh8[:, :, i], sg8[:, :, i], dot)
    for o in (1, 2, 4):
        dot = dot + dot[:, lane ^ o]
    dot = dot[:, :1]
    if mut != "rsqrt_eps":
        dot = torch.where(nrm < 1e-12, torch.zeros_like(dot), dot)
    return store((sg - xh * dot) * inv, BF16), dy * xh


def ce_replica(x, lab, C, Cp, gs, mut=None):
    rows = x.shape[0]
    Cs = Cp if mut == "softmax_cp" else C
    v = torch.full((rows, R.CE_SLOTS * 32), float("-inf"))
    v[:, :Cs] = x[:, :Cs]
    mx = v.max(1, keepdim=True).values
    e = torch.exp(v - mx).view(rows, R.CE_SLOTS, 32)
    se = torch.zeros(rows, 32)
    for i in range(R.CE_SLOTS):
        se = se + e[:, i]
    se = butterfly(se)[:, None]
    inv = gs / se
    g = e.view(rows, -1)[:, :Cp] * inv
    g[:, Cs:] = 0
    if mut != "no_label":
        g[torch.arange(rows), lab.clamp_min(0)] -= gs
    g[lab == -100] = 0
    loss = ((mx[:, 0] + torch.log(se[:, 0])) - x[torch.arange(rows), lab.clamp_min(0)]) * (lab != -100)
    return store(g, BF16), loss


# ------------------------------------------------------------------------------------------------ fixed cases
def ln_rows(M, D, seed):
    """randn rows with an exact-zero row (a pad row), |mean| / std = 1e3, a near-constant row (std 1e-3), one outlier."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, D, generator=g) * 3 + 0.5
    x[1] = 0
    x[2] = 1e3 + torch.randn(D, generator=g)
    x[3] = 0.25 + 1e-3 * torch.randn(D, generator=g)
    x[4, D // 3] = 200.0
    return x


def ln_gamma(D, seed, big=False):
    g = 1 + 0.3 * torch.randn(D, generator=torch.Generator().manual_seed(seed + 1))
    if big:
        g[D // 2:D // 2 + 8] = 1e5         # drives fp16 y past 65504
    return g


LN_CASES = [(6, 64), (7, 132), (6, 1024), (5, 2048)]


@pytest.mark.parametrize("M,D", LN_CASES)
@pytest.mark.parametrize("y_dtype", [BF16, F16])
def test_ln_fwd_reference_matches_torch_and_replica(M, D, y_dtype):
    from oracle import restatement
    x, g = ln_rows(M, D, D), ln_gamma(D, D, big=y_dtype == F16)
    ref = R.ln_fwd_ref(x, g, y_dtype)
    want = F.layer_norm(x.double(), (D,), g.double(), None, 1e-5)
    assert torch.allclose(R.clamp16(want, y_dtype), ref["y"], rtol=1e-12, atol=1e-12)
    assert torch.allclose(restatement.layer_norm(x.double(), g.double()), ref["ycopy"], rtol=1e-12, atol=1e-12)
    y, mean, rstd = ln_fwd_replica(x, g, D, y_dtype)
    r = R.check(y, ref["y"], ref["y_bound"], "y")
    R.check(mean, ref["mean"], ref["mean_bound"], "mean")
    R.check(rstd, ref["rstd"], ref["rstd_bound"], "rstd")
    assert r >= 0.4, r                                      # a 16-bit store reaches most of its half ulp
    if y_dtype == F16:
        assert float(y.float().abs().max()) == R.FP16_MAX  # saturated, not inf
    assert float(rstd[1]) == pytest.approx(1e-5 ** -0.5, rel=1e-6) and bool((y[1] == 0).all())


@pytest.mark.parametrize("mut", ["var_d1", "eps6", "eps_out", "rz"])
@pytest.mark.parametrize("M,D", LN_CASES)
def test_ln_fwd_mutations_exceed_the_bound(M, D, mut):
    x, g = ln_rows(M, D, D), ln_gamma(D, D)
    ref = R.ln_fwd_ref(x, g, BF16)
    y, mean, rstd = ln_fwd_replica(x, g, D, BF16, mut=mut)
    worst = max(R.ratio(y, ref["y"], ref["y_bound"]), R.ratio(rstd, ref["rstd"], ref["rstd_bound"]))
    assert worst > 1.0, (mut, worst)


def _ln_bwd_case(M, D, seed):
    gen = torch.Generator().manual_seed(seed + 7)
    x, g = ln_rows(M, D, seed), ln_gamma(D, seed)
    _, mean, rstd = ln_fwd_replica(x, g, D, BF16)
    stats = torch.stack([mean, rstd], 1)
    dy = torch.randn(M, D, generator=gen).to(BF16)
    dres = torch.randn(M, D, generator=gen)
    draw = torch.randn(M, D, generator=gen).to(BF16)
    return x, g, stats, dy, dres, draw


@pytest.mark.parametrize("M,D", LN_CASES)
def test_ln_bwd_reference_matches_autograd_and_replica(M, D):
    x, g, stats, dy, dres, draw = _ln_bwd_case(M, D, D)
    # float64 statistics: the reference is then exactly the gradient of F.layer_norm
    x64 = x.double().requires_grad_(True)
    g64 = g.double().requires_grad_(True)
    F.layer_norm(x64, (D,), g64, None, 1e-5).backward(dy.double())
    st64 = torch.stack([x.double().mean(1), 1 / torch.sqrt(x.double().var(1, unbiased=False) + 1e-5)], 1)
    perm = torch.tensor([M - 1 - i if i % 2 else -1 for i in range(M)], dtype=torch.int32)
    ref = R.ln_bwd_ref(dy, x, st64, g, dres=dres, draw=draw, dgamma0=torch.ones(D))
    assert torch.allclose(ref["dx"], x64.grad + dres.double() + draw.double(), rtol=1e-10, atol=1e-10)
    assert torch.allclose(ref["dgamma"], g64.grad + 1, rtol=1e-10, atol=1e-10)
    refp = R.ln_bwd_ref(dy, x, st64, g, src_row=perm)
    want = torch.zeros(M, D, dtype=F64)
    has = perm >= 0
    x2 = x.double().requires_grad_(True)
    F.layer_norm(x2, (D,), g.double(), None, 1e-5).backward(dy.double()[perm.long().clamp_min(0)] * has[:, None])
    want = x2.grad
    assert torch.allclose(refp["dx"], want, rtol=1e-10, atol=1e-10)
    # replica (fp32 statistics as the forward stores them)
    ref = R.ln_bwd_ref(dy, x, stats, g, dres=dres, draw=draw)
    dx, dg = ln_bwd_replica(dy, x, stats, g, D, dres, draw)
    r = R.check(dx, ref["dx"], ref["dx_bound"], "dx")
    rb = R.check(dx.to(BF16), ref["dx"], ref["dx_bf16_bound"], "dx_bf16")
    R.check(dg, ref["dgamma"], ref["dgamma_bound"], "dgamma")
    assert r >= 0.01 and rb >= 0.4, (r, rb)


@pytest.mark.parametrize("mut", ["no_s1", "no_s2"])
@pytest.mark.parametrize("M,D", LN_CASES)
def test_ln_bwd_mutations_exceed_the_bound(M, D, mut):
    x, g, stats, dy, _, _ = _ln_bwd_case(M, D, D)
    ref = R.ln_bwd_ref(dy, x, stats, g)
    dx, _ = ln_bwd_replica(dy, x, stats, g, D, mut=mut)
    assert R.ratio(dx, ref["dx"], ref["dx_bound"]) > 1.0


def test_ln_bwd_finite_differences():
    M, D = 3, 12
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(M, D, generator=gen, dtype=F64)
    g = torch.randn(D, generator=gen, dtype=F64)
    dy = torch.randn(M, D, generator=gen).to(BF16)
    st = torch.stack([x.mean(1), 1 / torch.sqrt(x.var(1, unbiased=False) + 1e-5)], 1)
    ref = R.ln_bwd_ref(dy, x, st, g)
    L = lambda xx, gg: float((R.ln_fwd_ref(xx, gg, F32)["ycopy"] * dy.double()).sum())
    h = 1e-6
    for _ in range(4):
        vx = torch.randn(M, D, generator=gen, dtype=F64)
        vg = torch.randn(D, generator=gen, dtype=F64)
        fd = (L(x + h * vx, g + h * vg) - L(x - h * vx, g - h * vg)) / (2 * h)
        an = float((ref["dx"] * vx).sum() + (ref["dgamma"] * vg).sum())
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)), (fd, an)


# ------------------------------------------------------------------------------------------------ q/k l2norm
def qk_vectors(n, seed):
    """n 64-vectors in bf16: random, exact zero, sub-1e-12 norms (0.3e-12 and 0.8e-12), a large one."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(n, 64, generator=g)
    v[1] = 0
    v[2] = v[2] / v[2].norm() * 0.3e-12
    v[3] = v[3] / v[3].norm() * 0.8e-12
    v[4] *= 1e3
    return v.to(BF16)


def test_qk_reference_matches_normalize_and_replica():
    M, h = 6, 3
    gen = torch.Generator().manual_seed(2)
    q = torch.cat([qk_vectors(M, 1), qk_vectors(M, 2), torch.randn(M, 64, generator=gen).to(BF16)], 1)
    kv = torch.cat([qk_vectors(M, 3), torch.randn(M, 64, generator=gen).to(BF16)], 1)
    qs, ks = 1 + 0.5 * torch.rand(64, generator=gen), 1 + 0.5 * torch.rand(64, generator=gen)
    dqn, dkvn = torch.randn(M, h * 64, generator=gen), torch.randn(M, 128, generator=gen)
    fw = R.qk_fwd_ref(q, kv, qs, ks, h)
    bw = R.qk_bwd_ref(dqn, dkvn, q, kv, qs, ks, h, dq_scale0=torch.ones(64))
    q64 = q.double().view(M, h, 64).requires_grad_(True)
    k64 = kv.double()[:, :64].clone().requires_grad_(True)
    qs64, ks64 = qs.double().requires_grad_(True), ks.double().requires_grad_(True)
    yq = F.normalize(q64, dim=-1) * qs64
    yk = F.normalize(k64, dim=-1) * ks64
    assert torch.allclose(yq.reshape(M, -1), fw["qn"], rtol=1e-12, atol=0)
    assert torch.allclose(yk, fw["kvn"][:, :64], rtol=1e-12, atol=0) and torch.equal(fw["kvn"][:, 64:], kv.double()[:, 64:])
    ((yq.reshape(M, -1) * dqn.double()).sum() + (yk * dkvn.double()[:, :64]).sum()).backward()
    assert torch.allclose(bw["dq"], q64.grad.reshape(M, -1), rtol=1e-10, atol=0)
    assert torch.allclose(bw["dkv"][:, :64], k64.grad, rtol=1e-10, atol=0)
    assert torch.equal(bw["dkv"][:, 64:], dkvn.double()[:, 64:])
    assert torch.allclose(bw["dq_scale"], qs64.grad + 1, rtol=1e-10) and torch.allclose(bw["dk_scale"], ks64.grad, rtol=1e-10)
    # replicas: each q / k vector on its own
    for v, s, d, y64, yb, dx64, dxb in (
            (q.view(-1, 64), qs, dqn.view(-1, 64), fw["qn"].view(-1, 64), fw["qn_bound"].view(-1, 64), bw["dq"].view(-1, 64),
             bw["dq_bound"].view(-1, 64)),
            (kv[:, :64], ks, dkvn[:, :64], fw["kvn"][:, :64], fw["kvn_bound"][:, :64], bw["dkv"][:, :64], bw["dkv_bound"][:, :64])):
        y = qk_replica(v, s)
        dx, _ = qk_replica(v, s, d)
        assert R.check(y, y64, yb, "qn") >= 0.3
        assert R.check(dx, dx64, dxb, "dq") >= 0.3
        y, dxm = qk_replica(v, s, mut="rsqrt_eps"), qk_replica(v, s, d, mut="rsqrt_eps")[0]
        assert max(R.ratio(y, y64, yb), R.ratio(dxm, dx64, dxb)) > 1.0
    # below the clamp the gradient is s dy / eps: the fixed case has vectors there with a nonzero dy
    assert float(q.view(-1, 64)[3].float().norm()) < 1e-12 and float(dqn.view(-1, 64)[3].abs().max()) > 0


def test_qk_scale_sums_against_replica():
    M, h = 40, 2
    gen = torch.Generator().manual_seed(9)
    q = torch.cat([qk_vectors(M, 4), qk_vectors(M, 5)], 1)
    kv = torch.cat([qk_vectors(M, 6), torch.randn(M, 64, generator=gen).to(BF16)], 1)
    qs, ks = torch.rand(64, generator=gen) + 0.5, torch.rand(64, generator=gen) + 0.5
    dqn, dkvn = torch.randn(M, h * 64, generator=gen), torch.randn(M, 128, generator=gen)
    bw = R.qk_bwd_ref(dqn, dkvn, q, kv, qs, ks, h)
    _, pq = qk_replica(q.view(-1, 64), qs, dqn.view(-1, 64))
    _, pk = qk_replica(kv[:, :64], ks, dkvn[:, :64])
    dqs, dks = torch.zeros(64), torch.zeros(64)
    for i in range(pq.shape[0]):
        dqs = dqs + pq[i]
    for i in range(pk.shape[0]):
        dks = dks + pk[i]
    R.check(dqs, bw["dq_scale"], bw["dq_scale_bound"], "dq_scale")
    R.check(dks, bw["dk_scale"], bw["dk_scale_bound"], "dk_scale")


# ------------------------------------------------------------------------------------------------ cross entropy
def ce_case(C, Cp, rows, seed):
    """logits [rows, Cp] (finite padding: a kernel that read it would change the result), labels with 0, C - 1 and
    -100, a dominant +1e4 logit, a row of equal logits."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, Cp, generator=g) * 6
    lab = torch.randint(0, C, (rows,), generator=g)
    lab[0], lab[1], lab[4] = 0, C - 1, -100
    x[2, min(17, C - 1)] = 1e4
    x[3, :C] = 0.75
    return x, lab


@pytest.mark.parametrize("C,Cp", [(2, 8), (33, 64), (101, 128), (1025, 1088)])
def test_ce_reference_matches_torch_and_replica(C, Cp):
    rows, gs, ls = 21, 0.37, 0.5
    x, lab = ce_case(C, Cp, rows, C)
    ref = R.ce_ref(x, lab, C, Cp, grad_scale=gs, loss_scale=ls)
    x64 = x[:, :C].double().requires_grad_(True)
    lossv = F.cross_entropy(x64, lab, ignore_index=-100, reduction="none")
    assert torch.allclose(ref["loss"], lossv.detach(), rtol=1e-12, atol=1e-12)
    (lossv.sum() * gs).backward()
    assert torch.allclose(ref["dlogits"][:, :C], x64.grad, rtol=1e-10, atol=1e-15)
    assert bool((ref["dlogits"][:, C:] == 0).all()) and ref["count"] == rows - 1
    assert ref["total"] == pytest.approx(float(lossv.sum()) * ls, rel=1e-12)
    g, loss = ce_replica(x, lab, C, Cp, gs)
    assert R.check(g, ref["dlogits"], ref["dlogits_bound"], "dlogits") >= 0.3
    R.check(loss, ref["loss"], ref["loss_bound"], "loss")
    for mut in ("softmax_cp", "no_label"):
        gm, _ = ce_replica(x, lab, C, Cp, gs, mut=mut)
        assert R.ratio(gm, ref["dlogits"], ref["dlogits_bound"]) > 1.0, mut


def test_ce_strided_labels():
    plane = torch.arange(60, dtype=torch.int32).view(3, 20)
    lab = R.ce_labels(plane[0, 5:], 12, label_stride=3, rows_per_batch=4, batch_stride=20)
    want = torch.stack([plane[b, 5 + 3 * t] for b in range(3) for t in range(4)]).long()
    assert torch.equal(lab, want)
    assert torch.equal(R.ce_labels(plane.view(-1)[:7], 7), plane.view(-1)[:7].long())


def test_ce_finite_differences():
    C, rows = 7, 3
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(rows, C, generator=gen, dtype=F64)
    lab = torch.tensor([0, 6, 3])
    ref = R.ce_ref(x, lab, C, C, grad_scale=1.0)
    h, v = 1e-6, torch.randn(rows, C, generator=gen, dtype=F64)
    L = lambda xx: float(R.ce_ref(xx, lab, C, C, grad_scale=1.0)["loss"].sum())
    fd = (L(x + h * v) - L(x - h * v)) / (2 * h)
    assert abs(fd - float((ref["dlogits"] * v).sum())) <= 1e-7


# ------------------------------------------------------------------------------------------------ bookkeeping
def test_launch_restatements():
    # launch_ln_bwd: 4 blocks per SM of 8 warps up to D = 512, 2 at D = 1024 (NCHUNK 8), 1 of 4 warps above
    assert R.ln_bwd_launch(1, 64, 132) == (1, 8, 8)
    assert R.ln_bwd_launch(132 * 4 * 8 + 1, 64, 132) == ((132 * 4 * 8 + 1 + 8) // 9, 9, 8)
    assert R.ln_bwd_launch(16384, 1024, 132)[2] == 8 and R.ln_bwd_launch(16384, 2048, 132) == (132, 125, 4)
    assert [R.ln_nchunk(D) for D in (4, 128, 132, 256, 260, 512, 516, 1024, 1028, 2048)] == [1, 1, 2, 2, 4, 4, 8, 8, 16, 16]
    assert R.qk_bwd_launch(10, 3, 132) == (2, 1) and R.qk_bwd_launch(100000, 8, 132) == (1056, 30)


def test_scatter_reference():
    dt0 = torch.randn(5, 8, dtype=F64)
    src = torch.tensor([1, -1, 1, 3, 1], dtype=torch.int32)
    dx = torch.randn(5, 8, dtype=F64)
    t, b = R.scatter_ref(dt0, src, dx, 0.5)
    want = dt0.clone()
    for m in range(5):
        if src[m] >= 0:
            want[src[m]] += 0.5 * dx[m]
    assert torch.allclose(t, want, rtol=1e-14) and bool((b[[0, 2, 4]] == 0).all()) and bool((b[[1, 3]] > 0).all())
