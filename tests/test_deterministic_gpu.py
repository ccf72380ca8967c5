"""Deterministic mode: with torch.use_deterministic_algorithms(True) the training step runs the fixed-order kernel
variants (include/omlm_b200.h, *_det) and gives bit-identical results for identical inputs on one GPU model.

Every test here turns the switch on through the `det` fixture, which restores it afterwards, so the other test files
run in the default mode.  Reference values that go through torch's own CUDA kernels are computed with the switch off
(`switch(False)`): this file tests the library, not torch's deterministic kernels."""
import contextlib
import glob
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "tiny_*.pt")))


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


@contextlib.contextmanager
def switch(on):
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def cos(a, b):
    a, b = a.double().cpu().reshape(-1), b.double().cpu().reshape(-1)
    return float((a @ b) / (a.norm() * b.norm()).clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------ kernel variants
def _attn_inputs(B, N, h, seed):
    from open_musiclm_b200 import lib
    g = torch.Generator(device="cuda").manual_seed(seed)
    M = B * N
    q = F.normalize(torch.randn(M, h, 64, device="cuda", generator=g), dim=-1).reshape(M, h * 64).bfloat16()
    k = F.normalize(torch.randn(M, 64, device="cuda", generator=g), dim=-1)
    kv = torch.cat([k, torch.randn(M, 64, device="cuda", generator=g)], 1).bfloat16()
    table = torch.randn(h, N, device="cuda", generator=g)
    key_mask = (torch.rand(B, N, device="cuda", generator=g) > 0.1).to(torch.uint8)
    key_mask[:, 0] = 1
    o = torch.empty(M, h * 64, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(M * h, device="cuda")
    lib.attn_fwd_tc(q, kv, table, key_mask, o, lse, B, N, h)
    d_o = (torch.randn(M, h * 64, device="cuda", generator=g) * 0.1).bfloat16()
    return q, kv, table, key_mask, o, lse, d_o


@pytest.mark.parametrize("B,N,h", [(16, 1024, 8), (16, 2048, 8), (16, 1024, 16), (4, 1000, 8)])
def test_attn_bwd_det_matches_default_and_repeats_bit_identically(det, B, N, h):
    from open_musiclm_b200 import lib
    q, kv, table, key_mask, o, lse, d_o = _attn_inputs(B, N, h, seed=B * N + h)
    M = B * N

    def run(ws):
        dq = torch.empty(M, h * 64, device="cuda")
        dkv = torch.empty(M, 128, device="cuda")
        dt = torch.full((h, N), 0.5, device="cuda")           # accumulated into (+=)
        dsum = torch.empty(M * h, device="cuda")
        lib.attn_bwd_tc(q, kv, d_o, o, lse, table, key_mask, dsum, dq, dkv, dt, B, N, h, det=ws)
        return dq, dkv, dt

    ref = run(None)
    ws = lib.AttnBwdDetWorkspace("cuda", B, N, h)
    outs = [run(ws) for _ in range(3)]
    assert not ws.error()
    for a, b in zip(outs[0], ref):
        assert torch.isfinite(a).all()
        assert rel(a, b) <= 1e-5, rel(a, b)                    # same arithmetic, another fp32 summation order
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b)


def test_wgrad_det_matches_torch_and_repeats(det):
    """The weight-gradient GEMM at the cfg2 w2 shape (16384 rows, 1024 x 2730 out), which the cost model splits."""
    import open_musiclm_b200 as O
    from open_musiclm_b200 import lib
    from open_musiclm_b200.engine import Engine
    g = torch.Generator(device="cuda").manual_seed(7)
    K, m, n, npad = 16384, 1024, 2730, 2816
    dy = torch.randn(K, m, device="cuda", generator=g).bfloat16()
    x = torch.randn(K, npad, device="cuda", generator=g).bfloat16()
    base = torch.randn(m, n, device="cuda", generator=g)
    with switch(False):
        ref = base.double() + dy.double().T @ x[:, :n].double()

    class _E:             # the engine's split choice without a model
        _tile_cost, bwd_max_ctas = Engine._tile_cost, 0
        _num_sms = Engine._num_sms
    part = torch.empty(Engine.DET_WGRAD_PART_BYTES // 4, device="cuda")
    outs = []
    for _ in range(3):
        out = base.clone()
        calls = []
        real = lib.call
        lib.call = lambda name, *a: (calls.append((name, a)), real(name, *a))[1]
        try:
            Engine._wgrad(_E(), dy, x, out, m, npad, det_part=part, n_valid=n)
        finally:
            lib.call = real
        (name, args), = calls
        assert name == "omlm_gemm16_splitk_det"
        splits = args[13].value
        # more than one split after the library's clamp: the partial slices and the split-order reduction ran
        assert lib.gemm_splitk_det_workspace(m, npad, K, splits, n_valid=n) > 0, splits
        outs.append(out)
    assert rel(outs[0], ref) <= 1e-5, rel(outs[0], ref)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_small_reductions_det(det):
    """embed_scatter_add (repeated rows, start-token-like rows), grad_sumsq and cross entropy: the fixed-order variants
    against float64 torch, and bit-identical on repeats."""
    from open_musiclm_b200 import lib
    g = torch.Generator(device="cuda").manual_seed(11)
    rows, M, D = 300, 16 * 1024, 1024
    src = torch.randint(-1, rows, (M,), device="cuda", generator=g, dtype=torch.int32)
    src[::1024] = 5                                            # one row with a contribution from every "sequence"
    dx = torch.randn(M, D, device="cuda", generator=g)
    base = torch.randn(rows, D, device="cuda", generator=g)
    marks = lib.embed_row_markers(rows, "cuda")
    with switch(False):
        ok = src >= 0
        ref = base.double().index_add(0, src[ok].long(), dx[ok].double() * 0.1)
    outs = []
    for _ in range(3):
        t = base.clone()
        lib.embed_scatter_add(t, src, dx, 0.1, first=marks)
        outs.append(t)
    assert rel(outs[0], ref) <= 1e-6 and torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    assert bool((marks == 0x7FFFFFFF).all())
    # grad_sumsq
    arena = torch.randn(50_000_003 // 4 * 4 + 3, device="cuda", generator=g)
    part = torch.empty(4 * lib.num_sms(), device="cuda", dtype=torch.float64)
    sums = []
    for _ in range(3):
        acc = torch.full((1,), 2.0, device="cuda", dtype=torch.float64)
        lib.grad_sumsq(arena, acc, prescale=0.5, part=part)
        sums.append(acc)
    with switch(False):
        ref = 2.0 + float(((arena.double() * 0.5) ** 2).sum())
    assert abs(float(sums[0]) - ref) <= 1e-6 * ref and torch.equal(sums[0], sums[1]) and torch.equal(sums[0], sums[2])
    # cross entropy: loss sum and rows counted
    R_, C = 5000, 1025
    logits = torch.randn(R_, 1088, device="cuda", generator=g)
    labels = torch.randint(0, C, (R_,), device="cuda", generator=g, dtype=torch.int32)
    labels[::7] = -100
    cpart = torch.empty(2 * ((R_ + 7) // 8), device="cuda")
    accs = []
    for _ in range(3):
        acc = torch.zeros(2, device="cuda")
        lib.cross_entropy(logits, labels, C, acc, loss_scale=0.25, part=cpart)
        accs.append(acc)
    with switch(False):
        keep = labels != -100
        ref = F.cross_entropy(logits[keep, :C].double(), labels[keep].long(), reduction="sum") * 0.25
    assert abs(float(accs[0][0]) - float(ref)) <= 1e-5 * abs(float(ref)) and float(accs[0][1]) == float(keep.sum())
    assert torch.equal(accs[0], accs[1]) and torch.equal(accs[0], accs[2])


# ------------------------------------------------------------------------------------------------ partial-row variants
# Each at the cfg2 shapes: against the default entry point (same per-element code; the reduced outputs differ only in
# the fp32 summation order), against float64 torch at the tolerances of tests/test_kernels_gpu.py, and three calls
# bit-identical.
@pytest.mark.parametrize("variant", ["dres_draw", "src_row"])
def test_layernorm_bwd_det_cfg2(det, variant):
    from open_musiclm_b200 import lib
    M, D = 16384, 1024
    g = torch.Generator(device="cuda").manual_seed(21)
    x = torch.randn(M, D, device="cuda", generator=g) * 3 + 0.5
    gamma = 1 + 0.2 * torch.randn(D, device="cuda", generator=g)
    y = torch.empty(M, D, device="cuda", dtype=torch.bfloat16)
    stats = torch.empty(M, 2, device="cuda")
    lib.layernorm_fwd(x, gamma, y, None, stats)
    dres = draw = src = None
    if variant == "dres_draw":
        dy = torch.randn(M, D, device="cuda", generator=g).bfloat16()
        dres = torch.randn(M, D, device="cuda", generator=g)
        draw = torch.randn(M, D, device="cuda", generator=g).bfloat16()
        dy_full = dy.double()
    else:                 # permuted dy rows, every other x row without a gradient (the logit-head gather)
        src = torch.full((M,), -1, device="cuda", dtype=torch.int32)
        src[::2] = torch.arange(M // 2, device="cuda", dtype=torch.int32).flip(0)
        dy = torch.randn(M // 2, D, device="cuda", generator=g).bfloat16()
        dy_full = torch.zeros(M, D, device="cuda", dtype=torch.float64)
        dy_full[::2] = dy[src[::2].long()].double()
    part = torch.empty(4 * lib.num_sms() * D, device="cuda")

    def run(p):
        dx = torch.empty(M, D, device="cuda")
        dg = torch.full((D,), 0.5, device="cuda")                    # accumulated into (+=)
        lib.layernorm_bwd(dy, x, stats, gamma, dx, dg, dres=dres, draw=draw, src_row=src, part=p)
        return dx, dg
    ref_dx, ref_dg = run(None)
    outs = [run(part) for _ in range(3)]
    with switch(False):
        xd, gd = x.double().requires_grad_(True), gamma.double().requires_grad_(True)
        F.layer_norm(xd, (D,), gd, None, 1e-5).backward(dy_full)
        t_dx = xd.grad + (dres.double() + draw.double() if dres is not None else 0)
    dx, dg = outs[0]
    assert torch.equal(dx, ref_dx) and rel(dg, ref_dg) <= 1e-5, rel(dg, ref_dg)
    assert rel(dx, t_dx) < 1e-5 and rel(dg - 0.5, gd.grad) < 1e-4, (rel(dx, t_dx), rel(dg - 0.5, gd.grad))
    for o in outs[1:]:
        assert torch.equal(o[0], dx) and torch.equal(o[1], dg)


@pytest.mark.parametrize("h", [8, 16])
def test_qk_l2norm_bwd_det_cfg2(det, h):
    from open_musiclm_b200 import lib
    M = 16384
    g = torch.Generator(device="cuda").manual_seed(h)
    q = torch.randn(M, h * 64, device="cuda", generator=g).bfloat16()
    kv = torch.randn(M, 128, device="cuda", generator=g).bfloat16()
    qs = 1 + 0.3 * torch.randn(64, device="cuda", generator=g)
    ks = 1 + 0.3 * torch.randn(64, device="cuda", generator=g)
    dqn = torch.randn(M, h * 64, device="cuda", generator=g)
    dkvn = torch.randn(M, 128, device="cuda", generator=g)
    part = torch.empty(8 * lib.num_sms() * 128, device="cuda")

    def run(p):
        dq, dkv = torch.empty_like(q), torch.empty_like(kv)
        dqs, dks = torch.full((64,), 0.5, device="cuda"), torch.full((64,), -0.5, device="cuda")
        lib.qk_l2norm_bwd(dqn, dkvn, q, kv, qs, ks, dq, dkv, dqs, dks, h, part=p)
        return dq, dkv, dqs, dks
    ref = run(None)
    outs = [run(part) for _ in range(3)]
    with switch(False):
        qf, kvf = q.double().requires_grad_(True), kv.double().requires_grad_(True)
        qsd, ksd = qs.double().requires_grad_(True), ks.double().requires_grad_(True)
        qr = F.normalize(qf.view(M, h, 64), dim=-1) * qsd
        kr = F.normalize(kvf[:, :64], dim=-1) * ksd
        ((qr.reshape(M, -1) * dqn.double()).sum() + (kr * dkvn[:, :64].double()).sum()).backward()
    dq, dkv, dqs, dks = outs[0]
    assert torch.equal(dq, ref[0]) and torch.equal(dkv, ref[1])
    assert rel(dqs, ref[2]) <= 1e-5 and rel(dks, ref[3]) <= 1e-5
    assert rel(dq, qf.grad) < 4e-3 and rel(dkv[:, :64], kvf.grad[:, :64]) < 4e-3
    assert rel(dqs - 0.5, qsd.grad) < 1e-4 and rel(dks + 0.5, ksd.grad) < 1e-4, (rel(dqs - 0.5, qsd.grad), rel(dks + 0.5, ksd.grad))
    for o in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(o, outs[0]))


def _ileave_cols(F_, Fp):
    """canonical column (value c | gate F+c) -> column of the interleaved [M, 2Fp] layout."""
    c = torch.arange(F_)
    a = (c // 128) * 256 + (c % 128)
    return torch.cat([a, a + 128])


@pytest.mark.parametrize("conv,drop_p,gemm_parts", [(True, 0.1, True), (True, 0.0, False), (False, 0.1, False), (False, 0.0, True)],
                         ids=["conv-drop-gemmparts", "conv-nodrop-ownpass", "plain-drop-ownpass", "plain-nodrop-gemmparts"])
def test_ffn_mid_bwd_det_cfg2(det, conv, drop_p, gemm_parts):
    """B=16, N=1024, d=1024, F=2730, Fp=2816, fp16 forward activations.  conv=False is the plain FeedForward (taps pinned
    to (0, 0, 1), no dconv_w); gemm_parts: the LayerNorm row sums come from the d_hn GEMM's epilogue (rowstat_parts > 0),
    else from the kernel's own statistics pass."""
    from open_musiclm_b200 import lib
    B, N, d, F_ = 16, 1024, 1024, 2730
    Fp, M, adt = 2816, 16 * 1024, torch.float16
    g = torch.Generator(device="cuda").manual_seed(31)
    xn = torch.randn(M, d, device="cuda", generator=g).to(adt)
    W1 = (torch.rand(2 * F_, d, device="cuda", generator=g) * 2 - 1) / math.sqrt(d)
    if conv:
        cw = (torch.rand(2 * F_, 3, device="cuda", generator=g) * 2 - 1) / math.sqrt(3)
    else:
        cw = torch.zeros(2 * F_, 3, device="cuda")
        cw[:, 2] = 1.0
    gam = 1 + 0.2 * torch.randn(F_, device="cuda", generator=g)
    w1p = torch.empty(2 * Fp, d, device="cuda", dtype=adt)
    cwp, gp = torch.empty(2 * Fp, 3, device="cuda"), torch.empty(Fp, device="cuda")
    lib.pack(W1, d, 2 * F_, d, w1p, 2 * Fp, d, split_dst=-1, split_src=F_)
    lib.pack(cw, 3, 2 * F_, 3, cwp, 2 * Fp, 3, split_dst=-1, split_src=F_)
    lib.pack(gam, F_, 1, F_, gp, 1, Fp)
    u = torch.empty(M, 2 * Fp, device="cuda", dtype=adt)
    h = torch.empty(M, Fp, device="cuda", dtype=adt)
    rowsum = torch.empty(M, Fp // 128, 2, device="cuda")
    lib.gemm_ffn_up(xn, w1p, cwp, u, h, rowsum, N, Fp)
    hn, hn_b = torch.empty(M, Fp, device="cuda", dtype=adt), torch.empty(M, Fp, device="cuda", dtype=torch.bfloat16)
    stats = torch.empty(M, 2, device="cuda")
    seed = torch.tensor([99], dtype=torch.int64, device="cuda")
    kbits = torch.zeros(M, Fp // 8, device="cuda", dtype=torch.uint8) if drop_p > 0 else None
    lib.ffn_norm_fwd(h, rowsum, gp, hn, stats, F_, Fp, drop_p, seed, 3, keep_bits=kbits, hn_copy=hn_b)
    if gemm_parts:        # dhn = dx W2 with the row sums taken in the GEMM's epilogue
        dx = torch.randn(M, d, device="cuda", generator=g).bfloat16()
        w2 = ((torch.rand(d, Fp, device="cuda", generator=g) * 2 - 1) / math.sqrt(d)).bfloat16()
        w2[:, F_:] = 0
        dhn = torch.empty(M, Fp, device="cuda", dtype=torch.bfloat16)
        rowstat = torch.empty(M, Fp // 128, 2, device="cuda")
        lib.gemm_rowstat(dx, w2, dhn, hn_b, gp, rowstat, b_mn=True, M=M, N=Fp, K=d, keep_bits=kbits,
                         keep_scale=1.0 / (1.0 - drop_p) if drop_p > 0 else 1.0)
        parts = Fp // 128
    else:
        dhn = torch.zeros(M, Fp, device="cuda", dtype=torch.bfloat16)
        dhn[:, :F_] = torch.randn(M, F_, device="cuda", generator=g).bfloat16()
        rowstat = torch.empty(M, 2, device="cuda")
        parts = 0
    part = torch.empty(B * (N // 128) * 7 * F_, device="cuda")

    def run(p):
        du = torch.empty(M, 2 * Fp, device="cuda", dtype=torch.bfloat16)
        dg = torch.full((F_,), 0.5, device="cuda")
        dcw = torch.full((2 * F_, 3), -0.25, device="cuda") if conv else None
        lib.ffn_mid_bwd(dhn, hn_b, u, stats, cwp, gp, rowstat, du, dg, dcw, B, N, F_, Fp, drop_p, keep_bits=kbits,
                        rowstat_parts=parts, part=p)
        return du, dg, dcw
    ref = run(None)
    outs = [run(part) for _ in range(3)]
    cols = _ileave_cols(F_, Fp).to("cuda")
    with switch(False):   # float64 restatement of the conv / GEGLU / LayerNorm / dropout forward, backward by autograd
        uf = u[:, cols].double().requires_grad_(True)
        cwr, gr = cw.double().requires_grad_(True), gam.double().requires_grad_(True)
        up = F.pad(uf.view(B, N, 2 * F_), (0, 0, 2, 0))
        y = up[:, 0:-2] * cwr[:, 0] + up[:, 1:-1] * cwr[:, 1] + up[:, 2:] * cwr[:, 2]
        hmid = F.gelu(y[..., F_:]) * y[..., :F_]
        out = F.layer_norm(hmid, (F_,), gr, None, 1e-5).reshape(M, F_)
        if drop_p > 0:
            keep = ((kbits[:, :, None] >> torch.arange(8, device="cuda", dtype=torch.uint8)) & 1).bool().reshape(M, Fp)[:, :F_]
            out = out * keep / (1 - drop_p)
        out.backward(dhn[:, :F_].double())
    du, dg, dcw = outs[0]
    assert torch.equal(du, ref[0]) and rel(dg, ref[1]) <= 1e-5, rel(dg, ref[1])
    assert rel(du[:, cols], uf.grad) < 1.5e-2 and rel(dg - 0.5, gr.grad) < 8e-3, (rel(du[:, cols], uf.grad), rel(dg - 0.5, gr.grad))
    if conv:
        assert rel(dcw, ref[2]) <= 1e-5 and rel(dcw + 0.25, cwr.grad) < 1.5e-2, (rel(dcw, ref[2]), rel(dcw + 0.25, cwr.grad))
    for o in outs[1:]:
        assert torch.equal(o[0], du) and torch.equal(o[1], dg) and (not conv or torch.equal(o[2], dcw))


def test_sgemm_small_det_relpos_shapes(det):
    """The rel-pos MLP weight gradients of cfg2 (N = 1024, h = 8, Hr = 512): dW4 = dT^T a3 and dW1 = dz^T arange."""
    from open_musiclm_b200 import lib
    N, h, Hr = 1024, 8, 512
    g = torch.Generator(device="cuda").manual_seed(41)
    dT = torch.randn(h, N, device="cuda", generator=g)
    a3 = torch.randn(N, Hr, device="cuda", generator=g)
    dz = torch.randn(N, Hr, device="cuda", generator=g)
    rp_in = torch.arange(N, device="cuda", dtype=torch.float32)[:, None]
    base4, base1 = torch.randn(h, Hr, device="cuda", generator=g), torch.randn(Hr, 1, device="cuda", generator=g)

    def run(det_):
        w4, w1 = base4.clone(), base1.clone()
        lib.sgemm_small(dT, (N, 1), a3, (Hr, 1), w4, (Hr, 1), h, Hr, N, accumulate=True, det=det_)
        lib.sgemm_small(dz, (1, Hr), rp_in, (1, 1), w1, (1, 1), Hr, 1, N, accumulate=True, det=det_)
        return w4, w1
    ref = run(False)
    outs = [run(True) for _ in range(3)]
    with switch(False):
        t4 = base4.double() + dT.double() @ a3.double()
        t1 = base1.double() + dz.double().t() @ rp_in.double()
    assert rel(outs[0][0], ref[0]) <= 1e-5 and rel(outs[0][1], ref[1]) <= 1e-5
    assert rel(outs[0][0], t4) < 1e-5 and rel(outs[0][1], t1) < 1e-5
    for o in outs[1:]:
        assert torch.equal(o[0], outs[0][0]) and torch.equal(o[1], outs[0][1])


# ------------------------------------------------------------------------------------------------ whole training steps
def _cfg2_batches(n, B=16, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [[t.cuda() for t in (torch.randint(0, 1024, (B,) + s, generator=g) for s in [(12,), (197,), (270, 3)])] for _ in range(n)]


def _trainer(seed=0, depth=6, heads=8, use_cuda_graph=True, mask_prob=0.15):
    import open_musiclm_b200 as O
    torch.manual_seed(seed)
    m = O.create_coarse_transformer(dim=1024, depth=depth, heads=heads, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1,
                                    grad_shrink_alpha=0.1).cuda()
    return O.HotPathTrainer(m, cross_entropy_loss_weights=[0.0, 0.0, 1.0], lr=3e-4, lr_warmup=100, wd=0.01, max_grad_norm=0.5,
                            use_cuda_graph=use_cuda_graph, mask_prob=mask_prob)


def _run(tr, batches):
    losses, norms = [], []
    for b in batches:
        losses.append(tr.train_step([b]).clone())
        norms.append(tr.grad_norm().clone())
    torch.cuda.synchronize()
    return losses, norms


def _assert_same_state(ta, tb):
    for name in ("arena_p", "adam_m", "adam_v"):
        assert torch.equal(getattr(ta.eng, name), getattr(tb.eng, name)), name


@pytest.mark.parametrize("depth,heads", [(6, 8), (2, 16)], ids=["cfg2", "depth2_h16"])
def test_two_trainers_same_seed_bit_identical(det, depth, heads):
    batches = _cfg2_batches(5)
    ta, tb = _trainer(depth=depth, heads=heads), _trainer(depth=depth, heads=heads)
    la, na = _run(ta, batches)
    lb, nb = _run(tb, batches)
    assert all(torch.equal(x, y) for x, y in zip(la, lb)), (la, lb)
    assert all(torch.equal(x, y) for x, y in zip(na, nb)), (na, nb)
    assert all(bool(torch.isfinite(x)) for x in la + na)
    _assert_same_state(ta, tb)
    assert ta._graphs and all(st["graphs"] is not None for st in ta._graphs.values())        # steps 3-5 were replayed
    # eager steps equal graph-replayed steps.  Without the forgetful mask: a captured graph keeps the mask's draw index
    # of its capture (the host-side counter), so with a mask eager and replayed steps draw different masks in any mode
    tg = _trainer(depth=depth, heads=heads, mask_prob=0.0)
    te = _trainer(depth=depth, heads=heads, use_cuda_graph=False, mask_prob=0.0)
    lg, ng = _run(tg, batches)
    le, ne = _run(te, batches)
    assert all(torch.equal(x, y) for x, y in zip(lg, le)) and all(torch.equal(x, y) for x, y in zip(ng, ne)), (lg, le)
    _assert_same_state(tg, te)
    for tr in (ta, tb, tg, te):
        for ws in tr.eng._ws.values():
            if "det_attn" in ws:
                assert not ws["det_attn"].error()


def test_resume_is_bit_identical(det):
    """test_trainer_state_dict_round_trip's scenario with the switch on: the resumed run equals the uninterrupted one."""
    import open_musiclm_b200 as O
    kw = dict(dim=128, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=64, num_clap_quantizers=4,
              attn_dropout=0.0, ff_dropout=0.1)
    g = torch.Generator().manual_seed(3)
    batches = [[torch.randint(0, 64, s, generator=g).cuda() for s in [(2, 4), (2, 20)]] for _ in range(6)]

    def fresh():
        torch.manual_seed(0)
        m = O.create_semantic_transformer(**kw).cuda()
        return m, O.HotPathTrainer(m, cross_entropy_loss_weights=[0.0, 1.0], lr=1e-3, lr_warmup=4, wd=0.01, use_cuda_graph=False)
    m_a, tr_a = fresh()
    for b in batches[:3]:
        tr_a.train_step([b])
    ck_model = {k: v.clone() for k, v in m_a.state_dict().items()}
    ck_opt = tr_a.state_dict()
    la = [tr_a.train_step([b]).clone() for b in batches[3:]]
    m_b, tr_b = fresh()
    m_b.load_state_dict(ck_model)
    tr_b.load_state_dict(ck_opt)
    lb = [tr_b.train_step([b]).clone() for b in batches[3:]]
    assert all(torch.equal(x, y) for x, y in zip(la, lb)), (la, lb)
    for (k, va), (_, vb) in zip(m_a.state_dict().items(), m_b.state_dict().items()):
        assert torch.equal(va, vb), k
    _assert_same_state(tr_a, tr_b)


# ------------------------------------------------------------------------------------------------ parity under the switch
def _build(fx):
    import open_musiclm_b200 as O
    fn = {"semantic": O.create_semantic_transformer, "coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}[fx["stage"]]
    m = fn(**fx["kwargs"])
    m.load_state_dict(fx["state_dict"], strict=True)
    return m.cuda().eval()


def _check_grads(got, gold, tag):
    """The tolerances of tests/test_parity_gpu.py: cos >= 0.999, rel <= 2e-2 (rel-pos MLP: 0.995 / 1e-1; its analytically
    zero output bias is bounded by the gradient scale of the same layer)."""
    w3 = next((g for k, g in gold.items() if k.endswith("rel_pos_bias.net.3.weight") and g is not None), None)
    bad = []
    for k, g in gold.items():
        mine = got[k]
        if g is None:
            assert mine is None or float(mine.abs().max()) == 0.0, (tag, k)
            continue
        if k.endswith("rel_pos_bias.net.3.bias"):
            if not float(mine.double().norm()) <= 0.05 * (float(w3.norm()) if w3 is not None else 1.0):
                bad.append(k)
            continue
        if float(g.norm()) < 1e-6:
            continue
        c_min, r_max = (0.995, 1e-1) if "rel_pos_bias" in k else (0.999, 2e-2)
        if not (cos(mine, g) >= c_min and rel(mine, g) <= r_max):
            bad.append((k, cos(mine, g), rel(mine, g)))
    assert not bad, (tag, bad)


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_fixture_parity_under_the_switch(det, path):
    import open_musiclm_b200 as O
    fx = torch.load(path, weights_only=False)
    m = _build(fx)
    ids = [t.cuda() for t in fx["ids"]]
    logits = m(all_token_ids=ids, self_attn_mask=fx["key_mask"].cuda())
    for a, b in zip(logits, fx["logits"]):
        assert rel(a.detach(), b) <= 1e-2
    with switch(False):           # torch's cross entropy has no deterministic CUDA kernel: the loss and d loss / d logits
        total, running = 0, 0.0    # are torch's; the library's backward below runs with the switch on
        for lg, lb, w in zip(logits, fx["labels"], fx["ce_weights"]):
            if w > 0:
                running = running + F.cross_entropy(lg.permute(0, 2, 1), lb.cuda()) * lb.numel() * w
                total += lb.numel()
        loss = running / total
        live = [lg for lg in logits if lg is not None and lg.requires_grad]
        dl = torch.autograd.grad(loss, live, retain_graph=True, allow_unused=True)
    assert abs(float(loss) - float(fx["loss"])) / float(fx["loss"]) <= 1e-2
    pairs = [(a, g) for a, g in zip(live, dl) if g is not None]
    torch.autograd.backward([a for a, _ in pairs], [g for _, g in pairs])
    _check_grads({k: p.grad for k, p in m.named_parameters()}, fx["grads"], "api")
    m2 = _build(fx)
    tr = O.HotPathTrainer(m2, cross_entropy_loss_weights=fx["ce_weights"], lr=3e-4, lr_warmup=10, wd=1e-2)
    toks = [t.cuda() for t in fx["tokens"]]
    l_eval = tr.eval_loss(toks)
    assert abs(float(l_eval) - float(fx["loss"])) / float(fx["loss"]) <= 1e-2
    tr.eng.arena_g.zero_()
    tr._micro_batch(toks, False, 0, True, det=True)
    gold = {k: (g if g is not None else torch.zeros_like(fx["state_dict"][k])) for k, g in fx["grads"].items()}
    _check_grads({k: tr.eng.gview[k] for k, _ in m2.named_parameters()}, gold, "trainer")


# ------------------------------------------------------------------------------------------------ toggling, eval, generate
def test_toggling_recaptures_and_off_mode_issues_default_entry_points():
    """One process, switch on -> off -> on.  Graphs are re-captured per mode; off-mode steps issue exactly the entry
    points a trainer that never saw the switch issues, and the toggled process still matches the fixture."""
    import open_musiclm_b200 as O
    from open_musiclm_b200 import lib
    path = [p for p in GOLD if p.endswith("tiny_coarse.pt")][0]
    fx = torch.load(path, weights_only=False)
    gold = {k: (g if g is not None else torch.zeros_like(fx["state_dict"][k])) for k, g in fx["grads"].items()}
    batches = _cfg2_batches(8, B=4, seed=2)

    def record(fn):
        names, real = [], lib.call
        lib.call = lambda name, *a: (names.append(name), real(name, *a))[1]
        try:
            fn()
        finally:
            lib.call = real
        return names

    def fixture_pass(t):
        """eval loss + gradients of the fixture batch, each reading the switch as a step does"""
        toks = [x.cuda() for x in fx["tokens"]]
        loss = float(t.eval_loss(toks))
        t.eng.arena_g.zero_()
        t._micro_batch(toks, False, 0, True, det=torch.are_deterministic_algorithms_enabled())
        grads = {k: t.eng.gview[k].clone() for k, _ in t.transformer.named_parameters()}
        t.eng.arena_g.zero_()
        assert abs(loss - float(fx["loss"])) / float(fx["loss"]) <= 1e-2
        _check_grads(grads, gold, "fixture")

    # reference entry-point sequences from trainers that never see the switch (second passes: no one-time packing)
    with switch(False):
        t0 = _trainer(depth=2, heads=8, mask_prob=0.0)
        t0.train_step([batches[4]])
        names_t0 = record(lambda: t0.train_step([batches[5]]))
        f0 = O.HotPathTrainer(_build(fx), cross_entropy_loss_weights=fx["ce_weights"], lr=3e-4, lr_warmup=10, wd=1e-2)
        fixture_pass(f0)
        names_f0 = record(lambda: fixture_pass(f0))
        del t0, f0

    tr = _trainer(depth=2, heads=8, mask_prob=0.0)     # no forgetful mask: see test_two_trainers_same_seed_bit_identical
    tx = O.HotPathTrainer(_build(fx), cross_entropy_loss_weights=fx["ce_weights"], lr=3e-4, lr_warmup=10, wd=1e-2)
    with switch(True):
        on_names = record(lambda: tr.train_step([batches[0]]))           # eager steps 1-2, then the capture
        for b in batches[1:4]:
            tr.train_step([b])
        fixture_pass(tx)
    assert any(n.endswith("_det") for n in on_names)
    with switch(False):
        tr.train_step([batches[4]])                                       # new key: eager steps in the default mode
        off_names = record(lambda: tr.train_step([batches[5]]))
        tr.train_step([batches[6]])                                       # ... then the capture
        fixture_pass(tx)                                                  # the toggled process matches the fixture
        off_fix = record(lambda: fixture_pass(tx))
    assert off_names == names_t0 and not any(n.endswith("_det") for n in off_names)
    assert off_fix == names_f0
    assert {k[0] for k in tr._graphs} == {True, False}
    assert all(st["graphs"] is not None for st in tr._graphs.values())
    # back on: from a saved state, the toggled trainer and a fresh on-mode trainer take bit-identical steps
    with switch(True):
        fixture_pass(tx)
        ck_model = {k: v.clone() for k, v in tr.transformer.state_dict().items()}
        ck_opt = tr.state_dict()
        lt = [tr.train_step([b]).clone() for b in batches[:4]]
        tf = _trainer(depth=2, heads=8, seed=1, mask_prob=0.0)
        tf.transformer.load_state_dict(ck_model)
        tf.load_state_dict(ck_opt)
        lf = [tf.train_step([b]).clone() for b in batches[:4]]
        assert all(torch.equal(x, y) for x, y in zip(lt, lf)), (lt, lf)
        _assert_same_state(tr, tf)
    tr.eng.check_errors()


def test_eval_and_generate_under_the_switch(det):
    import open_musiclm_b200 as O
    tr = _trainer(depth=2, heads=8)
    b = _cfg2_batches(1, B=4, seed=9)[0]
    l1, l2 = tr.eval_loss(b).clone(), tr.eval_loss(b).clone()
    assert bool(torch.isfinite(l1)) and torch.equal(l1, l2)
    w = O.TokenConditionedTransformerWrapper(transformer=tr.transformer.eval(), unique_consecutive=False)
    g = torch.Generator().manual_seed(5)
    cond = [torch.randint(0, 1024, (4, 12), generator=g).cuda(), torch.randint(0, 1024, (4, 20), generator=g).cuda()]
    uni = torch.rand(8 * 3, 4, 1025, generator=g).clamp_(1e-6, 1 - 1e-6)
    on = w.generate(conditioning_token_ids=cond, max_time_steps=8, uniform_noise=uni)
    with switch(False):
        off = w.generate(conditioning_token_ids=cond, max_time_steps=8, uniform_noise=uni)
    assert torch.equal(on, off)
