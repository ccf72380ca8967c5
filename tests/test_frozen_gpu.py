"""Fine-tuning with frozen parameters on the H100 path: the kernels' null parameter-gradient outputs, the attention
backward without the bias gradient, and the trainer / API path with parameters frozen by requires_grad=False.

Bit-identity is asserted wherever the library promises a fixed order (deterministic mode, and kernels without float
atomics on the compared outputs).  The default-mode attention backward adds dQ and dK|dV with atomics in arrival order,
so there the two variants are compared up to fp32 reordering."""
import contextlib
import glob
import os

import pytest
import torch
import torch.nn.functional as F

import optim_reference as OR
from test_attention_reference_gpu import CASES as ATTN_CASES, make_inputs
from test_deterministic_gpu import _build, _check_grads
from test_optim_reference_gpu import _check_update, _spy

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = {os.path.basename(p)[:-3]: p for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "tiny_*.pt"))}


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as _lib
    _lib.load()
    return _lib


@contextlib.contextmanager
def switch(on):
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------ attention backward
def _attn_both(lib, B, N, h, mask, bias, qk, det):
    """(dq, dkv) with a bias table and with dtable = None, from the same inputs."""
    qn, kvn, table, key_mask, d_o = make_inputs(B, N, h, mask, bias, qk, seed=B * 7919 + N * 31 + h)
    M = B * N
    out = torch.empty(M, h * 64, device=DEV, dtype=torch.bfloat16)
    lse = torch.empty(M * h, device=DEV)
    lib.attn_fwd_tc(qn, kvn, table, key_mask, out, lse, B, N, h)
    res = []
    for with_table in (True, False):
        dq = torch.full((M, h * 64), float("nan"), device=DEV)
        dkv = torch.full((M, 128), float("nan"), device=DEV)
        dt = torch.zeros(h, table.shape[1], device=DEV) if with_table else None
        ws = lib.AttnBwdDetWorkspace(DEV, B, N, h) if det else None
        lib.attn_bwd_tc(qn, kvn, d_o, out, lse, table, key_mask, torch.empty(M * h, device=DEV), dq, dkv, dt, B, N, h, det=ws)
        torch.cuda.synchronize()
        if ws is not None:
            assert not ws.error()
        res.append((dq, dkv))
    return res


def _assert_same(res, det, tag):
    (dq1, dkv1), (dq0, dkv0) = res
    assert bool(torch.isfinite(dq0).all()) and bool(torch.isfinite(dkv0).all()), tag
    if det:
        assert bits_equal(dq0, dq1) and bits_equal(dkv0, dkv1), tag
    else:
        assert rel(dq0, dq1) <= 1e-5 and rel(dkv0, dkv1) <= 1e-5, (tag, rel(dq0, dq1), rel(dkv0, dkv1))


@pytest.mark.parametrize("det", [True, False], ids=["det", "default"])
@pytest.mark.parametrize("B,N,h,mask,bias,qk", [c for c in ATTN_CASES if c[2] <= 58],
                         ids=[f"B{c[0]}-N{c[1]}-h{c[2]}-{c[3]}-{c[4]}-{c[5]}" for c in ATTN_CASES if c[2] <= 58])
def test_attn_bwd_without_table_matches(lib, B, N, h, mask, bias, qk, det):
    """dtable = None: dQ and dK|dV equal the call with a table (bit for bit in deterministic mode)."""
    _assert_same(_attn_both(lib, B, N, h, mask, bias, qk, det), det, (B, N, h))


@pytest.mark.parametrize("B,N,h", [(2, 700, 3), (1, 1024, 8), (1, 260, 12)])
def test_attn_bwd_without_table_at_forced_chunk_lengths(lib, monkeypatch, B, N, h):
    for T in (1, 3, 16):
        monkeypatch.setenv("OMLM_ATTN_BWD_T", str(T))
        _assert_same(_attn_both(lib, B, N, h, "rand", "rand", "rand", True), True, (B, N, h, T))


# ------------------------------------------------------------------------------------------------ null gradient outputs
GUARD = 12345.0


def _guarded(n):
    """A buffer of n floats inside guard values: (view, whole)."""
    whole = torch.full((n + 64,), GUARD, device=DEV)
    return whole[32:32 + n], whole


def _guard_ok(whole, n):
    return bool((whole[:32] == GUARD).all()) and bool((whole[32 + n:] == GUARD).all())


@pytest.mark.parametrize("det", [True, False], ids=["det", "default"])
@pytest.mark.parametrize("M,D", [(1000, 128), (777, 1024), (64, 200)])
def test_layernorm_bwd_null_dgamma(lib, M, D, det):
    g = torch.Generator(device=DEV).manual_seed(M + D)
    x = torch.randn(M, D, device=DEV, generator=g) * 2 + 0.5
    gamma = torch.rand(D, device=DEV, generator=g) + 0.5
    y = torch.empty(M, D, device=DEV, dtype=torch.bfloat16)
    stats = torch.empty(M, 2, device=DEV)
    lib.layernorm_fwd(x, gamma, y, None, stats)
    dy = torch.randn(M, D, device=DEV, generator=g).bfloat16()
    dres = torch.randn(M, D, device=DEV, generator=g)
    draw = torch.randn(M, D, device=DEV, generator=g).bfloat16()
    part = torch.empty(4 * lib.num_sms() * max(D, 128), device=DEV) if det else None
    outs = []
    for null in (False, True):
        dx = torch.full((M, D), float("nan"), device=DEV)
        dxb = torch.empty(M, D, device=DEV, dtype=torch.bfloat16)
        dg, whole = _guarded(D)
        dg.fill_(0.25)
        lib.layernorm_bwd(dy, x, stats, gamma, dx, None if null else dg, dres=dres, draw=draw, dx_bf16=dxb, part=part)
        torch.cuda.synchronize()
        assert _guard_ok(whole, D)
        outs.append((dx, dxb, dg))
    assert bits_equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert bool((outs[1][2] == 0.25).all()) and not bool((outs[0][2] == 0.25).all())


@pytest.mark.parametrize("det", [True, False], ids=["det", "default"])
@pytest.mark.parametrize("which", ["q", "k", "both"])
def test_qk_l2norm_bwd_null_scales(lib, which, det):
    M, h = 3000, 3
    g = torch.Generator(device=DEV).manual_seed(7)
    q_raw = torch.randn(M, h * 64, device=DEV, generator=g).bfloat16()
    kv_raw = torch.randn(M, 128, device=DEV, generator=g).bfloat16()
    qs = torch.rand(64, device=DEV, generator=g) + 0.5
    ks = torch.rand(64, device=DEV, generator=g) + 0.5
    dqn = torch.randn(M, h * 64, device=DEV, generator=g)
    dkvn = torch.randn(M, 128, device=DEV, generator=g)
    part = torch.empty(8 * lib.num_sms() * 128, device=DEV) if det else None

    def run(null_q, null_k):
        dq_raw = torch.empty(M, h * 64, device=DEV, dtype=torch.bfloat16)
        dkv_raw = torch.empty(M, 128, device=DEV, dtype=torch.bfloat16)
        (dqs, wq), (dks, wk) = _guarded(64), _guarded(64)
        dqs.fill_(0.5); dks.fill_(-0.5)
        lib.qk_l2norm_bwd(dqn, dkvn, q_raw, kv_raw, qs, ks, dq_raw, dkv_raw, None if null_q else dqs, None if null_k else dks, h, part=part)
        torch.cuda.synchronize()
        assert _guard_ok(wq, 64) and _guard_ok(wk, 64)
        return dq_raw, dkv_raw, dqs, dks

    full = run(False, False)
    part_run = run(which in ("q", "both"), which in ("k", "both"))
    assert torch.equal(full[0], part_run[0]) and torch.equal(full[1], part_run[1])
    for i, null in ((2, which in ("q", "both")), (3, which in ("k", "both"))):
        init = 0.5 if i == 2 else -0.5
        if null:
            assert bool((part_run[i] == init).all())
        elif det:
            assert bits_equal(part_run[i], full[i])
        else:
            assert rel(part_run[i], full[i]) <= 1e-5


@pytest.mark.parametrize("det", [True, False], ids=["det", "default"])
@pytest.mark.parametrize("which", ["gamma", "conv", "both"])
def test_ffn_mid_bwd_null_outputs(lib, which, det):
    B, N, F_, Fp = 2, 300, 200, 256
    M = B * N
    g = torch.Generator(device=DEV).manual_seed(11)
    dhn = torch.randn(M, Fp, device=DEV, generator=g).bfloat16()
    hn = torch.randn(M, Fp, device=DEV, generator=g).bfloat16()
    u = torch.randn(M, 2 * Fp, device=DEV, generator=g).bfloat16()
    stats = torch.stack([torch.randn(M, device=DEV, generator=g) * 0.1, torch.rand(M, device=DEV, generator=g) + 0.5], 1).contiguous()
    conv = torch.randn(2 * Fp, 3, device=DEV, generator=g) * 0.5
    gamma = torch.zeros(Fp, device=DEV)
    gamma[:F_] = torch.rand(F_, device=DEV, generator=g) + 0.5
    part = torch.empty(B * ((N + 127) // 128) * 7 * F_, device=DEV) if det else None

    def run(null_g, null_c):
        du = torch.empty(M, 2 * Fp, device=DEV, dtype=torch.bfloat16)
        rowstat = torch.empty(M, 2, device=DEV)
        (dg, wg), (dc, wc) = _guarded(F_), _guarded(6 * F_)
        dg.fill_(0.5); dc.fill_(-0.5)
        lib.ffn_mid_bwd(dhn, hn, u, stats, conv, gamma, rowstat, du, None if null_g else dg, None if null_c else dc, B, N, F_, Fp,
                        part=part)
        torch.cuda.synchronize()
        assert _guard_ok(wg, F_) and _guard_ok(wc, 6 * F_)
        return du, dg, dc

    full = run(False, False)
    got = run(which in ("gamma", "both"), which in ("conv", "both"))
    assert torch.equal(full[0], got[0])
    for i, null, init in ((1, which in ("gamma", "both"), 0.5), (2, which in ("conv", "both"), -0.5)):
        if null:
            assert bool((got[i] == init).all())
        elif det:
            assert bits_equal(got[i], full[i])
        else:
            assert rel(got[i], full[i]) <= 1e-5


# ------------------------------------------------------------------------------------------------ trainer
def _names(m):
    return [n for n, _ in m.named_parameters()]


def pattern(kind, names, depth):
    """Parameter names frozen by each pattern."""
    rows = ("embeddings.", "absolute_position_embeddings.", "start_tokens.")
    if kind == "rows":                      # (a) embeddings (+ absolute positions) and start tokens
        return {n for n in names if n.startswith(rows)}
    if kind == "emb":                       # the token embeddings only: start tokens and positions still train
        return {n for n in names if n.startswith("embeddings.")}
    if kind == "relpos":                    # (b) the relative-position bias parameters
        return {n for n in names if n.startswith("transformer.rel_pos_bias.")}
    if kind == "top":                       # (c) everything but the top layer and the heads
        return {n for n in names if not n.startswith((f"transformer.layers.{depth - 1}.", "logit_weights."))}
    if kind == "heads":                     # (d) only the heads trainable
        return {n for n in names if not n.startswith("logit_weights.")}
    raise ValueError(kind)


def _model(fx, frozen):
    m = _build(fx)
    for n, p in m.named_parameters():
        p.requires_grad_(n not in frozen)
    return m


def _trainer(fx, frozen, graph=False, mask_prob=0.15):
    import open_musiclm_b200 as O
    return O.HotPathTrainer(_model(fx, frozen), cross_entropy_loss_weights=fx["ce_weights"], lr=1e-3, lr_warmup=3, wd=1e-2,
                            max_grad_norm=0.5, grad_accum_every=1, mask_prob=mask_prob, use_cuda_graph=graph)


def _batch(fx, step):
    g = torch.Generator().manual_seed(500 + step)
    return [[torch.randint(0, 64, tuple(t.shape), generator=g).cuda() for t in fx["tokens"]]]


PATTERNS = [("tiny_coarse", k) for k in ("rows", "relpos", "top", "heads")] + \
           [("tiny_coarse", "emb"), ("tiny_semantic", "top"), ("tiny_fine", "rows"), ("tiny_nobias_abspos", "emb"), ("tiny_plainff_t5", "top"), ("tiny_plainff_t5", "relpos"),
            ("tiny_nobias_abspos", "top"), ("tiny_nobias_abspos", "rows")]


@pytest.mark.parametrize("fx_name,kind", PATTERNS, ids=[f"{a}-{b}" for a, b in PATTERNS])
def test_trainer_frozen_deterministic(lib, fx_name, kind):
    """Deterministic mode: after the first step the trainable gradients equal an unfrozen twin's bit for bit; over four
    steps the frozen ranges of arena_g, arena_p, adam_m and adam_v do not change, and every update is within the float64
    reference's per-element scale."""
    fx = torch.load(GOLD[fx_name], weights_only=False)
    names = _names(_build(fx))
    frozen = pattern(kind, names, fx["kwargs"]["depth"])
    with switch(True):
        tf, tu = _trainer(fx, frozen), _trainer(fx, set())
        assert frozen <= tf.frozen and not (tf.frozen - frozen - tu.frozen)
        sf, su = _spy(tf), _spy(tu)
        eng = tf.eng
        spans = [(eng.layout[n], eng.layout[n] + eng.pview[n].numel()) for n in tf.frozen]
        before = [x.clone() for x in (eng.arena_p, eng.adam_m, eng.adam_v)]
        for step in range(4):
            mb = _batch(fx, step)
            tf.train_step(mb)
            if step == 0:
                tu.train_step(mb)
            torch.cuda.synchronize()
            assert int(eng.err_flag.item()) == 0
            g = sf[step][1]
            for a, b in spans:
                assert not bool(g[a:b].any()), (step, a, b)
                for x0, x in zip(before, (eng.arena_p, eng.adam_m, eng.adam_v)):
                    assert bits_equal(x0[a:b], x[a:b]), (step, a, b)
            if step == 0:
                gu = su[0][1]
                for n in names:
                    if n not in tf.frozen:
                        o, k = eng.layout[n], eng.pview[n].numel()
                        assert bits_equal(g[o:o + k], gu[o:o + k]), n
            _check_update(lib, tf, sf[step], step)


def test_trainer_frozen_graph_matches_eager_and_flags_are_read_once(lib):
    """The CUDA-graph trainer equals its eager twin bit for bit (no forgetful mask: a captured graph keeps the mask
    stream's host-side draw count, as in test_optim_reference_gpu.py); a requires_grad change afterwards raises."""
    fx = torch.load(GOLD["tiny_coarse"], weights_only=False)
    frozen = pattern("top", _names(_build(fx)), fx["kwargs"]["depth"])
    with switch(True):
        tg, te = _trainer(fx, frozen, graph=True, mask_prob=0.0), _trainer(fx, frozen, graph=False, mask_prob=0.0)
        for step in range(5):
            mb = _batch(fx, step)
            tg.train_step(mb)
            te.train_step(mb)
            torch.cuda.synchronize()
            for a, b in ((tg.eng.arena_p, te.eng.arena_p), (tg.eng.adam_m, te.eng.adam_m), (tg.eng.adam_v, te.eng.adam_v)):
                assert bits_equal(a, b), step
        assert tg._graphs and all(st["graphs"] is not None for st in tg._graphs.values())
    p = dict(tg.transformer.named_parameters())["transformer.layers.0.0.to_q.weight"]
    p.requires_grad_(True)
    with pytest.raises(RuntimeError, match="requires_grad changed"):
        tg.train_step(_batch(fx, 9))


def _api_grads(m, fx):
    ids = [t.cuda() for t in fx["ids"]]
    logits = m(all_token_ids=ids, self_attn_mask=fx["key_mask"].cuda())
    with switch(False):           # torch's cross entropy has no deterministic CUDA kernel: d loss / d logits are torch's,
        total, loss = 0, 0.0      # the library's backward below runs in the caller's mode
        for lg, lb, w in zip(logits, fx["labels"], fx["ce_weights"]):
            if w > 0:
                loss = loss + F.cross_entropy(lg.permute(0, 2, 1), lb.cuda()) * lb.numel() * w
                total += lb.numel()
        live = [lg for lg in logits if lg is not None and lg.requires_grad]
        dl = torch.autograd.grad(loss / total, live, allow_unused=True)
    pairs = [(a, g) for a, g in zip(live, dl) if g is not None]
    torch.autograd.backward([a for a, _ in pairs], [g for _, g in pairs])
    torch.cuda.synchronize()
    return {n: p.grad for n, p in m.named_parameters()}


@pytest.mark.parametrize("fx_name,kind", [("tiny_coarse", "top"), ("tiny_coarse", "relpos"), ("tiny_plainff_t5", "top"),
                                          ("tiny_nobias_abspos", "rows")])
@pytest.mark.parametrize("det", [True, False], ids=["det", "default"])
def test_api_path_frozen(lib, fx_name, kind, det):
    """loss.backward() leaves grad None on frozen parameters; the others equal the unfrozen model's (bit for bit in
    deterministic mode) and the reference fixture's within the parity bounds."""
    fx = torch.load(GOLD[fx_name], weights_only=False)
    names = _names(_build(fx))
    frozen = pattern(kind, names, fx["kwargs"]["depth"])
    with switch(det):
        gf = _api_grads(_model(fx, frozen), fx)
        gu = _api_grads(_model(fx, set()), fx)
    for n in names:
        if n in frozen:
            assert gf[n] is None, n
        elif det:
            assert bits_equal(gf[n], gu[n]), n
    _check_grads({n: g for n, g in gf.items() if n not in frozen}, {n: g for n, g in fx["grads"].items() if n not in frozen}, "frozen api")


def test_api_path_frozen_after_the_engine_exists(lib):
    """Freezing after a forward pass (the engine and its arena views exist): the frozen gradients are None."""
    fx = torch.load(GOLD["tiny_coarse"], weights_only=False)
    m = _build(fx)
    with torch.no_grad():
        m(all_token_ids=[t.cuda() for t in fx["ids"]], self_attn_mask=fx["key_mask"].cuda())
    frozen = pattern("rows", _names(m), fx["kwargs"]["depth"])
    for n, p in m.named_parameters():
        p.requires_grad_(n not in frozen)
    g = _api_grads(m, fx)
    assert all((g[n] is None) == (n in frozen) for n in g)


@pytest.mark.parametrize("fx_name,kind", [("tiny_coarse", "rows"), ("tiny_coarse", "top"), ("tiny_plainff_t5", "heads")])
def test_trainer_frozen_default_mode(lib, fx_name, kind):
    """Default mode: the trainable gradients of a step match the unfrozen twin's within the parity bounds; frozen ranges
    stay bit-unchanged."""
    fx = torch.load(GOLD[fx_name], weights_only=False)
    names = _names(_build(fx))
    frozen = pattern(kind, names, fx["kwargs"]["depth"])
    with switch(False):
        tf, tu = _trainer(fx, frozen), _trainer(fx, set())
        sf, su = _spy(tf), _spy(tu)
        p0 = tf.eng.arena_p.clone()
        mb = _batch(fx, 0)
        tf.train_step(mb)
        tu.train_step(mb)
        torch.cuda.synchronize()
    eng = tf.eng
    got = {n: sf[0][1][eng.layout[n]:eng.layout[n] + eng.pview[n].numel()].view(eng.pview[n].shape) for n in names}
    ref = {n: (None if n in tf.frozen else su[0][1][eng.layout[n]:eng.layout[n] + eng.pview[n].numel()].view(eng.pview[n].shape))
           for n in names}
    _check_grads(got, ref, "default-mode trainer")
    for n in tf.frozen:
        o, k = eng.layout[n], eng.pview[n].numel()
        assert bits_equal(p0[o:o + k], eng.arena_p[o:o + k]), n
