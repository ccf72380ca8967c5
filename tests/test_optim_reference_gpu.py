"""The optimiser step on the GPU against float64 (tests/optim_reference.py): grad_sumsq and adamw_step within their
derived error scales, the re-pack of the master weights bit for bit against a torch reconstruction, the engine's packed
buffers and arena after steps, and the trainer's trajectory and checkpoint files against the reference's optimizer."""
import pytest
import torch

import optim_reference as OR

pytestmark = pytest.mark.gpu
DEV = "cuda"
TINY = dict(dim=128, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=64, acoustic_codebook_size=64,
            num_clap_quantizers=4, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1)
CE = [0.0, 0.0, 1.0]


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as L
    L.device_check()
    return L


def _mixed_magnitudes(n, seed, lo=-20, hi=15):
    gen = torch.Generator().manual_seed(seed)
    e = torch.rand(n, generator=gen, dtype=torch.float64) * (hi - lo) + lo
    return (torch.randn(n, generator=gen, dtype=torch.float64).sign() * 10.0 ** e).float().to(DEV)


def _sumsq(lib, g, prescale, det):
    acc = torch.zeros(1, device=DEV, dtype=torch.float64)
    part = torch.empty(4 * lib.num_sms(), device=DEV, dtype=torch.float64) if det else None
    lib.grad_sumsq(g, acc, prescale=prescale, part=part)
    return float(acc)


# ------------------------------------------------------------------------------------------------ grad_sumsq
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 7, 4099, 3_000_003])
@pytest.mark.parametrize("prescale", [1.0, 0.125])
@pytest.mark.parametrize("det", [False, True], ids=["atomic", "det"])
def test_grad_sumsq_within_bound(lib, n, prescale, det):
    """Every n & 3 tail, a size where every thread loops, magnitudes 1e-20 ... 1e15; det repeats bit-identical."""
    g = _mixed_magnitudes(n, n)
    blocks, _ = OR.sumsq_grid(n, lib.num_sms())
    for gg in (g, g * 1e-15, g.abs().clamp_max(1e-18)):                 # the sum dominated by large, mid and tiny terms
        got, want = _sumsq(lib, gg, prescale, det), OR.sumsq(gg, prescale)
        assert abs(got - want) <= OR.sumsq_bound(gg, prescale, blocks), (got, want)
        if det:
            assert _sumsq(lib, gg, prescale, det) == got


def test_grad_sumsq_at_the_cfg4_arena_size(lib):
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=24, heads=16, num_coarse_quantizers=3).cuda()
    n = m.engine.n_params_arena
    del m
    torch.cuda.empty_cache()
    assert n > 200_000_000
    g = torch.randn(n, device=DEV) * 1e-3
    blocks, _ = OR.sumsq_grid(n, lib.num_sms())
    want, bound = OR.sumsq(g), OR.sumsq_bound(g, 1.0, blocks)
    for det in (False, True):
        got = _sumsq(lib, g, 1.0, det)
        assert abs(got - want) <= bound, (det, got, want, bound)


# ------------------------------------------------------------------------------------------------ adamw_step
CASES = [dict(t=1, fac=1e-7, wd=0.01, max_norm=0.5), dict(t=2, fac=0.3, wd=0.0, max_norm=1e6),
         dict(t=10, fac=1.0, wd=0.01, max_norm=None), dict(t=1000, fac=1.0, wd=0.01, max_norm=1e-4, prescale=1 / 3, gscale=1e-8),
         dict(t=100000, fac=1.0, wd=0.01, max_norm=0.5, prescale=0.125)]


def _adamw_run(lib, case, n, n_decay):
    p, g, m, v = OR.adamw_cases(n, seed=case["t"] + n, device=DEV)
    g = g * case.get("gscale", 1.0)
    pre = case.get("prescale", 1.0)
    kw = dict(t=case["t"], lr=3e-4 * case["fac"], wd=case["wd"], n_decay=n_decay, max_grad_norm=case["max_norm"], prescale=pre)
    S = OR.sumsq(g, pre)
    hyper = torch.tensor(OR.hyper_vector(t=kw["t"], lr=kw["lr"], wd=kw["wd"], max_grad_norm=kw["max_grad_norm"], prescale=pre),
                         dtype=torch.float32, device=DEV)
    acc = torch.tensor([S], dtype=torch.float64, device=DEV)
    pk, mk, vk = p.clone(), m.clone(), v.clone()
    lib.adamw_step(pk, g, mk, vk, n_decay, hyper, acc)
    want = OR.adamw_update(p, g, m, v, **kw)[:3]
    bound = OR.adamw_bound(p, g, m, v, **kw, sumsq_value=S)
    return (pk, mk, vk), want, bound, (p, g, m, v, hyper, acc)


@pytest.mark.parametrize("n", [7003, 1_200_007], ids=["one-pass", "grid-stride"])
@pytest.mark.parametrize("which", range(6), ids=["nd0", "nd1", "nd63", "nd64", "nd-n-1", "nd-n"])
@pytest.mark.parametrize("case", CASES, ids=[f"t{c['t']}" for c in CASES])
def test_adamw_step_componentwise(lib, n, which, case):
    """p, m and v of every element within the derived scale: n_decay at every edge, n below and above the grid-stride
    threshold, t up to 1e5, warm-up factor 1e-7, clip active / inactive / disabled, prescale 1/3 and 1/8, gradients 0,
    subnormal, 1e-12, 1, 1e4, v = 0 (denominator exactly eps) and v ~ eps^2."""
    n_decay = [0, 1, 63, 64, n - 1, n][which]
    got, want, bound, _ = _adamw_run(lib, case, n, n_decay)
    for name, x, w, b in zip("pmv", got, want, bound):
        err = (x.double() - w).abs()
        bad = err > b
        assert not bool(bad.any()), (name, int(bad.sum()), float((err / b.clamp_min(1e-300)).max()))


def test_adamw_shard_split_is_bit_identical(lib):
    """AdamW over arena parts [a, b) with n_decay' = max(0, min(b - a, n_decay - a)) (the sharded update, the frozen-head
    gaps) equals the whole-arena launch bit for bit."""
    n, n_decay = 1_200_007, 700_001
    (pk, mk, vk), _, _, (p, g, m, v, hyper, acc) = _adamw_run(lib, CASES[0], n, n_decay)
    ps, ms, vs = p.clone(), m.clone(), v.clone()
    cuts = [0, 63, 4096, 700_000, 700_001, 700_002, 1_000_000, n]
    for a, b in zip(cuts[:-1], cuts[1:]):
        lib.adamw_step(ps[a:b], g[a:b], ms[a:b], vs[a:b], max(0, min(b - a, n_decay - a)), hyper, acc)
    for x, y in ((ps, pk), (ms, mk), (vs, vk)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


# ------------------------------------------------------------------------------------------------ pack
FMTS = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}


def _convert(x, dt):
    """fp32 -> dt as the pack kernels convert: round to nearest even; fp16 saturates finite (satfinite), keeps NaN."""
    return x.clamp(-65504.0, 65504.0).to(dt) if dt == torch.float16 else x.to(dt)


def _bits(x):
    return x.view(torch.int16 if x.element_size() == 2 else torch.int32)


def _assert_bits(got, want, what=""):
    gn, wn = got.float().isnan(), want.float().isnan()
    assert torch.equal(gn, wn), what
    assert torch.equal(_bits(got)[~gn], _bits(want)[~wn]), what


def _reconstruct(src, rows_valid, cols_valid, rows_p, cols_p, split_dst, split_src):
    """dst[r, c] = src[map(r), c] (include/omlm_b200.h), zero elsewhere; src [rows, src_ld] fp32."""
    r = torch.arange(rows_p, device=src.device)
    if split_dst > 0:
        half, rr = r // split_dst, r % split_dst
        sr = half * split_src + rr
        live = (rr < split_src) & (sr < rows_valid)
    elif split_dst < 0:
        w = r % 256
        ch = (r // 256) * 128 + w % 128
        sr = (w // 128) * split_src + ch
        live = (ch < split_src) & (sr < rows_valid)
    else:
        sr, live = r, r < rows_valid
    out = torch.zeros(rows_p, cols_p, device=src.device)
    out[live, :cols_valid] = src[sr[live], :cols_valid]
    return out


def _special_src(rows, ld, seed):
    """Random values with ±0, fp32 / fp16 / bf16 subnormals, ±inf, NaN, 65504 ... 70000 and bf16 / fp16 ties mixed in."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(rows * ld, generator=gen)
    sp = torch.tensor([0.0, -0.0, 1e-40, -3e-39, 1e-6, -5e-8, float("inf"), float("-inf"), float("nan"), 65504.0, -65519.0,
                       65520.0, 70000.0, -1e30, 1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 1 + 2 ** -11, 1 + 3 * 2 ** -11, 2.0 ** -126])
    pick = torch.rand(rows * ld, generator=gen) < 0.3
    x[pick] = sp[torch.randint(0, len(sp), (int(pick.sum()),), generator=gen)]
    return x.view(rows, ld).to(DEV)


def _dst(rows_p, cols_p, dt, misalign):
    """A destination filled with NaN bits; misalign: starts one element past a 16-byte boundary (scalar stores)."""
    buf = torch.full((rows_p * cols_p + 8,), float("nan"), device=DEV).to(dt)
    o = 1 if misalign else 0
    return buf[o:o + rows_p * cols_p].view(rows_p, cols_p)


# (rows_valid, cols_valid, src_ld, rows_p, cols_p, split_dst, split_src): plain with row and column padding, per-head
# padding, GEGLU interleave with F = 200 and 130 (not multiples of 128), cols_p not a multiple of 4 (scalar stores),
# odd src_ld (scalar loads), one-quad and exactly-one-unit (1024 quads) jobs
GEOMS = [(70, 52, 52, 80, 64, 0, 0), (5, 7, 9, 8, 8, 0, 0), (3 * 37, 48, 48, 3 * 64, 48, 64, 37), (400, 24, 24, 512, 24, -1, 200),
         (260, 3, 3, 512, 3, -1, 130), (9, 13, 13, 9, 13, 0, 0), (64, 64, 64, 64, 64, 0, 0), (1, 4, 4, 1, 4, 0, 0),
         (1, 200, 200, 1, 256, 0, 0)]


@pytest.mark.parametrize("geom", GEOMS, ids=[f"g{i}" for i in range(len(GEOMS))])
@pytest.mark.parametrize("fmt", list(FMTS))
@pytest.mark.parametrize("misalign", [False, True], ids=["vec", "scalar"])
def test_pack_single_bit_exact(lib, geom, fmt, misalign):
    rv, cv, ld, rp, cp, sd, ss = geom
    src = _special_src(rv, ld, hash(geom) & 0xffff)
    dst = _dst(rp, cp, FMTS[fmt], misalign)
    lib.pack(src, ld, rv, cv, dst, rp, cp, sd, ss)
    _assert_bits(dst, _convert(_reconstruct(src, rv, cv, rp, cp, sd, ss), FMTS[fmt]), (geom, fmt))


def _table_jobs(njobs, seed):
    """Job geometries cycling through GEOMS and large multi-unit jobs, formats and dual destinations in both pairings."""
    jobs = []
    for j in range(njobs):
        if j % 7 == 3:
            geom = (300, 64, 64, 300, 64, 0, 0)                        # 4800 quads: several units, ends mid-unit
        elif j % 11 == 5:
            geom = (128, 64, 64, 128, 64, 0, 0)                        # ends exactly on a unit boundary
        else:
            geom = GEOMS[j % len(GEOMS)]
        kind = j % 5
        fmt, fmt2 = [("bf16", None), ("f16", None), ("f32", None), ("f16", "bf16"), ("bf16", "f16")][kind]
        jobs.append((geom, fmt, fmt2, (j // 5) % 2 == 1))
    return jobs


@pytest.mark.parametrize("njobs", [1, 512, 513])
def test_pack_table_bit_exact(lib, njobs):
    """PackTable: 1, 512 and 513 jobs (two launches); small jobs between multi-unit ones, jobs ending on a unit
    boundary, every format, dual destinations both ways, vector and scalar paths; padding exactly +0."""
    tab = lib.PackTable(torch.device(DEV))
    outs = []
    for j, (geom, fmt, fmt2, mis) in enumerate(_table_jobs(njobs, 0)):
        rv, cv, ld, rp, cp, sd, ss = geom
        src = _special_src(rv, ld, j)
        dst = _dst(rp, cp, FMTS[fmt], mis)
        dst2 = _dst(rp, cp, FMTS[fmt2], mis) if fmt2 else None
        tab.add(src, ld, rv, cv, dst, rp, cp, split_dst=sd, split_src=ss, dst2=dst2)
        outs.append((src, geom, dst, dst2))
    assert tab.n_jobs == njobs and len(tab.chunks) == (njobs + 511) // 512
    tab.run()
    torch.cuda.synchronize()
    for j, (src, (rv, cv, ld, rp, cp, sd, ss), dst, dst2) in enumerate(outs):
        ref = _reconstruct(src, rv, cv, rp, cp, sd, ss)
        _assert_bits(dst, _convert(ref, dst.dtype), j)
        if dst2 is not None:
            _assert_bits(dst2, _convert(ref, dst2.dtype), (j, "dst2"))


@pytest.mark.parametrize("geom", GEOMS, ids=[f"g{i}" for i in range(len(GEOMS))])
def test_unpack_add_inverts_pack(lib, geom):
    rv, cv, ld, rp, cp, sd, ss = geom
    src = torch.randn(rv, ld, device=DEV)
    packed = torch.empty(rp, cp, device=DEV)
    lib.pack(src, ld, rv, cv, packed, rp, cp, sd, ss)
    base = torch.randn(rv, ld, device=DEV)
    acc = base.clone()
    lib.unpack_add(packed, rp, cp, acc, ld, rv, cv, sd, ss)
    want = base.clone()
    want[:, :cv] += src[:, :cv]
    assert torch.equal(acc, want)


# ------------------------------------------------------------------------------------------------ engine state
def _engine_model(monkeypatch, act16, d, L, conv_ff=True):
    import open_musiclm_b200 as O
    monkeypatch.setenv("OMLM_ACT16", act16)
    torch.manual_seed(0)
    kw = dict(TINY, dim=d, depth=L, heads=2 if d == 128 else 8)
    if d != 128:
        kw.update(clap_codebook_size=1024, semantic_codebook_size=1024, acoustic_codebook_size=1023)
    m = O.create_coarse_transformer(**kw, use_conv_ff=conv_ff).cuda()
    return m


def _tokens(m, B=2, seed=1234):
    g = torch.Generator().manual_seed(seed)
    cb = [s.codebook_size for s in m.engine.seqs]
    return [torch.randint(0, c, s, generator=g).cuda() for c, s in zip(cb, [(B, 4), (B, 11), (B, 10, 3)])]


def _check_packed(eng):
    pv, d, HD, F, Fp = eng.pview, eng.d, eng.HD, eng.F, eng.Fp
    bf = torch.bfloat16
    for l, pk in enumerate(eng.pk):
        p = f"transformer.layers.{l}."
        fk = eng.ffk
        wq = _reconstruct(pv[p + "0.to_q.weight"], HD, d, HD, d, 0, 0)
        w1 = _reconstruct(pv[p + fk["w1"]], 2 * F, d, 2 * Fp, d, -1, F)
        w2 = _reconstruct(pv[p + fk["w2"]], d, F, d, Fp, 0, 0)
        for k, ref in (("wq", wq), ("w1", w1), ("w2", w2)):
            _assert_bits(pk[k], _convert(ref, eng.a16), (l, k))
            _assert_bits(pk[k + "_b"], _convert(ref, bf), (l, k + "_b"))
        _assert_bits(pk["wkv_b"], _convert(pv[p + "0.to_kv.weight"], bf), (l, "wkv_b"))
        _assert_bits(pk["wo_b"], _convert(pv[p + "0.to_out.0.weight"], bf), (l, "wo_b"))
        if fk["conv"] is not None:
            conv = _reconstruct(pv[p + fk["conv"]].reshape(2 * F, 3), 2 * F, 3, 2 * Fp, 3, -1, F)
        else:
            conv = torch.zeros(2 * Fp, 3, device=DEV)
            conv[:, 2] = 1.0
        _assert_bits(pk["conv"], conv, (l, "conv"))
        _assert_bits(pk["gin"], _reconstruct(pv[p + fk["gin"]].reshape(1, F), 1, F, 1, Fp, 0, 0).reshape(-1), (l, "gin"))
    for s, seq in enumerate(eng.seqs):
        q, C, Cp = seq.num_quantizers, eng.C[s], eng.Cp[s]
        ref = _reconstruct(pv[f"logit_weights.{s}"].reshape(q * C, d), q * C, d, q * Cp, d, Cp, C)
        _assert_bits(eng.pk_logit[s].view(-1, d), _convert(ref, eng.a16), ("logit", s))
        _assert_bits(eng.pk_logit_b[s].view(-1, d), _convert(ref, bf), ("logit_b", s))
    if eng.bias_type == "continuous":
        Hr, T = eng.Hr, eng.Hr8
        for j in (1, 2):
            w = pv[f"transformer.rel_pos_bias.net.{j}.0.weight"]
            hi = w.to(bf)
            lo = (w - hi.float()).to(bf)
            ref = torch.zeros(Hr, 3 * T, device=DEV, dtype=bf)
            ref[:, :Hr], ref[:, T:T + Hr], ref[:, 2 * T:2 * T + Hr] = hi, lo, hi
            _assert_bits(eng.pk_rp[j - 1], ref, ("rp", j))


@pytest.mark.parametrize("act16", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", [(128, 2, True), (1024, 2, True), (128, 2, False)], ids=["tiny", "d1024", "plainff"])
def test_engine_state_after_steps(lib, monkeypatch, act16, shape):
    """After optimiser steps: every packed buffer equals its reconstruction from the master weights bit for bit; the
    arena's alignment gaps are exactly 0 in p, g, m and v; every ndim >= 2 parameter lies below n_decay, the rest above."""
    import open_musiclm_b200 as O
    d, L, conv_ff = shape
    m = _engine_model(monkeypatch, act16, d, L, conv_ff)
    tr = O.HotPathTrainer(m, cross_entropy_loss_weights=CE, lr=1e-3, wd=0.01, use_cuda_graph=False)
    toks = _tokens(m)
    for _ in range(2):
        tr.train_step([toks])
    eng = tr.eng
    eng.refresh_packed(force=True)
    torch.cuda.synchronize()
    _check_packed(eng)
    used = torch.zeros(eng.n_params_arena, dtype=torch.bool, device=DEV)
    for n, p in m.named_parameters():
        o = eng.layout[n]
        used[o:o + p.numel()] = True
        assert (o + p.numel() <= eng.n_decay) if p.ndim >= 2 else (o >= eng.n_decay), n
    for buf in (eng.arena_p, eng.arena_g, eng.adam_m, eng.adam_v):
        assert not bool(buf[~used].any())


# ------------------------------------------------------------------------------------------------ trainer trajectory
def _trainer(wd, max_norm, graph, **kw):
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_coarse_transformer(**TINY).cuda()
    return O.HotPathTrainer(m, cross_entropy_loss_weights=CE, lr=1e-3, lr_warmup=5, wd=wd, max_grad_norm=max_norm,
                            grad_accum_every=2, mask_prob=0.0, use_cuda_graph=graph, **kw)


def _spy(tr):
    """Records (p, g, m, v) of the arena before each optimiser update of an eager trainer."""
    eng, snaps, orig = tr.eng, [], tr._update_body

    def body(det):
        snaps.append(tuple(x.clone() for x in (eng.arena_p, eng.arena_g, eng.adam_m, eng.adam_v)))
        orig(det)
    tr._update_body = body
    return snaps


def _batches(step):
    g = torch.Generator().manual_seed(100 + step)
    return [[torch.randint(0, 64, s, generator=g).cuda() for s in [(2, 4), (2, 11), (2, 10, 3)]] for _ in range(2)]


def _frozen_spans(tr):
    eng = tr.eng
    return [(eng.layout[n], eng.layout[n] + eng.pview[n].numel()) for n in tr.frozen]


def _check_update(lib, tr, snap, step):
    """One recorded update of the trainer against the float64 reference from its own pre-step state."""
    eng = tr.eng
    p, g, m, v = snap
    frozen = _frozen_spans(tr)
    kw = dict(t=step + 1, lr=tr.lr * OR.lr_factor(step, tr.lr_warmup), wd=tr.wd, n_decay=eng.n_decay,
              max_grad_norm=tr.max_grad_norm, frozen=frozen)
    blocks, _ = OR.sumsq_grid(eng.n_params_arena, lib.num_sms())
    S = OR.sumsq(g)
    eS = OR.sumsq_bound(g, 1.0, blocks)
    want = OR.adamw_update(p, g, m, v, **kw)[:3]
    bound = OR.adamw_bound(p, g, m, v, **kw, sumsq_value=S, sumsq_err=eS)
    for name, x, w, b in zip("pmv", (eng.arena_p, eng.adam_m, eng.adam_v), want, bound):
        err = (x.double() - w).abs()
        assert not bool((err > b).any()), (step, name, float((err / b.clamp_min(1e-300)).max()))
    if tr.max_grad_norm is not None:
        norm = float(tr.grad_norm())
        assert abs(norm - S ** 0.5) <= (eS / (2 * S) + 2 * OR.U) * S ** 0.5


@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("max_norm", [1e-4, 1e6, None], ids=["clip-all", "clip-none", "no-clip"])
def test_trainer_trajectory(lib, wd, max_norm):
    """Deterministic mode, grad_accum_every 2, warm-up 5, 12 steps: the CUDA-graph trainer (eager, capture, replays)
    equals an eager twin bit for bit at every step; every twin update is within the float64 reference's scale from its
    own pre-step state, and so is grad_norm(); the heads of the zero-weighted sequences are bit-unchanged."""
    torch.use_deterministic_algorithms(True)
    try:
        tg, te = _trainer(wd, max_norm, True), _trainer(wd, max_norm, False)
        snaps = _spy(te)
        heads0 = {n: te.eng.pview[n].clone() for n in te.frozen}
        assert te.frozen == {"logit_weights.0", "logit_weights.1"}
        for step in range(12):
            mbs = _batches(step)
            tg.train_step(mbs)
            te.train_step(mbs)
            torch.cuda.synchronize()
            for a, b in ((tg.eng.arena_p, te.eng.arena_p), (tg.eng.adam_m, te.eng.adam_m), (tg.eng.adam_v, te.eng.adam_v)):
                assert torch.equal(a.view(torch.int32), b.view(torch.int32)), step
            _check_update(lib, te, snaps[step], step)
        assert tg._graphs and all(st["graphs"] is not None for st in tg._graphs.values())
        for tr in (tg, te):
            for n, h0 in heads0.items():
                o = tr.eng.layout[n]
                assert torch.equal(tr.eng.pview[n], h0), n
                assert not bool(tr.eng.adam_m[o:o + h0.numel()].any()) and not bool(tr.eng.adam_v[o:o + h0.numel()].any())
    finally:
        torch.use_deterministic_algorithms(False)


# ------------------------------------------------------------------------------------------------ checkpoints
@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_checkpoint_loads_into_the_reference_optimizer(lib, tmp_path, wd):
    """save() after 3 steps loads into the optimizer and LinearLR the reference builds (Adam with one group at wd 0);
    one float64 step of that optimizer with the trainer's next gradient equals the trainer's next update within the
    scale; frozen heads carry no optimizer state."""
    tr = _trainer(wd, 0.5, False)
    eng = tr.eng
    for step in range(3):
        tr.train_step(_batches(step))
    paths = [str(tmp_path / f) for f in ("model.pt", "optim.pt", "sched.pt")]
    tr.save(*paths)
    names = [n for n, _ in tr.transformer.named_parameters()]
    params = [torch.nn.Parameter(tr.eng.pview[n].detach().double().cpu().clone()) for n in names]
    # built as the reference's trainer builds them, then loaded in its order (trainer.py:226-236, 371-387)
    opt = OR.reference_optimizer(params, lr=tr.lr, wd=wd)
    sched = torch.optim.lr_scheduler.LinearLR(opt, start_factor=1e-7, end_factor=1.0, total_iters=tr.lr_warmup)
    opt.load_state_dict(torch.load(paths[1]))
    sched.load_state_dict(torch.load(paths[2]))
    assert sched.last_epoch == 3
    for n, p in zip(names, params):
        assert (p in opt.state) == (n not in tr.frozen), n
    snaps = _spy(tr)
    tr.train_step(_batches(3))
    _, g, _, _ = snaps[0]
    for n, p in zip(names, params):
        o = eng.layout[n]
        p.grad = None if n in tr.frozen else g[o:o + p.numel()].view(p.shape).double().cpu()
    torch.nn.utils.clip_grad_norm_([p for p in params if p.grad is not None], 0.5)
    opt.step()
    sched.step()
    p0, g0, m0, v0 = snaps[0]
    kw = dict(t=4, lr=tr.lr * OR.lr_factor(3, tr.lr_warmup), wd=wd, n_decay=eng.n_decay, max_grad_norm=0.5,
              frozen=_frozen_spans(tr))
    blocks, _ = OR.sumsq_grid(eng.n_params_arena, lib.num_sms())
    bound = OR.adamw_bound(p0, g0, m0, v0, **kw, sumsq_value=OR.sumsq(g0), sumsq_err=OR.sumsq_bound(g0, 1.0, blocks))
    for n, p in zip(names, params):
        o = eng.layout[n]
        err = (eng.pview[n].double().cpu() - p.detach()).abs().reshape(-1)
        b = bound[0][o:o + p.numel()].cpu()
        # the reference step ran from the saved fp32 state in float64: its own distance to adamw_update is float64 rounding
        assert bool((err <= b + 1e-12 * p.detach().abs().reshape(-1)).all()), (n, float((err / b.clamp_min(1e-300)).max()))


def test_trainer_loads_a_one_group_adam_file(lib, tmp_path):
    """A wd = 0 checkpoint as the reference writes it (Adam, one group, no state for heads without gradient)."""
    tr = _trainer(0.0, 0.5, False)
    names = [n for n, _ in tr.transformer.named_parameters()]
    params = [torch.nn.Parameter(tr.eng.pview[n].detach().cpu().clone()) for n in names]
    opt = torch.optim.Adam(params, lr=tr.lr, betas=(0.9, 0.99), eps=1e-8)
    sched = torch.optim.lr_scheduler.LinearLR(opt, start_factor=1e-7, end_factor=1.0, total_iters=tr.lr_warmup)
    gen = torch.Generator().manual_seed(5)
    for n, p in zip(names, params):
        p.grad = None if n in tr.frozen else torch.randn(p.shape, generator=gen)
    opt.step()
    sched.step()
    paths = [str(tmp_path / f) for f in ("model.pt", "optim.pt", "sched.pt")]
    torch.save({k: v.detach().clone() for k, v in tr.transformer.state_dict().items()}, paths[0])
    torch.save(opt.state_dict(), paths[1])
    torch.save(sched.state_dict(), paths[2])
    assert tr.load(*paths) == 1
    eng = tr.eng
    for n, p in zip(names, params):
        o = eng.layout[n]
        st = opt.state.get(p)
        m = eng.adam_m[o:o + p.numel()].view(p.shape).cpu()
        v = eng.adam_v[o:o + p.numel()].view(p.shape).cpu()
        if st is None:
            assert not bool(m.any()) and not bool(v.any()), n
        else:
            assert torch.equal(m, st["exp_avg"]) and torch.equal(v, st["exp_avg_sq"]), n
