"""Token log-probabilities of KV-cache generation on the H100: the sampler's two outputs against the float64 statements
of tests/logprob_reference.py under their derived bounds (tokens bit-identical to the sampler without them), the per-row
prefix kernel against ce_ref, and generate / GenerationSession end to end: tokens and Engine.seed unchanged by
return_logprobs, graph replay equal to eager, seeded rows equal to the row alone, session rows equal to generate, and
the teacher-forced idiom against the decode's values."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from logprob_reference import model_logprob, sample_logprob  # noqa: E402
from norm_loss_reference import ce_labels, ce_ref  # noqa: E402
from test_generate_ragged_gpu import _model, _prompts  # noqa: E402
from test_sampling_nucleus_cpu import edge_logits  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as L
    L.device_check()
    return L


def _close(got, want, bound):
    """got (fp32) within bound of want (float64); NaN where want is NaN."""
    got, want = got.double().cpu(), want.double().cpu()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    err = (got - want).abs()[~nan]
    assert bool((err <= bound[~nan]).all()), float((err - bound[~nan]).max())


def _sample(lib, x, k, T, allow, top_p, noise, logprob, rows=None):
    B, C = x.shape
    tokens, lp, slp = lib.logprob_buffers(B, 4, DEV)
    if not logprob:
        lp = slp = None
    next_row = torch.zeros(B, device=DEV, dtype=torch.int32)
    counters = torch.tensor([2, 0], device=DEV, dtype=torch.int32)
    uni = seed = seeds = None
    if noise == "uniform":
        uni = torch.rand(3, B, C, generator=torch.Generator().manual_seed(C)).clamp_min(1e-6).to(DEV)
    elif noise == "engine":
        seed = torch.tensor([1234], device=DEV, dtype=torch.int64)
    else:
        seeds = torch.arange(B, device=DEV, dtype=torch.int64) * 7919 + 5
    kw = dict(rows) if rows else dict(top_p=top_p)
    lib.sample(x, C, k, T, allow, uni, seed, tokens, next_row, 3, counters, None, B, seeds=seeds, logprobs=lp, sample_logprobs=slp, **kw)
    torch.cuda.synchronize()
    return tokens[:, 2], (lp[:, 2] if logprob else None), (slp[:, 2] if logprob else None), next_row, counters


@pytest.mark.parametrize("noise", ["uniform", "engine", "seeds"])
@pytest.mark.parametrize("C", [2, 65, 1025, 16384])
def test_sampler_logprobs_against_float64(lib, C, noise):
    g = torch.Generator().manual_seed(C)
    x = edge_logits(24, C, g).to(DEV)
    for k in sorted({1, max(1, C // 10), C}):
        for top_p in (None, 0.5, 0.9):
            for T in (0.4, 1.0, 2.0):
                for allow in (False, True):
                    tok0, _, _, nr0, c0 = _sample(lib, x, k, T, allow, top_p, noise, False)
                    tok, lp, slp, nr, c = _sample(lib, x, k, T, allow, top_p, noise, True)
                    assert torch.equal(tok, tok0) and torch.equal(nr, nr0) and torch.equal(c, c0)
                    ok = (tok >= 0) & (tok < C)     # a row with no finite candidate score has no token
                    okc = ok.cpu()
                    t = tok.clamp(0, C - 1)
                    v, bnd = model_logprob(x, t)
                    _close(lp[ok], v[okc], bnd[okc])
                    v, bnd = sample_logprob(x, t, k, T, allow, top_p)
                    _close(slp[ok], v[okc], bnd[okc])


@pytest.mark.parametrize("C", [65, 1025, 16384])
def test_sampler_logprobs_per_row_arguments(lib, C):
    """Per-row k, T and top_p: each row's values equal the single-value call with that row's scalars, bit for bit."""
    g = torch.Generator().manual_seed(C + 1)
    B = 12
    x = edge_logits(B, C, g).to(DEV)
    ks = [max(1, (b * C) // B) for b in range(B)]
    Ts = [0.4 + 0.15 * b for b in range(B)]
    ps = [(None, 0.5, 0.9)[b % 3] for b in range(B)]
    rows = dict(top_k_rows=torch.tensor(ks, device=DEV, dtype=torch.int32), temperature_rows=torch.tensor(Ts, device=DEV),
                top_p_rows=torch.tensor([1.0 if p is None else p for p in ps], device=DEV))
    tok, lp, slp, _, _ = _sample(lib, x, 1, 1.0, False, None, "seeds", True, rows=rows)
    for b in range(B):
        t1, lp1, slp1, _, _ = _sample(lib, x, ks[b], Ts[b], False, ps[b], "seeds", True)
        assert int(tok[b]) == int(t1[b])
        for u, v in ((lp[b], lp1[b]), (slp[b], slp1[b])):
            assert float(u) == float(v) or (math.isnan(float(u)) and math.isnan(float(v)))


@pytest.mark.parametrize("C", [2, 65, 1280, 1281, 4099, 65536])
def test_token_logprob_against_ce_ref(lib, C):
    """omlm_token_logprob through the strided label view (3 heads' interleaved labels, 5 rows per sequence) equals the
    negated ce_ref row loss within its bound, and 0 for labels outside [0, C)."""
    g = torch.Generator().manual_seed(C)
    B, cnt, q = 6, 5, 3
    ld = (C + 3) // 4 * 4
    x = torch.zeros(B * cnt, ld)
    x[:, :C] = torch.randn(B * cnt, C, generator=g) * 3
    lab = torch.randint(0, C, (B, cnt * q + q), generator=g, dtype=torch.int32)
    lab[0, 1], lab[1, 4] = -100, C                          # ignored, out of range
    qi = 1
    xd, labd = x.to(DEV), lab.to(DEV)
    out = torch.full((B * cnt,), 7.0, device=DEV)
    lib.token_logprob(xd, labd.view(-1)[qi:], C, out, label_stride=q, rows_per_batch=cnt, batch_stride=cnt * q + q)
    torch.cuda.synchronize()
    l = ce_labels(lab.view(-1)[qi:], B * cnt, q, cnt, cnt * q + q)
    valid = (l >= 0) & (l < C)
    ref = ce_ref(x, torch.where(valid, l, torch.full_like(l, -100)), C, C, grad_scale=0.0)
    got = out.cpu().double()
    assert bool((got[~valid] == 0).all())
    assert bool(((got + ref["loss"]).abs()[valid] <= ref["loss_bound"][valid]).all())


@pytest.mark.parametrize("C", [65, 1025, 1281])
def test_token_logprob_flat_labels_against_ce_ref(lib, C):
    """omlm_token_logprob with one flat label per row, as a session's packed prefill scores its prefixes (rows of a
    logits buffer wider than C, -100 on the next-token rows): the negated ce_ref row loss within its bound, 0 for
    labels outside [0, C), and nothing written past the rows."""
    g = torch.Generator().manual_seed(C + 1)
    rows, ld = 37, (C + 63) // 64 * 64
    x = torch.full((rows, ld), float("nan"))
    x[:, :C] = torch.randn(rows, C, generator=g) * 3
    lab = torch.randint(0, C, (rows,), generator=g, dtype=torch.int32)
    lab[:3], lab[10] = -100, C
    out = torch.full((rows + 2,), 7.0, device=DEV)
    lib.token_logprob(x.to(DEV), lab.to(DEV), C, out, rows=rows)
    torch.cuda.synchronize()
    l = lab.long()
    valid = (l >= 0) & (l < C)
    ref = ce_ref(x, torch.where(valid, l, torch.full_like(l, -100)), C, C, grad_scale=0.0)
    got = out.cpu().double()
    assert bool((got[rows:] == 7.0).all())
    assert bool((got[:rows][~valid] == 0).all())
    assert bool(((got[:rows] + ref["loss"]).abs()[valid] <= ref["loss_bound"][valid]).all())


# ------------------------------------------------------------------------------------------------ generate / session
def _gen(w, cond, pred, **kw):
    return w.generate(conditioning_token_ids=cond, pred_token_ids=pred, **kw)


@pytest.mark.parametrize("stage,B,seeded", [("coarse", 3, False), ("coarse", 20, False), ("semantic", 3, True),
                                            ("coarse", 17, True)])
def test_tokens_and_seed_do_not_change(stage, B, seeded):
    m, w, _, _ = _model(stage)
    g = torch.Generator().manual_seed(B)
    cond, pred, q = _prompts(B, stage, 3, 64, g)
    kw = dict(max_time_steps=9, temperature=0.8, filter_thres=0.5)
    if seeded:
        kw["seeds"] = list(range(100, 100 + B))
    extras = [dict(), dict(top_p=0.9), dict(pred_lengths=[1 + b % 3 for b in range(B)]),
              dict(temperature=[0.5 + 0.1 * b for b in range(B)]),
              # the longest prefix belongs to a row that samples nothing (max_time_steps equal to its length)
              dict(pred_lengths=[3] + [1 + b % 2 for b in range(1, B)], max_time_steps=[3] + [5] * (B - 1))]
    if not seeded:
        n_new = 6 * q
        extras.append(dict(uniform_noise=torch.rand(n_new, B, 65, generator=g).clamp_min(1e-6)))
    for extra in extras:
        args = {**kw, **extra}
        if "uniform_noise" in extra:
            args["max_time_steps"] = 9
        e0 = m.engine.seed.clone()          # a device counter, advanced in place by unseeded calls
        base = _gen(w, cond, pred, **args)
        e1 = m.engine.seed.clone()
        m.engine.seed.copy_(e0)             # the same Engine.seed stream for both calls
        tok, lp, slp = _gen(w, cond, pred, return_logprobs=True, **args)
        assert torch.equal(m.engine.seed, e1) and torch.equal(e1, e0 + (0 if seeded else 1))
        assert torch.equal(tok, base)
        assert lp.shape == slp.shape == tok.shape and lp.dtype == torch.float32
        gone = tok == -1
        assert bool((lp[gone] == 0).all()) and bool((slp[gone] == 0).all())
        assert bool((lp[~gone] <= 0).all())


def test_graph_equals_trace_and_decode_values():
    """Replay and eager give bit-identical arrays; the sampled tokens' values equal the float64 statements of the
    traced rows within the derived bounds; prefix sample_logprobs are 0."""
    m, w, _, _ = _model("coarse")
    g = torch.Generator().manual_seed(5)
    B = 4
    cond, pred, q = _prompts(B, "coarse", 2, 64, g)
    kw = dict(max_time_steps=7, temperature=0.7, filter_thres=0.6, top_p=0.9, seeds=[11, 12, 13, 14], allow_eos_in_output=True,
              include_eos_in_output=True)
    a = _gen(w, cond, pred, return_logprobs=True, **kw)
    trace = []
    b = _gen(w, cond, pred, return_logprobs=True, trace_logits=trace, **kw)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    tok, lp, slp = (t.reshape(B, -1) for t in a)
    C = 65
    k = max(int((1 - 0.6) * C), 1)
    p0 = 2 * q
    assert bool((slp[:, :p0] == 0).all())
    for s, row in enumerate(trace):
        p = p0 + s
        live = tok[:, p] >= 0
        if not bool(live.any()):
            continue
        allow = (p % q) == q - 1
        v, bnd = model_logprob(row, tok[:, p].clamp_min(0))
        _close(lp[live, p], v[live.cpu()], bnd[live.cpu()])
        v, bnd = sample_logprob(row, tok[:, p].clamp_min(0), k, 0.7, allow, 0.9)
        _close(slp[live, p], v[live.cpu()], bnd[live.cpu()])


def test_teacher_forced_idiom_matches_the_decode():
    """Scoring the generated sequence teacher-forced returns the same tokens and sample_logprobs 0; its logprobs are
    the forward rows' log-softmax within ce_ref's bound, and differ from the decode's by at most 2 max |dl| (dl = decode
    row minus forward row of the same position) plus both rounding bounds."""
    from norm_loss_reference import ce_ref
    m, w, _, _ = _model("coarse")
    g = torch.Generator().manual_seed(9)
    B, C = 3, 65
    cond, pred, q = _prompts(B, "coarse", 1, 64, g)
    trace = []
    tok, lp, _ = _gen(w, cond, pred, max_time_steps=6, seeds=[1, 2, 3], return_logprobs=True, trace_logits=trace)
    tok2, lp2, slp2 = _gen(w, cond, tok, max_time_steps=6, return_logprobs=True)
    assert torch.equal(tok2, tok) and bool((slp2 == 0).all())
    flat = tok.reshape(B, -1)
    n = flat.shape[1]
    ids = [torch.cat([c.reshape(B, -1), torch.full((B, 1), e, device=DEV)], 1) for c, e in zip(cond, w.eos_ids)]
    rows = m(all_token_ids=ids + [flat], return_only_final_seq_logits=True)[-1][:, :n, :C].float()
    live = (flat >= 0).cpu()
    ce = ce_ref(rows.reshape(-1, C).cpu(), flat.clamp_min(0).reshape(-1).cpu(), C, C, grad_scale=0.0)
    lp2f, lpf = lp2.reshape(B, -1).cpu().double(), lp.reshape(B, -1).cpu().double()
    cb = ce["loss_bound"].view(B, n)
    assert bool((((lp2f + ce["loss"].view(B, n)).abs() <= cb) | ~live).all())
    for s_, row in enumerate(trace):
        p = q + s_
        d = (row.cpu().double() - rows[:, p].cpu().double()).abs().max(1).values
        _, bnd = model_logprob(row, flat[:, p].clamp_min(0))
        assert bool((((lpf[:, p] - lp2f[:, p]).abs() <= 2 * d + bnd + cb[:, p]) | ~live[:, p]).all())


@pytest.mark.parametrize("stage,B,dim,heads", [("coarse", 17, 128, 2), ("semantic", 40, 128, 2), ("coarse", 256, 128, 2),
                                               ("coarse", 20, 1024, 8), ("coarse", 20, 1024, 16)])
def test_seeded_rows_equal_the_row_alone(stage, B, dim, heads):
    m, w, _, _ = _model(stage, dim=dim, heads=heads)
    g = torch.Generator().manual_seed(B)
    cond, pred, q = _prompts(B, stage, 3, 64, g)
    seeds = [1000 + 3 * b for b in range(B)]
    lengths = [b % 4 for b in range(B)]
    kw = dict(max_time_steps=6, temperature=0.9, filter_thres=0.5, top_p=0.9, return_logprobs=True)
    tok, lp, slp = _gen(w, cond, pred, seeds=seeds, pred_lengths=lengths, **kw)
    for b in sorted({0, 1, B // 2, B - 1}):
        n = lengths[b]
        t1, l1, s1 = w.generate(conditioning_token_ids=[t[b:b + 1] for t in cond], pred_token_ids=pred[b:b + 1, :n] if n else None,
                                seeds=[seeds[b]], **kw)
        W = t1.shape[1]
        assert torch.equal(tok[b, :W], t1[0]) and torch.equal(lp[b, :W], l1[0]) and torch.equal(slp[b, :W], s1[0])


@pytest.mark.parametrize("stage", ["coarse", "semantic"])
def test_session_rows_equal_generate(stage):
    import open_musiclm_b200 as O
    m, w, _, _ = _model(stage)
    g = torch.Generator().manual_seed(3)
    q = 3 if stage == "coarse" else 1
    sess = O.GenerationSession(w, slots=4, max_positions=64, return_logprobs=True, max_queue=8)
    reqs = []
    for i in range(6):
        cond, pred, _ = _prompts(1, stage, 1 + i % 3, 64, g)
        reqs.append(dict(conditioning_token_ids=cond, pred_token_ids=pred if q > 1 else pred.view(1, -1, 1), seed=50 + i, max_time_steps=4 + i % 3, temperature=0.8, top_p=(None, 0.9)[i % 2]))
    handles = [sess.add(**r) for r in reqs]
    done = {}
    while not sess.idle:
        sess.step()
        done.update(sess.finished())
    done.update(sess.finished())
    for h, r in zip(handles, reqs):
        r = dict(r)
        seed = r.pop("seed")
        want = w.generate(seeds=[seed], return_logprobs=True, **r)
        for x, y in zip(done[h], want):
            assert torch.equal(x, y[0])


# ------------------------------------------------------------------------------------------------ the reference
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("case", ["semantic", "coarse", "fine_eos"])
def test_reference_fixture_end_to_end(case):
    """generate on the reference's weights, prompt and uniforms (tests/golden/logprobs_*.pt): the reference's tokens;
    each value within 2 max_c |dl_c| (divided by T for sample_logprobs, compared where both rows give the same candidate
    set) plus the rounding bound, dl = the engine's row minus the reference's row of that position."""
    import open_musiclm_b200 as O
    from logprob_reference import candidate_set
    from norm_loss_reference import ce_ref
    fx = torch.load(os.path.join(GOLD, f"logprobs_{case}.pt"), weights_only=False)
    fn = {"semantic": O.create_semantic_transformer, "coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}[fx["stage"]]
    m = fn(**fx["kwargs"])
    m.load_state_dict(torch.load(os.path.join(GOLD, fx["weights"]), weights_only=False)["state_dict"], strict=True)
    m = m.cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    cond = [t.cuda() for t in fx["cond"]]
    prefix = None if fx["prefix"] is None else fx["prefix"].cuda()
    trace = []
    tok, lp, slp = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=fx["max_time_steps"],
                              filter_thres=fx["filter_thres"], temperature=fx["temperature"], uniform_noise=fx["uniforms"],
                              include_eos_in_output=fx["include_eos_in_output"], allow_eos_in_output=fx["allow_eos_in_output"],
                              return_logprobs=True, trace_logits=trace)
    assert torch.equal(tok.cpu(), fx["out"])
    B, q = tok.shape[0], tok.shape[2]
    tok, lp, slp = (t.reshape(B, -1).cpu() for t in (tok, lp, slp))
    C = fx["rows"].shape[-1]
    k, T = max(int((1 - fx["filter_thres"]) * C), 1), fx["temperature"]
    n_pre = 0 if prefix is None else prefix[0].numel()
    for s, row in enumerate(trace):
        p = n_pre + s
        live = tok[:, p] >= 0
        ref_row = fx["rows"][s]
        d = (row.cpu().double() - ref_row.double()).abs().max(1).values
        t = fx["sampled"][s]
        v, bnd = model_logprob(row, t)
        assert bool((((lp[:, p].double() - fx["logprobs"][s]).abs() <= 2 * d + bnd) | ~live).all())
        allow = bool(fx["allow_eos_in_output"]) and p % q == q - 1
        same = (candidate_set(row.cpu(), k, T, allow, None) == candidate_set(ref_row, k, T, allow, None)).all(1)
        v, bnd = sample_logprob(row, t, k, T, allow, None)
        assert bool((((slp[:, p].double() - fx["sample_logprobs"][s]).abs() <= 2 * d / T + bnd) | ~live | ~same).all())
        assert int((live & same).sum()) > 0 or not bool(live.any())
    if n_pre:
        ids = [torch.cat([c.reshape(B, -1), torch.full((B, 1), e, device=DEV)], 1) for c, e in zip(cond, w.eos_ids)]
        rows = m(all_token_ids=ids + [prefix.reshape(B, -1)], return_only_final_seq_logits=True)[-1][:, :n_pre, :C].float().cpu()
        d = (rows.double() - fx["prefix_rows"].double()).abs().amax((1, 2))
        ce = ce_ref(rows.reshape(-1, C), fx["prefix"].reshape(-1), C, C, grad_scale=0.0)
        bound = 2 * d[:, None] + ce["loss_bound"].view(B, n_pre)
        assert bool(((lp[:, :n_pre].double() - fx["prefix_logprobs"]).abs() <= bound).all())
        assert bool((slp[:, :n_pre] == 0).all())


def test_absolute_positions_tokens_do_not_change():
    m, w, _, _ = _model("coarse", use_absolute_position_embeddings=True, max_absolute_position_embeddings=64)
    g = torch.Generator().manual_seed(4)
    cond, pred, q = _prompts(5, "coarse", 2, 64, g)
    for kw in (dict(seeds=[1, 2, 3, 4, 5]), dict(seeds=[1, 2, 3, 4, 5], pred_lengths=[0, 1, 2, 1, 0])):
        base = _gen(w, cond, pred, max_time_steps=6, **kw)
        tok, lp, slp = _gen(w, cond, pred, max_time_steps=6, return_logprobs=True, **kw)
        assert torch.equal(tok, base) and bool((lp[tok == -1] == 0).all())
