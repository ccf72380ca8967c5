"""Codebooks of any size, and of different sizes in different sequences, on the H100 path.

  a. the cross-entropy entry points for C > 1280 (the streaming kernel) against float64: losses, gradients, the zero
     padding tail, ignored rows, the strided label view, the deterministic variant and CUDA-graph replay;
  b. the fused training step (HotPathTrainer) against the reference's fixtures tests/golden/cbsize_*.pt and against the
     CPU oracle at model scale (d = 1024, a 4096-entry semantic codebook), in both modes;
  c. generation with a 1500 / 2048-entry predicted codebook: the reference's tokens, seeded rows that do not depend on
     the batch, and the three-stage MusicLM chain against the oracle-backed chain;
  d. the token store's 16-bit arrays with ids up to 16383."""
import contextlib
import os
import random
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(__file__)
sys.path.insert(0, HERE)
import codebook_fixtures as CF  # noqa: E402
import norm_loss_reference as NL  # noqa: E402
GOLD = os.path.join(HERE, "golden")
TRAIN = [os.path.join(GOLD, f"cbsize_{n}.pt") for n in ("semantic", "coarse")]
GEN = [os.path.join(GOLD, f"cbsize_gen_{n}.pt") for n in ("semantic", "semantic_b20")]


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@contextlib.contextmanager
def switch(on):
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def _round_up(x, m):
    return (x + m - 1) // m * m


# ------------------------------------------------------------------------------------------------ a. the kernel
def _ce_case(C, rows, seed):
    """logits [rows, Cp] fp32 with NaN in the padding columns (they must never be read), labels with 0 and C - 1,
    every fifth row ignored, one row with a +1e4 logit and one row of equal logits."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    Cp = _round_up(C, 64)
    logits = torch.randn(rows, Cp, device=DEV, generator=g) * 6
    logits[:, C:] = float("nan")
    labels = torch.randint(0, C, (rows,), device=DEV, generator=g, dtype=torch.int32)
    labels[0] = 0
    if rows > 1:
        labels[1] = C - 1
    if rows > 5:
        labels[4::5] = -100
    if rows > 2:
        logits[2, 17] = 1e4                     # one dominant class (label elsewhere: a loss of ~1e4)
    if rows > 3:
        logits[3, :C] = 0.75                    # all classes equal: loss log(C), gradient 1/C
    return logits, labels, Cp


def _ce_reference(logits, labels, C, gs, chunk=512):
    """float64 reference in chunks of rows (bounded memory): yields (first row, dlogits [rows, C], kept-row mask, loss sum
    over the kept rows)."""
    for r0 in range(0, logits.shape[0], chunk):
        x = logits[r0:r0 + chunk, :C].double()
        lb = labels[r0:r0 + chunk].long()
        keep = lb != -100
        lse = torch.logsumexp(x, 1)
        safe = lb.clamp_min(0)
        loss = lse - x.gather(1, safe[:, None])[:, 0]
        p = torch.exp(x - lse[:, None])
        p.scatter_add_(1, safe[:, None], -torch.ones_like(p[:, :1]))
        p *= gs
        p[~keep] = 0
        yield r0, p, keep, float(loss[keep].sum())


@pytest.mark.parametrize("rows", [1, 7, 333, 8000])
@pytest.mark.parametrize("C", [1281, 1345, 2049, 4097, 16384, 65536])
def test_cross_entropy_any_class_count_vs_float64(C, rows):
    from open_musiclm_b200 import lib
    logits, labels, Cp = _ce_case(C, rows, seed=C + rows)
    gs, ls = 0.37, 0.5
    acc = torch.zeros(2, device=DEV)
    dl = torch.full((rows, Cp), 7.0, device=DEV, dtype=torch.bfloat16)
    lib.cross_entropy(logits, labels, C, acc, grad_scale=gs, dlogits=dl, loss_scale=ls)
    total = 0.0
    kept = 0
    for r0, p, keep, loss in _ce_reference(logits, labels, C, gs):
        rows_c = p.shape[0]
        # every element within the bound both cross-entropy kernels are held to (tests/norm_loss_reference.py)
        ref = NL.ce_ref(logits[r0:r0 + rows_c], labels[r0:r0 + rows_c].long(), C, Cp, grad_scale=gs)
        NL.check(dl[r0:r0 + rows_c], ref["dlogits"], ref["dlogits_bound"], f"C={C} dlogits rows {r0}+")
        total += loss
        kept += int(keep.sum())
        if not bool(keep.all()):
            assert float(dl[r0:r0 + rows_c][~keep].abs().max()) == 0.0        # ignored rows: exact zeros
    ref = total * ls
    assert abs(float(acc[0]) - ref) <= 1e-5 * abs(ref), (float(acc[0]), ref)
    assert float(acc[1]) == kept
    if Cp > C:
        assert float(dl[:, C:].abs().max()) == 0.0
    if rows > 3:                                  # equal logits: loss log C, softmax 1/C
        one = torch.zeros(2, device=DEV)
        lib.cross_entropy(logits[3:4], labels[3:4], C, one)
        assert abs(float(one[0]) - np.log(C)) <= 1e-5 * np.log(C)


def test_cross_entropy_strided_label_view_large_C():
    """The trainer's label view: rows ordered (sequence b, step t) of one logit-head group, labels at plane[b, off + qi + q t]."""
    from open_musiclm_b200 import lib
    torch.manual_seed(3)
    C = 2049
    Cp = _round_up(C, 64)
    B, cnt, q, qi, off = 9, 37, 3, 1, 5
    plane = torch.randint(0, C, (B, off + q * cnt + 2), device=DEV, dtype=torch.int32)
    plane[2, off + qi + q * 4] = -100
    lg = torch.randn(B * cnt, Cp, device=DEV) * 4
    acc = torch.zeros(2, device=DEV)
    dl = torch.empty(B * cnt, Cp, device=DEV, dtype=torch.bfloat16)
    lib.cross_entropy(lg, plane[0, off + qi:], C, acc, grad_scale=0.5, dlogits=dl, rows=B * cnt, label_stride=q, rows_per_batch=cnt,
                      batch_stride=plane.stride(0), loss_scale=0.25)
    lab = plane[:, off + qi::q][:, :cnt].reshape(-1).long()
    x = lg[:, :C].double().requires_grad_(True)
    ref = 0.25 * F.cross_entropy(x, lab, ignore_index=-100, reduction="sum")
    r = float(ref.detach())
    assert abs(float(acc[0]) - r) <= 1e-5 * r and float(acc[1]) == B * cnt - 1
    (ref * 2.0).backward()                       # d(0.5 * sum) / dx = 2 * d(0.25 * sum) / dx
    assert rel(dl[:, :C], x.grad) <= 4e-3 and float(dl[:, C:].abs().max()) == 0.0
    assert float(dl[2 * cnt + 4].abs().max()) == 0.0


@pytest.mark.parametrize("C", [1281, 4097, 16385])
def test_cross_entropy_det_and_graph_replay(C):
    """omlm_cross_entropy_det: bit-identical on repeat, equal to the default entry point up to fp32 summation order,
    the same dlogits bit for bit; a CUDA-graph replay of either call equals the eager call."""
    from open_musiclm_b200 import lib
    rows = 5000
    logits, labels, Cp = _ce_case(C, rows, seed=11)
    part = torch.empty(2 * ((rows + 7) // 8), device=DEV)

    def run(det, acc, dl):
        acc.zero_()
        lib.cross_entropy(logits, labels, C, acc, grad_scale=0.1, dlogits=dl, loss_scale=0.25, part=part if det else None)

    outs = []
    for det in (True, True, False):
        acc, dl = torch.zeros(2, device=DEV), torch.empty(rows, Cp, device=DEV, dtype=torch.bfloat16)
        run(det, acc, dl)
        outs.append((acc, dl))
    (a0, d0), (a1, d1), (a2, d2) = outs
    assert torch.equal(a0, a1) and torch.equal(d0, d1)
    assert torch.equal(d0, d2) and float(a0[1]) == float(a2[1])
    assert abs(float(a0[0]) - float(a2[0])) <= 1e-6 * abs(float(a2[0]))
    for det, (acc_e, dl_e) in ((True, outs[0]), (False, outs[2])):
        acc, dl = torch.zeros(2, device=DEV), torch.empty(rows, Cp, device=DEV, dtype=torch.bfloat16)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            run(det, acc, dl)                                  # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            run(det, acc, dl)
        dl.fill_(7.0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(dl, dl_e)
        if det:
            assert torch.equal(acc, acc_e)
        else:
            assert float(acc[1]) == float(acc_e[1]) and abs(float(acc[0]) - float(acc_e[0])) <= 1e-6 * abs(float(acc_e[0]))


def test_cross_entropy_layout_checks():
    """The streaming kernel's 128-bit loads and 16-byte stores need aligned rows: misaligned layouts are argument errors."""
    from open_musiclm_b200 import lib
    C, rows = 2049, 8
    logits = torch.randn(rows, 2112, device=DEV)
    labels = torch.zeros(rows, device=DEV, dtype=torch.int32)
    acc = torch.zeros(2, device=DEV)
    with pytest.raises(lib.OmlmError):
        lib.cross_entropy(torch.randn(rows, 2050, device=DEV), labels, C, acc)                    # ld % 4 != 0
    with pytest.raises(lib.OmlmError):
        lib.cross_entropy(logits[:, 1:], labels, C, acc)                                           # misaligned rows
    with pytest.raises(lib.OmlmError):
        lib.cross_entropy(logits, labels, C, acc, dlogits=torch.empty(rows, 2050, device=DEV, dtype=torch.bfloat16)[:, :2049])
    lib.cross_entropy(logits, labels, C, acc, dlogits=torch.empty(rows, 2112, device=DEV, dtype=torch.bfloat16))
    torch.cuda.synchronize()
    assert float(acc[1]) == rows


# ------------------------------------------------------------------------------------------------ b. fused training step
def _fixture_oracle(fx):
    """The fixture's model on the GPU, its CPU weights, and the oracle's fp32 loss, logits and every gradient on them."""
    from oracle import restatement as R
    from test_codebooks_cpu import cfg_of
    m = CF.model_of(fx)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    names = [k for k, _ in m.named_parameters()]
    sd_g = {k: (v.clone().requires_grad_(True) if k in names else v) for k, v in sd.items()}
    loss, logits, *_ = R.loss_and_logits(cfg_of(fx, ce_weights=fx["ce_weights"]), sd_g, [t.numpy() for t in fx["tokens"]])
    loss.backward()
    grads = {k: (sd_g[k].grad if sd_g[k].grad is not None else torch.zeros_like(sd[k])) for k in names}
    return m.cuda().eval(), float(loss.detach()), [l.detach() for l in logits], grads


def _vs_reference_samples(got, fx, tag):
    """Every gradient against the reference's recorded entries and norm (the rel-L2 bounds of tests/test_parity_gpu.py;
    rel-pos MLP 1e-1; the analytically zero rel_pos_bias.net.3.bias is bounded in check_grads against the oracle)."""
    bad = []
    for k, s in fx["grads"].items():
        if s is None or s["norm"] < 1e-6 or k.endswith("rel_pos_bias.net.3.bias"):
            continue
        tol = 1e-1 if "rel_pos_bias" in k else 2e-2
        r, n = CF.rel_to(got[k], s), CF.norm_rel(got[k], s)
        if not (r <= tol and n <= tol):
            bad.append((k, r, n))
    assert not bad, (tag, bad)


@pytest.mark.parametrize("path", TRAIN, ids=[os.path.basename(p) for p in TRAIN])
def test_codebook_fixture_api_and_fused_trainer_vs_reference(path):
    """The reference-API forward / backward and HotPathTrainer's fused step (token plan, per-sequence embedding rows and
    eos ids, head packing [q, Cp, d], CE over C = 1501 / Cp = 1536, head wgrad with row_split = Cp) against the
    reference's loss and recorded logit / gradient entries, and against the oracle's full logits and gradients."""
    import open_musiclm_b200 as O
    from test_parity_gpu import check_grads
    fx = torch.load(path, weights_only=False)
    m, loss_o, logits_o, grads_o = _fixture_oracle(fx)
    assert abs(loss_o - float(fx["loss"])) <= 1e-5 * float(fx["loss"])
    logits = m(all_token_ids=[t.cuda() for t in fx["ids"]], self_attn_mask=fx["key_mask"].cuda())
    for a, b, s in zip(logits, logits_o, fx["logits"]):
        assert a.shape == b.shape and rel(a.detach(), b) <= 1e-2 and CF.rel_to(a, s) <= 1e-2
    total, running = 0, 0.0
    for lg, lb, w in zip(logits, fx["labels"], fx["ce_weights"]):
        if w > 0:
            running = running + F.cross_entropy(lg.permute(0, 2, 1), lb.cuda()) * lb.numel() * w
            total += lb.numel()
    loss = running / total
    assert abs(float(loss.detach()) - float(fx["loss"])) / float(fx["loss"]) <= 1e-2
    loss.backward()
    got = {k: p.grad for k, p in m.named_parameters()}
    check_grads(got, grads_o, "api")
    _vs_reference_samples(got, fx, "api")
    m2 = CF.model_of(fx).cuda().eval()
    eng = m2.engine
    assert eng.C == [cb + 1 for cb in fx["codebooks"]] and eng.Cp == [_round_up(cb + 1, 64) for cb in fx["codebooks"]]
    tr = O.HotPathTrainer(m2, cross_entropy_loss_weights=fx["ce_weights"], lr=3e-4, lr_warmup=10, wd=1e-2)
    toks = [t.cuda() for t in fx["tokens"]]
    for det in (False, True):
        with switch(det):
            assert abs(float(tr.eval_loss(toks)) - float(fx["loss"])) / float(fx["loss"]) <= 1e-2
            eng.arena_g.zero_()
            tr._micro_batch(toks, False, 0, True, det=det)
            got = {k: eng.gview[k] for k, _ in m2.named_parameters()}
            check_grads(got, grads_o, f"fused det={det}")
            _vs_reference_samples(got, fx, f"fused det={det}")
            eng.arena_g.zero_()
    eng.check_errors()


def test_codebook_fixture_optimizer_steps():
    import open_musiclm_b200 as O
    from open_musiclm_b200 import lib
    fx = torch.load(TRAIN[0], weights_only=False)
    m = CF.model_of(fx)
    p0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m = m.cuda().eval()
    tr = O.HotPathTrainer(m, cross_entropy_loss_weights=fx["ce_weights"], lr=3e-4, lr_warmup=10, wd=1e-2, max_grad_norm=0.5)
    toks = [t.cuda() for t in fx["tokens"]]
    eng = tr.eng
    for gold in fx["opt_steps"]:
        loss = tr._micro_batch(toks, False, 0, True)
        assert abs(float(loss) - float(gold["loss"])) / float(gold["loss"]) <= 1e-2
        tr._set_hyper()
        eng.sumsq.zero_()
        lib.grad_sumsq(eng.arena_g, eng.sumsq)
        assert abs(float(tr.grad_norm()) - float(gold["grad_norm"])) / float(gold["grad_norm"]) <= 2e-2
        lib.adamw_step(eng.arena_p, eng.arena_g, eng.adam_m, eng.adam_v, eng.n_decay, tr.hyper, eng.sumsq)
        eng.arena_g.zero_(); eng.refresh_packed(force=True); tr.steps += 1
        if gold["params"] is not None:
            num = den = 0.0
            for k, s in gold["params"].items():
                if fx["grads"][k] is not None and fx["grads"][k]["norm"] < 1e-6:
                    continue    # gradient is rounding noise (softmax-invariant bias): Adam turns its sign into +-lr
                d_ref = (s["val"] - CF.at(p0[k], s)).double(); d_got = (CF.at(eng.pview[k], s) - CF.at(p0[k], s)).double()
                num += float((d_ref * d_got).sum()); den += float(d_ref.norm() ** 2)
                assert CF.rel_to(eng.pview[k], s) <= 1e-3, k
            assert num / den > 0.97


def _semantic_4096(seed=0):
    import open_musiclm_b200 as O
    torch.manual_seed(seed)
    return O.create_semantic_transformer(dim=1024, depth=2, heads=8, clap_codebook_size=1024, semantic_codebook_size=4096,
                                         num_clap_quantizers=12, attn_dropout=0.0, ff_dropout=0.1)


def _semantic_4096_cfg(ce_weights=(0.0, 1.0)):
    from oracle import restatement as R
    return R.Cfg(seqs=[R.SeqInfo(1024, 12), R.SeqInfo(4096, 1)], dim=1024, depth=2, heads=8, ce_weights=list(ce_weights))


def _semantic_4096_tokens(B, seed=1234):
    g = torch.Generator().manual_seed(seed)
    sem = torch.randint(0, 4096, (B, 241), generator=g)
    sem[0, -1] = 4095
    return [torch.randint(0, 1024, (B, 12), generator=g), sem]


def test_semantic_codebook_4096_model_scale_vs_oracle():
    """d = 1024, L = 2, h = 8, clap 1024 x 12, semantic codebook 4096 (C = 4097, Cp = 4160): logits, loss and every
    gradient against the fp32 CPU oracle, then two optimiser steps against the oracle's clip + AdamW."""
    import open_musiclm_b200 as O
    from open_musiclm_b200 import lib
    from oracle import restatement as R
    from test_parity_gpu import _forward_vs_oracle, _grads_vs_oracle
    cfg = _semantic_4096_cfg()
    toks = _semantic_4096_tokens(2)
    m, tr, sd = _forward_vs_oracle(_semantic_4096(), cfg, toks, [0.0, 1.0], "sem4096")
    assert tr.eng.C == [1025, 4097] and tr.eng.Cp == [1088, 4160]
    _grads_vs_oracle(m, tr, sd, cfg, toks, "sem4096")
    # two optimiser steps (eval semantics), the oracle stepping its own fp32 gradients
    names = [k for k, _ in m.named_parameters()]
    params = {k: sd[k].clone() for k in names}
    state = {}
    tr2 = O.HotPathTrainer(m, cross_entropy_loss_weights=[0.0, 1.0], lr=3e-4, lr_warmup=10, wd=1e-2, max_grad_norm=0.5)
    eng = tr2.eng
    for it in range(2):
        osd = {k: (params[k].clone().requires_grad_(True) if k in params else v) for k, v in sd.items()}
        loss_ref = R.loss_and_logits(cfg, osd, [t.numpy() for t in toks])[0]
        loss_ref.backward()
        norm_ref = R.clip_and_adamw(params, {k: osd[k].grad for k in names}, state, step=it, lr=3e-4, wd=1e-2, warmup_iters=10)
        eng.arena_g.zero_()
        loss = tr2._micro_batch([t.cuda() for t in toks], False, 0, True)
        assert abs(float(loss) - float(loss_ref)) <= 1e-2 * float(loss_ref)
        tr2._set_hyper()
        eng.sumsq.zero_()
        lib.grad_sumsq(eng.arena_g, eng.sumsq)
        assert abs(float(tr2.grad_norm()) - norm_ref) <= 2e-2 * norm_ref
        lib.adamw_step(eng.arena_p, eng.arena_g, eng.adam_m, eng.adam_v, eng.n_decay, tr2.hyper, eng.sumsq)
        eng.arena_g.zero_(); eng.refresh_packed(force=True); tr2.steps += 1
    num = den = 0.0
    for k in names:
        if k.endswith("rel_pos_bias.net.3.bias"):
            continue    # analytically zero gradient (test_parity_gpu.py): Adam turns its rounding noise into +-lr
        d_ref = (params[k] - sd[k]).double(); d_got = (eng.pview[k].cpu() - sd[k]).double()
        num += float((d_ref * d_got).sum()); den += float(d_ref.norm() ** 2)
        assert rel(eng.pview[k], params[k]) <= 1e-3, k
    print("sem4096: update direction agreement", num / den)
    assert num / den > 0.95
    eng.check_errors()


def test_semantic_codebook_4096_deterministic_and_graph():
    """Under torch.use_deterministic_algorithms(True): two trainers take bit-identical steps (eager, then replayed from
    the captured graph), and graph-replayed steps equal eager ones."""
    import open_musiclm_b200 as O
    g = torch.Generator().manual_seed(5)
    batches = []
    for _ in range(4):
        t = _semantic_4096_tokens(4, seed=int(torch.randint(0, 1 << 30, (1,), generator=g)))
        batches.append([x.cuda() for x in t])

    def trainer(use_cuda_graph=True):
        return O.HotPathTrainer(_semantic_4096().cuda(), cross_entropy_loss_weights=[0.0, 1.0], lr=3e-4, lr_warmup=100, wd=0.01,
                                max_grad_norm=0.5, use_cuda_graph=use_cuda_graph, mask_prob=0.0)

    def run(tr):
        out = [tr.train_step([b]).clone() for b in batches]
        torch.cuda.synchronize()
        return out

    with switch(True):
        ta, tb, te = trainer(), trainer(), trainer(use_cuda_graph=False)
        la, lb, le = run(ta), run(tb), run(te)
        assert ta._graphs and all(st["graphs"] is not None for st in ta._graphs.values())
        assert all(torch.equal(x, y) for x, y in zip(la, lb)), (la, lb)
        assert all(torch.equal(x, y) for x, y in zip(la, le)), (la, le)
        assert all(bool(torch.isfinite(x)) for x in la)
        for name in ("arena_p", "adam_m", "adam_v"):
            assert torch.equal(getattr(ta.eng, name), getattr(tb.eng, name)), name
            assert torch.equal(getattr(ta.eng, name), getattr(te.eng, name)), name
    # default mode: graph and eager steps agree up to the fp32 atomics
    tg, tx = trainer(), trainer(use_cuda_graph=False)
    lg, lx = run(tg), run(tx)
    assert all(abs(float(x) - float(y)) <= 1e-3 * abs(float(y)) for x, y in zip(lg, lx)), (lg, lx)


def test_semantic_codebook_2048_trains_and_generates():
    """A semantic stage built with semantic_codebook_size = 2048 (C = 2049) trains through HotPathTrainer.train_step,
    eagerly and from the graph, in both modes, through the reference wrapper's forward(return_loss=True), and
    generates."""
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_semantic_transformer(dim=256, depth=2, heads=4, semantic_codebook_size=2048, attn_dropout=0.0, ff_dropout=0.1).cuda()
    g = torch.Generator().manual_seed(2)
    batch = [torch.randint(0, 1024, (4, 12), generator=g).cuda(), torch.randint(0, 2048, (4, 120), generator=g).cuda()]
    for det in (False, True):
        with switch(det):
            tr = O.HotPathTrainer(m, cross_entropy_loss_weights=[0.0, 1.0], lr=1e-3, lr_warmup=0, wd=0.01)
            l0 = float(tr.eval_loss(batch))
            losses = [float(tr.train_step([batch])) for _ in range(5)]       # steps 3-5 replay the captured graph
            assert tr._graphs and all(np.isfinite(x) for x in losses)
            assert float(tr.eval_loss(batch)) < l0, (l0, losses)
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    loss, _, _ = w(all_token_ids=batch, return_loss=True)
    assert np.isfinite(float(loss))
    out = w.generate(conditioning_token_ids=[batch[0][:2]], max_time_steps=10)
    assert out.shape == (2, 10, 1) and int(out.max()) < 2048
    m.engine.check_errors()


# ------------------------------------------------------------------------------------------------ c. generation
def _fixture_model(fx):
    return CF.model_of(fx).cuda().eval()


def _oracle_cfg(fx):
    from test_codebooks_cpu import cfg_of
    return cfg_of(fx)


@pytest.mark.parametrize("path", GEN, ids=[os.path.basename(p) for p in GEN])
def test_generate_codebook_1500_matches_reference_tokens(path):
    """The reference's generate with a 1500-entry predicted codebook (top_k = int(0.1 * 1501) = 150), on the SIMT decode
    path (B = 2) and the tensor-core path (B = 20): token for token, except after a draw where the oracle's best and
    second-best noisy scores are within 5e-2 (a near tie that 16-bit logits may break the other way)."""
    import open_musiclm_b200 as O
    from oracle import restatement as R
    fx = torch.load(path, weights_only=False)
    m = _fixture_model(fx)
    assert m.engine.C[-1] == 1501 and m.engine.Cp[-1] == 1536
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    kw = dict(conditioning_token_ids=[t.cuda() for t in fx["cond"]], max_time_steps=fx["max_time_steps"], filter_thres=fx["filter_thres"],
              temperature=fx["temperature"], uniform_noise=CF.uniforms(fx))
    trace = []
    out_eager = w.generate(trace_logits=trace, **kw)
    out_graph = w.generate(**kw)
    assert torch.equal(out_eager, out_graph)
    gold = fx["out"]
    assert out_graph.shape == gold.shape
    if torch.equal(out_graph.cpu(), gold):
        print(os.path.basename(path), "all", gold.numel(), "tokens identical to the reference's")
        return
    uni = CF.uniforms(fx)
    sd = {k: v.detach().clone() for k, v in CF.model_of(fx).state_dict().items()}
    _, otrace = R.generate(_oracle_cfg(fx), sd, [t.numpy() for t in fx["cond"]], lambda s, shape: uni[s],
                           max_time_steps=fx["max_time_steps"], filter_thres=fx["filter_thres"], temperature=fx["temperature"],
                           return_trace=True)
    mine, ref = out_graph.cpu().reshape(gold.shape[0], -1), gold.reshape(gold.shape[0], -1)
    for b in range(mine.shape[0]):
        diff = (mine[b] != ref[b]).nonzero()
        if len(diff):
            s = int(diff[0])
            gap = float(otrace[s][1][b])
            assert gap < 5e-2, (os.path.basename(path), b, s, gap)
            assert rel(trace[s][b].cpu()[torch.isfinite(otrace[s][0][b])], otrace[s][0][b][torch.isfinite(otrace[s][0][b])]) < 1e-2
            print(f"{os.path.basename(path)}: sequence {b} left the reference trajectory at token {s} (near tie, gap {gap:.3e})")


def test_seeded_rows_do_not_depend_on_the_batch_codebook_2048():
    """Seeded generation with C = 2049: a target (prompt, seed) at the first, a middle and the last row of batches of 17
    and 40 samples the tokens it samples alone (B = 1), bit for bit, on both decode paths."""
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_semantic_transformer(dim=512, depth=2, heads=8, semantic_codebook_size=2048, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    g = torch.Generator().manual_seed(7)
    tc = torch.randint(0, 1024, (1, 12), generator=g).cuda()
    tp = torch.randint(0, 2048, (1, 5, 1), generator=g).cuda()
    tp[0, 0, 0] = 2047
    tseed, steps, T = 0x5EED_2048, 12, 0.9
    ref = w.generate(conditioning_token_ids=[tc], pred_token_ids=tp, max_time_steps=steps, temperature=T, seeds=[tseed])
    for B in (17, 40):
        cond = torch.randint(0, 1024, (B, 12), generator=g).cuda()
        prefix = torch.randint(0, 2048, (B, 5, 1), generator=g).cuda()
        seeds = [int(x) for x in torch.randint(0, 2 ** 62, (B,), generator=g)]
        rows = sorted({0, B // 2, B - 1})
        for r in rows:
            cond[r], prefix[r], seeds[r] = tc[0], tp[0], tseed
        out = w.generate(conditioning_token_ids=[cond], pred_token_ids=prefix, max_time_steps=steps, temperature=T, seeds=seeds)
        for r in rows:
            assert torch.equal(out[r], ref[0]), (B, r)
    assert int(ref.max()) < 2048


class _WideNoise:
    """A NoiseStream for stages of different class counts: uniforms [n, b, C_max] handed out in order; each stage's
    generate keeps the first C columns of its draws (see _narrow)."""

    def __init__(self, uniforms):
        self.u, self.at = uniforms, 0

    def take(self, n):
        assert self.at + n <= self.u.shape[0], "noise stream exhausted"
        out = self.u[self.at:self.at + n]
        self.at += n
        return out


def _narrow(wrapper, log, trace=None):
    """Wrap wrapper.generate: the uniforms narrowed to its class count; the new tokens of every call logged."""
    orig = wrapper.generate
    C = wrapper.token_sequences[-1].codebook_size + 1

    def gen(**kw):
        kw["uniform_noise"] = kw["uniform_noise"][..., :C].contiguous()
        out = orig(**kw)
        init = 0 if kw.get("pred_token_ids") is None else kw["pred_token_ids"].shape[1]
        log.append(out[:, init:].reshape(out.shape[0], -1).cpu())
        return out
    wrapper.generate = gen


def test_three_stage_generation_with_a_2048_semantic_codebook():
    """MusicLM.generate_tokens with a 2048-entry semantic codebook shared by the semantic stage (predicted, C = 2049) and
    the coarse stage (conditioning, eos 2048), acoustic codebook 64: the decode-path chain against the oracle-backed
    chain under the same noise -- same number of draws, same shape, the same tokens up to the first near tie."""
    import open_musiclm_b200 as O
    from oracle import restatement as R
    from test_stages_cpu import OracleWrapper
    common = dict(dim=64, depth=1, heads=2, attn_dropout=0.0, ff_dropout=0.1)
    kws = {"semantic": dict(clap_codebook_size=64, semantic_codebook_size=2048, num_clap_quantizers=4),
           "coarse": dict(clap_codebook_size=64, semantic_codebook_size=2048, acoustic_codebook_size=64, num_clap_quantizers=4,
                          num_coarse_quantizers=3),
           "fine": dict(clap_codebook_size=64, acoustic_codebook_size=64, num_clap_quantizers=4, num_coarse_quantizers=3,
                        num_fine_quantizers=5)}
    seqs = {"semantic": [(64, 4), (2048, 1)], "coarse": [(64, 4), (2048, 1), (64, 3)], "fine": [(64, 4), (64, 3), (64, 5)]}
    fns = {"semantic": O.create_semantic_transformer, "coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}
    models, sds = {}, {}
    for i, (k, fn) in enumerate(fns.items()):
        torch.manual_seed(10 + i)
        mdl = fn(**common, **kws[k])
        sds[k] = {n: v.clone() for n, v in mdl.state_dict().items()}
        models[k] = mdl.cuda().eval()
    args = dict(output_seconds=3, semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5,
                semantic_steps_per_second=6, acoustic_steps_per_second=8)
    g = torch.Generator().manual_seed(3)
    clap = torch.randint(0, 64, (2, 4), generator=g)
    uniforms = torch.rand(400, 2, 2049, generator=g).clamp_(1e-6, 1 - 1e-6)
    mlm = O.MusicLM(semantic_transformer=models["semantic"], coarse_transformer=models["coarse"], fine_transformer=models["fine"])
    log = []
    for st in (mlm.semantic, mlm.coarse, mlm.fine):
        _narrow(st.transformer_wrapper, log)
    noise = _WideNoise(uniforms)
    out = mlm.generate_tokens(clap_token_ids=clap.cuda(), noise=noise, **args)
    wr = {k: OracleWrapper(R.Cfg(seqs=[R.SeqInfo(c, q) for c, q in seqs[k]], dim=64, depth=1, heads=2), sds[k]) for k in fns}
    olog = []
    for k in fns:
        _narrow(wr[k], olog)
    ref_chain = O.MusicLM(stages=(O.SemanticStage(semantic_transformer=None, wrapper=wr["semantic"]),
                                  O.CoarseStage(coarse_transformer=None, wrapper=wr["coarse"]), O.FineStage(fine_transformer=None, wrapper=wr["fine"])))
    onoise = _WideNoise(uniforms)
    ref = ref_chain.generate_tokens(clap_token_ids=clap, noise=onoise, **args)
    assert noise.at == onoise.at and out.shape == ref.shape and len(log) == len(olog)
    assert int(log[0].max()) >= 1024                     # semantic ids beyond the 1024 of every other test
    if torch.equal(out.cpu(), ref):
        print("three-stage generation, semantic codebook 2048: all", out.numel(), "tokens identical to the oracle chain's")
        return
    min_gap = min(w_.min_gap for w_ in wr.values())
    assert min_gap < 5e-2, ("tokens differ from the oracle chain without a near tie", min_gap)
    print(f"three-stage generation left the oracle trajectory; smallest oracle top-2 gap {min_gap:.3e}")


# ------------------------------------------------------------------------------------------------ d. token store
def test_token_store_round_trips_ids_up_to_16383():
    from open_musiclm_b200 import data as D
    from test_data_cpu import host_store, synth_items
    items = synth_items(4, seed=5)
    rng = np.random.default_rng(1)
    for it in items:
        it["semantic"] = rng.integers(0, 16384, it["semantic"].shape).astype(np.uint16)
        it["coarse"] = rng.integers(0, 16384, it["coarse"].shape).astype(np.uint16)
    items[0]["semantic"][0, 0] = 16383
    for stage in ("semantic", "coarse"):
        dev = D.TokenStore.from_items(stage, [{c: it[c] for c in D.STAGE_COLUMNS[stage]} for it in items])
        host = host_store(stage, items)
        ids = [0, 3, 1, 0, 2]
        a = dev.sample_batch(len(ids), rng=random.Random(4), items=ids)
        b = host.sample_batch(len(ids), rng=random.Random(4), items=ids)
        for x, y in zip(a, b):
            assert x.dtype == torch.int64 and x.is_cuda and torch.equal(x.cpu(), y)
        assert int(a[1].max()) >= 8192 and int(a[1].min()) >= 0
    flat = D.TokenStore.from_items("semantic", [{c: it[c] for c in D.STAGE_COLUMNS["semantic"]} for it in items]).flat["semantic"]
    assert int(flat.cpu().numpy().view(np.uint16).max()) == 16383
