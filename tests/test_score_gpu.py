"""Teacher-forced scoring on the H100 (open_musiclm_b200/score.py): `wrapper.score` bit for bit the teacher-forced
generate call of each row alone (semantic, coarse and fine stages, ragged lengths, 1 to 300 rows, several packed
groups and one, d = 1024 at 8 and 16 heads, absolute positions, T5 and no bias, the plain FFN), Engine.seed and later
calls untouched; `MusicLM.score_tokens` on generate_tokens' songs at musiclm_small dims bit for bit the per-window
teacher-forced generate calls (a list of songs of 4 to 20 s, a prime, coarse_only), and within the step-versus-forward
bound of the log p generate reported while sampling those tokens."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from logprob_reference import model_logprob  # noqa: E402
from norm_loss_reference import ce_ref  # noqa: E402
from test_generate_ragged_gpu import _model  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _fine_model(dim=128, heads=2, cb=64, **kw):
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_fine_transformer(dim=dim, depth=2, heads=heads, clap_codebook_size=cb, acoustic_codebook_size=cb, num_clap_quantizers=4,
                                  num_coarse_quantizers=3, num_fine_quantizers=5, attn_dropout=0.0, ff_dropout=0.1, **kw).cuda().eval()
    return m, O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)


def _inputs(w, B, steps, g, n_cond=(4, 9)):
    seqs = w.token_sequences
    cond = [torch.randint(0, seqs[s].codebook_size, (B, n_cond[s] * (seqs[s].num_quantizers if s else 1)), generator=g).cuda()
            for s in range(len(seqs) - 1)]
    x = torch.randint(0, seqs[-1].codebook_size, (B, steps, seqs[-1].num_quantizers), generator=g).cuda()
    return cond, x


def _alone(w, cond, x, b, n):
    """Row b's teacher-forced generate call alone: [n, q] logprobs."""
    if n == 0:
        return torch.zeros(0, x.shape[2], device=DEV)
    return w.generate(conditioning_token_ids=[t[b:b + 1] for t in cond], pred_token_ids=x[b:b + 1, :n], max_time_steps=n,
                      return_logprobs=True)[1][0]


CASES = [("semantic", 1, 128, 2, None), ("coarse", 3, 128, 2, None), ("fine", 3, 128, 2, None), ("coarse", 40, 128, 2, None),
         ("semantic", 300, 128, 2, None), ("coarse", 20, 1024, 8, None), ("semantic", 20, 1024, 16, None),
         ("coarse", 17, 128, 2, "abspos"), ("semantic", 17, 128, 2, "t5"), ("coarse", 17, 128, 2, "none"), ("fine", 17, 128, 2, "plainff")]


@pytest.mark.parametrize("stage,B,dim,heads,variant", CASES, ids=[f"{s}-b{b}-d{d}-h{h}-{v or 'continuous'}" for s, b, d, h, v in CASES])
def test_score_is_each_row_alone(stage, B, dim, heads, variant):
    """Ragged rows (lengths 0 ... 9 steps): the default packing and a max_rows that forces several groups (and one that
    fits a single prompt only) give the same bits, and every checked row equals its teacher-forced generate call."""
    kw = dict(use_absolute_position_embeddings=True, max_absolute_position_embeddings=80) if variant == "abspos" else \
        dict(relative_position_bias_type=variant) if variant in ("t5", "none") else dict(use_conv_ff=False) if variant == "plainff" else {}
    cb = 64 if dim == 128 else 1024
    if stage == "fine":
        m, w = _fine_model(dim, heads, cb, **kw)
    else:
        m, w, _, _ = _model(stage, dim=dim, heads=heads, cb=cb, **kw)
    g = torch.Generator().manual_seed(B * 7 + heads)
    steps = 9
    cond, x = _inputs(w, B, steps, g)
    lengths = [(3 * b + 1) % (steps + 1) for b in range(B)] if B > 1 else [steps]
    seed0 = m.engine.seed.clone()
    lp = w.score(conditioning_token_ids=cond, pred_token_ids=x, pred_lengths=lengths)
    assert lp.shape == x.shape and lp.dtype == torch.float32
    P = sum(t.shape[1] + 2 for t in cond) + steps * x.shape[2] + 1
    for max_rows in (3 * P, 1):
        assert torch.equal(w.score(conditioning_token_ids=cond, pred_token_ids=x, pred_lengths=lengths, max_rows=max_rows), lp), max_rows
    assert torch.equal(m.engine.seed, seed0)
    rows = range(B) if B <= 20 else sorted({0, 1, 2, B // 2, B - 2, B - 1} | set(range(3, B, B // 8)))
    for b in rows:
        n = lengths[b]
        assert torch.equal(lp[b, :n], _alone(w, cond, x, b, n)), b
        assert bool((lp[b, n:] == 0).all()) and bool((lp[b, :n] <= 0).all())


def test_score_leaves_training_and_generation_alone():
    """In training mode, between seeded calls: scoring returns eval values, leaves the mode and Engine.seed, and the
    following unseeded generate and train_step give what they give without the scoring call."""
    import open_musiclm_b200 as O
    m, w, _, _ = _model("coarse")
    g = torch.Generator().manual_seed(1)
    cond, x = _inputs(w, 4, 5, g)
    ref = w.score(conditioning_token_ids=cond, pred_token_ids=x)
    batch = [cond[0], cond[1], x]
    state = {k: v.detach().clone() for k, v in m.state_dict().items()}

    def run(score_first):
        m.load_state_dict(state)
        m.engine.seed.fill_(77)
        m.train()
        if score_first:
            assert torch.equal(w.score(conditioning_token_ids=cond, pred_token_ids=x), ref)
            assert m.training and int(m.engine.seed) == 77
        out = w.generate(conditioning_token_ids=cond, max_time_steps=4)
        tr = O.HotPathTrainer(m, cross_entropy_loss_weights=[0.0, 0.0, 1.0], lr=3e-4, wd=1e-2)
        loss = float(tr.train_step([batch]))
        return out, loss

    (o0, l0), (o1, l1) = run(False), run(True)
    assert torch.equal(o0, o1) and l0 == l1
    m.load_state_dict(state)
    m.eval()


# ------------------------------------------------------------------------------------------------ songs
@pytest.fixture(scope="module")
def small_musiclm():
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    mk = dict(dim=1024, attn_dropout=0.0, ff_dropout=0.1, grad_shrink_alpha=0.1, depth=6, heads=8)
    return O.MusicLM(semantic_transformer=O.create_semantic_transformer(**mk).cuda().eval(),
                     coarse_transformer=O.create_coarse_transformer(**mk, num_coarse_quantizers=3).cuda().eval(),
                     fine_transformer=O.create_fine_transformer(**mk, num_coarse_quantizers=3, num_fine_quantizers=5).cuda().eval())


def _window_calls(plan, streams, clap):
    """Per window job that samples a kept token: (job, its conditioning, its prefix followed by those tokens, the
    prefix length, the stream steps a ... b - 1 of those tokens), cut from the whole generated streams."""
    from open_musiclm_b200.stages import STREAMS
    part = lambda ref: None if ref is None else streams[ref[0]][:, ref[1]:ref[2]]
    out = []
    for job in plan.jobs:
        name = STREAMS[job.stage]
        pre = part(job.prefix)
        plen = 0 if pre is None else pre.shape[1]
        a, b = job.dest + max(plen - job.drop, 0), job.dest + job.steps - job.drop
        if b <= a:
            continue
        tok = streams[name][:, a:b]
        cond = [clap] + ([] if job.cond is None else [part(job.cond)])
        full = tok if pre is None else torch.cat([pre, tok], 1)
        out.append((job, cond, full, plen, (a, b)))
    return out


def _streams(mlm, plan, sem, coarse, fine, primes):
    """The whole generated streams (the windows' frame) back from generate_tokens' outputs: the crops are prime steps."""
    from open_musiclm_b200.score import song_layouts
    qs = (1, 3, 5)
    tp = None if not primes else tuple(primes[k].shape[1] for k in ("prime_semantic_token_ids", "prime_coarse_token_ids", "prime_fine_token_ids"))
    lay = song_layouts(plan, tp, qs)
    out = {}
    for name, t, pk in (("semantic", sem, "prime_semantic_token_ids"), ("coarse", coarse, "prime_coarse_token_ids"), ("fine", fine, "prime_fine_token_ids")):
        if t is None:
            continue
        L = lay[name]
        head = primes[pk].reshape(1, -1, L.q)[:, L.tail:L.tail + L.lo] if L.lo else t[:, :0]
        out[name] = torch.cat([head, t[:, L.pre:]], 1)
    if primes:
        out.update(prime_semantic=primes["prime_semantic_token_ids"].reshape(1, -1, 1), prime_coarse=primes["prime_coarse_token_ids"],
                   prime_fine=primes["prime_fine_token_ids"])
    return out


def _check_song(mlm, lp, plan, streams, clap, outs, seed, top_p, check_decode):
    """Every window's scored positions equal its teacher-forced generate call; with check_decode, also the log p the
    seeded sampling call reported, within 2 max |dl| + both rounding bounds.  Returns the worst ratio of difference to
    bound."""
    from open_musiclm_b200.score import song_layouts
    from open_musiclm_b200.stages import STREAMS, window_seed
    stages = (mlm.semantic, mlm.coarse, mlm.fine)
    worst = 0.0
    for job, cond, full, plen, (a, b) in _window_calls(plan, streams, clap):
        name = STREAMS[job.stage]
        w = stages[job.stage].transformer_wrapper
        L = song_layouts(plan, outs["tp"], (1, 3, 5))[name]
        got = lp[job.stage][:, L.pre + a - L.lo:L.pre + b - L.lo]
        tf = w.generate(conditioning_token_ids=cond, pred_token_ids=full, max_time_steps=full.shape[1], return_logprobs=True)[1]
        assert torch.equal(got, tf[:, plen:]), (name, job.window)
        if not check_decode:
            continue
        trace = []
        tok, dlp, _ = w.generate(conditioning_token_ids=cond, pred_token_ids=None if plen == 0 else full[:, :plen],
                                 max_time_steps=job.max_time_steps, temperature=job.temperature, seeds=[window_seed(seed, job.stage, job.window)],
                                 top_p=top_p, return_logprobs=True, trace_logits=trace)
        q = full.shape[2]
        keep = slice(max(plen, job.drop) * q, None)
        assert torch.equal(tok.reshape(-1)[keep], full.reshape(-1)[plen * q:]), (name, job.window)
        C = w.token_sequences[-1].codebook_size + 1
        ids = [torch.cat([c.reshape(1, -1), torch.full((1, 1), e, device=DEV)], 1) for c, e in zip(cond, w.eos_ids)]
        flat = full.reshape(1, -1)
        with torch.no_grad():
            rows = w.transformer(all_token_ids=ids + [flat], return_only_final_seq_logits=True)[-1][0, :flat.shape[1], :C].float()
        ce = ce_ref(rows.cpu(), flat[0].cpu(), C, C, grad_scale=0.0)
        for s, row in enumerate(trace):
            p = plen * q + s
            d = float((row[0].cpu().double() - rows[p].cpu().double()).abs().max())
            _, bnd = model_logprob(row, flat[:, p])
            bound = 2 * d + float(bnd[0]) + float(ce["loss_bound"][p])
            diff = abs(float(dlp.reshape(-1)[p]) - float(tf.reshape(-1)[p]))
            worst = max(worst, diff / bound)
            assert diff <= bound, (name, job.window, s, diff, bound)
    return worst


def test_score_tokens_equals_the_windows(small_musiclm):
    mlm = small_musiclm
    g = torch.Generator().manual_seed(5)
    secs = [4, 11, 20]
    claps = [torch.randint(0, 1024, (1, 12), generator=g).cuda() for _ in secs]
    prime = dict(prime_semantic_token_ids=torch.randint(0, 1024, (1, 300), generator=g).cuda(),
                 prime_coarse_token_ids=torch.randint(0, 1024, (1, 450, 3), generator=g).cuda(),
                 prime_fine_token_ids=torch.randint(0, 1024, (1, 450, 5), generator=g).cuda())
    songs = []
    for i, (s, clap) in enumerate(zip(secs, claps)):
        p = prime if i == 1 else {}
        top_p = 0.9 if i == 2 else None
        _, sem, coarse, fine = mlm.generate_tokens(clap_token_ids=clap, seeds=[100 + i], output_seconds=s, return_all=True, top_p=top_p, **p)
        songs.append(dict(clap=clap, secs=s, primes=p, sem=sem, coarse=coarse, fine=fine, seed=100 + i, top_p=top_p))
    pr = lambda k: [s["primes"].get(k) for s in songs]
    seed0 = [w.transformer.engine.seed.clone() for w in (mlm.semantic.transformer_wrapper, mlm.coarse.transformer_wrapper,
                                                          mlm.fine.transformer_wrapper)]
    args = dict(clap_token_ids=[s["clap"] for s in songs], semantic_token_ids=[s["sem"] for s in songs],
                coarse_token_ids=[s["coarse"] for s in songs], fine_token_ids=[s["fine"] for s in songs], output_seconds=secs,
                prime_semantic_token_ids=pr("prime_semantic_token_ids"), prime_coarse_token_ids=pr("prime_coarse_token_ids"),
                prime_fine_token_ids=pr("prime_fine_token_ids"))
    lp = mlm.score_tokens(**args)
    for st in range(3):
        for a, b in zip(mlm.score_tokens(max_rows=2000, **args)[st], lp[st]):
            assert torch.equal(a, b)
    for w, s0 in zip((mlm.semantic.transformer_wrapper, mlm.coarse.transformer_wrapper, mlm.fine.transformer_wrapper), seed0):
        assert torch.equal(w.transformer.engine.seed, s0)
    from open_musiclm_b200.stages import plan_song
    worst = 0.0
    for i, s in enumerate(songs):
        tp = None if not s["primes"] else (300, 450, 450)
        plan = plan_song(output_seconds=s["secs"], prime_lengths=tp)
        streams = _streams(mlm, plan, s["sem"], s["coarse"], s["fine"], s["primes"])
        worst = max(worst, _check_song(mlm, [lp[st][i] for st in range(3)], plan, streams, s["clap"], dict(tp=tp), s["seed"], s["top_p"],
                                       check_decode=i != 1))
    print(f"METRIC score_vs_decode_worst_ratio {worst:.4f}")


def test_score_tokens_coarse_only(small_musiclm):
    mlm = small_musiclm
    g = torch.Generator().manual_seed(6)
    clap = torch.randint(0, 1024, (2, 12), generator=g).cuda()
    _, sem, _, _ = mlm.generate_tokens(clap_token_ids=clap, seeds=[7, 8], output_seconds=6, return_all=True)
    coarse = mlm.generate_tokens(clap_token_ids=clap, seeds=[7, 8], output_seconds=6, coarse_only=True)
    lp_sem, lp_coarse, lp_fine = mlm.score_tokens(clap_token_ids=clap, semantic_token_ids=sem, coarse_token_ids=coarse, output_seconds=6,
                                                  coarse_only=True)
    assert lp_fine is None and lp_sem.shape == sem.shape and lp_coarse.shape == coarse.shape
    from open_musiclm_b200.stages import plan_song
    plan = plan_song(output_seconds=6, coarse_only=True)
    for b in range(2):
        streams = _streams(mlm, plan, sem[b:b + 1], coarse[b:b + 1], None, {})
        _check_song(mlm, [lp_sem[b:b + 1], lp_coarse[b:b + 1], None], plan, streams, clap[b:b + 1], dict(tp=None), [7, 8][b], None,
                    check_decode=False)
