"""Training-mode steps against the fp32 oracle: FFN dropout and the forgetful causal mask, as the engine and the trainer
wire them, in the loss and every parameter gradient.

The masks of a step come from the device Philox streams (tests/train_mode_reference.py): the test reads the seed and
the stream id the step used, rebuilds both masks with the host replica, and checks
  * that the step drew exactly those masks: the keep bits of every layer (ws['keep'][l]) and the key mask token_plan
    returned (the conditioning pad / eos masking ANDed with the forgetful mask), bit for bit;
  * that it used them: its loss (rel 1e-2) and every parameter gradient (the bounds of test_parity_gpu.check_grads)
    against restatement.loss_and_logits under the same masks, by fp32 autograd.
The gradients are what has teeth: a wrong seed, stream id, layer stream, 1 / (1 - p) scale or a missing forgetful mask
moves every gradient outside the rel-pos MLP past the bounds, the median one by more than 3x (tests/test_train_mode_cpu.py),
and the loss by a few % only.  One wiring the gradients show only weakly, the 1 / (1 - p) of the row sums gemm_rowstat
takes for the LayerNorm backward, is checked on the sums themselves.

Covered: the trainer's eager micro-batch (the ffn_mid_bwd row-sum path at Fp % 256 != 0, the gemm_rowstat keep path
otherwise, fp16 and bf16 forward operands, default and deterministic kernels, p = 0.1 and 0.5), two accumulated
micro-batches, the model.train() API path with and without gradient, and the CUDA-graph train_step (the graph keeps
the stream id of its capture while the device seed advances).  Prints METRIC lines: the worst gradient per case."""
import contextlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(__file__))
import train_mode_reference as T  # noqa: E402
from test_parity_gpu import check_grads  # noqa: E402

from oracle import restatement as R  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD_DIR = os.path.join(os.path.dirname(__file__), "golden")
MASK_PROB = 0.15


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


# ------------------------------------------------------------------------------------------------ models
class Case:
    """Weights, tokens and oracle config of one model at one dropout probability."""

    def __init__(self, stage, kwargs, state_dict, tokens, ce_weights, cfg):
        self.stage, self.kwargs, self.sd, self.tokens, self.ce, self.cfg = stage, kwargs, state_dict, tokens, ce_weights, cfg
        self.B, self.N = tokens[0].shape[0], T.seq_len(cfg, [t.numpy() for t in tokens])


_SOURCES = {}


def _source(model):
    if model not in _SOURCES:
        if model.startswith("tiny_"):
            _SOURCES[model] = torch.load(os.path.join(GOLD_DIR, f"{model}.pt"), weights_only=False)
        else:
            # model scale: the coarse stage at d = 1024 (F = 2730, Fp = 2816), h = 8, depth 2, N = 501
            import open_musiclm_b200 as O
            kw = dict(dim=1024, depth=2, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1)
            torch.manual_seed(0)
            sd = {k: v.clone() for k, v in O.create_coarse_transformer(**kw).state_dict().items()}
            g = torch.Generator().manual_seed(1234)
            toks = [torch.randint(0, 1024, s, generator=g) for s in [(2, 12), (2, 100), (2, 128, 3)]]
            _SOURCES[model] = dict(stage="coarse", kwargs=kw, state_dict=sd, tokens=toks, ce_weights=[0.0, 0.0, 1.0])
    return _SOURCES[model]


def case_of(model, p) -> Case:
    fx = _source(model)
    kw = dict(fx["kwargs"], ff_dropout=p)
    if model.startswith("tiny_"):
        cfg = T.cfg_of(fx, p, MASK_PROB)
    else:
        cfg = R.coarse_cfg(depth=2, ff_dropout=p, mask_prob=MASK_PROB, ce_weights=list(fx["ce_weights"]))
    return Case(fx["stage"], kw, fx["state_dict"], fx["tokens"], fx["ce_weights"], cfg)


def build(case, act16, monkeypatch, train=True):
    import open_musiclm_b200 as O
    monkeypatch.setenv("OMLM_ACT16", act16)        # read when the engine is built
    fn = {"semantic": O.create_semantic_transformer, "coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}[case.stage]
    m = fn(**case.kwargs)
    m.load_state_dict(case.sd, strict=True)
    m = m.cuda().train(train)
    assert m.engine.a16 == {"fp16": torch.float16, "bf16": torch.bfloat16}[act16]
    assert m.engine.drop_p == case.cfg.ff_dropout
    return m


def record_key_masks(monkeypatch):
    """Every key mask lib.token_plan returns, in call order (the tensor itself: a captured graph rewrites it)."""
    from open_musiclm_b200 import lib
    masks, orig = [], lib.token_plan

    def token_plan(*a, **k):
        out = orig(*a, **k)
        masks.append(out[2])
        return out
    monkeypatch.setattr(lib, "token_plan", token_plan)
    return masks


def train_workspace(eng):
    return next(w for k, w in eng._ws.items() if k[2])


# ------------------------------------------------------------------------------------------------ checks
_ORACLE = {}


def oracle(case, model, seed, stream, tokens=None, tag=""):
    """restatement step of `case` under the replica masks of (seed, stream id), cached per model and masks."""
    key = (model, case.cfg.ff_dropout, seed, stream, tag)
    if key not in _ORACLE:
        toks = [t.numpy() for t in (tokens if tokens is not None else case.tokens)]
        _ORACLE[key] = T.oracle_step(case.cfg, case.sd, toks, T.replica_forget(seed, stream, case.B, case.N, MASK_PROB),
                                     T.replica_keeps(seed, case.cfg, case.B, case.N))
    return _ORACLE[key]


def assert_keep_bits(ws, case, seed, tag):
    Fp, F_ = T.padded_width(case.cfg), case.cfg.ff_inner
    for l in range(case.cfg.depth):
        got = T.unpack_keep(ws["keep"][l])[:, :F_]
        ref = T.replica_keep_rows(seed, l, case.B, case.N, Fp, case.cfg.ff_dropout)[:, :F_]
        assert np.array_equal(got, ref), (tag, l, int((got != ref).sum()))


def assert_key_mask(key_mask, case, seed, stream, tag, tokens=None):
    toks = [t.numpy() for t in (tokens if tokens is not None else case.tokens)]
    _, ref, _ = R.prepare_ids(case.cfg, toks, True, T.replica_forget(seed, stream, case.B, case.N, MASK_PROB))
    got = key_mask.bool().cpu().numpy()
    assert np.array_equal(got, ref), (tag, int((got != ref).sum()))


def assert_row_sums(eng, ws, case, tag):
    """The partial row sums gemm_rowstat wrote for layer 0 (the last layer the backward pass visits) against float64
    sums of the same bf16 operands: part j of row m holds (1 / (1 - p) sum_c gamma_c keep_c dhn_c, sum_c dhn_c hn_c)
    over its 128 channels c.  The dropout scale reaches the LayerNorm backward only through the first sum, as a row-mean
    correction the gradients show weakly (a scale of 1 passes their bounds at p = 0.1), so it is checked here."""
    M, Fp = ws["dhn"].shape
    P = Fp // 128
    dhn = ws["dhn"].double().cpu().view(M, P, 128)
    hn = ws["hn"][0].double().cpu().view(M, P, 128)
    gamma = eng.pk[0]["gin"].double().cpu().view(P, 128)
    keep = torch.from_numpy(T.unpack_keep(ws["keep"][0])).double().view(M, P, 128)
    got = ws["rowstat"].double().cpu()
    r1 = rel(got[..., 0], (gamma * keep * dhn).sum(-1) / (1.0 - case.cfg.ff_dropout))
    r2 = rel(got[..., 1], (dhn * hn).sum(-1))
    print(f"METRIC train-mode {tag} layer-0 row sums: rel {r1:.3e} (gamma keep dhn / (1 - p)), {r2:.3e} (dhn hn)")
    assert r1 <= 1e-2 and r2 <= 1e-2, (tag, r1, r2)


def grads_of(m, names_from):
    return {k: names_from[k].clone() for k, _ in m.named_parameters()}


def compare_grads(got, gold, tag, act16="fp16"):
    """check_grads, with the bf16 bound under bf16 forward operands; prints the worst gradient in and outside the
    rel-pos MLP."""
    worst = {}
    for k, g in gold.items():
        if g is None or k.endswith("rel_pos_bias.net.3.bias") or float(g.norm()) < 1e-6:
            continue
        a, b = got[k].double().cpu().reshape(-1), g.double().reshape(-1)
        c = float((a @ b) / (a.norm() * b.norm()).clamp_min(1e-30))
        r = float((a - b).norm() / b.norm().clamp_min(1e-30))
        grp = "relpos" if "rel_pos_bias" in k else "other"
        wc, wr = worst.get(grp, ((1.0, ""), (0.0, "")))
        worst[grp] = (min(wc, (c, k)), max(wr, (r, k)))
    for grp, ((c, kc), (r, kr)) in sorted(worst.items()):
        print(f"METRIC train-mode {tag} grads[{grp}]: worst cos {c:.6f} ({kc}), worst rel {r:.3e} ({kr})")
    check_grads(got, gold, tag, bound=(T.GRAD_COS, T.GRAD_REL if act16 == "fp16" else T.GRAD_REL_BF16))


MODELS = ["tiny_coarse", "tiny_plainff_t5", "conv_d1024"]


def eager_step(case, act16, det, monkeypatch, **trainer_kw):
    """One training-mode micro-batch of a fresh trainer: (model, trainer, key masks, loss)."""
    import open_musiclm_b200 as O
    m = build(case, act16, monkeypatch)
    tr = O.HotPathTrainer(m, cross_entropy_loss_weights=case.ce, mask_prob=MASK_PROB, use_cuda_graph=False, **trainer_kw)
    masks = record_key_masks(monkeypatch)
    tr.eng.arena_g.zero_()
    with switch(det):
        tr._fwd_bwd_body([[t.cuda() for t in case.tokens]], det)
    torch.cuda.synchronize()
    return m, tr, masks, float(tr.loss_acc[0, 0])


# ------------------------------------------------------------------------------------------------ (a) eager trainer
@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
@pytest.mark.parametrize("act16", ["fp16", "bf16"])
@pytest.mark.parametrize("model", MODELS)
def test_trainer_micro_batch_matches_oracle_under_its_masks(model, act16, det, p, monkeypatch):
    """HotPathTrainer, one micro-batch in training mode: the masks it drew are the replica's at (eng.seed, _mask_draws),
    and its loss and every gradient are the oracle's under those masks."""
    case = case_of(model, p)
    m, tr, masks, loss = eager_step(case, act16, det, monkeypatch)
    eng = tr.eng
    seed, stream = int(eng.seed.item()), tr._mask_draws
    assert stream == 1 and len(masks) == 1
    tag = f"{model}-{act16}-{'det' if det else 'default'}-p{p}"
    ws = train_workspace(eng)
    assert_keep_bits(ws, case, seed, tag)
    assert_key_mask(masks[0], case, seed, stream, tag)
    if T.padded_width(case.cfg) % 256 == 0:      # the gemm_rowstat path (else ffn_mid_bwd sums the rows itself)
        assert_row_sums(eng, ws, case, tag)
    loss_ref, _, _, grads_ref = oracle(case, model, seed, stream)
    assert abs(loss - loss_ref) / loss_ref <= 1e-2, (tag, loss, loss_ref)
    compare_grads(grads_of(m, eng.gview), grads_ref, tag, act16)


@pytest.mark.parametrize("model", MODELS)
def test_oracle_under_the_next_seed_fails_the_bounds(model, monkeypatch):
    """Negative control of the test above: the same GPU step against the oracle fed the masks of seed + 1 fails the
    gradient bounds, every gradient outside the rel-pos MLP by at least 3x."""
    case = case_of(model, 0.1)
    m, tr, _, _ = eager_step(case, "fp16", False, monkeypatch)
    seed, stream = int(tr.eng.seed.item()), tr._mask_draws
    got = grads_of(m, tr.eng.gview)
    _, _, _, wrong = oracle(case, model, seed + 1, stream)
    errs = T.grad_errors(got, wrong)
    smallest = min(r for _, _, r in errs)
    print(f"METRIC train-mode {model} against the seed+1 oracle: smallest gradient rel {smallest:.3e}, "
          f"median {float(np.median([r for _, _, r in errs])):.3e}")
    assert smallest >= 3 * T.GRAD_REL, [(k, r) for k, _, r in errs if r < 3 * T.GRAD_REL]
    with pytest.raises(AssertionError):
        check_grads(got, wrong, f"{model}-seed+1")


# ------------------------------------------------------------------------------------------------ (b) accumulation
@pytest.mark.parametrize("model", ["tiny_coarse", "tiny_plainff_t5"])
def test_two_accumulated_micro_batches_match_the_oracle_mean(model, monkeypatch):
    """grad_accum_every = 2: each micro-batch draws its own (seed, stream id) masks, and the accumulated gradient is the
    mean of the oracle's two gradients under them."""
    import open_musiclm_b200 as O
    case = case_of(model, 0.1)
    g = torch.Generator().manual_seed(77)
    cb = case.kwargs.get("clap_codebook_size", 64)
    mbs = [case.tokens, [torch.randint(0, cb, tuple(t.shape), generator=g) for t in case.tokens]]
    m = build(case, "fp16", monkeypatch)
    tr = O.HotPathTrainer(m, cross_entropy_loss_weights=case.ce, mask_prob=MASK_PROB, grad_accum_every=2, use_cuda_graph=False)
    eng = tr.eng
    masks = record_key_masks(monkeypatch)
    seed0, draws0 = int(eng.seed.item()), tr._mask_draws
    eng.arena_g.zero_()
    tr._fwd_bwd_body([[t.cuda() for t in mb] for mb in mbs], False)
    assert int(eng.seed.item()) == seed0 + 2 and tr._mask_draws == draws0 + 2 and len(masks) == 2
    refs = []
    for i, mb in enumerate(mbs):
        seed, stream = seed0 + 1 + i, draws0 + 1 + i
        assert_key_mask(masks[i], case, seed, stream, f"{model} micro-batch {i}", tokens=mb)
        refs.append(oracle(case, model, seed, stream, tokens=mb, tag=f"mb{i}"))
        got_loss = float(tr.loss_acc[i, 0])
        assert abs(got_loss - refs[i][0]) / refs[i][0] <= 1e-2, (i, got_loss, refs[i][0])
    assert_keep_bits(train_workspace(eng), case, seed0 + 2, f"{model} micro-batch 1")
    gold = {k: (None if a is None else 0.5 * (a + refs[1][3][k])) for k, a in refs[0][3].items()}
    compare_grads(grads_of(m, eng.gview), gold, f"{model}-accum2")


# ------------------------------------------------------------------------------------------------ (c) API path
@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("model", ["tiny_coarse", "tiny_plainff_t5"])
def test_api_forward_backward_in_train_mode(model, p, monkeypatch):
    """model.train() forward on the eval fixture's ids and key mask (no forgetful mask on this path, as in the
    reference), the wrapper's cross entropy, backward: dropout under (eng.seed, layer) in the forward and the same keep
    bits in the backward.  Then a torch.no_grad() forward in training mode, which runs every layer in one workspace
    (keep[0] reused), against the oracle's logits at the next seed."""
    fx = _source(model)
    case = case_of(model, p)
    m = build(case, "fp16", monkeypatch, train=True)
    eng = m.engine
    ids = [t.cuda() for t in fx["ids"]]
    key_mask = fx["key_mask"].cuda()
    B, N = fx["key_mask"].shape
    logits = m(all_token_ids=ids, self_attn_mask=key_mask)
    seed = int(eng.seed.item())
    assert seed == 1
    keeps = T.replica_keeps(seed, case.cfg, B, N)
    ws = train_workspace(eng)
    for l in range(case.cfg.depth):
        assert torch.equal(T.keep_bnf(T.unpack_keep(ws["keep"][l]), B, N, case.cfg.ff_inner), keeps[l]), l
    st = T.trainable_state(case.sd)
    np_ids = [t.numpy() for t in fx["ids"]]
    ref_logits = R.forward_logits(case.cfg, st, np_ids, fx["key_mask"].numpy(), drop_keeps=keeps)

    def ce(all_logits, to):
        total, running = 0, 0.0
        for lg, lb, w in zip(all_logits, fx["labels"], fx["ce_weights"]):
            if w > 0:
                running = running + F.cross_entropy(lg.permute(0, 2, 1), lb.to(to)) * lb.numel() * w
                total += lb.numel()
        return running / total
    for a, b in zip(logits, ref_logits):
        assert a.shape == b.shape and rel(a.detach(), b.detach()) <= 1e-2, rel(a.detach(), b.detach())
    loss, loss_ref = ce(logits, "cuda"), ce(ref_logits, "cpu")
    assert abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach()) <= 1e-2
    loss.backward()
    loss_ref.backward()
    gold = {k: (st[k].grad if st[k].grad is not None else torch.zeros_like(st[k])) for k, _ in m.named_parameters()}
    compare_grads({k: p_.grad for k, p_ in m.named_parameters()}, gold, f"api-{model}-p{p}")
    # no gradient: the one-layer workspace, each layer's keep bits drawn into keep[0] under its own stream
    with torch.no_grad():
        out = m(all_token_ids=ids, self_attn_mask=key_mask)
        ref = R.forward_logits(case.cfg, case.sd, np_ids, fx["key_mask"].numpy(), drop_keeps=T.replica_keeps(seed + 1, case.cfg, B, N))
    assert int(eng.seed.item()) == seed + 1
    for a, b in zip(out, ref):
        r = rel(a, b)
        print(f"METRIC train-mode api-{model}-p{p} no-grad logits rel {r:.3e}")
        assert r <= 1e-2, r


# ------------------------------------------------------------------------------------------------ (d) CUDA graph
def test_graph_replays_draw_new_masks_under_the_captured_stream_id(monkeypatch):
    """train_step's contract for the masks: the two eager steps per shape draw under (seed, stream id) = (s0 + i,
    i) for i = 1, 2; the captured graph holds the stream id of its capture (the host-side _mask_draws at capture, 3, is
    a kernel argument), while the device seed it increments advances on every replay.  So each replay draws new keep
    bits and a new forgetful mask, and both are the replica's at (that replay's seed, 3)."""
    import open_musiclm_b200 as O
    case = case_of("tiny_coarse", 0.1)
    m = build(case, "fp16", monkeypatch)
    tr = O.HotPathTrainer(m, cross_entropy_loss_weights=case.ce, mask_prob=MASK_PROB, use_cuda_graph=True)
    eng = tr.eng
    masks = record_key_masks(monkeypatch)
    toks = [t.cuda() for t in case.tokens]
    s0 = int(eng.seed.item())
    seen = []
    for step in range(5):
        tr.train_step([toks])
        seed = int(eng.seed.item())
        assert seed == s0 + 1 + step
        stream = min(step + 1, 3)              # two eager steps and the capture draw a stream id each, replays none
        assert len(masks) == stream and tr._mask_draws == stream
        assert (next(iter(tr._graphs.values()))["graphs"] is None) == (step < 2)
        tag = f"train_step {step}"
        ws = train_workspace(eng)
        assert_keep_bits(ws, case, seed, tag)
        assert_key_mask(masks[min(step, 2)], case, seed, stream, tag)
        seen.append((ws["keep"][0].clone(), masks[min(step, 2)].clone()))
    for (ka, ma), (kb, mb) in zip(seen[2:], seen[3:]):
        assert not torch.equal(ka, kb) and not torch.equal(ma, mb)
