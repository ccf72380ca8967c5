"""Codebooks of different sizes in different sequences, above 1024 entries: the oracle restatement against the REAL
reference's outputs recorded by tools/make_golden_codebooks.py (tests/golden/cbsize_*.pt, in the compact form of
tests/codebook_fixtures.py), at the tolerances of tests/test_oracle_cpu.py.  The oracle's Cfg carries one
SeqInfo(codebook_size, num_quantizers) per sequence, so each fixture's per-sequence sizes go straight into it."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

from oracle import restatement as R

sys.path.insert(0, os.path.dirname(__file__))
import codebook_fixtures as CF  # noqa: E402

HERE = os.path.join(os.path.dirname(__file__), "golden")
TRAIN = [os.path.join(HERE, f"cbsize_{n}.pt") for n in ("semantic", "coarse")]
GEN = sorted(glob.glob(os.path.join(HERE, "cbsize_gen_*.pt")))
QUANT = {"semantic": ("num_clap_quantizers", None), "coarse": ("num_clap_quantizers", None, "num_coarse_quantizers"),
         "fine": ("num_clap_quantizers", "num_coarse_quantizers", "num_fine_quantizers")}


def cfg_of(fx, **extra):
    """Cfg with the fixture's per-sequence codebook sizes (fx["codebooks"])."""
    kw = fx["kwargs"]
    nq = [kw[k] if k is not None else 1 for k in QUANT[fx["stage"]]]
    seqs = [R.SeqInfo(cb, q) for cb, q in zip(fx["codebooks"], nq)]
    return R.Cfg(seqs=seqs, dim=kw["dim"], depth=kw["depth"], heads=kw["heads"], ff_dropout=kw["ff_dropout"],
                 grad_shrink_alpha=kw["grad_shrink_alpha"], **extra)


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def test_fixtures_cover_large_and_mixed_codebooks():
    """What the fixtures are for: a 1500-entry sequence whose drawn ids go past 1024 (up to 1499) next to 64-entry ones,
    and, in the coarse fixture, the 1500-entry sequence as conditioning (its eos 1500 masked out of the keys)."""
    sem, coarse = (torch.load(p, weights_only=False) for p in TRAIN)
    assert sem["codebooks"] == [64, 1500] and coarse["codebooks"] == [64, 1500, 64]
    for fx in (sem, coarse):
        for t, cb in zip(fx["tokens"], fx["codebooks"]):
            assert int(t.min()) >= 0 and int(t.max()) == cb - 1
        assert int(fx["tokens"][1].max()) >= 1024
        assert fx["logits"][1]["shape"][-1] == 1501 or fx["ce_weights"][1] == 0.0
    assert not bool(coarse["key_mask"].all())           # the conditioning eos ids are masked


def _state(fx):
    """The fixture's weights (rebuilt, SHA-checked) as the oracle's flat dict."""
    return {k: v.detach().clone() for k, v in CF.model_of(fx).state_dict().items()}


def _check_sampled(got, s, tol, name):
    if s["norm"] < 1e-6:
        # e.g. rel_pos_bias.net.3.bias: a per-head constant cancels in the softmax, gradient is rounding noise
        assert float(got.norm()) < 1e-5, name
        return
    assert CF.rel_to(got, s) < tol, (name, CF.rel_to(got, s))
    assert CF.norm_rel(got, s) < tol, (name, CF.norm_rel(got, s))


@pytest.mark.parametrize("path", TRAIN, ids=[os.path.basename(p) for p in TRAIN])
def test_restatement_matches_reference_codebook_fixture(path):
    fx = torch.load(path, weights_only=False)
    cfg = cfg_of(fx, ce_weights=fx["ce_weights"])
    sd = {k: v.clone().requires_grad_(v.is_floating_point() and not k.endswith("beta")) for k, v in _state(fx).items()}
    loss, logits, labels, ids, mask = R.loss_and_logits(cfg, sd, [t.numpy() for t in fx["tokens"]])
    for a, b in zip(ids, fx["ids"]):
        assert np.array_equal(a, b.numpy())
    assert np.array_equal(mask, fx["key_mask"].numpy())
    for a, b in zip(labels, fx["labels"]):
        assert np.array_equal(a, b.numpy())
    for i, (a, s) in enumerate(zip(logits, fx["logits"])):
        _check_sampled(a.detach(), s, 2e-5, f"logits {i}")
    assert abs(float(loss.detach()) - float(fx["loss"])) / abs(float(fx["loss"])) < 1e-5
    loss.backward()
    for k, s in fx["grads"].items():
        g = sd[k].grad
        if s is None:
            assert g is None or float(g.abs().max()) == 0.0, k
        else:
            _check_sampled(g, s, 2e-4, k)


def test_restatement_optimizer_steps_codebook_fixture():
    fx = torch.load(TRAIN[0], weights_only=False)
    assert len(fx["opt_steps"]) == 2
    cfg = cfg_of(fx, ce_weights=fx["ce_weights"])
    sd0 = _state(fx)
    params = {k: v.clone() for k, v in sd0.items() if not k.endswith("beta")}
    toks = [t.numpy() for t in fx["tokens"]]
    state = {}
    for it, gold in enumerate(fx["opt_steps"]):
        sd = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        for k, v in sd0.items():
            if k.endswith("beta"):
                sd[k] = v
        loss, *_ = R.loss_and_logits(cfg, sd, toks)
        loss.backward()
        grads = {k: sd[k].grad for k in params}
        assert abs(float(loss.detach()) - float(gold["loss"])) / float(gold["loss"]) < 1e-4
        norm = R.clip_and_adamw(params, grads, state, step=it, lr=3e-4, wd=1e-2, warmup_iters=10)
        assert abs(norm - float(gold["grad_norm"])) / float(gold["grad_norm"]) < 1e-4
        if gold["params"] is not None:
            for k, s in gold["params"].items():
                if fx["grads"][k] is not None and fx["grads"][k]["norm"] < 1e-6:
                    continue    # gradient is rounding noise (softmax-invariant bias): Adam turns its sign into +-lr
                assert CF.rel_to(params[k], s) < 1e-5, k


@pytest.mark.parametrize("path", GEN, ids=[os.path.basename(p) for p in GEN])
def test_generate_restatement_reproduces_reference_tokens_codebook_fixture(path):
    fx = torch.load(path, weights_only=False)
    assert fx["codebooks"][-1] == 1500 and fx["noise_shape"][-1] == 1501
    uni = CF.uniforms(fx)
    out = R.generate(cfg_of(fx), _state(fx), [t.numpy() for t in fx["cond"]], lambda step, shape: uni[step],
                     max_time_steps=fx["max_time_steps"], filter_thres=fx["filter_thres"], temperature=fx["temperature"],
                     include_eos_in_output=fx["include_eos_in_output"], allow_eos_in_output=fx["allow_eos_in_output"])
    assert out.shape == fx["out"].shape and torch.equal(out, fx["out"])
    assert int(fx["out"].max()) >= 1024                  # sampled ids past the 1024 of every other fixture
