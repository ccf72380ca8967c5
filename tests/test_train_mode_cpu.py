"""Training-mode steps on the CPU: the oracle under the masks the REAL reference drew, the mask layouts the GPU tests
convert between, and the wrong masks the GPU comparison must be able to tell apart.

  * tests/golden/train_mode.pt (oracle/make_golden_train.py) holds a `.train()` step of the reference wrapper with
    FFN dropout and the forgetful causal mask on, and the masks it drew.  Given those masks the restatement reproduces
    the loss and every gradient (its norm and a seeded sample of its entries) at the thresholds of
    test_restatement_matches_reference_fixture.
  * The replica's keep bits and forgetful mask convert to the reference's layouts and back without loss.
  * Negative controls: a step under plausibly wrong masks (the next seed, the next stream id, no 1 / (1 - p), the
    layers' streams swapped, no forgetful mask) moves every gradient outside the rel-pos bias past the loosest GPU
    parity bound (bf16 forward operands), and the median one by at least 3x that bound.  A bound loosened so far that
    one of these faults passes fails here."""
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_train as MG
from oracle import restatement as R
import train_mode_reference as T

GOLD_DIR = os.path.join(os.path.dirname(__file__), "golden")
TRAIN = torch.load(os.path.join(GOLD_DIR, "train_mode.pt"), weights_only=False)
CASES = sorted(TRAIN)


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def source(case):
    fx = torch.load(os.path.join(GOLD_DIR, f"{case['source']}.pt"), weights_only=False)
    assert MG.state_sha(fx["state_dict"]) == case["state_sha"]
    return fx


def test_fixture_covers_both_ffn_paths_and_both_rates():
    assert {(c["source"], c["ff_dropout"]) for c in TRAIN.values()} == {(s, p) for s in MG.SOURCES for p in MG.DROPOUTS}


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_reference_training_step(name):
    case = TRAIN[name]
    fx = source(case)
    cfg = T.cfg_of(fx, case["ff_dropout"], case["mask_prob"])
    toks = [t.numpy() for t in fx["tokens"]]
    B, N = toks[0].shape[0], T.seq_len(cfg, toks)
    forget = case["forget"].numpy()
    # the reference's forgetful mask: num_drop positions per row over the whole sequence, never the first
    assert forget.shape == (B, N) and forget[:, 0].all() and ((~forget).sum(1) == T.num_drop(N, case["mask_prob"])).all()
    assert len(case["keeps"]) == cfg.depth and all(k.shape == (B, N, cfg.ff_inner) for k in case["keeps"])
    # the masks matter: the step differs from the eval step of the same weights and tokens
    assert abs(case["loss"] - float(fx["loss"])) / float(fx["loss"]) > 1e-3
    loss, logits, mask, grads = T.oracle_step(cfg, fx["state_dict"], toks, forget, case["keeps"])
    assert np.array_equal(mask, fx["key_mask"].numpy() & forget)
    for a, b in zip(logits, case["logits"]):
        assert a.shape == b.shape and rel(a, b) < 2e-5
    assert abs(loss - case["loss"]) / abs(case["loss"]) < 1e-5
    for k, gref in case["grads"].items():      # per gradient: its norm and a seeded sample of its entries
        g = grads[k]
        if gref is None:
            assert g is None or float(g.abs().max()) == 0.0, k
        elif gref["norm"] < 1e-6:
            assert float(g.norm()) < 1e-5, k          # rel_pos_bias.net.3.bias: analytically zero
        else:
            sample = g.reshape(-1)[MG.grad_sample_index(g.numel(), k)]
            assert abs(float(g.double().norm()) - gref["norm"]) / gref["norm"] < 2e-4, k
            assert rel(sample, gref["sample"]) < 2e-4, (k, rel(sample, gref["sample"]))


@pytest.mark.parametrize("name", CASES)
def test_mask_layouts_round_trip(name):
    case = TRAIN[name]
    fx = source(case)
    cfg = T.cfg_of(fx, case["ff_dropout"])
    B, N, F = case["keeps"][0].shape
    Fp = T.padded_width(cfg)
    assert F == cfg.ff_inner and Fp % 128 == 0 and Fp - F < 128
    # reference [B, N, F] -> engine bits [B N, Fp / 8] -> [B, N, F]
    for k in case["keeps"]:
        bits = T.pack_keep(T.keep_rows(k, Fp))
        assert bits.dtype == np.uint8 and bits.shape == (B * N, Fp // 8)
        assert torch.equal(T.keep_bnf(T.unpack_keep(bits), B, N, F), k)
        assert torch.equal(T.keep_bnf(T.unpack_keep(torch.from_numpy(bits)), B, N, F), k)
    # replica rows -> engine bits -> rows, and the bit order: bit i of byte j is channel 8 j + i, row b N + n is (b, n)
    seed = 12345 + (7 << 32)
    full = T.replica_keep_rows(seed, 1, B, N, Fp, case["ff_dropout"])
    bits = T.pack_keep(full)
    assert np.array_equal(T.unpack_keep(bits), full)
    keeps = T.replica_keeps(seed, cfg, B, N)
    assert keeps[1].dtype == torch.bool and keeps[1].shape == (B, N, F)
    for b, n, j, i in ((0, 0, 0, 0), (B - 1, N // 2, 3, 5), (1, N - 1, F // 8 - 1, 7)):
        assert bool(bits[b * N + n, j] >> i & 1) == bool(full[b * N + n, 8 * j + i]) == bool(keeps[1][b, n, 8 * j + i])
    assert torch.equal(T.replica_keeps(seed, cfg, B, N, layers=[1, 0])[0], keeps[1])
    kept = float(torch.cat([k.reshape(-1) for k in keeps]).float().mean())
    assert abs(kept - (1 - case["ff_dropout"])) < 0.03
    # replica forgetful mask -> the [B, N] bool prepare_ids takes: num_drop dropped per row, never position 0
    forget = T.replica_forget(seed, 3, B, N, 0.15)
    assert forget.dtype == bool and forget.shape == (B, N) and forget[:, 0].all()
    assert ((~forget).sum(1) == T.num_drop(N, 0.15)).all()
    _, mask, _ = R.prepare_ids(cfg, [t.numpy() for t in fx["tokens"]], True, forget)
    assert np.array_equal(mask, fx["key_mask"].numpy() & forget)


WRONG = ["next seed", "next stream", "no 1/(1-p)", "layers swapped", "no forgetful mask"]


def wrong_step(variant, cfg, sd, toks, seed, stream):
    B, N = toks[0].shape[0], T.seq_len(cfg, toks)
    forget = T.replica_forget(seed + (variant == "next seed"), stream + (variant == "next stream"), B, N, cfg.mask_prob)
    keeps = T.replica_keeps(seed + (variant == "next seed"), cfg, B, N,
                            layers=list(reversed(range(cfg.depth))) if variant == "layers swapped" else None)
    return T.oracle_step(cfg, sd, toks, None if variant == "no forgetful mask" else forget, keeps, scale=variant != "no 1/(1-p)")


@pytest.mark.parametrize("variant", WRONG)
@pytest.mark.parametrize("name", CASES)
def test_wrong_masks_move_every_gradient_past_the_bound(name, variant):
    case = TRAIN[name]
    fx = source(case)
    cfg = T.cfg_of(fx, case["ff_dropout"])
    assert cfg.depth == 2                  # "layers swapped" exchanges two different streams
    toks = [t.numpy() for t in fx["tokens"]]
    seed, stream = 5 + (3 << 32), 2
    right = wrong_step(None, cfg, fx["state_dict"], toks, seed, stream)
    wrong = wrong_step(variant, cfg, fx["state_dict"], toks, seed, stream)
    errs = T.grad_errors(wrong[3], right[3])
    assert len(errs) >= 20
    assert T.GRAD_REL_BF16 >= T.GRAD_REL
    passing = [(k, round(c, 5), round(r, 4)) for k, c, r in errs if c >= T.GRAD_COS and r <= T.GRAD_REL_BF16]
    assert not passing, (variant, passing)
    median = float(np.median([r for _, _, r in errs]))
    print(f"{name} {variant}: median gradient rel {median:.3f}, smallest {min(r for _, _, r in errs):.3f}, "
          f"loss rel {abs(wrong[0] - right[0]) / right[0]:.2e}")
    assert median >= 3 * T.GRAD_REL_BF16, (variant, median)
