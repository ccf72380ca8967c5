"""bench.py's training step at its own batch, sequence by sequence, against the fp32 oracle (oracle/restatement.py).

test_parity_gpu.py checks cfg2 and cfg3 at batch 1 - 2 with whole-tensor norms.  bench.py times batch 16 (cfg2, the
headline) and 8 (cfg3, the fine stage with the remainder heads), and one whole-tensor rel-L2 dilutes an error confined to
one sequence by sqrt(B): a batch-indexing bug in the last sequence would pass it (tests/test_bench_step_cpu.py).  Here
each workload is built as bench.py builds it (COMMON, TRAIN, synth_batch), at depth 1 (the per-layer forms repeat
unchanged across layers), and checked at bench.py's batch:
  * logits of the API forward in eval mode, for every sequence b and every returned tensor, rel-L2 <= 1e-2 each, and
    each sequence's cross entropy, rel <= 1e-2;
  * the trainer's eager training-mode micro-batch (FFN dropout 0.1, forgetful mask 0.15), in both OMLM_ACT16 modes and
    both kernel modes: the masks it drew equal the host replica's at its seed and stream id, and its loss and every
    parameter gradient equal the oracle's under those masks (test_parity_gpu.check_grads' bounds)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(__file__))
import test_train_mode_gpu as TM  # noqa: E402

import bench  # noqa: E402
from oracle import restatement as R  # noqa: E402

pytestmark = pytest.mark.gpu
SEQ_BOUND = 1e-2        # logits rel-L2 per sequence and per returned tensor; CE rel per sequence
WORKLOADS = ["cfg2", "cfg3"]


def per_sequence_rel(got, ref):
    """rel-L2 of got against ref for each sequence b (dim 0): [B] floats."""
    d = (got.double().cpu() - ref.double().cpu()).flatten(1).norm(dim=1)
    return (d / ref.double().cpu().flatten(1).norm(dim=1).clamp_min(1e-30)).tolist()


def whole_rel(got, ref):
    return float((got.double().cpu() - ref.double().cpu()).norm() / ref.double().cpu().norm().clamp_min(1e-30))


def sequence_fails(got, ref, tag, bound=SEQ_BOUND):
    """The sequences whose rel-L2 reaches the bound, as messages."""
    return [f"{tag} sequence {b}: rel-L2 {r:.3e} >= {bound:.0e}" for b, r in enumerate(per_sequence_rel(got, ref)) if not r < bound]


# ------------------------------------------------------------------------------------------------ the workloads
_CASES = {}


def case_of(key):
    """bench.py's workload `key` at depth 1: weights of torch.manual_seed(0) (as bench.measure), one batch of synth_batch
    at the workload's batch and shapes, the oracle config with the same ce weights, dropout 0.1 and mask_prob 0.15."""
    if key not in _CASES:
        import open_musiclm_b200 as O
        wl = bench.WORKLOADS[key]
        kw = dict(bench.COMMON, **dict(wl["model"], depth=1))
        make = {"coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}[wl["stage"]]
        torch.manual_seed(0)
        sd = {k: v.clone() for k, v in make(**kw).state_dict().items()}
        toks = bench.synth_batch(wl["batch"], torch.Generator().manual_seed(1234), wl["shapes"])
        m = wl["model"]
        common = dict(dim=kw["dim"], depth=1, heads=m["heads"], n_clap_q=wl["shapes"][0][0], ff_dropout=kw["ff_dropout"],
                      mask_prob=TM.MASK_PROB, grad_shrink_alpha=kw["grad_shrink_alpha"], ce_weights=list(bench.TRAIN["ce_weights"]))
        cfg = (R.coarse_cfg(n_coarse_q=m["num_coarse_quantizers"], **common) if wl["stage"] == "coarse" else
               R.fine_cfg(n_coarse_q=m["num_coarse_quantizers"], n_fine_q=m["num_fine_quantizers"], **common))
        _CASES[key] = TM.Case(wl["stage"], kw, sd, toks, list(bench.TRAIN["ce_weights"]), cfg)
        assert (_CASES[key].B, _CASES[key].N) == (wl["batch"], wl["N"])
    return _CASES[key]


_EVAL = {}


def eval_oracle(key):
    if key not in _EVAL:
        c = case_of(key)
        with torch.no_grad():
            _EVAL[key] = R.loss_and_logits(c.cfg, c.sd, [t.numpy() for t in c.tokens])
    return _EVAL[key]


def per_sequence_ce(logits, labels, weights):
    """The wrapper's token-count-weighted cross entropy of each sequence b alone: [B] floats."""
    B = labels[0].shape[0]
    out = []
    for b in range(B):
        num = den = 0.0
        for lg, lb, w in zip(logits, labels, weights):
            if w > 0 and lg is not None:
                lab = torch.from_numpy(np.asarray(lb[b])).long().reshape(-1)
                num += w * float(F.cross_entropy(lg[b].double().cpu().reshape(-1, lg.shape[-1]), lab, reduction="sum"))
                den += lab.numel()
        out.append(num / den)
    return out


# ------------------------------------------------------------------------------------------------ the tests
@pytest.mark.parametrize("act16", ["fp16", "bf16"])
@pytest.mark.parametrize("key", WORKLOADS)
def test_bench_forward_per_sequence_vs_oracle(key, act16, monkeypatch):
    """The API forward (eval) on the ids and key mask the oracle prepared: every returned tensor of every sequence and
    every sequence's cross entropy within 1e-2 of the oracle's."""
    c = case_of(key)
    m = TM.build(c, act16, monkeypatch, train=False)
    _, logits_ref, labels, ids, mask = eval_oracle(key)
    with torch.no_grad():
        logits = m(all_token_ids=[torch.from_numpy(i).cuda() for i in ids], self_attn_mask=torch.from_numpy(mask).cuda())
    torch.cuda.synchronize()
    fails = []
    assert len(logits) == len(logits_ref)
    for s, (a, b) in enumerate(zip(logits, logits_ref)):
        assert a.shape == b.shape, (key, s, a.shape, b.shape)
        r = per_sequence_rel(a, b)
        print(f"METRIC bench {key} {act16} logits[{s}]: worst sequence rel-L2 {max(r):.3e} (sequence {int(np.argmax(r))}), "
              f"whole {whole_rel(a, b):.3e}")
        fails += sequence_fails(a, b, f"{key} {act16} logits[{s}]")
    got = per_sequence_ce([lg.detach() for lg in logits], labels, c.ce)
    want = per_sequence_ce(logits_ref, labels, c.ce)
    r = [abs(x - y) / abs(y) for x, y in zip(got, want)]
    print(f"METRIC bench {key} {act16} per-sequence CE: worst rel {max(r):.3e} (sequence {int(np.argmax(r))})")
    fails += [f"{key} {act16} sequence {b}: CE {x:.6f}, oracle {y:.6f}" for b, (x, y, e) in enumerate(zip(got, want, r))
              if not e <= SEQ_BOUND]
    assert not fails, "\n".join(fails)


_TRAIN = {}


@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
@pytest.mark.parametrize("act16", ["fp16", "bf16"])
@pytest.mark.parametrize("key", WORKLOADS)
def test_bench_training_step_every_gradient_vs_oracle(key, act16, det, monkeypatch):
    """The trainer's eager micro-batch at bench.py's batch in training mode: the keep bits of the layer and the key mask
    are the replica's at (eng.seed, stream id); the loss and every parameter gradient are the oracle's under them."""
    c = case_of(key)
    m, tr, masks, loss = TM.eager_step(c, act16, det, monkeypatch)
    eng = tr.eng
    seed, stream = int(eng.seed.item()), tr._mask_draws
    assert stream == 1 and len(masks) == 1
    tag = f"bench-{key}-{act16}-{'det' if det else 'default'}"
    TM.assert_keep_bits(TM.train_workspace(eng), c, seed, tag)
    TM.assert_key_mask(masks[0], c, seed, stream, tag)
    if (seed, stream) not in _TRAIN.setdefault(key, {}):     # every fresh trainer draws the same masks: one oracle run each
        _TRAIN[key][(seed, stream)] = TM.T.oracle_step(c.cfg, c.sd, [t.numpy() for t in c.tokens],
                                                       TM.T.replica_forget(seed, stream, c.B, c.N, TM.MASK_PROB),
                                                       TM.T.replica_keeps(seed, c.cfg, c.B, c.N))
    loss_ref, _, _, grads_ref = _TRAIN[key][(seed, stream)]
    print(f"METRIC bench {tag} loss {loss:.6f} oracle {loss_ref:.6f}")
    assert abs(loss - loss_ref) / loss_ref <= 1e-2, (tag, loss, loss_ref)
    TM.compare_grads(TM.grads_of(m, eng.gview), grads_ref, tag, act16)
