"""Prefixes of different lengths in one generate call (`generate(pred_lengths=...)`), host side: the argument checks,
the float restatement that defines a ragged batch's tokens (oracle/restatement.py's generate run one row at a time) and
the stage wrappers' plumbing.  tests/test_generate_ragged_gpu.py runs the decode path against the same restatement."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import open_musiclm_b200 as O
from oracle import restatement as R
from open_musiclm_b200.decode import check_pred_lengths


# ------------------------------------------------------------------------------------------------ the restatement
def ragged_reference(cfg, sd, cond, uniform, pred, lengths, max_time_steps, return_trace=False, **kw):
    """The tokens a ragged batch must give: row b is oracle generate on that row alone, with its first lengths[b] time
    steps of pred as the prefix and slices 0, 1, ... of uniform[:, b] as its Gumbel draws; rows are right-padded with
    -1 to the widest row.  cond: list of [B, n] arrays, pred: [B, steps, q] array, uniform: [n_new_max, B, C] tensor.
    return_trace: also the per-row traces of oracle generate (logits, top-2 gap of every sampled token)."""
    B = cond[0].shape[0]
    q = cfg.seqs[-1].num_quantizers
    rows, traces = [], []
    for b in range(B):
        pb = np.asarray(pred)[b:b + 1, :lengths[b]]
        out, trace = R.generate(cfg, sd, [np.asarray(t)[b:b + 1] for t in cond], lambda s, shape, b=b: uniform[s, b][None],
                                pred_token_ids=pb, max_time_steps=max_time_steps, return_trace=True, **kw)
        rows.append(out.reshape(-1))
        traces.append(trace)
    width = max(max_time_steps, max(lengths)) * q
    res = torch.full((B, width), -1, dtype=torch.int64)
    for b, r in enumerate(rows):
        res[b, :r.numel()] = r
    res = res.view(B, -1, q)
    return (res, traces) if return_trace else res


def tiny_coarse(seed=0):
    cfg = R.coarse_cfg(dim=64, depth=1, heads=2, codebook=16, n_clap_q=2, n_coarse_q=3)
    return cfg, R.init_state(cfg, seed)


def _inputs(B, n_sem, steps, C, n_new, seed):
    g = torch.Generator().manual_seed(seed)
    cond = [torch.randint(0, 16, (B, 2), generator=g).numpy(), torch.randint(0, 16, (B, n_sem), generator=g).numpy()]
    pred = torch.randint(0, 16, (B, steps, 3), generator=g).numpy()
    uni = torch.rand(n_new, B, C, generator=g).clamp_(1e-6, 1 - 1e-6)
    return cond, pred, uni


def test_reference_of_equal_lengths_is_the_batched_generate():
    """With every row at the full prefix length the restatement is oracle generate on the whole batch."""
    cfg, sd = tiny_coarse()
    T, steps = 4, 2
    cond, pred, uni = _inputs(3, 5, steps, 17, (T - steps) * 3, 1)
    batched = R.generate(cfg, sd, cond, lambda s, shape: uni[s], pred_token_ids=pred, max_time_steps=T)
    assert torch.equal(ragged_reference(cfg, sd, cond, uni, pred, [steps] * 3, T), batched)


def test_reference_rows_follow_their_own_length():
    """Row 0 with no prefix is generate without pred_token_ids, a full-prefix row past max_time_steps is its prefix
    (then -1), and a row reads only its first n_new slices of the uniform stream: the others can hold anything."""
    cfg, sd = tiny_coarse(3)
    T, steps = 3, 4
    lengths = [0, 2, 4, 1]
    n_new_b = [max(0, (T - n) * 3) for n in lengths]
    cond, pred, uni = _inputs(4, 3, steps, 17, max(n_new_b), 2)
    pred[1, 2:] = -1                                         # padding is never read
    out = ragged_reference(cfg, sd, cond, uni, pred, lengths, T)
    assert out.shape == (4, 4, 3)
    alone = R.generate(cfg, sd, [t[:1] for t in cond], lambda s, shape: uni[s, :1], pred_token_ids=None, max_time_steps=T)
    assert torch.equal(out[0, :T], alone[0])
    assert torch.equal(out[0, T:], torch.full((1, 3), -1))
    assert torch.equal(out[2], torch.from_numpy(pred[2]))    # 4 steps > max_time_steps: nothing sampled
    assert torch.equal(out[1, :2], torch.from_numpy(pred[1, :2])) and torch.equal(out[3, :1], torch.from_numpy(pred[3, :1]))
    assert bool((out[1, T:] == -1).all()) and bool((out[3, T:] == -1).all())
    other = uni.clone()
    for b, k in enumerate(n_new_b):
        other[k:, b] = torch.rand(other.shape[0] - k, other.shape[2], generator=torch.Generator().manual_seed(b))
    assert torch.equal(ragged_reference(cfg, sd, cond, other, pred, lengths, T), out)


# ------------------------------------------------------------------------------------------------ argument checks
def test_check_pred_lengths():
    pred = torch.zeros(3, 5, 2, dtype=torch.int64)
    assert check_pred_lengths(None, pred, 3) is None
    assert check_pred_lengths(None, None, 3) is None
    assert check_pred_lengths([5, 5, 5], pred, 3) is None                          # nothing ragged
    assert check_pred_lengths(torch.tensor([5, 5, 5]), pred, 3) is None
    assert check_pred_lengths([0, 5, 2], pred, 3) == [0, 5, 2]
    assert check_pred_lengths(torch.tensor([0, 5, 2]), pred, 3) == [0, 5, 2]
    assert check_pred_lengths(np.array([1, 2, 3]), pred, 3) == [1, 2, 3]
    assert check_pred_lengths((np.int32(4), 3, 0), pred, 3) == [4, 3, 0]
    assert check_pred_lengths([2, 2, 2], pred, 3) == [2, 2, 2]                     # equal, but shorter than the prefix


BAD = [
    ("count", dict(pred_lengths=[1, 2])),
    ("count", dict(pred_lengths=[1, 2, 3, 4])),
    ("count", dict(pred_lengths=torch.tensor([1, 2]))),
    ("range", dict(pred_lengths=[1, 6, 2])),
    ("range", dict(pred_lengths=[-1, 2, 2])),
    ("range", dict(pred_lengths=torch.tensor([0, 0, 9]))),
    ("type", dict(pred_lengths=[1.0, 2, 3])),
    ("type", dict(pred_lengths=[1, "2", 3])),
    ("type", dict(pred_lengths=torch.tensor([1.0, 2.0, 3.0]))),
    ("type", dict(pred_lengths=torch.tensor([1, 2, 3], dtype=torch.int32))),
    ("type", dict(pred_lengths=torch.tensor([[1, 2, 3]]))),
    ("bool", dict(pred_lengths=[True, 2, 3])),
    ("bool", dict(pred_lengths=[1, 2, False])),
    ("missing", dict(pred_lengths=[1, 2, 3], pred_token_ids=None)),
]


@pytest.mark.parametrize("what,kw", BAD, ids=[f"{w}-{i}" for i, (w, _) in enumerate(BAD)])
def test_bad_pred_lengths_raise_before_anything_runs(what, kw):
    """Every bad pred_lengths is a ValueError from generate before it touches the engine (on this CPU-only model the
    engine's first use raises OmlmError, so reaching it would fail the test)."""
    m = O.create_coarse_transformer(dim=64, depth=1, heads=2, clap_codebook_size=16, semantic_codebook_size=16,
                                    acoustic_codebook_size=16, num_clap_quantizers=2, num_coarse_quantizers=3)
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    args = dict(conditioning_token_ids=[torch.zeros(3, 2, dtype=torch.int64), torch.zeros(3, 4, dtype=torch.int64)],
                pred_token_ids=torch.zeros(3, 5, 3, dtype=torch.int64), max_time_steps=8)
    args.update(kw)
    with pytest.raises(ValueError, match="pred_lengths"):
        w.generate(**args)
    # a good value gets past the check, to the engine
    args.update(pred_lengths=[0, 5, 3], pred_token_ids=torch.zeros(3, 5, 3, dtype=torch.int64))
    with pytest.raises(O.lib.OmlmError):
        w.generate(**args)


# ------------------------------------------------------------------------------------------------ stage plumbing
class RecordingWrapper:
    """Stands in for TokenConditionedTransformerWrapper: records each generate call's keywords and returns zeros."""

    def __init__(self, q, cb, log):
        self.token_sequences = [SimpleNamespace(codebook_size=cb, num_quantizers=q)] * 3
        self.device = torch.device("cpu")
        self.q, self.log = q, log

    def generate(self, *, conditioning_token_ids, pred_token_ids=None, max_time_steps, **kw):
        self.log.append(dict(kw, pred_token_ids=pred_token_ids, max_time_steps=max_time_steps))
        return torch.zeros(conditioning_token_ids[0].shape[0], max_time_steps, self.q, dtype=torch.int64)


def test_stage_wrappers_pass_pred_lengths_and_take_the_longest_row_of_noise():
    log = []
    stages = [O.SemanticStage(semantic_transformer=None, wrapper=RecordingWrapper(1, 16, log)),
              O.CoarseStage(coarse_transformer=None, wrapper=RecordingWrapper(3, 16, log)),
              O.FineStage(fine_transformer=None, wrapper=RecordingWrapper(5, 16, log))]
    clap, sem, coarse = torch.zeros(2, 4, dtype=torch.int64), torch.zeros(2, 6, dtype=torch.int64), torch.zeros(2, 6, 3, dtype=torch.int64)
    calls = [(stages[0], dict(clap_token_ids=clap, semantic_token_ids=torch.zeros(2, 5, dtype=torch.int64)), 1),
             (stages[1], dict(clap_token_ids=clap, semantic_token_ids=sem, coarse_token_ids=torch.zeros(2, 5, 3, dtype=torch.int64)), 3),
             (stages[2], dict(clap_token_ids=clap, coarse_token_ids=coarse, fine_token_ids=torch.zeros(2, 5, 5, dtype=torch.int64)), 5)]
    for st, args, q in calls:
        lengths = [1, 4]
        noise = O.NoiseStream(torch.rand(100, 2, 17))
        st.generate(max_time_steps=7, noise=noise, pred_lengths=lengths, **args)
        assert log[-1]["pred_lengths"] == lengths
        assert log[-1]["uniform_noise"].shape[0] == (7 - 1) * q == noise.at            # the row that samples most
        # seeded, without a noise stream: handed through as is
        st.generate(max_time_steps=7, pred_lengths=torch.tensor([5, 0]), seeds=[1, 2], **args)
        assert torch.equal(log[-1]["pred_lengths"], torch.tensor([5, 0])) and log[-1]["seeds"] == [1, 2]
        # a bad value raises before the stream is touched
        noise = O.NoiseStream(torch.rand(100, 2, 17))
        with pytest.raises(ValueError, match="pred_lengths"):
            st.generate(max_time_steps=7, noise=noise, pred_lengths=[1, 9], **args)
        assert noise.at == 0
