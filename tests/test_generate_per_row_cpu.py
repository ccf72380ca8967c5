"""Sampling arguments per row in one generate call (`generate(temperature=[...], filter_thres=[...], top_p=[...],
max_time_steps=[...])`), host side: the argument checks and the collapse of equal values, the float restatement that
defines a per-row batch's tokens (oracle generate run one row at a time with that row's scalars, through
ragged_reference for ragged prefixes) and the stage wrappers' plumbing.  tests/test_generate_per_row_gpu.py runs the
decode path against the same restatement."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import open_musiclm_b200 as O  # noqa: E402
from oracle import restatement as R  # noqa: E402
from open_musiclm_b200.decode import check_sampling_rows  # noqa: E402
from test_generate_ragged_cpu import RecordingWrapper, _inputs, ragged_reference, tiny_coarse  # noqa: E402


# ------------------------------------------------------------------------------------------------ the restatement
def per_row_reference(cfg, sd, cond, uniform, pred, lengths, max_time_steps, temperature, filter_thres, return_trace=False, **kw):
    """The tokens a batch with per-row sampling arguments must give: row b is ragged_reference of that row alone (oracle
    generate with its first lengths[b] steps of pred as the prefix, slices 0, 1, ... of uniform[:, b]) at the scalars
    max_time_steps[b], temperature[b] and filter_thres[b]; rows are right-padded with -1 to the widest row,
    max over b of max(max_time_steps[b], lengths[b]) steps.  cond: list of [B, n] arrays, pred: [B, steps, q] array,
    uniform: [n_new_max, B, C] tensor; lengths, max_time_steps, temperature, filter_thres: B values each.
    return_trace: also the per-row traces of oracle generate."""
    B = cond[0].shape[0]
    q = cfg.seqs[-1].num_quantizers
    rows, traces = [], []
    for b in range(B):
        out, tr = ragged_reference(cfg, sd, [np.asarray(t)[b:b + 1] for t in cond], uniform[:, b:b + 1], np.asarray(pred)[b:b + 1],
                                   [lengths[b]], max_time_steps[b], return_trace=True, temperature=float(temperature[b]),
                                   filter_thres=float(filter_thres[b]), **kw)
        rows.append(out.reshape(-1))
        traces.append(tr[0])
    width = max(max(t, n) for t, n in zip(max_time_steps, lengths)) * q
    res = torch.full((B, width), -1, dtype=torch.int64)
    for b, r in enumerate(rows):
        res[b, :r.numel()] = r
    res = res.view(B, -1, q)
    return (res, traces) if return_trace else res


def test_reference_of_equal_values_is_the_batched_generate():
    """With every row at the same arguments and the full prefix, the restatement is oracle generate on the whole batch;
    with ragged prefixes it is ragged_reference."""
    cfg, sd = tiny_coarse()
    T, steps = 4, 2
    cond, pred, uni = _inputs(3, 5, steps, 17, (T - steps) * 3, 1)
    batched = R.generate(cfg, sd, cond, lambda s, shape: uni[s], pred_token_ids=pred, max_time_steps=T, temperature=0.7,
                         filter_thres=0.5)
    assert torch.equal(per_row_reference(cfg, sd, cond, uni, pred, [steps] * 3, [T] * 3, [0.7] * 3, [0.5] * 3), batched)
    lengths = [0, 2, 1]
    cond, pred, uni = _inputs(3, 5, steps, 17, T * 3, 2)
    assert torch.equal(per_row_reference(cfg, sd, cond, uni, pred, lengths, [T] * 3, [0.7] * 3, [0.5] * 3),
                       ragged_reference(cfg, sd, cond, uni, pred, lengths, T, temperature=0.7, filter_thres=0.5))


def test_reference_rows_follow_their_own_arguments():
    """Each row is oracle generate of that row alone with its own temperature, top-k share and length; a row whose
    max_time_steps does not pass its prefix is its prefix, then -1; a row reads only its first n_new slices."""
    cfg, sd = tiny_coarse(5)
    steps = 2
    lengths = [2, 2, 1, 0]
    T = [5, 2, 3, 4]
    temps, thres = [0.3, 1.0, 2.5, 0.9], [0.0, 0.9, 0.5, 0.7]
    n_new_b = [max(0, (t - n) * 3) for t, n in zip(T, lengths)]
    cond, pred, uni = _inputs(4, 3, steps, 17, max(n_new_b), 3)
    out = per_row_reference(cfg, sd, cond, uni, pred, lengths, T, temps, thres)
    assert out.shape == (4, 5, 3)
    for b in range(4):
        pb = pred[b:b + 1, :lengths[b]] if lengths[b] else None
        alone = R.generate(cfg, sd, [t[b:b + 1] for t in cond], lambda s, shape, b=b: uni[s, b][None], pred_token_ids=pb,
                           max_time_steps=T[b], temperature=temps[b], filter_thres=thres[b])
        w = alone.shape[1]
        assert torch.equal(out[b, :w], alone[0]) and bool((out[b, w:] == -1).all()), b
    assert torch.equal(out[1, :2], torch.from_numpy(pred[1])) and bool((out[1, 2:] == -1).all())     # samples nothing
    other = uni.clone()
    for b, k in enumerate(n_new_b):
        other[k:, b] = torch.rand(other.shape[0] - k, other.shape[2], generator=torch.Generator().manual_seed(b))
    assert torch.equal(per_row_reference(cfg, sd, cond, other, pred, lengths, T, temps, thres), out)


# ------------------------------------------------------------------------------------------------ argument checks
def test_check_sampling_rows_forms_and_collapse():
    C = 17
    # single values pass through as today (top_k None: computed from filter_thres where generate needs it)
    assert check_sampling_rows(3, C, 0.7, 0.9, None, 8) == (0.7, None, None, 8)
    assert check_sampling_rows(3, C, 0.7, 0.9, 1.0, 8) == (0.7, None, None, 8)
    assert check_sampling_rows(3, C, 0.7, 0.9, 0.5, 8)[2] == 0.5
    # lists, tuples and tensors of equal values are that single value
    assert check_sampling_rows(3, C, [0.7] * 3, (0.5,) * 3, [None, 1, 1.0], torch.tensor([8, 8, 8])) == (0.7, 8, None, 8)
    assert check_sampling_rows(3, C, torch.full((3,), 0.5), torch.full((3,), 0.5, dtype=torch.float64), torch.ones(3), [4] * 3) \
        == (0.5, 8, None, 4)
    assert check_sampling_rows(3, C, 1.0, [0.9, 0.92, 0.95], 0.5, 8)[1] == 1                        # the same k = 1
    # per-row values
    temp, k, p, steps = check_sampling_rows(3, C, [0.5, 1, np.float32(2.0)], [0.0, 0.5, 0.9], (None, 0.9, 1e-7),
                                            torch.tensor([0, 3, 9]))
    assert temp == [0.5, 1.0, 2.0] and k == [17, 8, 1] and p == [None, 0.9, 1e-7] and steps == [0, 3, 9]
    assert check_sampling_rows(2, C, torch.tensor([0.3, 0.1], dtype=torch.float64), 0.9, torch.tensor([1.0, 0.25]), 8)[0::2] \
        == ([0.3, 0.1], [None, 0.25])
    assert check_sampling_rows(3, C, 0.7, [-0.05, 0.5, 1.5], None, 8)[1] == [17, 8, 1]  # k = C at the edge
    assert check_sampling_rows(2, C, torch.tensor(0.5), 0.9, None, 8)[0].dim() == 0                  # a 0-d tensor is one value


BAD = [
    ("temperature", [0.5, 1.0]), ("temperature", torch.tensor([0.5, 1.0, 1.0, 1.0])), ("temperature", [True, 1.0, 1.0]),
    ("temperature", ["1", 1.0, 1.0]), ("temperature", [None, 1.0, 1.0]), ("temperature", [math.nan, 1.0, 1.0]),
    ("temperature", [math.inf, 1.0, 1.0]), ("temperature", [0.0, 1.0, 1.0]), ("temperature", [1.0, -0.5, 1.0]),
    ("temperature", torch.tensor([1, 1, 2])), ("temperature", torch.ones(1, 3)), ("temperature", torch.tensor([1.0, math.nan, 1.0])),
    ("filter_thres", [0.9, 0.9]), ("filter_thres", [math.nan, 0.9, 0.9]), ("filter_thres", [0.9, -math.inf, 0.9]),
    ("filter_thres", [0.9, 0.9, -0.1]), ("filter_thres", [False, 0.9, 0.9]), ("filter_thres", ["0.9", 0.9, 0.9]),
    ("filter_thres", torch.tensor([0, 0, 1])),
    ("top_p", [0.5, 0.5]), ("top_p", [0.0, 0.5, 0.5]), ("top_p", [0.5, 1.5, 0.5]), ("top_p", [math.nan, 0.5, 0.5]),
    ("top_p", [True, 0.5, 0.5]), ("top_p", ["0.9", 0.5, 0.5]), ("top_p", torch.tensor([0.5, 2.0, 0.5])),
    ("top_p", torch.tensor([1, 1, 1])), ("top_p", torch.tensor([0.5, -0.5, 0.5])),
    ("max_time_steps", [8, 8]), ("max_time_steps", [8.0, 8, 8]), ("max_time_steps", [True, 8, 8]), ("max_time_steps", [8, -1, 8]),
    ("max_time_steps", ["8", 8, 8]), ("max_time_steps", torch.tensor([8.0, 8.0, 9.0])),
    ("max_time_steps", torch.tensor([8, 8, 9], dtype=torch.int32)), ("max_time_steps", torch.tensor([[8, 8, 9]])),
]


@pytest.mark.parametrize("name,value", BAD, ids=[f"{n}-{i}" for i, (n, _) in enumerate(BAD)])
def test_bad_per_row_values_raise_before_anything_runs(name, value):
    """Every bad per-row value is a ValueError naming its keyword, from generate before it touches the engine (on this
    CPU-only model the engine's first use raises OmlmError, so reaching it would fail the test)."""
    m = O.create_coarse_transformer(dim=64, depth=1, heads=2, clap_codebook_size=16, semantic_codebook_size=16,
                                    acoustic_codebook_size=16, num_clap_quantizers=2, num_coarse_quantizers=3)
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    args = dict(conditioning_token_ids=[torch.zeros(3, 2, dtype=torch.int64), torch.zeros(3, 4, dtype=torch.int64)],
                pred_token_ids=torch.zeros(3, 5, 3, dtype=torch.int64), max_time_steps=8)
    with pytest.raises(ValueError, match=name):
        w.generate(**dict(args, **{name: value}))
    # good per-row values of every keyword get past the checks, to the engine
    good = dict(temperature=[0.5, 1.0, 2.0], filter_thres=torch.tensor([0.0, 0.5, 0.9]), top_p=[None, 0.9, 1],
                max_time_steps=torch.tensor([0, 6, 9]))
    with pytest.raises(O.lib.OmlmError):
        w.generate(**dict(args, **good))


# ------------------------------------------------------------------------------------------------ stage plumbing
class PerRowRecordingWrapper(RecordingWrapper):
    """RecordingWrapper whose output is as wide as the longest row's max_time_steps."""

    def generate(self, *, conditioning_token_ids, pred_token_ids=None, max_time_steps, **kw):
        steps = max_time_steps if isinstance(max_time_steps, int) else max(int(v) for v in max_time_steps)
        super().generate(conditioning_token_ids=conditioning_token_ids, pred_token_ids=pred_token_ids, max_time_steps=steps, **kw)
        self.log[-1]["max_time_steps"] = max_time_steps
        return torch.zeros(conditioning_token_ids[0].shape[0], steps, self.q, dtype=torch.int64)


def test_stage_wrappers_pass_per_row_values_and_take_the_longest_row_of_noise():
    log = []
    stages = [O.SemanticStage(semantic_transformer=None, wrapper=PerRowRecordingWrapper(1, 16, log)),
              O.CoarseStage(coarse_transformer=None, wrapper=PerRowRecordingWrapper(3, 16, log)),
              O.FineStage(fine_transformer=None, wrapper=PerRowRecordingWrapper(5, 16, log))]
    clap, sem, coarse = torch.zeros(2, 4, dtype=torch.int64), torch.zeros(2, 6, dtype=torch.int64), torch.zeros(2, 6, 3, dtype=torch.int64)
    calls = [(stages[0], dict(clap_token_ids=clap, semantic_token_ids=torch.zeros(2, 5, dtype=torch.int64)), 1),
             (stages[1], dict(clap_token_ids=clap, semantic_token_ids=sem, coarse_token_ids=torch.zeros(2, 5, 3, dtype=torch.int64)), 3),
             (stages[2], dict(clap_token_ids=clap, coarse_token_ids=coarse, fine_token_ids=torch.zeros(2, 5, 5, dtype=torch.int64)), 5)]
    for st, args, q in calls:
        per_row = dict(temperature=[0.5, 1.5], filter_thres=(0.9, 0.5), top_p=torch.tensor([0.9, 1.0]))
        noise = O.NoiseStream(torch.rand(100, 2, 17))
        st.generate(max_time_steps=[9, 6], noise=noise, **per_row, **args)
        rec = log[-1]
        assert rec["max_time_steps"] == [9, 6] and rec["temperature"] == [0.5, 1.5] and rec["filter_thres"] == (0.9, 0.5)
        assert torch.equal(rec["top_p"], per_row["top_p"])
        assert rec["uniform_noise"].shape[0] == (9 - 5) * q == noise.at                # the row that samples most
        # with pred_lengths: the longest row is the one with the most steps left
        noise = O.NoiseStream(torch.rand(100, 2, 17))
        st.generate(max_time_steps=torch.tensor([3, 7]), pred_lengths=[1, 4], noise=noise, **args)
        assert noise.at == (7 - 4) * q and torch.equal(log[-1]["max_time_steps"], torch.tensor([3, 7]))
        # seeded, without a noise stream: handed through as is
        st.generate(max_time_steps=[2, 8], seeds=[1, 2], **per_row, **args)
        assert log[-1]["max_time_steps"] == [2, 8] and log[-1]["seeds"] == [1, 2]
        # a bad value raises before the stream is touched
        for bad in (dict(temperature=[1.0, -1.0]), dict(top_p=[0.5, 2.0]), dict(filter_thres=[0.9]), dict(max_time_steps=[9, -1])):
            noise = O.NoiseStream(torch.rand(100, 2, 17))
            with pytest.raises(ValueError, match=next(iter(bad))):
                st.generate(**dict(dict(max_time_steps=9), **bad), noise=noise, **args)
            assert noise.at == 0
