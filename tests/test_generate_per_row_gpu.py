"""Sampling arguments per row in one generate call on the H100: omlm_sample_rows against the host references
(nucleus_reference, the Philox replicas) and against the single-value samplers row by row, bit for bit; equal values
bit-identical to the single-value call; every seeded row of a mixed batch bit-identical to that row alone with its own
scalars, on both decode paths; unseeded rows against the float restatement of tests/test_generate_per_row_cpu.py."""
import itertools
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from test_generate_per_row_cpu import per_row_reference  # noqa: E402
from test_generate_ragged_gpu import NEAR_TIE, _alone, _model, _prompts, rel  # noqa: E402
from test_generate_seeded_cpu import seeded_uniforms  # noqa: E402
from test_philox_cpu import sampler_uniforms  # noqa: E402
from test_sampling_nucleus_cpu import edge_logits  # noqa: E402
from test_sampling_nucleus_gpu import check_nucleus  # noqa: E402
from test_stages_cpu import oracle_cfg  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = -7


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as L
    L.device_check()
    return L


# ------------------------------------------------------------------------------------------------ 1. the sampler kernel
def _launch(lib, x, C, mode, seed, seeds, uniform, allow, k=1, T=1.0, top_p=None, rows=None, step=0):
    """One sampler launch at sample index `step` on logits x [B, C]; rows: dict of per-row device arrays
    (omlm_sample_rows), else the single-value entry point for (k, T, top_p)."""
    B = x.shape[0]
    tokens = torch.full((B, step + 1), SENTINEL, device=DEV, dtype=torch.int64)
    counters = torch.tensor([step, 0], device=DEV, dtype=torch.int32)
    next_row = torch.full((B,), SENTINEL, device=DEV, dtype=torch.int32)
    kw = dict(seeds=seeds) if mode == "per_sequence" else {}
    lib.sample(x, C, k, T, allow, uniform if mode == "uniform" else None, seed if mode == "engine_seed" else None, tokens, next_row,
               5, counters, None, B, top_p=top_p, **kw, **(rows or {}))
    torch.cuda.synchronize()
    assert counters.tolist() == [step + 1, 0]
    ok = tokens[:, step] < C                     # a row where no class can win (a NaN temperature) has no table row
    assert torch.equal(next_row.long()[ok], tokens[ok, step] + 5)
    return tokens[:, step]


def _row_uniforms(mode, uni, seed, seeds, step, B, C):
    if mode == "uniform":
        return uni[step].cpu()
    if mode == "engine_seed":
        return torch.from_numpy(sampler_uniforms(seed, step, B, C))
    return torch.from_numpy(np.stack([seeded_uniforms(s, step, C) for s in seeds]))


def _kernel_case(C, mode, B=30):
    g = torch.Generator().manual_seed(C * 3 + len(mode))
    x = edge_logits(B, C, g, scale=4.0)
    x[6] = -torch.linspace(0, 300, C)[torch.randperm(C, generator=g)]       # exp underflows below the maximum's 300 / T
    x[6, 0] = 0.0
    ks = [1, C, 2, max(C // 2, 1)] + [int(v) for v in torch.randint(1, C + 1, (B - 4,), generator=g)]
    ks[6] = C
    temps = [float(v) for v in torch.logspace(math.log10(0.05), math.log10(5.0), B)[torch.randperm(B, generator=g)]]
    temps[6] = 1.0
    tops = [(None, 1.0, 1e-7, 0.9)[b % 4] for b in range(B)]
    tops[6] = None
    seed = 0x0123456789ABCDEF
    seeds = [int(v) for v in torch.randint(-2 ** 62, 2 ** 62, (B,), generator=g)]
    uni = torch.rand(3, B, C, generator=g, device="cpu").to(DEV)
    return x, ks, temps, tops, seed, seeds, uni


def _rows(ks, temps, tops, nucleus=True):
    return dict(top_k_rows=torch.tensor(ks, device=DEV, dtype=torch.int32),
                temperature_rows=torch.tensor(temps, device=DEV, dtype=torch.float32),
                top_p_rows=torch.tensor([1.0 if p is None else p for p in tops], device=DEV, dtype=torch.float32) if nucleus else None)


@pytest.mark.parametrize("mode", ["uniform", "engine_seed", "per_sequence"])
@pytest.mark.parametrize("C", [65, 1025, 16384])
def test_sample_rows_equals_the_references_row_by_row(lib, C, mode):
    """30 rows per launch with their own k (1 ... C), temperature (0.05 ... 5) and top_p (None, 1.0, 1e-7 and 0.9 mixed
    in one launch), on edge rows (ties, +-0.0, -inf, equal maxima, NaN) and a row whose top-k logits span 300 (p
    underflows to 0; it has top_p None in a nucleus launch); eos forbidden and allowed, sample indices 0 and 2.  Each
    row's token is bit-identical to the single-value sampler's (omlm_sample[_seeded] for None / 1.0, omlm_sample_nucleus
    otherwise) for that row's scalars, and equals the float64 reference under the host replica of the stream."""
    from open_musiclm_b200.decode import seeds_tensor
    x, ks, temps, tops, seed, seeds, uni = _kernel_case(C, mode)
    B = x.shape[0]
    xd = x.to(DEV)
    seed_t, seeds_t = torch.tensor([seed - 2 ** 64 if seed >= 2 ** 63 else seed], device=DEV), seeds_tensor(seeds, B, DEV)
    loose = 0
    for nucleus, allow, step in itertools.product((True, False), (False, True), (0, 2)):
        row_tops = tops if nucleus else [None] * B
        got = _launch(lib, xd, C, mode, seed_t, seeds_t, uni, allow, rows=_rows(ks, temps, row_tops, nucleus), step=step).cpu()
        u = _row_uniforms(mode, uni, seed, seeds, step, B, C)
        for r in range(B):
            single = _launch(lib, xd, C, mode, seed_t, seeds_t, uni, allow, k=ks[r], T=temps[r], top_p=row_tops[r], step=step)
            assert int(got[r]) == int(single[r]), (C, mode, nucleus, allow, step, r, ks[r], temps[r], row_tops[r])
            top = None if row_tops[r] in (None, 1.0) else row_tops[r]
            loose += check_nucleus(got[r:r + 1], x[r:r + 1], u[r:r + 1], ks[r], float(np.float32(temps[r])), allow, top, (C, mode, r))
    print(f"C = {C}, {mode}: {loose} rows accepted at a top_p boundary or a near tie")


def test_sample_rows_out_of_range_values_stay_in_bounds(lib):
    """Values generate never passes: k below 1 samples as k = 1 and above C as k = C; top_p outside (0, 1), NaN and
    inf included, samples without a nucleus; a NaN, zero, negative or infinite temperature finishes the launch and
    leaves the other rows' tokens as they are."""
    C, B = 1025, 16
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, C, generator=g).to(DEV)
    uni = torch.rand(1, B, C, generator=g).to(DEV)
    ks = [0, -3, -2 ** 31, C + 50, 2 ** 31 - 1, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7]
    tops = [None] * 5 + [math.nan, -1.0, 2.0, 0.0, math.inf, None, None, None, None, 0.5, 0.5]
    temps = [1.0] * 10 + [math.nan, 0.0, -1.0, math.inf, 0.7, 0.7]
    got = _launch(lib, x, C, "uniform", None, None, uni, False, rows=_rows(ks, temps, tops)).cpu()
    clamped = [1, 1, 1, C, C] + [7] * 11
    for r in range(B):
        if 10 <= r < 14:
            continue
        top = tops[r] if tops[r] is not None and 0 < tops[r] < 1 else None
        single = _launch(lib, x, C, "uniform", None, None, uni, False, k=clamped[r], T=temps[r], top_p=top)
        assert int(got[r]) == int(single[r]), r


def test_sample_rows_graph_replay_equals_eager(lib):
    C, B = 1025, 40
    x, ks, temps, tops, seed, seeds, uni = _kernel_case(C, "engine_seed", B)
    xd, rows = x.to(DEV), _rows(ks, temps, tops)
    s = torch.tensor([77], device=DEV, dtype=torch.int64)

    def run(tokens, counters, next_row):
        lib.sample(xd, C, 1, 1.0, False, None, s, tokens, next_row, 0, counters, None, B, **rows)

    bufs = [torch.full((B, 4), SENTINEL, device=DEV, dtype=torch.int64), torch.zeros(2, device=DEV, dtype=torch.int32),
            torch.zeros(B, device=DEV, dtype=torch.int32)]
    for _ in range(4):
        run(*bufs)
    eager = bufs[0].clone()
    bufs[0].fill_(SENTINEL)
    bufs[1].zero_()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run(*bufs)
    bufs[0].fill_(SENTINEL)
    bufs[1].zero_()
    for _ in range(4):
        graph.replay()
    torch.cuda.synchronize()
    assert bufs[1].tolist() == [4, 0] and torch.equal(bufs[0], eager)


# ------------------------------------------------------------------------------------------------ 2. collapse
@pytest.mark.parametrize("top_p", [None, 0.85])
@pytest.mark.parametrize("seeded", [False, True])
@pytest.mark.parametrize("B", [3, 20])
def test_equal_values_are_the_single_value_call(B, seeded, top_p):
    """Lists and tensors of equal values for all four keywords give the tokens and traced logits of the single-value
    call, bit for bit (Engine.seed reset before each unseeded call), traced and from CUDA graphs."""
    m, w, _, _ = _model()
    eng = m.engine
    g = torch.Generator().manual_seed(B + 2 * seeded)
    cond, pred, _ = _prompts(B, "coarse", 3, 64, g)
    kw = dict(conditioning_token_ids=cond, pred_token_ids=pred)
    if seeded:
        kw["seeds"] = [int(v) for v in torch.randint(0, 2 ** 62, (B,), generator=g)]
    single = dict(temperature=0.8, filter_thres=0.7, top_p=top_p, max_time_steps=7)
    forms = {"single": single,
             "list": dict(temperature=[0.8] * B, filter_thres=(0.7,) * B, top_p=[top_p] * B, max_time_steps=[7] * B),
             "tensor": dict(temperature=torch.full((B,), 0.8, dtype=torch.float64), filter_thres=torch.full((B,), 0.7, dtype=torch.float64),
                            top_p=torch.full((B,), 1.0 if top_p is None else top_p, dtype=torch.float64),
                            max_time_steps=torch.full((B,), 7, dtype=torch.int64))}
    s0 = eng.seed.clone()
    runs = {}
    for name, args in forms.items():
        for mode in ("trace", "graph"):
            eng.seed.copy_(s0)
            tr = [] if mode == "trace" else None
            runs[name, mode] = (w.generate(trace_logits=tr, **args, **kw), tr)
    for name in ("list", "tensor"):
        for mode in ("trace", "graph"):
            assert torch.equal(runs[name, mode][0], runs["single", mode][0]), (name, mode)
        tr, tr0 = runs[name, "trace"][1], runs["single", "trace"][1]
        assert len(tr) == len(tr0) and all(torch.equal(a, b) for a, b in zip(tr, tr0))


# ------------------------------------------------------------------------------------------------ 3. row alone, seeded
def _mixed_args(B, g, T, with_top_p=True):
    """Per-row temperature (0.3 ... 2), filter_thres, top_p and max_time_steps, all differing between rows; row 1
    (when B > 1) samples nothing."""
    temps = [round(0.3 + 1.7 * float(v), 4) for v in torch.rand(B, generator=g)]
    thres = [(0.0, 0.5, 0.9, 0.8, 0.95)[b % 5] for b in range(B)]
    tops = [(None, 0.9, 1e-7, 1.0, 0.5, 0.75)[b % 6] for b in range(B)] if with_top_p else [None] * B
    steps = [T - (b % 3) for b in range(B)]
    if B > 1:
        steps[1] = 0
    return temps, thres, tops, steps


SEEDED_CASES = [("coarse", 2, False, False), ("coarse", 17, True, False), ("coarse", 40, False, True), ("coarse", 256, True, False),
                ("semantic", 2, True, True), ("semantic", 17, False, False), ("semantic", 40, True, False)]


@pytest.mark.parametrize("stage,B,ragged,abs_pos", SEEDED_CASES,
                         ids=[f"{s}-B{B}-{'ragged' if r else 'full'}-{'abspos' if a else 'relpos'}" for s, B, r, a in SEEDED_CASES])
def test_seeded_rows_equal_each_row_alone(stage, B, ragged, abs_pos):
    """A seeded batch with per-row temperature, filter_thres, top_p and max_time_steps (a row that samples nothing
    included), with and without ragged pred_lengths and absolute positions: every row's tokens and the traced logits of
    its own steps are bit-identical to that row alone with its scalars; eager and graph runs of the batch agree.  At
    B = 256 every 16th row and the special rows are compared."""
    steps_pre, T = (5, 8) if stage == "coarse" else (9, 14)
    q = 3 if stage == "coarse" else 1
    extra = dict(use_absolute_position_embeddings=True, max_absolute_position_embeddings=T * q + 1) if abs_pos else {}
    m, w, _, _ = _model(stage, dim=256, heads=4, **extra)
    g = torch.Generator().manual_seed(B * 5 + ragged + 2 * abs_pos)
    cond, pred, q = _prompts(B, stage, steps_pre, 64, g)
    temps, thres, tops, steps = _mixed_args(B, g, T)
    lengths = [[0, steps_pre, 1, 3][b % 4] for b in range(B)] if ragged else None
    seeds = [int(v) for v in torch.randint(0, 2 ** 62, (B,), generator=g)]
    kw = dict(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=lengths, seeds=seeds, temperature=temps, filter_thres=thres,
              top_p=tops, max_time_steps=torch.tensor(steps))
    tr = []
    out = w.generate(trace_logits=tr, **kw)
    assert torch.equal(w.generate(**kw), out)
    assert torch.equal(w.generate(use_cuda_graph=False, **kw), out)
    n_b = lengths or [steps_pre] * B
    assert out.shape == (B, max(max(t, n) for t, n in zip(steps, n_b)), q)
    rows = range(B) if B <= 40 else sorted(set(range(0, B, 16)) | {1, 2, 3, 4, 5, B - 1})
    for b in rows:
        atr = []
        alone = _alone(w, cond, pred, b, n_b[b], seeds=[seeds[b]], trace_logits=atr, temperature=temps[b], filter_thres=thres[b],
                       top_p=tops[b], max_time_steps=steps[b])
        width = alone.shape[1]
        assert torch.equal(out[b, :width], alone[0]), (B, b)
        assert bool((out[b, width:] == -1).all()), (B, b)
        assert len(atr) == max(0, (steps[b] - n_b[b]) * q)
        for s, lg in enumerate(atr):
            assert torch.equal(tr[s][b], lg[0]), (B, b, s)


def test_per_row_absolute_position_limit():
    """With absolute positions the limit applies per row to the rows that sample: a batch whose longest row reaches
    max_absolute_position_embeddings exactly generates, every row equal to the row alone; one more step on row 2 raises
    IndexError naming it before anything runs (Engine.seed unchanged), whatever row 1, which samples nothing, holds."""
    T, q = 5, 3
    lim = T * q - 1
    m, w, _, _ = _model(use_absolute_position_embeddings=True, max_absolute_position_embeddings=lim)
    eng = m.engine
    g = torch.Generator().manual_seed(12)
    B = 4
    cond, pred, _ = _prompts(B, "coarse", 2, 64, g)
    steps, temps = [T, 1, T - 1, 3], [0.5, 0.9, 1.3, 2.0]
    seeds = [5, 6, 7, 8]
    out = w.generate(conditioning_token_ids=cond, pred_token_ids=pred, max_time_steps=steps, temperature=temps, seeds=seeds)
    for b in range(B):
        alone = _alone(w, cond, pred, b, 2, max_time_steps=steps[b], temperature=temps[b], seeds=[seeds[b]])
        assert torch.equal(out[b, :alone.shape[1]], alone[0]) and bool((out[b, alone.shape[1]:] == -1).all()), b
    seed = eng.seed.clone()
    with pytest.raises(IndexError, match=r"row 2 reaches 17 tokens"):
        w.generate(conditioning_token_ids=cond, pred_token_ids=pred, max_time_steps=[T - 1, 1, T + 1, 3], temperature=temps)
    assert torch.equal(eng.seed, seed)
    with pytest.raises(ValueError, match="temperature"):
        w.generate(conditioning_token_ids=cond, pred_token_ids=pred, max_time_steps=steps, temperature=[1.0, 0.0, 1.0, 1.0])
    assert torch.equal(eng.seed, seed)


@pytest.mark.parametrize("heads", [8, 16])
def test_per_row_coarse_at_model_width_equals_single_rows(heads):
    """Coarse stage at d = 1024, depth 2, h = 8 and 16: one seeded call of 5 rows with their own arguments (ragged
    prefixes too) against each row alone."""
    m, w, _, _ = _model(dim=1024, depth=2, heads=heads, cb=1024)
    g = torch.Generator().manual_seed(heads)
    B, steps_pre, T = 5, 6, 8
    cond, pred, q = _prompts(B, "coarse", steps_pre, 1024, g, n_cond=(12, 40))
    lengths = [0, 6, 3, 1, 5]
    temps, thres, tops, steps = _mixed_args(B, g, T)
    seeds = [int(v) for v in torch.randint(0, 2 ** 62, (B,), generator=g)]
    out = w.generate(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=lengths, seeds=seeds, temperature=temps,
                     filter_thres=thres, top_p=tops, max_time_steps=steps)
    for b, n in enumerate(lengths):
        alone = _alone(w, cond, pred, b, n, seeds=[seeds[b]], temperature=temps[b], filter_thres=thres[b], top_p=tops[b],
                       max_time_steps=steps[b])
        assert torch.equal(out[b, :alone.shape[1]], alone[0]) and bool((out[b, alone.shape[1]:] == -1).all()), (heads, b)


# ------------------------------------------------------------------------------------------------ 4. row alone, unseeded
def _compare_rows(name, out, trace, ref, otraces, lengths, steps, ks, q):
    """Row by row, the sampled tokens against the restatement of that row alone, up to a near tie (after which that row
    is not compared), with the logits along the shared trajectory within 1e-2; masked post-eos tokens match as -1.  A
    near tie is a top-2 gap of the oracle's noisy scores below NEAR_TIE, or, since 16-bit logits may order two values
    at the top-k boundary the other way (the smaller k, the likelier), the row's k-th and (k+1)-th oracle logits within
    NEAR_TIE of each other."""
    exact = total = 0
    for b, (n, T, kk) in enumerate(zip(lengths, steps, ks)):
        k = max(0, (T - n) * q)
        mine, gold = out[b].reshape(-1).cpu(), ref[b].reshape(-1)
        assert torch.equal(mine[:n * q], gold[:n * q]) and torch.equal(mine[n * q + k:], gold[n * q + k:]), (name, b)
        total += k
        for s in range(k):
            if gold[n * q + s] == -1:
                assert mine[n * q + s] == -1, (name, b, s)
                exact += 1
                continue
            if mine[n * q + s] != gold[n * q + s]:
                gap = float(otraces[b][s][1][0])
                top = otraces[b][s][0][0].sort(descending=True).values
                kgap = float(top[kk - 1] - top[kk]) if kk < top.numel() else float("inf")
                assert min(gap, kgap) < NEAR_TIE, (name, b, s, int(mine[n * q + s]), int(gold[n * q + s]), gap, kgap)
                print(f"{name}: row {b} left the restatement's trajectory at token {s} (near tie, gaps {gap:.3e}, {kgap:.3e})")
                break
            exact += 1
            lg, og = trace[s][b].cpu(), otraces[b][s][0][0]
            fin = torch.isfinite(og)
            assert rel(lg[fin], og[fin]) < 1e-2, (name, b, s, rel(lg[fin], og[fin]))
    print(f"{name}: {exact} of {total} sampled tokens identical to the restatement's")
    assert exact >= 0.8 * total


UNSEEDED_CASES = [(stage, B, ragged) for stage in ("coarse", "semantic") for B in (4, 20) for ragged in (False, True)]


@pytest.mark.parametrize("stage,B,ragged", UNSEEDED_CASES,
                         ids=[f"{s}-B{B}-{'ragged' if r else 'full'}" for s, B, r in UNSEEDED_CASES])
def test_unseeded_rows_match_the_restatement(stage, B, ragged):
    """uniform_noise with per-row temperature, filter_thres and max_time_steps (ragged prefixes too), against
    per_row_reference: SIMT decode at B = 4, tensor-core decode at B = 20; graph and eager runs agree."""
    steps_pre, T = (4, 6) if stage == "coarse" else (9, 14)
    m, w, sd, args = _model(stage)
    g = torch.Generator().manual_seed(3 * B + ragged)
    cond, pred, q = _prompts(B, stage, steps_pre, 64, g)
    temps, thres, _, steps = _mixed_args(B, g, T, with_top_p=False)
    lengths = [(3 * b) % (steps_pre + 1) for b in range(B)] if ragged else [steps_pre] * B
    for b, n in enumerate(lengths):
        pred[b, n:] = -1                          # padding is never read (nothing is padding without pred_lengths)
    n_new = max(max(0, (t - n) * q) for t, n in zip(steps, lengths))
    uni = torch.rand(n_new, B, 65, generator=g).clamp_(1e-6, 1 - 1e-6)
    kw = dict(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=lengths if ragged else None, max_time_steps=steps,
              uniform_noise=uni, temperature=temps, filter_thres=thres, allow_eos_in_output=True)
    trace = []
    out = w.generate(trace_logits=trace, **kw)
    assert torch.equal(w.generate(**kw), out) and torch.equal(w.generate(use_cuda_graph=False, **kw), out)
    assert len(trace) == n_new
    cfg = oracle_cfg(stage, dict(args, num_coarse_quantizers=3))
    ref, otraces = per_row_reference(cfg, sd, [t.cpu().numpy() for t in cond], uni, pred.cpu().numpy(), lengths, steps, temps, thres,
                                     return_trace=True, allow_eos_in_output=True)
    assert out.shape == ref.shape
    ks = [max(int((1 - t) * 65), 1) for t in thres]
    _compare_rows(f"{stage} B={B}{' ragged' if ragged else ''}", out, trace, ref, otraces, lengths, steps, ks, q)
