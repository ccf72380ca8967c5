"""Nucleus (top-p) sampling on the H100: omlm_sample_nucleus against the float64 reference of
tests/test_sampling_nucleus_cpu.py on supplied uniforms and on both Philox streams (host replicas), its counters and
CUDA-graph replay; generate(top_p=...) end to end, bit-identity of top_p None / 1.0 with a call without it, batch
invariance of seeded generation, and the three stages through MusicLM.generate_tokens.
A kernel token may differ from the reference's only (a) where a class's float64 mass above lies within 1e-5 (relative)
of top_p: either membership of that value is accepted, and the token must be the reference's choice under one of them;
or (b) at a near tie of the noisy scores (within 1e-5 * max(1, |best|), fp32 against float64)."""
import itertools
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from test_generate_seeded_cpu import seeded_uniforms  # noqa: E402
from test_philox_cpu import sampler_uniforms  # noqa: E402
from test_sampling_nucleus_cpu import edge_logits, nucleus_reference, prepare  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = -7


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as L
    L.device_check()
    return L


def check_nucleus(tokens, logits, uniform, k, T, allow_eos, top_p, what=""):
    """tokens [B] against the float64 reference; returns the number of rows accepted under (a) or (b) of the module
    docstring.  Rows whose top-k set holds NaN logits only have no reference token and are not compared."""
    ref = nucleus_reference(logits, uniform, k, T, allow_eos, top_p)
    x = prepare(logits, allow_eos)
    raw = x / T - torch.log(-torch.log(uniform.double().cpu() + 1e-20) + 1e-20)
    raw = torch.where(torch.isnan(raw), torch.full_like(raw, -math.inf), raw)
    tokens = tokens.cpu()
    loose = 0
    for b in range(tokens.shape[0]):
        t, r = int(tokens[b]), int(ref.token[b])
        if r < 0 or t == r:
            continue
        # candidate nuclei: the reference's, and every prefix by value through the masses within 1e-5 of top_p
        cands = [ref.nuc[b]]
        if ref.top_p is not None:
            ab, tp = ref.above[b], ref.top_p
            amb = ref.kept[b] & ~torch.isnan(x[b]) & ((ab - tp).abs() <= 1e-5 * tp)
            base = ref.nuc[b] & ~amb
            cands.append(base)
            for a in torch.unique(ab[amb]).tolist():
                cands.append(base | (amb & (ab <= a)))
        ok = False
        for n in cands:
            if not bool(n[t]):
                continue
            best = float(torch.where(n, raw[b], torch.full_like(raw[b], -math.inf)).max())
            if float(raw[b, t]) >= best - 1e-5 * max(1.0, abs(best)):
                ok = True
                break
        assert ok, (what, "row", b, "kernel", t, "float64", r, "above", float(ref.above[b, t]) if t < x.shape[1] else None,
                    float(ref.above[b, r]))
        loose += 1
    return loose


def sample(lib, logits, C, k, T, allow_eos, top_p, uniform=None, seed=None, seeds=None, tokens=None, counters=None, pos=None,
           next_row=None, row_offset=0):
    B = logits.shape[0]
    tokens = torch.full((B, 1), SENTINEL, device=DEV, dtype=torch.int64) if tokens is None else tokens
    counters = torch.zeros(2, device=DEV, dtype=torch.int32) if counters is None else counters
    next_row = torch.full((B,), SENTINEL, device=DEV, dtype=torch.int32) if next_row is None else next_row
    lib.sample(logits, C, k, T, allow_eos, uniform, seed, tokens, next_row, row_offset, counters, pos, B, seeds=seeds, top_p=top_p)
    return tokens, counters, next_row


def padded(x, ld):
    buf = torch.full((x.shape[0], ld), math.nan, device=DEV, dtype=torch.float32)
    buf[:, :x.shape[1]] = x
    return buf


TOP_P = (1e-7, 0.05, 0.5, 0.9, 0.999999)


# ------------------------------------------------------------------------------------------------ supplied uniforms
@pytest.mark.parametrize("C", [2, 3, 1025, 2049, 4097, 16384])
def test_nucleus_sampler_matches_float64_on_supplied_uniforms(lib, C):
    """k in {1, 0.1 C, C} x top_p in {1e-7, 0.05, 0.5, 0.9, 0.999999} x T in {0.4, 0.95, 1, 2} x eos allowed or not;
    12 rows per launch of the edge kinds of edge_logits (ties at the nucleus boundary, +-0.0, -inf, equal maxima, NaN),
    every other launch with a row pitch of C + 5 (NaN in between)."""
    g = torch.Generator().manual_seed(C)
    loose = total = 0
    for i, (k, top_p, T, allow) in enumerate(itertools.product(sorted({1, max(int(0.1 * C), 1), C}), TOP_P, (0.4, 0.95, 1.0, 2.0),
                                                                (False, True))):
        B = 12
        x = edge_logits(B, C, g, scale=(3.0, 0.5, 8.0)[i % 3])
        u = torch.rand(1, B, C, generator=g)
        xd, ud = x.to(DEV), u.to(DEV)
        tokens, counters, next_row = sample(lib, padded(xd, C + 5) if i % 2 else xd, C, k, T, allow, top_p, uniform=ud, row_offset=3)
        assert counters.tolist() == [1, 0]
        loose += check_nucleus(tokens[:, 0], x, u[0], k, T, allow, top_p, (C, k, top_p, T, allow))
        assert torch.equal(next_row, (tokens[:, 0] + 3).to(torch.int32))
        total += B
    print(f"C = {C}: {total} rows, {loose} accepted at the top_p boundary or a near tie")


def test_nucleus_narrows_the_draw(lib):
    """With a probe uniform of 1 - 2^-24 on class b in row b (every other uniform in [0.01, 0.5]), class b is sampled if
    and only if it is in N: the kernel's nucleus, read class by class, equals the reference's."""
    C = 64
    g = torch.Generator().manual_seed(64)
    for kind_row in range(6):
        x1 = edge_logits(6, C, g)[kind_row]
        x = x1[None].expand(C, C).contiguous()
        u = 0.01 + 0.49 * torch.rand(C, C, generator=g)
        u[torch.arange(C), torch.arange(C)] = 1.0 - 2.0 ** -24
        for k, top_p, allow in itertools.product((6, 32, C), (0.05, 0.5, 0.9), (False, True)):
            tokens, _, _ = sample(lib, x.to(DEV), C, k, 1.0, allow, top_p, uniform=u[None].to(DEV))
            ref = nucleus_reference(x, u, k, 1.0, allow, top_p)
            wins = tokens[:, 0].cpu() == torch.arange(C)
            expect = ref.nuc.diagonal()
            near = ref.kept.diagonal() & ((ref.above.diagonal() - ref.top_p).abs() <= 1e-5 * ref.top_p)
            assert torch.equal(wins | near, expect | near), (kind_row, k, top_p, allow, (wins != expect).nonzero().flatten().tolist())


# ------------------------------------------------------------------------------------------------ Philox streams
@pytest.mark.parametrize("seeded", [False, True], ids=["engine_seed", "per_sequence"])
def test_nucleus_philox_streams_equal_the_replicas(lib, seeded):
    """Three launches with pos given: tokens equal the reference under the replica's uniforms of each step (unseeded:
    counter (c, b, step, 0x5a17) under the engine seed; seeded: (c, step, 0, 0x5eed) under each row's seed), the step
    counter reaches 3 with the arrival counter back at 0, and pos advances by one per launch."""
    g = torch.Generator().manual_seed(7 + seeded)
    for C, B, k, T, top_p in [(65, 5, 6, 1.0, 0.5), (1025, 40, 102, 0.95, 0.9), (16384, 9, 1638, 0.4, 0.9), (2049, 17, 2049, 2.0, 0.999999)]:
        x = edge_logits(B, C, g)
        tokens = torch.full((B, 3), SENTINEL, device=DEV, dtype=torch.int64)
        counters = torch.zeros(2, device=DEV, dtype=torch.int32)
        pos = torch.tensor([100], device=DEV, dtype=torch.int32)
        seed = 0x0123456789ABCDEF
        seeds = [int(v) for v in torch.randint(0, 2 ** 62, (B,), generator=g)]
        from open_musiclm_b200.decode import seeds_tensor
        kw = dict(seeds=seeds_tensor(seeds, B, DEV)) if seeded else dict(seed=torch.tensor([seed], device=DEV, dtype=torch.int64))
        for _ in range(3):
            sample(lib, x.to(DEV), C, k, T, False, top_p, tokens=tokens, counters=counters, pos=pos, **kw)
        assert counters.tolist() == [3, 0] and int(pos) == 103
        for step in range(3):
            if seeded:
                u = torch.from_numpy(np.stack([seeded_uniforms(s, step, C) for s in seeds]))
            else:
                u = torch.from_numpy(sampler_uniforms(seed, step, B, C))
            check_nucleus(tokens[:, step], x, u, k, T, False, top_p, (seeded, C, step))


def test_nucleus_graph_replay_equals_eager(lib):
    C, B, k, T, top_p = 1025, 40, 102, 0.95, 0.9
    x = edge_logits(B, C, torch.Generator().manual_seed(3)).to(DEV)
    s = torch.tensor([77], device=DEV, dtype=torch.int64)
    eager = torch.full((B, 4), SENTINEL, device=DEV, dtype=torch.int64)
    counters = torch.zeros(2, device=DEV, dtype=torch.int32)
    for _ in range(4):
        sample(lib, x, C, k, T, False, top_p, seed=s, tokens=eager, counters=counters)
    tokens = torch.full((B, 4), SENTINEL, device=DEV, dtype=torch.int64)
    counters = torch.zeros(2, device=DEV, dtype=torch.int32)
    next_row = torch.zeros(B, device=DEV, dtype=torch.int32)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sample(lib, x, C, k, T, False, top_p, seed=s, tokens=tokens, counters=counters, next_row=next_row)
    tokens.fill_(SENTINEL)
    counters.zero_()
    for _ in range(4):
        graph.replay()
    torch.cuda.synchronize()
    assert counters.tolist() == [4, 0] and torch.equal(tokens, eager)


def test_nucleus_entry_point_rejects_bad_top_p(lib):
    x = torch.randn(2, 8, device=DEV)
    for bad in (0.0, 1.5, -0.5, math.nan):
        with pytest.raises(lib.OmlmError, match="top_p"):
            sample(lib, x, 8, 2, 1.0, False, bad, seed=torch.zeros(1, device=DEV, dtype=torch.int64))
    with pytest.raises(lib.OmlmError, match="exclude"):
        from open_musiclm_b200.decode import seeds_tensor
        sample(lib, x, 8, 2, 1.0, False, 0.5, uniform=torch.rand(1, 2, 8, device=DEV), seeds=seeds_tensor([1, 2], 2, DEV))


# ------------------------------------------------------------------------------------------------ generate
def _coarse(abs_pos=False):
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    kw = dict(use_absolute_position_embeddings=True, max_absolute_position_embeddings=32) if abs_pos else {}
    m = O.create_coarse_transformer(dim=1024, depth=2, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1,
                                    **kw).cuda().eval()
    return m, O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)


def _prompt(B, g):
    return ([torch.randint(0, 1024, (B, 12), generator=g).cuda(), torch.randint(0, 1024, (B, 20), generator=g).cuda()],
            torch.randint(0, 1024, (B, 2, 3), generator=g).cuda())


@pytest.fixture(scope="module")
def coarse():
    return _coarse()


def test_top_p_none_and_one_are_bit_identical_to_no_top_p(coarse):
    """On the SIMT path (B = 2) and the tensor-core path (B = 20), unseeded (engine seed reset before each call) and
    seeded: top_p=None and top_p=1.0 give the tokens of a call without top_p; values outside (0, 1] raise ValueError
    before anything runs and leave Engine.seed as it was."""
    m, w = coarse
    eng = m.engine
    g = torch.Generator().manual_seed(1)
    for B, seeded in itertools.product((2, 20), (False, True)):
        cond, prefix = _prompt(B, g)
        kw = dict(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=6, temperature=0.95)
        if seeded:
            kw["seeds"] = [int(v) for v in torch.randint(0, 2 ** 62, (B,), generator=g)]
        outs = []
        for extra in ({}, dict(top_p=None), dict(top_p=1.0)):
            eng.seed.fill_(0x5EED)
            outs.append(w.generate(**kw, **extra))
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), (B, seeded)
        eng.seed.fill_(0x5EED)
        nuc = w.generate(**kw, top_p=0.05)
        assert nuc.shape == outs[0].shape
    before = eng.seed.clone()
    cond, prefix = _prompt(2, g)
    for bad in (0.0, -0.1, 1.01, math.nan, True, "0.9"):
        with pytest.raises(ValueError, match="top_p"):
            w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=6, top_p=bad)
    assert torch.equal(eng.seed, before)


@pytest.mark.parametrize("abs_pos", [False, True], ids=["relpos", "abspos"])
@pytest.mark.parametrize("B", [2, 20])
def test_generate_tokens_equal_the_reference_on_traced_logits(B, abs_pos, coarse):
    """generate(top_p=..., uniform_noise=..., trace_logits=...): every sampled token is the float64 reference's choice
    from the logits it was sampled from (top-k 0.1 C, eos forbidden), at two nucleus masses and temperatures."""
    m, w = _coarse(abs_pos=True) if abs_pos else coarse
    g = torch.Generator().manual_seed(B + 10 * abs_pos)
    C, steps = 1025, 6
    k = max(int(0.1 * C), 1)
    for top_p, T in ((0.9, 0.95), (0.3, 0.4)):
        cond, prefix = _prompt(B, g)
        n_new = (steps - 2) * 3
        uni = torch.rand(n_new, B, C, generator=g)
        trace = []
        out = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=steps, temperature=T, top_p=top_p,
                         uniform_noise=uni, trace_logits=trace)
        flat = out.reshape(B, -1)[:, 6:]
        assert len(trace) == flat.shape[1] == n_new
        loose = sum(check_nucleus(flat[:, s], trace[s].cpu(), uni[s], k, T, False, top_p, (B, abs_pos, top_p, s)) for s in range(n_new))
        print(f"B = {B}, abs_pos = {abs_pos}, top_p = {top_p}: {loose} tokens accepted at a boundary or near tie")
        graph = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=steps, temperature=T, top_p=top_p,
                           uniform_noise=uni)
        eager = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=steps, temperature=T, top_p=top_p,
                           uniform_noise=uni, use_cuda_graph=False)
        assert torch.equal(graph, out) and torch.equal(eager, out)


def test_seeded_nucleus_generate_does_not_depend_on_the_batch(coarse):
    """A target (prompt, seed) at the first, a middle and the last row of batches of 17 and 40 samples, with top_p=0.9,
    the tokens it samples alone (B = 1), in CUDA-graph and eager runs."""
    m, w = coarse
    g = torch.Generator().manual_seed(17)
    tc, tp = _prompt(1, g)
    tseed = 0xC0FFEE_0123456789
    kw = dict(max_time_steps=6, temperature=0.95, top_p=0.9)
    ref = w.generate(conditioning_token_ids=tc, pred_token_ids=tp, seeds=[tseed], **kw)
    assert torch.equal(w.generate(conditioning_token_ids=tc, pred_token_ids=tp, seeds=[tseed], use_cuda_graph=False, **kw), ref)
    for B in (17, 40):
        cond, prefix = _prompt(B, g)
        seeds = torch.randint(-2 ** 62, 2 ** 62, (B,), generator=g, dtype=torch.int64)
        rows = sorted({0, B // 2, B - 1})
        for r in rows:
            cond[0][r], cond[1][r], prefix[r] = tc[0][0], tc[1][0], tp[0]
            seeds[r] = tseed - 2 ** 64            # the same 64 bits as the list entry of the single run
        out = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, seeds=seeds, **kw)
        assert torch.equal(w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, seeds=seeds, use_cuda_graph=False, **kw), out)
        for r in rows:
            assert torch.equal(out[r], ref[0]), (B, r)


# ------------------------------------------------------------------------------------------------ MusicLM
def test_musiclm_three_stages_with_per_stage_top_p():
    """MusicLM.generate_tokens(seeds=..., top_p=(0.95, 0.9, 0.8)) with the small stages of tests/golden/musiclm_windows.pt:
    two runs are identical, and each prompt's streams equal its single-prompt run."""
    import open_musiclm_b200 as O
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "musiclm_windows.pt"), weights_only=False)
    fns = {"semantic": O.create_semantic_transformer, "coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}
    models = {}
    for name, fn in fns.items():
        mdl = fn(**fx["kwargs"][name])
        mdl.load_state_dict(fx["state_dicts"][name], strict=True)
        models[name] = mdl.cuda().eval()
    mlm = O.MusicLM(semantic_transformer=models["semantic"], coarse_transformer=models["coarse"], fine_transformer=models["fine"])
    cb, nq = fx["kwargs"]["semantic"]["clap_codebook_size"], fx["kwargs"]["semantic"]["num_clap_quantizers"]
    clap = torch.randint(0, cb, (3, nq), generator=torch.Generator().manual_seed(9)).cuda()
    seeds = [5, 2 ** 64 - 1, 31337]
    kw = dict(seeds=seeds, top_p=(0.95, 0.9, 0.8), return_all=True, **fx["args"])
    batch = mlm.generate_tokens(clap_token_ids=clap, **kw)
    again = mlm.generate_tokens(clap_token_ids=clap, **kw)
    for a, r in zip(batch, again):
        assert torch.equal(a, r)
    for b in range(3):
        one = mlm.generate_tokens(clap_token_ids=clap[b:b + 1], seeds=[seeds[b]], top_p=(0.95, 0.9, 0.8), return_all=True, **fx["args"])
        for a, r in zip(batch, one):
            assert torch.equal(a[b:b + 1], r), b
