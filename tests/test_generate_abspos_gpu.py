"""Generation for models with absolute position embeddings (use_absolute_position_embeddings=True) on the H100 decode
path: the decode step's gather with a device-side position row (omlm_embed_gather_pos) against torch indexing, the
incremental step against the full forward at model scale, seeded generation across batch sizes, the reference's
bounds, the REAL reference's tokens (tests/golden/abspos_gen_*.pt) and three-stage windowed generation."""
import dataclasses
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from test_generate_abspos_cpu import ABS_GEN, abspos_cfg  # noqa: E402
from test_generate_seeded_cpu import seeded_uniforms  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
NEAR_TIE = 5e-2      # oracle top-2 gap below which 16-bit logits may legitimately sample the other token


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _fixture_wrapper(fx):
    import open_musiclm_b200 as O
    fn = {"semantic": O.create_semantic_transformer, "coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}[fx["stage"]]
    m = fn(**fx["kwargs"])
    m.load_state_dict(fx["state_dict"], strict=True)
    return O.TokenConditionedTransformerWrapper(transformer=m.cuda().eval(), unique_consecutive=False)


def _abs_coarse(depth=2, heads=8, dim=1024, **kw):
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=dim, depth=depth, heads=heads, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1,
                                    use_absolute_position_embeddings=True, **kw).cuda().eval()
    return m, O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)


def _compare_to_oracle(name, out, trace, ref, otrace, n_prefix):
    """Token for token up to near ties (after which that sequence is not compared), with the logits along the shared
    trajectory within 1e-2 of the oracle's: the rule of test_decode_gpu.test_generate_matches_reference_tokens_under_fixed_noise."""
    B = out.shape[0]
    mine, gold = out.cpu().reshape(B, -1)[:, n_prefix:], torch.as_tensor(ref).reshape(B, -1)[:, n_prefix:]
    exact = 0
    for b in range(B):
        for s in range(mine.shape[1]):
            if gold[b, s] == -1:          # after an eos both are masked
                assert mine[b, s] == -1
                exact += 1
                continue
            if mine[b, s] != gold[b, s]:
                gap = float(otrace[s][1][b])
                assert gap < NEAR_TIE, (name, b, s, int(mine[b, s]), int(gold[b, s]), gap)
                print(f"{name}: sequence {b} left the reference trajectory at token {s} (near tie, gap {gap:.3e})")
                break
            exact += 1
            lg, og = trace[s][b].cpu(), otrace[s][0][b]
            fin = torch.isfinite(og)
            assert rel(lg[fin], og[fin]) < 1e-2, (name, b, s, rel(lg[fin], og[fin]))
    print(f"{name}: {exact} of {mine.numel()} sampled tokens identical to the oracle's")
    assert exact >= 0.8 * mine.numel()


# ------------------------------------------------------------------------------------------------ a. the gather
@pytest.mark.parametrize("D", [64, 1024])
@pytest.mark.parametrize("B", [1, 17, 256])
def test_embed_gather_pos_matches_torch_indexing(B, D):
    """x[b] = table[next_row[b]] + table[row_base + *pos + offset], bit-exact against torch indexing, eagerly and from
    a captured CUDA graph whose position tensor is advanced between replays; a negative next_row adds nothing, and so
    does a position outside [0, pos_rows)."""
    from open_musiclm_b200 import lib
    g = torch.Generator(device=DEV).manual_seed(B * 7 + D)
    row_base, n_pos, off = 200, 90, -37
    table = torch.randn(row_base + n_pos + 10, D, device=DEV, generator=g)
    next_row = torch.randint(0, row_base, (B,), device=DEV, generator=g, dtype=torch.int32)
    if B > 1:
        next_row[B // 2] = -1
    pos = torch.zeros(1, device=DEV, dtype=torch.int32)
    x = torch.full((B, D), float("nan"), device=DEV)

    def expect(p):
        e = torch.where((next_row >= 0)[:, None], table[next_row.clamp_min(0).long()], torch.zeros((), device=DEV))
        j = p + off
        return e + table[row_base + j] if 0 <= j < n_pos else e

    for p in (37, 38, 37 + 50, 37 + n_pos - 1, 36, 37 + n_pos):
        pos.fill_(p)
        x.fill_(float("nan"))
        lib.embed_gather_pos(table, next_row, pos, off, row_base, n_pos, x)
        assert torch.equal(x, expect(p)), p
    pos.fill_(37)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lib.embed_gather_pos(table, next_row, pos, off, row_base, n_pos, x)
    for p in (37, 41, 37 + n_pos - 1, 60):
        pos.fill_(p)
        x.fill_(float("nan"))
        graph.replay()
        assert torch.equal(x, expect(p)), ("graph", p)


def test_embed_gather_pos_argument_checks():
    from open_musiclm_b200 import lib
    table = torch.randn(64, 8, device=DEV)
    rows = torch.zeros(2, device=DEV, dtype=torch.int32)
    pos = torch.zeros(1, device=DEV, dtype=torch.int32)
    with pytest.raises(lib.OmlmError, match="bad shape"):
        lib.embed_gather_pos(table, rows, pos, 0, 0, 8, torch.empty(2, 6, device=DEV))
    with pytest.raises(lib.OmlmError, match="position rows"):
        lib.embed_gather_pos(table, rows, pos, 0, 0, 0, torch.empty(2, 8, device=DEV))
    with pytest.raises(lib.OmlmError, match="position rows"):
        lib.embed_gather_pos(table, rows, pos, 0, -1, 8, torch.empty(2, 8, device=DEV))


# ------------------------------------------------------------------------------------------------ b. model scale
@pytest.mark.parametrize("B", [2, 20])
def test_incremental_step_with_absolute_positions_equals_full_forward(B):
    """Coarse stage with absolute positions (d = 1024, L = 2, h = 8), SIMT (B = 2) and tensor-core (B = 20) decode:
    the logits of every step against the full wgmma forward over the same prefix (the bound of
    test_incremental_step_equals_full_forward_at_model_scale), and eager and CUDA-graph steps sample the same tokens."""
    m, w = _abs_coarse()
    g = torch.Generator().manual_seed(5)
    cond = [torch.randint(0, 1024, (B, 12), generator=g).cuda(), torch.randint(0, 1024, (B, 40), generator=g).cuda()]
    prefix = torch.randint(0, 1024, (B, 3, 3), generator=g).cuda()
    trace = []
    out = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=9, trace_logits=trace)
    assert out.shape == (B, 9, 3) and int(out.min()) >= 0 and int(out.max()) < 1024
    flat = out.reshape(B, -1)
    ids_c = [torch.cat([t, torch.full((B, 1), 1024, device=DEV)], 1) for t in cond]
    worst = 0.0
    for s, lg in enumerate(trace):
        with torch.no_grad():
            full = m(all_token_ids=ids_c + [flat[:, :9 + s]], return_only_final_seq_logits=True)[-1][:, -1]
        worst = max(worst, rel(lg, full))
    print(f"B = {B}: decode vs full forward with absolute positions, worst logits rel-L2 over {len(trace)} steps: {worst:.2e}")
    assert worst < 5e-3
    n_new = 6 * 3
    uni = torch.rand(n_new, B, 1025, generator=g).clamp_(1e-6, 1 - 1e-6)
    eager = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=9, uniform_noise=uni, trace_logits=[])
    graph = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=9, uniform_noise=uni)
    assert torch.equal(eager, graph)


# ------------------------------------------------------------------------------------------------ c. seeded
def test_seeded_generate_with_absolute_positions_does_not_depend_on_the_batch():
    """A target (prompt, seed) at the first, a middle and the last row of batches of 3, 17 and 40 with random other
    rows: tokens and every trace_logits row bit-identical to the target alone (B = 1); eager and graph runs agree."""
    m, w = _abs_coarse()
    g = torch.Generator().manual_seed(7)
    steps, T = 6, 0.9
    tc = [torch.randint(0, 1024, (1, 12), generator=g).cuda(), torch.randint(0, 1024, (1, 20), generator=g).cuda()]
    tp = torch.randint(0, 1024, (1, 2, 3), generator=g).cuda()
    tseed = 0x5EED_AB5_0123
    ref_tr = []
    ref = w.generate(conditioning_token_ids=tc, pred_token_ids=tp, max_time_steps=steps, temperature=T, seeds=[tseed], trace_logits=ref_tr)
    assert torch.equal(w.generate(conditioning_token_ids=tc, pred_token_ids=tp, max_time_steps=steps, temperature=T, seeds=[tseed]), ref)
    for B in (3, 17, 40):
        cond = [torch.randint(0, 1024, (B, 12), generator=g).cuda(), torch.randint(0, 1024, (B, 20), generator=g).cuda()]
        prefix = torch.randint(0, 1024, (B, 2, 3), generator=g).cuda()
        seeds = [int(v) for v in torch.randint(0, 2 ** 62, (B,), generator=g)]
        rows = sorted({0, B // 2, B - 1})
        for r in rows:
            cond[0][r], cond[1][r], prefix[r] = tc[0][0], tc[1][0], tp[0]
            seeds[r] = tseed
        tr = []
        eager = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=steps, temperature=T, seeds=seeds, trace_logits=tr)
        graph = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=steps, temperature=T, seeds=seeds)
        assert torch.equal(eager, graph), B
        assert len(tr) == len(ref_tr)
        for r in rows:
            assert torch.equal(eager[r], ref[0]), (B, r)
            for s in range(len(tr)):
                assert torch.equal(tr[s][r], ref_tr[s][0]), (B, r, s)


@pytest.mark.parametrize("path", ABS_GEN, ids=[os.path.basename(p) for p in ABS_GEN])
def test_seeded_generate_with_absolute_positions_matches_the_oracle_under_the_replica_noise(path):
    """Seeded generate on the abspos fixtures' weights and prompts against the oracle (abs_pos=True) fed each row's
    replica uniforms."""
    from oracle import restatement as R
    fx = torch.load(path, weights_only=False)
    w = _fixture_wrapper(fx)
    B = fx["cond"][0].shape[0]
    seeds = [(0x9E3779B97F4A7C15 * (b + 1)) % 2 ** 64 for b in range(B)]
    C = fx["uniforms"].shape[-1]
    kw = dict(max_time_steps=fx["max_time_steps"], filter_thres=fx["filter_thres"], temperature=fx["temperature"],
              include_eos_in_output=fx["include_eos_in_output"], allow_eos_in_output=fx["allow_eos_in_output"])
    trace = []
    out = w.generate(conditioning_token_ids=[t.cuda() for t in fx["cond"]], pred_token_ids=None if fx["prefix"] is None else fx["prefix"].cuda(),
                     seeds=seeds, trace_logits=trace, **kw)
    noise = lambda s, shape: torch.from_numpy(np.stack([seeded_uniforms(sd, s, C) for sd in seeds]))
    ref, otrace = R.generate(abspos_cfg(fx), fx["state_dict"], [t.numpy() for t in fx["cond"]], noise,
                             pred_token_ids=None if fx["prefix"] is None else fx["prefix"].numpy(), return_trace=True, **kw)
    assert out.shape == ref.shape
    n_prefix = 0 if fx["prefix"] is None else fx["prefix"].shape[1] * out.shape[2]
    _compare_to_oracle(os.path.basename(path) + " (seeded)", out, trace, ref, otrace, n_prefix)


# ------------------------------------------------------------------------------------------------ d. bounds
def test_generate_bounds_are_the_reference_lookups():
    """max_absolute_position_embeddings = 16: a conditioning sequence of 16 tokens with its eos and a predicted sequence
    with prefix + n_new - 1 = 16 generate; one more raises IndexError before anything runs (Engine.seed unchanged); a
    call that samples nothing checks nothing."""
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_semantic_transformer(dim=64, depth=1, heads=2, clap_codebook_size=64, semantic_codebook_size=64, num_clap_quantizers=4,
                                      attn_dropout=0.0, use_absolute_position_embeddings=True, max_absolute_position_embeddings=16).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    eng = m.engine
    g = torch.Generator().manual_seed(3)
    ids = lambda n: torch.randint(0, 64, (2, n), generator=g).cuda()
    # conditioning: 15 ids + eos
    assert w.generate(conditioning_token_ids=[ids(15)], max_time_steps=4).shape == (2, 4, 1)
    seed = eng.seed.clone()
    with pytest.raises(IndexError, match="conditioning sequence 0 has 17 tokens"):
        w.generate(conditioning_token_ids=[ids(16)], max_time_steps=4)
    assert torch.equal(eng.seed, seed)
    # without the appended eos the same 16 ids fit
    assert w.generate(conditioning_token_ids=[ids(16)], max_time_steps=4, append_eos_to_conditioning_tokens=False).shape == (2, 4, 1)
    # predicted: prefix 5 + n_new 12 - 1 = 16
    pre = ids(5)
    out = w.generate(conditioning_token_ids=[ids(4)], pred_token_ids=pre, max_time_steps=17)
    assert out.shape == (2, 17, 1) and torch.equal(out[:, :5, 0], pre)
    seed = eng.seed.clone()
    with pytest.raises(IndexError, match="predicted sequence reaches 17 tokens"):
        w.generate(conditioning_token_ids=[ids(4)], pred_token_ids=pre, max_time_steps=18)
    with pytest.raises(IndexError, match="predicted sequence reaches 17 tokens"):
        w.generate(conditioning_token_ids=[ids(4)], max_time_steps=18, seeds=[1, 2])
    assert torch.equal(eng.seed, seed)
    # n_new = 0: no forward, nothing checked
    long = ids(20)
    assert torch.equal(w.generate(conditioning_token_ids=[ids(30)], pred_token_ids=long, max_time_steps=20)[..., 0], long)


# ------------------------------------------------------------------------------------------------ e. reference tokens
@pytest.mark.parametrize("path", ABS_GEN, ids=[os.path.basename(p) for p in ABS_GEN])
def test_generate_with_absolute_positions_matches_reference_tokens_under_fixed_noise(path):
    """wrapper.generate on the reference's weights, prompt and Gumbel noise stream (SIMT decode at B = 2, tensor-core
    decode at B = 20): eager and CUDA-graph runs agree, and the tokens equal the real reference's up to near ties."""
    from oracle import restatement as R
    from open_musiclm_b200.decode import SKINNY_MAX_BATCH
    fx = torch.load(path, weights_only=False)
    w = _fixture_wrapper(fx)
    B = fx["cond"][0].shape[0]
    print(os.path.basename(path), "tensor-core" if B > SKINNY_MAX_BATCH else "SIMT", "decode path")
    kw = dict(conditioning_token_ids=[t.cuda() for t in fx["cond"]], pred_token_ids=None if fx["prefix"] is None else fx["prefix"].cuda(),
              max_time_steps=fx["max_time_steps"], filter_thres=fx["filter_thres"], temperature=fx["temperature"],
              include_eos_in_output=fx["include_eos_in_output"], allow_eos_in_output=fx["allow_eos_in_output"], uniform_noise=fx["uniforms"])
    trace = []
    out_eager = w.generate(trace_logits=trace, **kw)
    out_graph = w.generate(**kw)
    assert torch.equal(out_eager, out_graph), "CUDA-graph replay and eager launches must sample the same tokens"
    gold = fx["out"]
    assert out_graph.shape == gold.shape and out_graph.dtype == torch.int64
    uni = fx["uniforms"]
    _, otrace = R.generate(abspos_cfg(fx), fx["state_dict"], [t.numpy() for t in fx["cond"]], lambda s, shape: uni[s],
                           pred_token_ids=None if fx["prefix"] is None else fx["prefix"].numpy(), max_time_steps=fx["max_time_steps"],
                           filter_thres=fx["filter_thres"], temperature=fx["temperature"], include_eos_in_output=fx["include_eos_in_output"],
                           allow_eos_in_output=fx["allow_eos_in_output"], return_trace=True)
    n_prefix = 0 if fx["prefix"] is None else fx["prefix"].shape[1] * gold.shape[2]
    _compare_to_oracle(os.path.basename(path), out_graph, trace, gold, otrace, n_prefix)


# ------------------------------------------------------------------------------------------------ f. windowing
def test_three_stage_windowed_generation_with_absolute_positions():
    """MusicLM.generate_tokens with three absolute-position stages (the stage shapes and noise stream of
    tests/golden/musiclm_windows.pt, random-init weights) on the decode path against the oracle-backed stages of
    tests/test_stages_cpu.py: every window's generate call counts positions from its own prompt.  The same number of
    draws, and the same tokens up to the first draw where the oracle's top-2 gap is a near tie."""
    import open_musiclm_b200 as O
    from oracle import restatement as R
    from test_stages_cpu import OracleWrapper, oracle_cfg
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "musiclm_windows.pt"), weights_only=False)
    # longest sequence any window feeds: a coarse window, 8 steps x 3 quantizers - 1 = 23 tokens
    abs_kw = dict(use_absolute_position_embeddings=True, max_absolute_position_embeddings=23)
    fns = {"semantic": O.create_semantic_transformer, "coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}
    models, sds = {}, {}
    torch.manual_seed(0)
    for k, fn in fns.items():
        m = fn(**fx["kwargs"][k], **abs_kw)
        sds[k] = {n: v.detach().clone() for n, v in m.state_dict().items()}
        models[k] = m.cuda().eval()
    mlm = O.MusicLM(semantic_transformer=models["semantic"], coarse_transformer=models["coarse"], fine_transformer=models["fine"])
    log = []
    for st in (mlm.semantic, mlm.coarse, mlm.fine):
        orig = st.transformer_wrapper.generate

        def shim(orig=orig, **kw):
            out = orig(**kw)
            init = 0 if kw.get("pred_token_ids") is None else kw["pred_token_ids"].shape[1]
            log.append(out[:, init:].reshape(out.shape[0], -1).cpu())
            return out
        st.transformer_wrapper.generate = shim
    noise = O.NoiseStream(fx["uniforms"])
    out = mlm.generate_tokens(clap_token_ids=fx["clap_ids"].cuda(), noise=noise, **fx["args"])
    assert noise.at == fx["uniforms"].shape[0] and out.shape == fx["out"].shape
    wr = {k: OracleWrapper(dataclasses.replace(oracle_cfg(k, fx["kwargs"][k]), abs_pos=True, max_abs_pos=23), sds[k]) for k in fns}
    olog, gaps = [], []
    for k in wr:
        def oshim(wrapper=wr[k], **kw):
            o, trace = R.generate(wrapper.cfg, wrapper.sd, [t.numpy() for t in kw["conditioning_token_ids"]], lambda s, shape: kw["uniform_noise"][s],
                                  pred_token_ids=None if kw.get("pred_token_ids") is None else kw["pred_token_ids"].numpy(),
                                  max_time_steps=kw["max_time_steps"], filter_thres=kw.get("filter_thres", 0.9),
                                  temperature=kw.get("temperature", 1.0), include_eos_in_output=kw.get("include_eos_in_output", False),
                                  return_trace=True)
            init = 0 if kw.get("pred_token_ids") is None else kw["pred_token_ids"].shape[1]
            olog.append(o[:, init:].reshape(o.shape[0], -1))
            gaps.append(torch.stack([gp for _, gp in trace], 1))          # [B, n_new]
            return o
        wr[k].generate = oshim
    ref_chain = O.MusicLM(stages=(O.SemanticStage(semantic_transformer=None, wrapper=wr["semantic"]),
                                  O.CoarseStage(coarse_transformer=None, wrapper=wr["coarse"]), O.FineStage(fine_transformer=None, wrapper=wr["fine"])))
    ref_noise = O.NoiseStream(fx["uniforms"])
    ref_out = ref_chain.generate_tokens(clap_token_ids=fx["clap_ids"], noise=ref_noise, **fx["args"])
    assert ref_noise.at == noise.at and ref_out.shape == out.shape and len(olog) == len(log)
    if torch.equal(out.cpu(), ref_out):
        print("three-stage generation with absolute positions: all", out.numel(), "tokens identical to the oracle's")
        return
    for call, (mine, ref, gap) in enumerate(zip(log, olog, gaps)):
        if torch.equal(mine, ref):
            continue
        diff = (mine != ref).nonzero()
        b, s = (int(v) for v in diff[diff[:, 1].argmin()])
        assert float(gap[b, s]) < NEAR_TIE, ("generate call", call, "sequence", b, "token", s, "gap", float(gap[b, s]))
        print(f"three-stage generation left the oracle trajectory in generate call {call} of {len(log)} at a near tie "
              f"(gap {float(gap[b, s]):.3e})")
        return
