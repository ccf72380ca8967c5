"""Seeded generation on the H100: the seeded sampler against float64 under the host replica's uniforms, the
batch-invariant decode GEMM, the prompt forward and the decode attention row for row across batch sizes, and
generate(seeds=...) / MusicLM.generate_tokens(seeds=...) end to end: a sequence's tokens and logits do not depend on
the batch it runs in."""
import glob
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(__file__))
from test_generate_seeded_cpu import seeded_uniforms  # noqa: E402
from test_sampling_gpu import check_tokens, padded_logits  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
GEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "gen_*.pt")))


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def replica(seeds, step, C):
    """[B, C] device uniforms of the seeded stream for the given per-row seeds at sample index `step`."""
    return torch.from_numpy(np.stack([seeded_uniforms(s, step, C) for s in seeds])).to(DEV)


def as_tensor(seeds):
    from open_musiclm_b200.decode import seeds_tensor
    return seeds_tensor(seeds, len(seeds), DEV)


# ------------------------------------------------------------------------------------------------ a. sampler
@pytest.mark.parametrize("C", [2, 1025, 16384])
@pytest.mark.parametrize("B", [1, 7, 256])
def test_seeded_sampler_is_the_float64_argmax_under_the_replica(B, C):
    """Several steps and k edges: tokens equal float64 top-k Gumbel-argmax under the replica's uniforms for each row's
    seed (up to near ties); a row equal in logits and seed to row 0 samples what row 0 samples, wherever it sits and in
    a one-row call."""
    from open_musiclm_b200 import lib
    g = torch.Generator().manual_seed(B * 31 + C)
    seeds = [int(v) for v in torch.randint(0, 2 ** 62, (B,), generator=g)]
    seeds[0] = 2 ** 64 - 12345                    # a seed above 2^63: read as raw bits
    if B > 1:
        seeds[-1] = seeds[0]
    steps = 4
    U = [replica(seeds, t, C) for t in range(steps)]
    ks = sorted({1, 2, max(int(0.1 * C), 1), C})
    near = 0
    for k in ks:
        for T, allow in ((1.0, False), (0.7, True)):
            x = torch.randn(steps, B, C, generator=g) * 3
            x[:, 1::3] = torch.round(x[:, 1::3])          # ties at the k-th value
            if B > 1:
                x[:, -1] = x[:, 0]
            x = x.to(DEV)
            tokens = torch.full((B, steps), -7, device=DEV, dtype=torch.int64)
            counters = torch.zeros(2, device=DEV, dtype=torch.int32)
            next_row = torch.empty(B, device=DEV, dtype=torch.int32)
            sd = as_tensor(seeds)
            one = torch.full((1, steps), -7, device=DEV, dtype=torch.int64)
            c1 = torch.zeros(2, device=DEV, dtype=torch.int32)
            for t in range(steps):
                lib.sample(padded_logits(x[t], C + 3), C, k, T, allow, None, None, tokens, next_row, 0, counters, None, B, seeds=sd)
                lib.sample(x[t, :1].contiguous(), C, k, T, allow, None, None, one, next_row[:1], 0, c1, None, 1, seeds=sd[:1])
            assert counters.tolist() == [steps, 0]
            for t in range(steps):
                n, _ = check_tokens(tokens[:, t], x[t], U[t], k, T, allow, (B, C, k, T, t))
                near += n
            assert torch.equal(tokens[-1], tokens[0]) and torch.equal(one[0], tokens[0])
    print(f"B = {B}, C = {C}: {near} tokens differ from float64 at a near tie")


def test_seeded_sampler_rejects_supplied_uniforms():
    from open_musiclm_b200 import lib
    x = torch.randn(2, 8, device=DEV)
    u = torch.rand(1, 2, 8, device=DEV)
    with pytest.raises(lib.OmlmError, match="exclude"):
        lib.sample(x, 8, 2, 1.0, False, u, None, torch.zeros(2, 1, device=DEV, dtype=torch.int64), torch.zeros(2, device=DEV, dtype=torch.int32),
                   0, torch.zeros(2, device=DEV, dtype=torch.int32), None, 2, seeds=as_tensor([1, 2]))


# ------------------------------------------------------------------------------------------------ b. invariant GEMM
# every decode GEMM (N, K) of musiclm_small (d 1024, h 8) and musiclm_large (h 16): wq, wkv, wo, w1, w2, logit head
SHAPES = [(512, 1024), (1024, 1024), (128, 1024), (1024, 512), (5632, 1024), (1024, 2816), (1088, 1024)]
BATCHES = [1, 2, 16, 17, 63, 64, 65, 128, 129, 256]


def _gemm_cases(N, K, wdt):
    """(prologue, A [256, K], kwargs with 256-row tensors, float64 reference before the output rounding)."""
    g = torch.Generator(device=DEV).manual_seed(N * 7 + K)
    R = 256
    W = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).to(wdt)
    Wd = W.double()
    x = torch.randn(R, K, device=DEV, generator=g) * 2 + 0.3
    gamma = 1 + 0.1 * torch.randn(K, device=DEV, generator=g)
    res = torch.randn(R, N, device=DEV, generator=g)
    a16 = x.to(wdt)
    out = [(0, a16, dict(addend=res), a16.double() @ Wd.t() + res.double()),
           (1, x, {}, x.to(wdt).double() @ Wd.t()),
           (2, x, dict(gamma=gamma), F.layer_norm(x, (K,), gamma, None, 1e-5).to(wdt).double() @ Wd.t())]
    if K % 128 == 0:
        Fl = K - 86
        hmid = torch.zeros(R, K, device=DEV)
        hmid[:, :Fl] = torch.randn(R, Fl, device=DEV, generator=g) * 3 + 1
        g3 = gamma.clone()
        g3[Fl:] = 0
        h16 = hmid.to(wdt)
        rowsum = torch.stack([h16.float().view(R, -1, 128).sum(-1), (h16.float() ** 2).view(R, -1, 128).sum(-1)], -1).contiguous()
        mean = h16.double()[:, :Fl].mean(-1, keepdim=True)
        var = h16.double()[:, :Fl].var(-1, unbiased=False, keepdim=True)
        hn = ((h16.double() - mean) * torch.rsqrt(var + 1e-5) * g3.double()).to(wdt).double()
        out.append((3, h16, dict(gamma=g3, rowsum=rowsum, n_real=Fl, addend=res), hn @ Wd.t() + res.double()))
    return W, out


@pytest.mark.parametrize("wdt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("N,K", SHAPES, ids=[f"{n}x{k}" for n, k in SHAPES])
def test_invariant_decode_gemm_rows_do_not_depend_on_the_batch(N, K, wdt):
    """Row r of a B-row omlm_decode_gemm_invariant call is bit-identical to the same row computed alone, for every B in
    BATCHES (batch padding 64, 128 and 256; one or two consumer warpgroups), fp32 and bf16 outputs; and every B stays
    within test_decode_gemm_against_torch's bounds of the float64 product."""
    from open_musiclm_b200 import lib
    W, cases = _gemm_cases(N, K, wdt)
    ws = lib.DecodeWorkspace(DEV, 256, [(N, K)], invariant=True)
    cut = lambda kw, B: {k: (v[:B] if isinstance(v, torch.Tensor) and v.dim() >= 2 else v) for k, v in kw.items()}
    for prologue, A, kw, ref in cases:
        for odt in (torch.float32, torch.bfloat16):
            single = torch.empty(256, N, device=DEV, dtype=odt)
            for r in range(256):
                lib.decode_gemm(A[r:r + 1], W, single[r:r + 1], prologue=prologue, ws=ws, invariant=True,
                                **{k: (v[r:r + 1] if isinstance(v, torch.Tensor) and v.dim() >= 2 else v) for k, v in kw.items()})
            tol = 1e-5 if (prologue == 0 and odt == torch.float32) else 2e-3
            for B in BATCHES:
                o = torch.full((B, N), float("nan"), device=DEV, dtype=odt)
                lib.decode_gemm(A[:B], W, o, prologue=prologue, ws=ws, invariant=True, **cut(kw, B))
                assert torch.equal(o, single[:B]), (prologue, odt, B, "rows differ from one-row calls",
                                                    (o != single[:B]).any(1).nonzero().flatten()[:8].tolist())
                r64 = ref[:B] if odt == torch.float32 else ref[:B].to(odt)
                assert rel(o, r64) < tol, (prologue, odt, B, rel(o, r64))


def test_invariant_workspace_is_at_least_the_default():
    from open_musiclm_b200 import lib
    for N, K in SHAPES:
        for B in (1, 64, 65, 256):
            assert lib.decode_gemm_workspace(B, N, K, invariant=True) >= (lib.decode_gemm_workspace(B, N, K) if B <= 64 else 0)
        assert lib.decode_gemm_workspace(40, N, K, invariant=True) == lib.decode_gemm_workspace(40, N, K)    # same split at Bp = 64


# ------------------------------------------------------------------------------------------------ c. prefill, attention
def _coarse(depth=2, heads=8, dim=1024):
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=dim, depth=depth, heads=heads, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    return m, O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)


@pytest.mark.parametrize("B", [40, 256])
def test_prompt_logits_do_not_depend_on_the_batch(B):
    """The prompt's last-position logits (Engine.forward_core, the first entry of trace_logits) of a sequence alone and
    at the first, a middle and the last row of a batch of B.  At B = 256 (M = 11008 rows) Engine._bn_for picks 256-wide
    tiles for the wo and w2 GEMMs, 128-wide ones at B = 1."""
    m, w = _coarse()
    g = torch.Generator().manual_seed(B)
    cond = [torch.randint(0, 1024, (B, 12), generator=g).cuda(), torch.randint(0, 1024, (B, 20), generator=g).cuda()]
    prefix = torch.randint(0, 1024, (B, 2, 3), generator=g).cuda()
    rows = (0, B // 2, B - 1)
    for r in rows[1:]:
        cond[0][r], cond[1][r], prefix[r] = cond[0][0], cond[1][0], prefix[0]
    M = B * (13 + 1 + 21 + 1 + 6 + 1)
    if B == 256:
        assert m.engine._bn_for(M, 1024, 512) == 256 and m.engine._bn_for(43, 1024, 512) == 128
    big, one = [], []
    w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=3, trace_logits=big, seeds=list(range(B)))
    w.generate(conditioning_token_ids=[c[:1] for c in cond], pred_token_ids=prefix[:1], max_time_steps=3, trace_logits=one, seeds=[0])
    for r in rows:
        assert torch.equal(big[0][r], one[0][0]), r


@pytest.mark.parametrize("N,K", [(512, 1024), (1024, 512), (1024, 2816)])
def test_gemm_tile_width_does_not_change_an_element(N, K):
    """The forward GEMM's elements are bit-identical with 128- and 256-wide tiles (the sum over K runs in the same
    k-block order), so the batch-dependent tile choice of Engine._bn_for leaves each prompt row's result unchanged."""
    from open_musiclm_b200 import lib
    g = torch.Generator(device=DEV).manual_seed(N + K)
    for dt in (torch.float16, torch.bfloat16):
        a = torch.randn(1000, K, device=DEV, generator=g).to(dt)
        b = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).to(dt)
        add = torch.randn(1000, N, device=DEV, generator=g)
        for odt, kw in ((torch.float32, dict(addend=add)), (torch.bfloat16, {})):
            outs = [lib.gemm(a, b, torch.empty(1000, N, device=DEV, dtype=odt), block_n=bn, **kw) for bn in (128, 256)]
            assert torch.equal(outs[0], outs[1]), (dt, odt)


@pytest.mark.parametrize("h", [1, 8, 16])
def test_attn_decode_mqa_rows_do_not_depend_on_the_batch(h):
    """A target sequence's output and appended cache row at rows 0, B // 2 and B - 1 of batches of B in {5, 16, 17, 200}
    (random other rows) against the target alone, at positions 0, 127, 128, 700 and 2047."""
    from open_musiclm_b200 import lib
    max_pos = 2048
    g = torch.Generator(device=DEV).manual_seed(h)

    def seqs(B):
        k = F.normalize(torch.randn(B, max_pos, 64, device=DEV, generator=g), dim=-1)
        cache = torch.cat([k, torch.randn(B, max_pos, 64, device=DEV, generator=g)], -1).to(torch.bfloat16)
        return cache, torch.randn(B, h * 64, device=DEV, generator=g).to(torch.bfloat16), torch.randn(B, 128, device=DEV, generator=g).to(torch.bfloat16)

    q_scale = 1 + 0.2 * torch.rand(64, device=DEV, generator=g)
    k_scale = 1 + 0.2 * torch.rand(64, device=DEV, generator=g)
    table = torch.randn(h, max_pos, device=DEV, generator=g) * 0.5
    tc, tq, tkv = seqs(1)
    for n in (0, 127, 128, 700, 2047):
        pos = torch.full((1,), n, device=DEV, dtype=torch.int32)
        c1, o1 = tc.clone(), torch.empty(1, h * 64, device=DEV, dtype=torch.bfloat16)
        lib.attn_decode_mqa(tq, tkv, q_scale, k_scale, c1, table, pos, max_pos, o1, h,
                            ws=lib.DecodeWorkspace(DEV, 1, [(1, 8)], max_pos=max_pos, heads=h))
        for B in (5, 16, 17, 200):
            cache, q, kv = seqs(B)
            rows = (0, B // 2, B - 1)
            for r in rows:
                cache[r], q[r], kv[r] = tc[0], tq[0], tkv[0]
            o = torch.empty(B, h * 64, device=DEV, dtype=torch.bfloat16)
            lib.attn_decode_mqa(q, kv, q_scale, k_scale, cache, table, pos, max_pos, o, h,
                                ws=lib.DecodeWorkspace(DEV, B, [(1, 8)], max_pos=max_pos, heads=h))
            for r in rows:
                assert torch.equal(o[r], o1[0]), (h, n, B, r, "output")
                assert torch.equal(cache[r], c1[0]), (h, n, B, r, "cache")


# ------------------------------------------------------------------------------------------------ d. end to end
def test_seeded_generate_does_not_depend_on_batch_row_or_execution():
    """coarse stage at d = 1024, h = 8: a target (prompt, seed) at the first, a middle and the last row of batches of
    1, 3, 16, 17, 40 and 256 with random other rows: its tokens and every trace_logits row are bit-identical to the
    target alone; eager and CUDA-graph runs agree; Engine.seed is untouched; another seed samples other tokens."""
    m, w = _coarse()
    eng = m.engine
    g = torch.Generator().manual_seed(7)
    steps, T = 6, 0.9
    tc = [torch.randint(0, 1024, (1, 12), generator=g).cuda(), torch.randint(0, 1024, (1, 20), generator=g).cuda()]
    tp = torch.randint(0, 1024, (1, 2, 3), generator=g).cuda()
    tseed = 0xC0FFEE_0123456789
    seed_before = eng.seed.clone()
    ref_tr = []
    ref = w.generate(conditioning_token_ids=tc, pred_token_ids=tp, max_time_steps=steps, temperature=T, seeds=[tseed], trace_logits=ref_tr)
    assert torch.equal(w.generate(conditioning_token_ids=tc, pred_token_ids=tp, max_time_steps=steps, temperature=T, seeds=[tseed]), ref)
    for B in (3, 16, 17, 40, 256):
        cond = [torch.randint(0, 1024, (B, 12), generator=g).cuda(), torch.randint(0, 1024, (B, 20), generator=g).cuda()]
        prefix = torch.randint(0, 1024, (B, 2, 3), generator=g).cuda()
        seeds = torch.randint(-2 ** 62, 2 ** 62, (B,), generator=g, dtype=torch.int64)
        rows = sorted({0, B // 2, B - 1})
        for r in rows:
            cond[0][r], cond[1][r], prefix[r] = tc[0][0], tc[1][0], tp[0]
            seeds[r] = tseed - 2 ** 64                 # the same 64 bits as the list entry of the single run
        tr = []
        eager = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=steps, temperature=T, seeds=seeds, trace_logits=tr)
        graph = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, max_time_steps=steps, temperature=T, seeds=seeds)
        assert torch.equal(eager, graph), B
        assert len(tr) == len(ref_tr)
        for r in rows:
            assert torch.equal(eager[r], ref[0]), (B, r)
            for s in range(len(tr)):
                assert torch.equal(tr[s][r], ref_tr[s][0]), (B, r, s)
    assert torch.equal(eng.seed, seed_before), "a seeded call must leave Engine.seed untouched"
    other = w.generate(conditioning_token_ids=tc, pred_token_ids=tp, max_time_steps=steps, temperature=T, seeds=[tseed + 1])
    assert not torch.equal(other, ref)


def test_seeded_generate_argument_errors():
    from open_musiclm_b200 import lib
    m, w = _coarse(depth=1, dim=64, heads=2)
    cond = [torch.randint(0, 64, (2, 4)).cuda(), torch.randint(0, 64, (2, 5)).cuda()]
    with pytest.raises(ValueError, match="exclude"):
        w.generate(conditioning_token_ids=cond, max_time_steps=2, seeds=[1, 2], uniform_noise=torch.rand(6, 2, 1025))
    with pytest.raises(ValueError, match="3 seeds for 2"):
        w.generate(conditioning_token_ids=cond, max_time_steps=2, seeds=[1, 2, 3])
    _, w17 = _coarse(depth=1, dim=64, heads=17)
    with pytest.raises(lib.OmlmError, match="at most 16 heads"):
        w17.generate(conditioning_token_ids=cond, max_time_steps=2, seeds=[1, 2])


# ------------------------------------------------------------------------------------------------ e. reference semantics
def _fixture_model(fx):
    import open_musiclm_b200 as O
    fn = {"semantic": O.create_semantic_transformer, "coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}[fx["stage"]]
    m = fn(**fx["kwargs"])
    m.load_state_dict(fx["state_dict"], strict=True)
    return m.cuda().eval()


@pytest.mark.parametrize("path", GEN, ids=[os.path.basename(p) for p in GEN])
def test_seeded_generate_matches_the_reference_under_the_replica_noise(path):
    """Seeded generate on the reference fixtures' weights and prompts equals the oracle's generate fed, for each row,
    the replica's uniforms of that row's seed: token for token up to near ties (oracle top-2 gap < 5e-2, after which
    that sequence is not compared), with matching logits along the shared trajectory."""
    import open_musiclm_b200 as O
    from oracle import restatement as R
    sys.path.insert(0, os.path.dirname(__file__))
    from test_decode_gpu import _oracle_cfg
    fx = torch.load(path, weights_only=False)
    m = _fixture_model(fx)
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    B = fx["cond"][0].shape[0]
    seeds = [(0x9E3779B97F4A7C15 * (b + 1)) % 2 ** 64 for b in range(B)]
    C = fx["uniforms"].shape[-1]
    kw = dict(pred_token_ids=None if fx["prefix"] is None else fx["prefix"].cuda(), max_time_steps=fx["max_time_steps"],
              filter_thres=fx["filter_thres"], temperature=fx["temperature"], include_eos_in_output=fx["include_eos_in_output"],
              allow_eos_in_output=fx["allow_eos_in_output"])
    trace = []
    out = w.generate(conditioning_token_ids=[t.cuda() for t in fx["cond"]], seeds=seeds, trace_logits=trace, **kw).cpu()
    noise = lambda s, shape: torch.from_numpy(np.stack([seeded_uniforms(sd, s, C) for sd in seeds]))
    ref, otrace = R.generate(_oracle_cfg(fx), fx["state_dict"], [t.numpy() for t in fx["cond"]], noise,
                             pred_token_ids=None if fx["prefix"] is None else fx["prefix"].numpy(), max_time_steps=fx["max_time_steps"],
                             filter_thres=fx["filter_thres"], temperature=fx["temperature"], include_eos_in_output=fx["include_eos_in_output"],
                             allow_eos_in_output=fx["allow_eos_in_output"], return_trace=True)
    ref = torch.as_tensor(ref)
    assert out.shape == ref.shape
    q = out.shape[2]
    n_prefix = 0 if fx["prefix"] is None else fx["prefix"].shape[1] * q
    mine, gold = out.reshape(B, -1)[:, n_prefix:], ref.reshape(B, -1)[:, n_prefix:]
    exact = 0
    for b in range(B):
        for s in range(mine.shape[1]):
            if gold[b, s] == -1:
                assert mine[b, s] == -1
                exact += 1
                continue
            if mine[b, s] != gold[b, s]:
                gap = float(otrace[s][1][b])
                assert gap < 5e-2, (os.path.basename(path), b, s, int(mine[b, s]), int(gold[b, s]), gap)
                break
            exact += 1
            lg, og = trace[s][b].cpu(), otrace[s][0][b]
            fin = torch.isfinite(og)
            assert rel(lg[fin], og[fin]) < 1e-2, (b, s, rel(lg[fin], og[fin]))
    print(f"{os.path.basename(path)}: {exact} of {mine.numel()} seeded tokens identical to the oracle's")
    assert exact >= 0.8 * mine.numel()


# ------------------------------------------------------------------------------------------------ f. MusicLM
def test_seeded_song_of_three_prompts_equals_three_single_prompt_songs():
    """MusicLM.generate_tokens(seeds=...) on the decode path with the small stages of tests/golden/musiclm_windows.pt:
    three prompts in one batch give, bit for bit, the three streams of three single-prompt runs."""
    import open_musiclm_b200 as O
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "musiclm_windows.pt"), weights_only=False)
    fns = {"semantic": O.create_semantic_transformer, "coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}
    models = {}
    for k, fn in fns.items():
        m = fn(**fx["kwargs"][k]); m.load_state_dict(fx["state_dicts"][k], strict=True); models[k] = m.cuda().eval()
    mlm = O.MusicLM(semantic_transformer=models["semantic"], coarse_transformer=models["coarse"], fine_transformer=models["fine"])
    cb, nq = fx["kwargs"]["semantic"]["clap_codebook_size"], fx["kwargs"]["semantic"]["num_clap_quantizers"]
    clap = torch.randint(0, cb, (3, nq), generator=torch.Generator().manual_seed(9)).cuda()
    seeds = [5, 2 ** 64 - 1, 31337]
    batch = mlm.generate_tokens(clap_token_ids=clap, seeds=seeds, return_all=True, **fx["args"])
    for b in range(3):
        one = mlm.generate_tokens(clap_token_ids=clap[b:b + 1], seeds=[seeds[b]], return_all=True, **fx["args"])
        for a, r in zip(batch, one):
            assert torch.equal(a[b:b + 1], r), b
    again = mlm.generate_tokens(clap_token_ids=clap[:1], seeds=[6], return_all=True, **fx["args"])
    assert not torch.equal(again[0], batch[0][:1])
