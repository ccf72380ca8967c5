"""Generation with more than 16 sequences: the tensor-core decode GEMM (csrc/decode_gemm.cu) against torch and against
skinny_gemm, the cache-sharing decode attention (attn_decode_mqa) against attn_decode, and generate() at B > 16 against
the B <= 16 path on the same sequences (sequences of a batch are independent).  The B = 20 token parity against the
real reference is tests/golden/gen_coarse_b20.pt, picked up by test_decode_gpu.py."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"

SHAPES = [(512, 1024), (128, 1024), (1024, 512), (5632, 1024), (1024, 2816), (1088, 1024), (192, 128)]


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _inputs(B, N, K, wdt):
    g = torch.Generator(device=DEV).manual_seed(B * 7919 + N + K)
    W = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).to(wdt)
    x = torch.randn(B, K, device=DEV, generator=g) * 2 + 0.3
    gamma = 1 + 0.1 * torch.randn(K, device=DEV, generator=g)
    res = torch.randn(B, N, device=DEV, generator=g)
    Fl = K - 86 if K % 128 == 0 else 0
    hmid = torch.zeros(B, K, device=DEV)
    if Fl:
        hmid[:, :Fl] = torch.randn(B, Fl, device=DEV, generator=g) * 3 + 1
    g3 = gamma.clone()
    g3[Fl:] = 0
    rowsum = torch.stack([hmid.view(B, -1, 128).sum(-1), (hmid ** 2).view(B, -1, 128).sum(-1)], -1).contiguous() if Fl else None
    return W, x, gamma, res, Fl, hmid, g3, rowsum


def _cases(B, N, K, wdt):
    """(prologue, A, kwargs, fp32 reference before the output rounding) for every prologue that applies to K."""
    W, x, gamma, res, Fl, hmid, g3, rowsum = _inputs(B, N, K, wdt)
    Wf = W.float()
    a16 = x.to(wdt)
    out = [(0, a16, dict(addend=res), a16.float() @ Wf.t() + res),
           (1, x, {}, x.to(wdt).float() @ Wf.t()),
           (2, x, dict(gamma=gamma), F.layer_norm(x, (K,), gamma, None, 1e-5).to(wdt).float() @ Wf.t())]
    if Fl:
        h16 = hmid.to(wdt)
        mean = hmid[:, :Fl].mean(-1, keepdim=True)
        var = hmid[:, :Fl].var(-1, unbiased=False, keepdim=True)
        hn = ((h16.float() - mean) * torch.rsqrt(var + 1e-5) * g3).to(wdt).float()
        out.append((3, h16, dict(gamma=g3, rowsum=rowsum, n_real=Fl, addend=res), hn @ Wf.t() + res))
    return W, out


@pytest.mark.parametrize("wdt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("N,K", SHAPES, ids=[f"{n}x{k}" for n, k in SHAPES])
@pytest.mark.parametrize("B", [1, 16, 17, 64, 100, 256])
def test_decode_gemm_against_torch(B, N, K, wdt):
    """Every prologue x output format against torch (skinny_gemm's tolerances); at B <= 16 also against skinny_gemm on
    the same inputs (only the fp32 accumulation order differs); a second call is bit-identical."""
    from open_musiclm_b200 import lib
    W, cases = _cases(B, N, K, wdt)
    ws = lib.DecodeWorkspace(DEV, B, [(N, K)])
    for prologue, A, kw, ref in cases:
        for odt in (torch.float32, torch.bfloat16, torch.float16):
            o = torch.full((B, N), float("nan"), device=DEV, dtype=odt)
            lib.decode_gemm(A, W, o, prologue=prologue, ws=ws, **kw)
            tol = 1e-5 if (prologue == 0 and odt == torch.float32) else 2e-3
            r = ref if odt == torch.float32 else ref.clamp(-65504, 65504).to(odt)
            assert torch.isfinite(o).all() and rel(o, r) < tol, (prologue, odt, rel(o, r))
            again = torch.empty_like(o)
            lib.decode_gemm(A, W, again, prologue=prologue, ws=ws, **kw)
            assert torch.equal(o, again), (prologue, odt, "repeated calls differ")
            if B <= 16:
                sk = torch.empty_like(o)
                lib.skinny_gemm(A, W, sk, prologue=prologue, **kw)
                assert rel(o, sk) < (1e-5 if odt == torch.float32 else 2e-3), (prologue, odt, rel(o, sk))


@pytest.mark.parametrize("n", [0, 127, 128, 1000, 2047])
@pytest.mark.parametrize("h", [2, 3, 8, 16])
@pytest.mark.parametrize("B", [17, 64])
def test_attn_decode_mqa_against_attn_decode(B, h, n):
    from open_musiclm_b200 import lib
    max_pos = 2048
    g = torch.Generator(device=DEV).manual_seed(B * 131 + h * 17 + n)
    k = F.normalize(torch.randn(B, max_pos, 64, device=DEV, generator=g), dim=-1) * (1 + 0.2 * torch.rand(64, device=DEV, generator=g))
    v = torch.randn(B, max_pos, 64, device=DEV, generator=g)
    cache0 = torch.cat([k, v], -1).to(torch.bfloat16)
    q_raw = torch.randn(B, h * 64, device=DEV, generator=g).to(torch.bfloat16)
    kv_raw = torch.randn(B, 128, device=DEV, generator=g).to(torch.bfloat16)
    q_scale = 1 + 0.2 * torch.rand(64, device=DEV, generator=g)
    k_scale = 1 + 0.2 * torch.rand(64, device=DEV, generator=g)
    table = torch.randn(h, max_pos, device=DEV, generator=g) * 0.5
    pos = torch.full((1,), n, device=DEV, dtype=torch.int32)
    c_ref, c_new = cache0.clone(), cache0.clone()
    o_ref = torch.empty(B, h * 64, device=DEV, dtype=torch.bfloat16)
    lib.attn_decode(q_raw, kv_raw, q_scale, k_scale, c_ref, table, pos, max_pos, o_ref, h)
    ws = lib.DecodeWorkspace(DEV, B, [(1, 8)], max_pos=max_pos, heads=h)
    outs = []
    for _ in range(2):
        c_new.copy_(cache0)
        o = torch.empty_like(o_ref)
        lib.attn_decode_mqa(q_raw, kv_raw, q_scale, k_scale, c_new, table, pos, max_pos, o, h, ws=ws)
        outs.append(o)
    assert torch.equal(c_new, c_ref), "the appended cache row must be bit-identical (and nothing else written)"
    assert torch.equal(outs[0], outs[1]), "repeated calls must be bit-identical"
    r = rel(outs[0], o_ref)
    err = (outs[0].float() - o_ref.float()).abs().max().item()
    assert r < 5e-3 and err <= 2e-2 * o_ref.float().abs().max().item(), (r, err)
    assert int(ws.counters.abs().sum()) == 0


def _noisy_top2_gap(lg, u, T, top_k):
    """Gap between the best and second-best Gumbel scores among the top-k logits (eos is never allowed here)."""
    lg = lg.double().clone()
    lg[:, -1] = -float("inf")
    kth = lg.topk(top_k, -1).values[:, -1:]
    s = lg / T - torch.log(-torch.log(u.double() + 1e-20) + 1e-20)
    s = s.masked_fill(lg < kth, -float("inf"))
    t2 = s.topk(2, -1).values
    return (t2[:, 0] - t2[:, 1]).cpu()


def test_batch_of_40_matches_three_batches_of_the_small_batch_path():
    """A model-scale stage (d = 1024, h = 8, L = 2) at B = 40 on the tensor-core path against the same sequences as
    batches of 16, 16 and 8 on the SIMT path, each with its own columns of the noise.  Tokens are equal except where
    the SIMT path's top-2 noisy scores are within 5e-2 (from there that sequence is no longer compared); the logits of
    every step agree to rel-L2 5e-3; eager and CUDA-graph runs sample the same tokens."""
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=2, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    g = torch.Generator().manual_seed(11)
    B, steps, T = 40, 8, 0.9
    cond = [torch.randint(0, 1024, (B, 12), generator=g).cuda(), torch.randint(0, 1024, (B, 20), generator=g).cuda()]
    prefix = torch.randint(0, 1024, (B, 2, 3), generator=g).cuda()
    n_new = (steps - 2) * 3
    uni = torch.rand(n_new, B, 1025, generator=g).clamp_(1e-6, 1 - 1e-6)
    kw = dict(max_time_steps=steps, temperature=T)
    tr = []
    big = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, uniform_noise=uni, trace_logits=tr, **kw)
    big_graph = w.generate(conditioning_token_ids=cond, pred_token_ids=prefix, uniform_noise=uni, **kw)
    assert torch.equal(big, big_graph), "CUDA-graph replay and eager launches must sample the same tokens"
    small, str_ = [], []
    for b0, b1 in ((0, 16), (16, 32), (32, 40)):
        t = []
        small.append(w.generate(conditioning_token_ids=[c[b0:b1] for c in cond], pred_token_ids=prefix[b0:b1],
                                uniform_noise=uni[:, b0:b1].contiguous(), trace_logits=t, **kw))
        str_.append(t)
    small = torch.cat(small, 0)
    strace = [torch.cat([t[s] for t in str_], 0) for s in range(n_new)]
    assert len(tr) == len(strace) == n_new
    top_k = max(int(0.1 * 1025), 1)
    mine, ref = big.reshape(B, -1)[:, 6:].cpu(), small.reshape(B, -1)[:, 6:].cpu()
    live = torch.ones(B, dtype=torch.bool)
    left = 0
    for s in range(n_new):
        rows = live.nonzero().flatten()
        if len(rows):
            r = rel(tr[s][rows.cuda()], strace[s][rows.cuda()])
            assert r <= 5e-3, (s, r)
        gap = _noisy_top2_gap(strace[s], uni[s].cuda(), T, top_k)
        for b in rows.tolist():
            if mine[b, s] != ref[b, s]:
                assert float(gap[b]) < 5e-2, (b, s, int(mine[b, s]), int(ref[b, s]), float(gap[b]))
                live[b] = False
                left += 1
    print(f"B = 40 against 16 + 16 + 8: {left} of {B} sequences left the small-batch trajectory at a near tie")


def test_incremental_step_equals_full_forward_at_batch_40():
    """musiclm_small coarse stage (d = 1024, L = 6, h = 8) at B = 40: the logits of every decode step against the full
    wgmma forward over the same prefix."""
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    g = torch.Generator().manual_seed(5)
    B = 40
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
    print("B = 40 decode vs full forward, worst logits rel-L2 over", len(trace), "steps:", worst)
    assert worst < 5e-3


def test_three_stage_generation_with_batch_20():
    """MusicLM.generate_tokens with 20 clips on random-init small stages: runs end to end (every stage on the batched
    path) and returns streams of the shapes a batch of 2 (the small-batch path) gives."""
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    common = dict(dim=64, depth=1, heads=2, clap_codebook_size=64, num_clap_quantizers=4, attn_dropout=0.0, ff_dropout=0.1)
    sem = O.create_semantic_transformer(semantic_codebook_size=64, **common).cuda().eval()
    coa = O.create_coarse_transformer(semantic_codebook_size=64, acoustic_codebook_size=64, num_coarse_quantizers=3, **common).cuda().eval()
    fin = O.create_fine_transformer(acoustic_codebook_size=64, num_coarse_quantizers=3, num_fine_quantizers=5, **common).cuda().eval()
    mlm = O.MusicLM(semantic_transformer=sem, coarse_transformer=coa, fine_transformer=fin)
    clap = torch.randint(0, 64, (20, 4), generator=torch.Generator().manual_seed(3)).cuda()
    args = dict(output_seconds=3, semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5,
                semantic_steps_per_second=6, acoustic_steps_per_second=8)
    out = mlm.generate_tokens(clap_token_ids=clap, return_all=True, **args)
    ref = mlm.generate_tokens(clap_token_ids=clap[:2], return_all=True, **args)
    outs, refs = (out, ref) if isinstance(out, (tuple, list)) else ((out,), (ref,))
    assert len(outs) == len(refs)
    for a, r in zip(outs, refs):
        assert a.shape[0] == 20 and a.shape[1:] == r.shape[1:], (a.shape, r.shape)
        valid = a[a >= 0]
        assert valid.numel() > 0 and int(valid.max()) < 64


def test_batch_limit_is_256_sequences():
    import open_musiclm_b200 as O
    from open_musiclm_b200 import lib
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=64, depth=1, heads=2, clap_codebook_size=64, semantic_codebook_size=64, acoustic_codebook_size=64,
                                    num_clap_quantizers=4, num_coarse_quantizers=3, attn_dropout=0.0).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    cond = lambda B: [torch.randint(0, 64, (B, 4)).cuda(), torch.randint(0, 64, (B, 5)).cuda()]
    with pytest.raises(lib.OmlmError, match="above 256"):
        w.generate(conditioning_token_ids=cond(257), max_time_steps=2)
    assert w.generate(conditioning_token_ids=cond(256), max_time_steps=2).shape == (256, 2, 3)
