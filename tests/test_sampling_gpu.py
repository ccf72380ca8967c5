"""The random and discrete kernels of generation and training against exact references:
  - omlm_sample (csrc/decode.cu): eos rule, exact top-k with its tie rule, Gumbel-argmax, against float64 torch written
    from utils.py:71-84, on supplied uniforms and on the device Philox stream (through the host replica of
    tests/test_philox_cpu.py), its counter protocol and CUDA-graph replay, and generate() on the default noise;
  - the dropout keep bits of omlm_ffn_norm_fwd and omlm_forgetful_mask, bit for bit against the replica;
  - omlm_decode_conv_geglu, fed one row at a time, against the float64 causal conv + exact-erf GEGLU of the sequence.
A sampled token may differ from the float64 one only where the best and second-best noisy scores are within
1e-5 * max(1, |best|) of each other (fp32 against float64 arithmetic); such near ties are counted and printed."""
import itertools
import math
import os
import sys

import numpy as np
import pytest
import torch
from scipy import stats

sys.path.insert(0, os.path.dirname(__file__))
from test_philox_cpu import dropout_keep, forgetful_mask, sampler_uniforms  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = -7
PROBE_U = 1.0 - 2.0 ** -24          # the largest float32 below 1: a noise of ~16.6 that outbids every other entry


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as L
    L.device_check()
    return L


# ------------------------------------------------------------------------------------------------ sampler reference
def ref_sample(logits, uniform, k, T, allow_eos):
    """float64 utils.py:71-84 on [B, C] logits and uniforms: eos -> -inf unless allowed, exactly k kept (equal values:
    lower index first; -0.0 equals +0.0), argmax of logits / T - log(-log(u + 1e-20) + 1e-20) over the kept entries.
    Returns (token, gap between the best and second-best kept scores, kept mask)."""
    x = logits.double() + 0.0                     # + 0.0 turns -0.0 into +0.0
    C = x.shape[1]
    if not allow_eos:
        x[:, C - 1] = -math.inf
    order = torch.sort(x, dim=1, descending=True, stable=True).indices
    kept = torch.zeros_like(x, dtype=torch.bool).scatter_(1, order[:, :k], True)
    score = x / T - torch.log(-torch.log(uniform.double() + 1e-20) + 1e-20)
    score = torch.where(kept, score, torch.full_like(score, -math.inf))
    top2 = torch.topk(score, 2, dim=1).values
    gap = torch.where(torch.isfinite(top2[:, 1]), top2[:, 0] - top2[:, 1], torch.full_like(top2[:, 0], math.inf))
    return score.argmax(1), gap, kept, top2[:, 0]


def check_tokens(tokens, logits, uniform, k, T, allow_eos, what=""):
    """tokens [B] (device) against the float64 reference; returns (number of near ties, kept mask)."""
    ref, gap, kept, best = ref_sample(logits, uniform, k, T, allow_eos)
    tokens = tokens.to(ref.device)
    tol = 1e-5 * best.abs().clamp_min(1.0)
    diff = tokens != ref
    near = gap < tol
    bad = diff & ~near
    assert not bad.any(), (what, "rows", bad.nonzero().flatten()[:8].tolist(), "kernel", tokens[bad][:8].tolist(),
                           "float64", ref[bad][:8].tolist(), "gap", gap[bad][:8].tolist())
    assert bool(kept.gather(1, tokens.long()[:, None]).all()), (what, "a token outside the top-k set")
    return int((diff & near).sum()), kept


def sample(lib, logits, C, k, T, allow_eos, uniform=None, seed=None, tokens=None, counters=None, pos=None, next_row=None,
           row_offset=0):
    B = logits.shape[0]
    tokens = torch.full((B, 1), SENTINEL, device=DEV, dtype=torch.int64) if tokens is None else tokens
    counters = torch.zeros(2, device=DEV, dtype=torch.int32) if counters is None else counters
    next_row = torch.full((B,), SENTINEL, device=DEV, dtype=torch.int32) if next_row is None else next_row
    lib.sample(logits, C, k, T, allow_eos, uniform, seed, tokens, next_row, row_offset, counters, pos, B)
    return tokens, counters, next_row


def padded_logits(x, ld):
    """[B, C] logits stored in a [B, ld] buffer whose unused columns hold NaN (they must never be read)."""
    B, C = x.shape
    buf = torch.full((B, ld), math.nan, device=DEV, dtype=torch.float32)
    buf[:, :C] = x
    return buf


def seed_tensor(seed):
    return torch.tensor([seed], dtype=torch.int64, device=DEV)


# ------------------------------------------------------------------------------------------------ supplied uniforms
@pytest.mark.parametrize("C", [2, 3, 64, 1025, 4097, 6145, 8193, 16384])
def test_sampler_matches_float64_on_supplied_uniforms(lib, C):
    """k in {1, 2, 0.1 C, C - 1, C} x T in {0.05, 1, 4} x eos allowed or not, over B in {1, 3, 40, 257} and row strides
    ld = C and ld = C + 37 (NaN in between).  One row in three has integer logits: many values tie at the k-th."""
    g = torch.Generator().manual_seed(C)
    ks = sorted({1, 2, max(int(0.1 * C), 1), C - 1, C})
    near = total = 0
    for i, (k, T, allow) in enumerate(itertools.product(ks, (0.05, 1.0, 4.0), (False, True))):
        B = (1, 3, 40, 257)[i % 4]
        ld = C + 37 if (i // 4) % 2 else C
        x = torch.randn(B, C, generator=g) * 3
        x[2::3] = torch.round(x[2::3])
        u = torch.rand(1, B, C, generator=g)
        x, u = x.to(DEV), u.to(DEV)
        tokens, counters, next_row = sample(lib, padded_logits(x, ld), C, k, T, allow, uniform=u)
        n, _ = check_tokens(tokens[:, 0], x, u[0], k, T, allow, (C, k, T, allow, B, ld))
        near += n
        total += B
        if not allow:
            assert int(tokens.max()) < C - 1
    print(f"C = {C}: {total} tokens, {near} differ from float64 at a near tie")


def _edge_rows(kind, C, g):
    """One [C] logits row of each edge case."""
    if kind == "ties":
        return torch.randint(0, 4, (C,), generator=g).float()
    if kind == "eos_max":
        x = torch.randint(0, 4, (C,), generator=g).float()
        x[C - 1] = 10.0
        return x
    if kind == "neg_inf":
        x = torch.randint(0, 4, (C,), generator=g).float()
        x[torch.randperm(C, generator=g)[: C // 3]] = -math.inf
        x[0] = 2.0                                  # at least one finite entry that is not eos
        return x
    if kind == "signed_zero":                      # the k-th value is a zero; +0.0 and -0.0 interleaved at random
        x = torch.where(torch.rand(C, generator=g) < 0.5, torch.tensor(0.0), torch.tensor(-0.0))
        x[torch.randperm(C - 1, generator=g)[:4]] = 1.0
        return x
    assert kind == "all_equal"
    return torch.full((C,), 0.5)


@pytest.mark.parametrize("C", [64, 1025])
@pytest.mark.parametrize("kind", ["ties", "eos_max", "neg_inf", "signed_zero", "all_equal"])
def test_sampler_keeps_exactly_the_top_k_set(lib, kind, C):
    """Which entries are kept, not only the argmax: row b repeats one edge-case logits row and gives class b the
    uniform 1 - 2^-24 (every other class a uniform in [0.01, 0.5]), so class b is sampled if and only if it is kept
    and finite.  Among equal values at the k-th the lower indices are kept, whatever the sign of a zero."""
    g = torch.Generator().manual_seed(C + len(kind))
    x1 = _edge_rows(kind, C, g)
    x = x1[None].expand(C, C).contiguous().to(DEV)
    u = (0.01 + 0.49 * torch.rand(1, C, C, generator=g))
    u[0, torch.arange(C), torch.arange(C)] = PROBE_U
    u = u.to(DEV)
    for k, allow in itertools.product(sorted({1, 6, max(int(0.1 * C), 1), C // 2, C - 1}), (False, True)):
        tokens, _, _ = sample(lib, x, C, k, 1.0, allow, uniform=u)
        _, kept = check_tokens(tokens[:, 0], x, u[0], k, 1.0, allow, (kind, C, k, allow))
        probe_wins = tokens[:, 0] == torch.arange(C, device=DEV)
        expect = kept.diagonal() & torch.isfinite(x1.to(DEV))
        if not allow:
            expect[C - 1] = False
        assert torch.equal(probe_wins, expect), (kind, C, k, allow, (probe_wins != expect).nonzero().flatten()[:8].tolist())
        assert int(kept.sum(1).min()) == k
        if kind == "eos_max" and not allow:
            assert int(tokens.max()) < C - 1


def test_sampler_signed_zero_rule(lib):
    """+0.0 and -0.0 are the same value: with k = 2 of [-0.0, +0.0, +0.0, -0.0, ...] the classes 0 and 1 are kept."""
    C = 8
    x1 = torch.tensor([-0.0, 0.0, 0.0, -0.0, -0.0, 0.0, -1.0, -1.0])
    x = x1[None].expand(C, C).contiguous().to(DEV)
    u = torch.full((1, C, C), 0.3)
    u[0, torch.arange(C), torch.arange(C)] = PROBE_U
    tokens, _, _ = sample(lib, x, C, 2, 1.0, True, uniform=u.to(DEV))
    wins = (tokens[:, 0].cpu() == torch.arange(C)).tolist()
    assert wins == [True, True, False, False, False, False, False, False], wins


# ------------------------------------------------------------------------------------------------ device Philox stream
@pytest.mark.parametrize("seed", [0, 7, 0x123456789ABCDEF0])
def test_sampler_philox_tokens_equal_the_replica(lib, seed):
    """Default noise: the tokens of three consecutive launches equal the float64 Gumbel-argmax over the replica's
    uniforms at steps 0, 1, 2 (counter (c, b, step, 0x5a17), key = the seed's two halves)."""
    g = torch.Generator().manual_seed(seed & 0xFFFF)
    near = 0
    for C, B, k, T, allow in [(64, 5, 6, 1.0, False), (1025, 40, 102, 0.7, True), (8193, 9, 819, 2.0, False)]:
        x = (torch.randn(B, C, generator=g) * 2).to(DEV)
        tokens = torch.full((B, 3), SENTINEL, device=DEV, dtype=torch.int64)
        counters = torch.zeros(2, device=DEV, dtype=torch.int32)
        for _ in range(3):
            sample(lib, x, C, k, T, allow, seed=seed_tensor(seed), tokens=tokens, counters=counters)
        for step in range(3):
            u = torch.from_numpy(sampler_uniforms(seed, step, B, C)).to(DEV)
            near += check_tokens(tokens[:, step], x, u, k, T, allow, (seed, C, step))[0]
    print(f"seed {seed:#x}: {near} near ties")


def _merged_chisquare(counts, expected):
    """chi-square p-value with every bin of expected count below 5 pooled into one bin."""
    small = expected < 5
    obs, exp = counts[~small].tolist(), expected[~small].tolist()
    if small.any():
        obs.append(counts[small].sum())
        exp.append(expected[small].sum())
    obs, exp = np.array(obs, dtype=np.float64), np.array(exp)
    return stats.chisquare(obs, exp * obs.sum() / exp.sum()).pvalue, len(obs)


@pytest.mark.parametrize("T", [0.7, 1.0, 2.0])
def test_sampler_philox_distribution_is_the_top_k_softmax(lib, T):
    """One realistic logits row (C = 1025, k = 102, eos forbidden and the largest logit) sampled 2048 rows x 16
    launches: the counts follow the exact float64 softmax over the top-k set (chi-square p > 1e-3, fixed seeds), and no
    class outside the set, eos included, is ever drawn."""
    C, k, B, L = 1025, 102, 2048, 16
    g = torch.Generator().manual_seed(11)
    x1 = torch.randn(C, generator=g) * 2.5
    x1[C - 1] = float(x1.max()) + 5
    x = x1[None].expand(B, C).contiguous().to(DEV)
    tokens = torch.full((B, L), SENTINEL, device=DEV, dtype=torch.int64)
    counters = torch.zeros(2, device=DEV, dtype=torch.int32)
    seed = seed_tensor(2024 + int(T * 10))
    for _ in range(L):
        sample(lib, x, C, k, T, False, seed=seed, tokens=tokens, counters=counters)
    counts = np.bincount(tokens.flatten().cpu().numpy(), minlength=C).astype(np.float64)
    xd = x1.double().clone()
    xd[C - 1] = -math.inf
    top = torch.topk(xd, k).indices.numpy()
    outside = np.ones(C, dtype=bool)
    outside[top] = False
    assert counts[outside].sum() == 0 and counts[C - 1] == 0
    p = torch.softmax(xd[top] / T, 0).numpy()
    pval, nbins = _merged_chisquare(counts[top], p * B * L)
    print(f"T = {T}: chi-square over {nbins} bins, p = {pval:.3g}")
    assert pval > 1e-3


def test_sampler_philox_steps_and_rows_are_independent(lib):
    """Six equally likely classes, 2048 rows x 16 launches: uniform marginal, and no dependence between the tokens of
    consecutive steps of one row or of neighbouring rows at one step (contingency chi-square, p > 1e-3)."""
    C, B, L = 6, 2048, 16
    x = torch.zeros(B, C, device=DEV)
    tokens = torch.full((B, L), SENTINEL, device=DEV, dtype=torch.int64)
    counters = torch.zeros(2, device=DEV, dtype=torch.int32)
    for _ in range(L):
        sample(lib, x, C, C, 1.0, True, seed=seed_tensor(31337), tokens=tokens, counters=counters)
    t = tokens.cpu().numpy()
    p_marg = stats.chisquare(np.bincount(t.flatten(), minlength=C)).pvalue
    steps = np.zeros((C, C))
    np.add.at(steps, (t[:, :-1].flatten(), t[:, 1:].flatten()), 1)
    rows = np.zeros((C, C))
    np.add.at(rows, (t[0::2].flatten(), t[1::2].flatten()), 1)
    p_steps, p_rows = stats.chi2_contingency(steps).pvalue, stats.chi2_contingency(rows).pvalue
    print(f"marginal p = {p_marg:.3g}, consecutive steps p = {p_steps:.3g}, neighbouring rows p = {p_rows:.3g}")
    assert min(p_marg, p_steps, p_rows) > 1e-3


# ------------------------------------------------------------------------------------------------ counters and graphs
@pytest.mark.parametrize("B", [1, 7, 300, 1000])
def test_sampler_counter_protocol(lib, B):
    """Each launch writes tokens[b, step] and nothing else of tokens, next_row = row_offset + token, advances step_ptr[0]
    by exactly one and leaves the arrival counter step_ptr[1] at 0; pos advances once per launch when given and is
    untouched otherwise."""
    C, k, seed = 64, 6, 5
    g = torch.Generator().manual_seed(B)
    x = (torch.randn(B, C, generator=g) * 2).to(DEV)
    tokens = torch.full((B, 9), SENTINEL, device=DEV, dtype=torch.int64)
    counters = torch.zeros(2, device=DEV, dtype=torch.int32)
    next_row = torch.full((B,), SENTINEL, device=DEV, dtype=torch.int32)
    pos = torch.tensor([40], device=DEV, dtype=torch.int32)
    for step in range(4):
        with_pos = step < 2
        sample(lib, x, C, k, 1.0, False, seed=seed_tensor(seed), tokens=tokens, counters=counters, next_row=next_row,
               pos=pos if with_pos else None, row_offset=1000 + step)
        assert counters.tolist() == [step + 1, 0]
        assert int(pos) == 40 + min(step + 1, 2)
        assert bool((tokens[:, step + 1:] == SENTINEL).all()) and bool((tokens[:, :step + 1] != SENTINEL).all())
        assert torch.equal(next_row.long(), 1000 + step + tokens[:, step])
        u = torch.from_numpy(sampler_uniforms(seed, step, B, C)).to(DEV)
        check_tokens(tokens[:, step], x, u, k, 1.0, False, ("protocol", B, step))


def test_sampler_graph_replay_follows_the_step_counter(lib):
    """One launch captured in a CUDA graph and replayed five times samples steps 0..4 of the Philox stream."""
    C, B, k, T, seed = 1025, 7, 102, 1.0, 77
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(B, C, generator=g) * 2).to(DEV)
    tokens = torch.full((B, 6), SENTINEL, device=DEV, dtype=torch.int64)
    counters = torch.zeros(2, device=DEV, dtype=torch.int32)
    next_row = torch.zeros(B, device=DEV, dtype=torch.int32)
    s = seed_tensor(seed)
    sample(lib, x, C, k, T, False, seed=s, tokens=tokens, counters=counters, next_row=next_row)   # warm-up (launch set-up)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sample(lib, x, C, k, T, False, seed=s, tokens=tokens, counters=counters, next_row=next_row)
    tokens.fill_(SENTINEL)
    counters.zero_()
    for _ in range(5):
        graph.replay()
    torch.cuda.synchronize()
    assert counters.tolist() == [5, 0] and bool((tokens[:, 5] == SENTINEL).all())
    for step in range(5):
        u = torch.from_numpy(sampler_uniforms(seed, step, B, C)).to(DEV)
        check_tokens(tokens[:, step], x, u, k, T, False, ("graph", step))


def test_generate_default_noise_is_the_replica_stream(lib):
    """generate() on the device Philox stream (small random-init coarse stage): every sampled token equals the float64
    sample from its own logits with the replica's uniforms at its own index in the call and the engine seed of the call;
    the seed advances by one per call, and CUDA-graph replay samples the eager tokens."""
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=128, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=64,
                                    acoustic_codebook_size=64, num_clap_quantizers=4, num_coarse_quantizers=3,
                                    attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    eng = m.engine
    g = torch.Generator().manual_seed(5)
    B, steps, T, C = 3, 5, 0.8, 65
    cond = [torch.randint(0, 64, (B, 4), generator=g).cuda(), torch.randint(0, 64, (B, 11), generator=g).cuda()]
    k = max(int(0.1 * C), 1)
    eng.seed.fill_(0x0BADC0DE12345)
    near = 0
    for call in range(2):
        seed = int(eng.seed)
        trace = []
        out = w.generate(conditioning_token_ids=cond, max_time_steps=steps, temperature=T, trace_logits=trace)
        assert int(eng.seed) == seed + 1
        flat = out.reshape(B, -1)
        assert len(trace) == flat.shape[1] == steps * 3
        for s, lg in enumerate(trace):
            u = torch.from_numpy(sampler_uniforms(seed, s, B, C)).to(DEV)
            near += check_tokens(flat[:, s], lg, u, k, T, False, ("generate", call, s))[0]
        eng.seed.fill_(seed)
        graph = w.generate(conditioning_token_ids=cond, max_time_steps=steps, temperature=T)
        assert torch.equal(graph, out)
    print(f"generate: {near} near ties")


# ------------------------------------------------------------------------------------------------ dropout and forgetful mask
@pytest.mark.parametrize("Fp", [128, 2816])
@pytest.mark.parametrize("drop_p", [0.1, 0.5])
def test_dropout_keep_bits_equal_the_replica(lib, drop_p, Fp):
    """ffn_norm_fwd's keep bits equal the replica for several seeds and layers, and hn is zero exactly where dropped."""
    M = 300
    g = torch.Generator().manual_seed(Fp)
    h = (torch.randn(M, Fp, generator=g) * 2 + 0.5).to(DEV).bfloat16()
    hf = h.float().view(M, Fp // 128, 128)
    rowsum = torch.stack([hf.sum(-1), (hf * hf).sum(-1)], -1).contiguous()
    gamma = (1 + 0.1 * torch.randn(Fp, generator=g)).to(DEV)
    for seed, layer in [(1, 0), (1, 5), (0x0123456789ABCDEF, 0), (42, 23)]:
        hn = torch.empty(M, Fp, device=DEV, dtype=torch.bfloat16)
        stats_ = torch.empty(M, 2, device=DEV)
        kbits = torch.zeros(M, Fp // 8, device=DEV, dtype=torch.uint8)
        lib.ffn_norm_fwd(h, rowsum, gamma, hn, stats_, Fp, Fp, drop_p, seed_tensor(seed), layer, keep_bits=kbits)
        keep = ((kbits[:, :, None] >> torch.arange(8, device=DEV, dtype=torch.uint8)) & 1).bool().reshape(M, Fp).cpu().numpy()
        ref = dropout_keep(seed, layer, np.arange(M), Fp, drop_p)
        assert np.array_equal(keep, ref), (seed, layer, int((keep != ref).sum()))
        zero = (hn == 0).cpu().numpy()
        assert zero[~ref].all() and zero[ref].mean() < 1e-3, (seed, layer)


@pytest.mark.parametrize("N", [2, 777, 12000])
def test_forgetful_mask_equals_the_replica(lib, N):
    """forgetful_mask equals the replica's ranking: the num_drop largest keys dropped, equal keys by position."""
    for seed, stream_id, num_drop in [(12345, 7, int(0.15 * N)), (0x0123456789ABCDEF, (5 << 32) + 3, N - 1), (9, 0, N // 2)]:
        num_drop = min(num_drop, N - 1)
        keep = lib.forgetful_mask(3, N, num_drop, seed_tensor(seed), stream_id, DEV).cpu().numpy()
        ref = forgetful_mask(seed, stream_id, 3, N, num_drop)
        assert np.array_equal(keep, ref), (N, seed, stream_id, num_drop, int((keep != ref).sum()))


# ------------------------------------------------------------------------------------------------ decode conv + GEGLU
def _ileave_cols(F_):
    """canonical column (value c | gate F + c) -> column of the interleaved [B, 2Fp] layout."""
    c = torch.arange(F_)
    a = (c // 128) * 256 + (c % 128)
    return torch.cat([a, a + 128])


def _ulp16(x, dt):
    """one unit in the last place of the 16-bit format at |x| (fp16 subnormals: 2^-24)."""
    mant, tiny = (10, -24) if dt == torch.float16 else (7, -133)
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(torch.clamp(e - mant, min=tiny))


@pytest.mark.parametrize("F_,Fp", [(170, 256), (256, 256)])
@pytest.mark.parametrize("adt", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_decode_conv_geglu_equals_the_float64_sequence(lib, adt, F_, Fp):
    """Rows of u fed one at a time from a zero state: h equals the float64 causal conv (zero left padding) + exact-erf
    GEGLU over the whole sequence within one 16-bit ulp (fp16: saturated at +-65504), padded channels are exactly 0,
    the row sums match float64, and after each step the state holds the last two u rows bit for bit."""
    conv_geglu_check(lib, adt, F_, Fp, 3, 7, F_ + (adt == torch.float16))


def conv_geglu_check(lib, adt, F_, Fp, B, T, seed):
    """decode_conv_geglu over T steps of B rows against the float64 sequence (the assertions of the test above)."""
    g = torch.Generator().manual_seed(seed)
    u_nat = (torch.randn(T, B, 2 * F_, generator=g) * 1.5)
    u_nat[T - 3, :, [0, 1, F_, F_ + 1]] = torch.tensor([1000.0, -1000.0, 1000.0, 1000.0])  # |h| ~ 1e5: the fp16 clamp
    u_nat = u_nat.to(adt)
    cw = (torch.rand(2 * F_, 3, generator=g) * 2 - 1) / math.sqrt(3)
    cw[[0, 1, F_, F_ + 1]] = torch.tensor([0.3, 0.3, 0.4])
    cw = cw.to(DEV)
    cwp = torch.empty(2 * Fp, 3, device=DEV)
    lib.pack(cw, 3, 2 * F_, 3, cwp, 2 * Fp, 3, split_dst=-1, split_src=F_)
    cols = _ileave_cols(F_).to(DEV)
    assert torch.equal(cwp[cols], cw)
    # the interleaved rows; padded columns hold finite junk (the zero padded weights must cancel it)
    u = (torch.randn(T, B, 2 * Fp, generator=g) * 4).to(adt).to(DEV)
    u[:, :, cols] = u_nat.to(DEV)
    # float64 reference over the whole sequence
    ud = torch.nn.functional.pad(u_nat.double().to(DEV), (0, 0, 0, 0, 2, 0))           # [T + 2, B, 2F]
    w = cw.double()
    y = ud[:-2] * w[:, 0] + ud[1:-1] * w[:, 1] + ud[2:] * w[:, 2]
    mag = ud[:-2].abs() * w[:, 0].abs() + ud[1:-1].abs() * w[:, 1].abs() + ud[2:].abs() * w[:, 2].abs()
    yv, yg = y[..., :F_], y[..., F_:]
    gelu = 0.5 * yg * (1 + torch.special.erf(yg / math.sqrt(2)))
    h_ref = gelu * yv
    m = gelu.abs() * mag[..., :F_] + yv.abs() * mag[..., F_:]                              # size of the fp32 terms
    state = torch.zeros(B, 2, 2 * Fp, device=DEV, dtype=adt)
    clamped = 0
    for t in range(T):
        h = torch.full((B, Fp), math.nan, device=DEV, dtype=adt)
        rowsum = torch.full((B, Fp // 128, 2), math.nan, device=DEV)
        lib.decode_conv_geglu(u[t].contiguous(), state, cwp, h, rowsum)
        exp = h_ref[t]
        if adt == torch.float16:
            clamped += int((exp.abs() > 65504).sum())
            exp = exp.clamp(-65504, 65504)
        err = (h[:, :F_].double() - exp).abs()
        bound = _ulp16(exp, adt) + 2e-6 * m[t]
        assert bool((err <= bound).all()), (t, float((err / bound).max()), (err > bound).nonzero()[:4].tolist())
        assert bool((h[:, F_:] == 0).all())
        hp = torch.zeros(B, Fp, device=DEV, dtype=torch.float64)
        hp[:, :F_] = h_ref[t]
        mp = torch.zeros_like(hp)
        mp[:, :F_] = m[t]
        hg, mg = hp.view(B, Fp // 128, 128), mp.view(B, Fp // 128, 128)
        s1, s2 = hg.sum(-1), (hg * hg).sum(-1)
        b1 = 2e-5 * (hg.abs().sum(-1) + mg.sum(-1)) + 1e-30
        b2 = 2e-5 * ((hg * hg).sum(-1) + (hg.abs() * mg).sum(-1)) + 1e-30
        assert bool(((rowsum[..., 0].double() - s1).abs() <= b1).all()), t
        assert bool(((rowsum[..., 1].double() - s2).abs() <= b2).all()), t
        prev = u[t - 1] if t >= 1 else torch.zeros_like(u[0])
        assert torch.equal(state[:, 0].view(torch.int16), prev.view(torch.int16)), t
        assert torch.equal(state[:, 1].view(torch.int16), u[t].view(torch.int16)), t
    if adt == torch.float16:
        assert clamped > 0
