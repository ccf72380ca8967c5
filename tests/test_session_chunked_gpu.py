"""Chunked prefill of a generation session on the H100: the attention with query offsets and K/V read from a cache
(rows past each visible end NaN) and the FFN-up with supplied conv history rows, bit-identical to the fixed-length
kernels on the whole sequence; and sessions with a prefill budget, whose every request equals generate alone."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from test_attention_reference_gpu import make_inputs  # noqa: E402
from test_generate_ragged_gpu import _model  # noqa: E402
from test_generate_session_gpu import _alone, _request, _run_schedule  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as L
    L.device_check()
    return L


def _unit(h):
    return 128 // math.gcd(h, 128)


# ------------------------------------------------------------------------------------------------ 1. attention
# (h, N); (3, 700): the d = 72 model's heads; (3, 100): a whole prompt shorter than U = 128; (8, 645), (16, 645): a final
# chunk shorter than U at p0 = 640, on the 64-row grid
CHUNK_ATTN = [(1, 1000), (2, 700), (6, 650), (8, 1000), (16, 700), (3, 700), (3, 100), (8, 645), (16, 645), (2, 40)]


def chunk_attn_chunks(h, N):
    """(p0, length) of the chunks of test_chunk_attention_is_the_whole_sequence: every U-aligned p0, every third chunk
    to the end of the sequence, the others 1 ... 5 units long."""
    U = _unit(h)
    g = torch.Generator().manual_seed(h)
    chunks = []
    for i, p0 in enumerate(range(0, N, U)):
        rem = N - p0
        n = rem if i % 3 == 0 else min(rem, U * int(torch.randint(1, 6, (1,), generator=g)))
        chunks.append((p0, n))
    return chunks


@pytest.mark.parametrize("h,N", CHUNK_ATTN)
def test_chunk_attention_is_the_whole_sequence(lib, h, N):
    """Chunks at every U-aligned p0 < N (non-final ones of whole units, final ones to the end, p0 = 0 among them),
    all in one launch: each chunk's keys come from its own slot of a cache-shaped buffer that holds the sequence's K/V
    up to the chunk's end and NaN after it.  out and lse2 equal attn_fwd_tc over the whole sequence."""
    from open_musiclm_b200.session import lpt_work
    U = _unit(h)
    qn, kvn, table, _, _ = make_inputs(1, N, h, None, "rand", "rand", seed=500 + h)
    o_ref = torch.empty(N, h * 64, device=DEV, dtype=torch.bfloat16)
    l_ref = torch.empty(N * h, device=DEV)
    lib.attn_fwd_tc(qn, kvn, table, None, o_ref, l_ref, 1, N, h)
    chunks = chunk_attn_chunks(h, N)
    n_max = N + 8
    cache = torch.full((len(chunks), n_max, 128), float("nan"), device=DEV, dtype=torch.bfloat16)
    for s, (p0, n) in enumerate(chunks):
        cache[s, :p0 + n] = kvn[:p0 + n]
    lens = [n for _, n in chunks]
    start = [sum(lens[:b]) for b in range(len(lens))]
    M = sum(lens)
    q = torch.cat([qn[p0:p0 + n] for p0, n in chunks])
    i32 = lambda v: torch.tensor(v, device=DEV, dtype=torch.int32)
    work = torch.from_numpy(lpt_work(lens, h, [p0 for p0, _ in chunks])).to(DEV).contiguous()
    out = torch.full((M, h * 64), 7.0, device=DEV, dtype=torch.bfloat16)
    lse = torch.full((M * h,), 7.0, device=DEV)
    lib.attn_fwd_tc_chunk(q, cache, table, work, i32(start), i32(lens), i32([p0 for p0, _ in chunks]),
                          i32([s * n_max for s in range(len(chunks))]), max(p0 + n for p0, n in chunks), out, lse, h)
    for s0, (p0, n) in zip(start, chunks):
        assert torch.equal(out[s0:s0 + n], o_ref[p0:p0 + n]), (h, p0, n)
        assert torch.equal(lse[s0 * h:(s0 + n) * h], l_ref[p0 * h:(p0 + n) * h]), (h, p0, n)


# ------------------------------------------------------------------------------------------------ 2. FFN up
CHUNK_FFN = [(192, 384), (1024, 2816), (72, 256)]          # (K, Fp); K = 72: a K tail, as the d = 72 model's


def chunk_ffn_chunks():
    """(p0, length) of the chunks of test_chunk_ffn_up_is_the_whole_sequence, in packing order."""
    return [(1, 1), (2, 1), (3, 2), (16, 3), (125, 1), (0, 130), (126, 7), (127, 126), (128, 127), (252, 148), (3, 300), (1, 2),
            (0, 34), (0, 3)]          # the last starts at packed row 882 = 7 x 126, on a tile seam and a slab edge


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("K,Fp", CHUNK_FFN)
def test_chunk_ffn_up_is_the_whole_sequence(lib, dt, K, Fp):
    """Chunks of one sequence at p0 in {1, 2, 3, U, 125, 126, 127, 128, 252} (and a p0 = 0 chunk), packed in one
    launch, each first row's conv history from two supplied rows of the whole run's u (a zero row before position 0):
    u, h and rowsum equal gemm_ffn_up on the whole sequence."""
    N = 400
    g = torch.Generator(device=DEV).manual_seed(K + (dt == torch.float16))
    xn = torch.randn(N, K, device=DEV, generator=g).to(dt)
    w1 = (torch.randn(2 * Fp, K, device=DEV, generator=g) / K ** 0.5).to(dt)
    conv = torch.randn(2 * Fp, 3, device=DEV, generator=g)
    u_ref, h_ref = torch.empty(N, 2 * Fp, device=DEV, dtype=dt), torch.empty(N, Fp, device=DEV, dtype=dt)
    r_ref = torch.empty(N, Fp // 128, 2, device=DEV)
    lib.gemm_ffn_up(xn, w1, conv, u_ref, h_ref, r_ref, N, Fp)
    chunks = chunk_ffn_chunks()
    lens = [n for _, n in chunks]
    M = sum(lens)
    hist = torch.zeros(2 * len(chunks), 2 * Fp, device=DEV, dtype=dt)
    hist_idx = torch.full((M,), -1, device=DEV, dtype=torch.int32)
    row = 0
    for c, (p0, n) in enumerate(chunks):
        for j in range(2):
            if p0 - 2 + j >= 0:
                hist[2 * c + j] = u_ref[p0 - 2 + j]
        if p0 > 0:
            hist_idx[row] = c
        row += n
    xp = torch.cat([xn[p0:p0 + n] for p0, n in chunks])
    row_pos = torch.cat([torch.arange(p0, p0 + n, device=DEV, dtype=torch.int32) for p0, n in chunks])
    u = torch.full((M, 2 * Fp), 3.0, device=DEV, dtype=dt)
    hh = torch.full((M, Fp), 3.0, device=DEV, dtype=dt)
    rs = torch.full((M, Fp // 128, 2), 3.0, device=DEV)
    lib.gemm_ffn_up_chunk(xp, w1, conv, u, hh, rs, row_pos, hist, hist_idx, Fp)
    s0 = 0
    for p0, n in chunks:
        assert torch.equal(u[s0:s0 + n], u_ref[p0:p0 + n]), (p0, n)
        assert torch.equal(hh[s0:s0 + n], h_ref[p0:p0 + n]), (p0, n)
        assert torch.equal(rs[s0:s0 + n], r_ref[p0:p0 + n]), (p0, n)
        s0 += n


# ------------------------------------------------------------------------------------------------ 3. sessions
def _long_requests(g, q, cb, n, max_steps, long_cond):
    """Requests whose conditioning is long enough that their prompts span several units."""
    shapes = [(2, long_cond)] + ([(3, 60)] if q == 3 else [])
    return [_request(g, q, cb, shapes, max_steps) for _ in range(n)]


SESSION_CASES = [("coarse", 1, 128, 2, False, 64, 3), ("coarse", 17, 128, 2, False, 192, 30), ("semantic", 40, 128, 2, False, 1000, 60),
                 ("coarse", 256, 128, 2, False, 4096, 280), ("semantic", 17, 128, 2, False, 64, 24), ("coarse", 17, 128, 2, True, 192, 24),
                 ("coarse", 5, 1024, 8, False, 16, 8), ("semantic", 5, 1024, 16, False, 24, 8), ("coarse", 40, 128, 2, False, 1000, 50),
                 ("semantic", 17, 128, 4, True, 4096, 24)]


@pytest.mark.parametrize("stage,slots,dim,heads,abs_pos,budget,n_req", SESSION_CASES,
                         ids=[f"{s}-slots{n}-d{d}-h{h}-{'abspos' if a else 'relpos'}-rows{b}" for s, n, d, h, a, b, _ in SESSION_CASES])
def test_chunked_sessions_equal_generate_alone(stage, slots, dim, heads, abs_pos, budget, n_req):
    """A random join schedule with prompts longer than the budget (prefill_rows in {U, 3U, 1000, 4096}): every request's
    tokens and traced logits equal generate alone with its seed, and graphs stay within 2 (q + 2)."""
    import open_musiclm_b200 as O
    q = 3 if stage == "coarse" else 1
    max_steps = 5 if stage == "coarse" else 10
    cb = 64 if dim == 128 else 1024
    extra = dict(use_absolute_position_embeddings=True, max_absolute_position_embeddings=400) if abs_pos else {}
    m, w, _, _ = _model(stage, dim=dim, heads=heads, cb=cb, **extra)
    g = torch.Generator().manual_seed(slots * 13 + budget + heads)
    reqs = _long_requests(g, q, cb, n_req, max_steps, 300)
    trace = dim == 1024 or slots in (1, 17)
    sess = O.GenerationSession(w, slots=slots, max_positions=512, max_queue=8, trace_logits=trace, prefill_rows=budget)
    assert sess.sched.unit == _unit(heads)
    traces = {} if trace else None
    got = _run_schedule(sess, reqs, g, traces)
    if not trace:
        assert sess.graph_count <= 2 * (q + 2)
    for i, r in enumerate(reqs):
        tr = [] if trace else None
        alone = _alone(w, r, tr)
        assert torch.equal(got[i], alone[0]), i
        if trace:
            assert traces[i].shape[0] == len(tr) and all(torch.equal(traces[i][s], tr[s][0]) for s in range(len(tr))), i


@pytest.mark.parametrize("stage,budget", [("coarse", 64), ("semantic", 192)])
def test_chunked_logprobs_equal_the_unchunked_session(stage, budget):
    """With return_logprobs (prefixes that chunks split), every request's (tokens, logprobs, sample_logprobs) equals
    the unchunked session's, which equals generate alone."""
    import open_musiclm_b200 as O
    q = 3 if stage == "coarse" else 1
    m, w, _, _ = _model(stage)
    outs = []
    for rows in (None, budget):
        g = torch.Generator().manual_seed(77)
        reqs = _long_requests(g, q, 64, 12, 5 if q == 3 else 10, 200)
        for r in reqs[::2]:                    # long prefixes, so that a chunk boundary falls inside them
            r["pred_token_ids"] = torch.randint(0, 64, (1, 70 // q, q) if q > 1 else (1, 70, 1), generator=g).cuda()[..., :q]
            r["max_time_steps"] = 70 // q + 3
        sess = O.GenerationSession(w, slots=4, max_positions=512, max_queue=16, return_logprobs=True, prefill_rows=rows)
        outs.append(_run_schedule(sess, reqs, g))
    for i in outs[0]:
        assert all(torch.equal(a, b) for a, b in zip(outs[0][i], outs[1][i])), i


def test_chunked_slot_reuse_and_three_stages():
    """Semantic, coarse and fine wrappers through one-slot and three-slot sessions with the smallest budget: a slot's
    occupants follow each other after chunked prefills, and each equals generate alone."""
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    kw = dict(dim=128, depth=2, heads=2, clap_codebook_size=64, num_clap_quantizers=4, attn_dropout=0.0, ff_dropout=0.0)
    models = {"semantic": (O.create_semantic_transformer(semantic_codebook_size=64, **kw), 1),
              "coarse": (O.create_coarse_transformer(semantic_codebook_size=64, acoustic_codebook_size=64, num_coarse_quantizers=3, **kw), 3),
              "fine": (O.create_fine_transformer(acoustic_codebook_size=64, num_coarse_quantizers=3, num_fine_quantizers=4, **kw), 4)}
    for name, (m, q) in models.items():
        m = m.cuda().eval()
        w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
        g = torch.Generator().manual_seed(len(name))
        shapes = [(100, 250)] + ([(6, 60)] if name == "coarse" else [(90, 90)] if name == "fine" else [])
        reqs = [_request(g, q, 64, shapes, 4) for _ in range(6)]
        if name == "fine":       # the coarse conditioning holds whole time steps of 3 quantizers
            for r in reqs:
                r["conditioning_token_ids"][1] = r["conditioning_token_ids"][1][:, :90]
        for slots in (1, 3):
            sess = O.GenerationSession(w, slots=slots, max_positions=512, max_queue=8, prefill_rows=64)
            got = _run_schedule(sess, reqs, g)
            for i, r in enumerate(reqs):
                assert torch.equal(got[i], _alone(w, r)[0]), (name, slots, i)
