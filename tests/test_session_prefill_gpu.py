"""Packed prefill of a generation session's joiners on the H100: the varlen attention and FFN-up kernels bit-identical
to the fixed-length kernels run on each sequence alone; the packed prefill's installed K/V rows, conv history,
next-token logits and prefix log-probabilities bit-identical to the one-row prefill; and mass joins (every slot filled
at one boundary, also split over a smaller packed workspace) bit-identical to generate alone."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from test_attention_reference_gpu import check, check_lse2, make_inputs, reference  # noqa: E402
from test_generate_ragged_gpu import _model  # noqa: E402
from test_generate_session_gpu import _alone, _request  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL_ROWS = 70


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as L
    L.device_check()
    return L


def _packed_arrays(lens, h):
    from open_musiclm_b200.session import lpt_work
    start = [sum(lens[:b]) for b in range(len(lens))]
    i32 = lambda v: torch.tensor(v, device=DEV, dtype=torch.int32)
    return i32(start), i32(lens), torch.from_numpy(lpt_work(lens, h)).to(DEV).contiguous(), start


# ------------------------------------------------------------------------------------------------ 1. attention
ATTN_LENS = {
    1: [1, 2, 127, 128, 129, 300, 1, 2048, 3],
    2: [1, 63, 64, 65, 2, 500, 3, 41],
    3: [1, 2, 127, 128, 129, 300, 5, 1000, 43],
    8: [1, 2, 15, 17, 127, 128, 129, 1, 2, 700, 1000],
    12: [2, 1, 9, 11, 127, 128, 129, 64, 1500, 1],
    16: [1, 7, 9, 2, 127, 128, 129, 2048, 1, 33],
}


# launches of more than 16 sequences, as scoring packs them; at h = 1 also more than 2^14 rows in all (the varlen
# kernels' row coordinates in their TMA maps)
ATTN_LENS_MANY = {
    1: [2048] * 8 + [1, 2, 127, 128, 129, 300, 3, 64, 65, 1000],
    2: [1, 63, 64, 65, 2, 500, 3, 41] * 3,
    3: [1, 2, 127, 128, 129, 300, 5, 1000, 43] * 2,
    16: [1, 7, 9, 2, 127, 128, 129, 2048, 1, 33] * 2,
}


@pytest.mark.parametrize("h", sorted(ATTN_LENS))
def test_varlen_attention_is_each_sequence_alone(lib, h):
    """Sequences packed without gaps (lengths 1, 2, 128/h +- 1, 127, 128, 129 and up to 2048): out and lse2 equal
    attn_fwd_tc on each sequence alone (B = 1, N = its length), the rows after the last sequence keep their sentinel,
    and one sequence's values lie within the float64 bounds of the fixed-length kernel."""
    _varlen_check(lib, h, ATTN_LENS[h], 77 + h)


@pytest.mark.parametrize("h", sorted(ATTN_LENS_MANY))
def test_varlen_attention_many_sequences(lib, h):
    """test_varlen_attention_is_each_sequence_alone's checks over 18 to 24 sequences in one launch, and past 2^14
    packed rows."""
    _varlen_check(lib, h, ATTN_LENS_MANY[h], 91 + h)


def _varlen_check(lib, h, lens, seed):
    M = sum(lens)
    qn, kvn, table, _, _ = make_inputs(1, M, h, None, "rand", "rand", seed=seed)
    seq_start, seq_len, work, start = _packed_arrays(lens, h)
    out = torch.full((M + SENTINEL_ROWS, h * 64), 7.0, device=DEV, dtype=torch.bfloat16)
    lse = torch.full(((M + SENTINEL_ROWS) * h,), 7.0, device=DEV)
    lib.attn_fwd_tc_varlen(qn, kvn, table, work, seq_start, seq_len, max(lens), out, lse, h)
    for s0, n in zip(start, lens):
        o1 = torch.full((n, h * 64), float("nan"), device=DEV, dtype=torch.bfloat16)
        l1 = torch.full((n * h,), float("nan"), device=DEV)
        lib.attn_fwd_tc(qn[s0:s0 + n].contiguous(), kvn[s0:s0 + n].contiguous(), table, None, o1, l1, 1, n, h)
        assert torch.equal(out[s0:s0 + n], o1), (h, s0, n)
        assert torch.equal(lse[s0 * h:(s0 + n) * h], l1), (h, s0, n)
    assert bool((out[M:] == 7.0).all()) and bool((lse[M * h:] == 7.0).all())
    b = max(range(len(lens)), key=lambda i: lens[i])
    s0, n = start[b], lens[b]
    ref = reference(qn[s0:s0 + n], kvn[s0:s0 + n], table, None, 1, n, h)
    fails = []
    check(fails, "fwd_tc", "out", out[s0:s0 + n], ref["out"].view(n, h * 64), 1, n, h, f"varlen h={h} len={n}")
    check_lse2(fails, "fwd_tc", lse[s0 * h:(s0 + n) * h].view(1, -1), ref["lse2"], f"varlen h={h} len={n}")
    assert not fails, "\n".join(fails)


# ------------------------------------------------------------------------------------------------ 2. FFN up
def _ffn_lens():
    """Sequence starts at every output-tile residue the history rows care about (global row % 126 in 0, 1, 2, 123,
    124, 125: tile offsets 2, 3, 4, 125, 126, 127 of the 128-row tile 126 i - 2 ...), with lengths 1 and 2 among them."""
    lens = [1, 2, 1, 1]
    row = sum(lens)
    for r in (123, 124, 125, 0, 1, 2, 125, 1):
        nxt = row + 1 + (r - row - 1) % 126
        lens.append(nxt - row)
        row = nxt
    return lens + [1, 2, 300, 2, 1, 129]


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("max_ctas", [1, 2, 7])
def test_varlen_ffn_up_is_each_sequence_alone(lib, dt, max_ctas):
    _varlen_ffn_case(lib, dt, max_ctas, 192, 384)


VARLEN_FFN = [(72, 256), (1024, 2816)]        # (K, Fp) of the d = 72 and cfg2 models: a K tail, and 22 channel groups


@pytest.mark.parametrize("K,Fp", VARLEN_FFN)
@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_varlen_ffn_up_at_model_widths(lib, dt, K, Fp):
    _varlen_ffn_case(lib, dt, 0, K, Fp)


def _varlen_ffn_case(lib, dt, max_ctas, K, Fp):
    """The sequences of _ffn_lens packed in one gemm_ffn_up_varlen launch: u, h and rowsum of each equal gemm_ffn_up on
    that sequence alone."""
    lens = _ffn_lens()
    M = sum(lens)
    g = torch.Generator(device=DEV).manual_seed(max_ctas + (dt == torch.float16))
    xn = torch.randn(M, K, device=DEV, generator=g).to(dt)
    w1 = (torch.randn(2 * Fp, K, device=DEV, generator=g) / K ** 0.5).to(dt)
    conv = torch.randn(2 * Fp, 3, device=DEV, generator=g)
    row_pos = torch.cat([torch.arange(n, device=DEV, dtype=torch.int32) for n in lens])
    u = torch.full((M, 2 * Fp), 3.0, device=DEV, dtype=dt)
    hh = torch.full((M, Fp), 3.0, device=DEV, dtype=dt)
    rs = torch.full((M, Fp // 128, 2), 3.0, device=DEV)
    lib.gemm_ffn_up_varlen(xn, w1, conv, u, hh, rs, row_pos, Fp, max_ctas=max_ctas)
    s0 = 0
    for n in lens:
        u1, h1 = torch.empty(n, 2 * Fp, device=DEV, dtype=dt), torch.empty(n, Fp, device=DEV, dtype=dt)
        r1 = torch.empty(n, Fp // 128, 2, device=DEV)
        lib.gemm_ffn_up(xn[s0:s0 + n].contiguous(), w1, conv, u1, h1, r1, n, Fp)
        assert torch.equal(u[s0:s0 + n], u1) and torch.equal(hh[s0:s0 + n], h1) and torch.equal(rs[s0:s0 + n], r1), (s0, n)
        s0 += n


# ------------------------------------------------------------------------------------------------ 3. packed prefill
def _session_model(stage, dim, heads, variant):
    cb = 64 if dim == 128 else 1024
    kw = {}
    if variant == "abspos":
        kw = dict(use_absolute_position_embeddings=True, max_absolute_position_embeddings=200)
    elif variant in ("t5", "none"):
        kw = dict(relative_position_bias_type=variant)
    elif variant == "plainff":
        kw = dict(use_conv_ff=False)
    m, w, _, _ = _model(stage, dim=dim, heads=heads, cb=cb, **kw)
    return m, w, cb


PREFILL_CASES = [("coarse", 128, 2, "continuous", 1), ("coarse", 128, 2, "continuous", 17), ("semantic", 128, 2, "continuous", 64),
                 ("coarse", 128, 2, "abspos", 3), ("semantic", 128, 2, "t5", 17), ("coarse", 128, 2, "none", 3),
                 ("coarse", 128, 2, "plainff", 17), ("coarse", 1024, 8, "continuous", 3), ("semantic", 1024, 16, "continuous", 17),
                 ("semantic", 128, 2, "abspos", 64)]


@pytest.mark.parametrize("stage,dim,heads,variant,k", PREFILL_CASES, ids=[f"{s}-d{d}-h{h}-{v}-k{k}" for s, d, h, v, k in PREFILL_CASES])
def test_packed_prefill_is_each_prefill_alone(stage, dim, heads, variant, k):
    """k joiners with different conditioning lengths and prefixes of 0 ... 3 steps installed by one packed prefill:
    every layer's K/V rows, the conv history, the next-token logits row and the prefix log-probabilities equal the
    one-row prefill (decode.prefill with its _PromptCapture, decode.prefix_logprobs) of each joiner."""
    import open_musiclm_b200 as O
    from open_musiclm_b200.decode import prefill, prefix_logprobs
    from open_musiclm_b200.session import _SlotDecode
    m, w, cb = _session_model(stage, dim, heads, variant)
    q = 3 if stage == "coarse" else 1
    g = torch.Generator().manual_seed(k * 31 + heads)
    shapes = [(1, 40)] + ([(2, 60)] if stage == "coarse" else [])
    reqs = [_request(g, q, cb, shapes, 6) for _ in range(k)]
    for r in reqs:
        r["max_time_steps"] = 6
    sess = O.GenerationSession(w, slots=k + 2, max_positions=200, return_logprobs=True)
    for r in reqs:
        sess.add(**r)
    dec = sess._device_state()
    joined = sess.sched.admit()
    sess._install(joined)
    eng = sess.eng
    ref = _SlotDecode(eng, k + 2, 200, True)
    Cp = eng.Cp[-1]
    for row, r in zip(joined, reqs):
        a = row.payload
        cond = [t.reshape(1, -1) for t in r["conditioning_token_ids"]]
        prefix = a["prefix"]
        pl, ws = prefill(w, cond, prefix, True, ref, slice(row.slot, row.slot + 1), torch.full((1,), row.P, device=DEV))
        P, s = row.P, row.slot
        for l in range(eng.L):
            assert torch.equal(dec.cache[l][s, :P], ref.cache[l][s, :P]), (row.handle, l)
            assert torch.equal(dec.conv[l][s], ref.conv[l][s]), (row.handle, l)
        assert torch.equal(dec.logits[s, :Cp], ref.logits[s, :Cp]), row.handle
        if prefix.shape[1]:
            assert torch.equal(a["prefix_lp"], prefix_logprobs(eng, pl, ws, prefix, q, sess.C)[0]), row.handle
        else:
            assert a["prefix_lp"] is None


# ------------------------------------------------------------------------------------------------ 4. mass joins
MASS_CASES = [("coarse", 17, 0), ("semantic", 40, 0), ("coarse", 256, 0), ("semantic", 40, 150), ("coarse", 17, 60)]


@pytest.mark.parametrize("stage,slots,pack_rows", MASS_CASES, ids=[f"{s}-slots{n}-pack{p or 'default'}" for s, n, p in MASS_CASES])
def test_mass_joins_equal_generate_alone(monkeypatch, stage, slots, pack_rows):
    """Every slot filled at one boundary with requests of mixed shapes, then refilled as rows leave (pack_rows: a
    packed workspace of that many rows, so a boundary splits into several packed prefills): every request's tokens,
    traced logits and return_logprobs triple equal generate alone with its seed, and joins capture no graph."""
    import open_musiclm_b200 as O
    import open_musiclm_b200.session as S
    if pack_rows:
        monkeypatch.setattr(S, "PACK_ROWS", pack_rows)
    q = 3 if stage == "coarse" else 1
    m, w, _, _ = _model(stage)
    g = torch.Generator().manual_seed(slots + pack_rows)
    shapes = [(1, 9)] + ([(2, 14)] if stage == "coarse" else [])
    reqs = [_request(g, q, 64, shapes, 5) for _ in range(slots + slots // 2)]
    for trace, logprob in ((True, False), (False, True)):
        sess = O.GenerationSession(w, slots=slots, max_positions=64, max_queue=len(reqs), trace_logits=trace, return_logprobs=logprob)
        if pack_rows:
            assert min(max(64, pack_rows), slots * 64) < sum(sess._prompt_lengths([c.numel() + 1 for c in r["conditioning_token_ids"]], 0)[0]
                                                             for r in reqs[:slots])
        handles = [sess.add(**r) for r in reqs]
        out, traces, counts = {}, {}, []
        while not sess.idle:
            sess.step()
            done = sess.finished()
            out.update(done)
            if trace:
                traces.update({h: sess.traced_logits(h) for h in done})
            counts.append(sess.graph_count)
        assert len(out) == len(reqs)
        if not trace:
            assert counts[-1] <= 2 * (q + 2) and counts == sorted(counts)
        for h, r in zip(handles, reqs):
            tr = [] if trace else None
            alone = _alone(w, dict(r, return_logprobs=logprob), tr)
            if logprob:
                assert all(torch.equal(x, y[0]) for x, y in zip(out[h], alone)), h
            else:
                assert torch.equal(out[h], alone[0]), h
                assert traces[h].shape[0] == len(tr) and all(torch.equal(traces[h][s], tr[s][0]) for s in range(len(tr))), h
