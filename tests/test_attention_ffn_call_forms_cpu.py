"""Host parts of the attention / conv feed-forward call-form inventory (test_attention_ffn_call_forms_gpu.py): its
coverage keys on hand-made forms, the covered set that the explicit case lists produce, and the packed / chunked
float64 references against a brute-force per-sequence computation."""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(__file__))
import call_forms  # noqa: E402
import test_attention_ffn_call_forms_gpu as T  # noqa: E402

BF16, F16 = torch.bfloat16, torch.float16


def test_attention_keys_on_hand_made_forms():
    assert T.n_class(63) == (True, False, False, False)
    assert T.n_class(1024) == (False, True, True, False)
    assert T.n_class(2049) == (False, False, False, True)
    assert T.n_class(192) == (False, True, False, False)
    assert T.attn_key(3, 50, True, 50) == ("attn_fwd_tc", 3, (True, False, False, False), True, False)
    assert T.attn_key(8, 1024, False, 1100, det=True, dtable_null=True) == \
        ("attn_bwd_tc", 8, (False, True, True, False), False, True, True, True)
    assert T.varlen_keys(8, [1, 16, 300]) == {("attn_fwd_tc_varlen", 8, True), ("attn_fwd_tc_varlen", 8, False),
                                              ("attn_fwd_tc_varlen", 8, "sequences > 16", False)}
    assert ("attn_fwd_tc_varlen", 8, "sequences > 16", True) in T.varlen_keys(8, [20] * 17)
    # h = 3: U = 128; one chunk at p0 = 0, one short final chunk at p0 = 128 (on the 64 grid), the cache 512 rows a slot
    keys = T.chunk_keys(3, [(0, 128, 0), (128, 30, 512)], 1024)
    assert keys == {("attn_fwd_tc_chunk", 3, False, False, False, True), ("attn_fwd_tc_chunk", 3, True, True, False, True)}
    # h = 16: U = 8, p0 = 40 lies off the 64-row grid; a slot exactly as long as the chunk's end leaves no gap
    assert T.chunk_keys(16, [(40, 8, 0)], 48) == {("attn_fwd_tc_chunk", 16, False, True, True, False)}
    assert T.decode_key("attn_decode", 3, True, False) == ("attn_decode", True, None, False)
    assert [T.decode_key("attn_decode_mqa", h, True, True)[2] for h in (1, 3, 4, 5, 8, 9, 16)] == [4, 4, 4, 8, 8, 16, 16]


def test_ffn_keys_on_hand_made_forms():
    # starts 0, 50, 100, 150 of B = 4 sequences of 50 rows: 50 lies two rows past the 16-row slab edge at 48
    assert T.up_keys(BF16, 72, 192, 256, True, 4, 50) == {
        ("gemm_ffn_up", str(BF16), True, False, True, True, False, True, True),
        ("gemm_ffn_up", str(BF16), True, False, False, True, False, True, True),
        ("gemm_ffn_up", str(BF16), True, False, False, False, False, True, True)}
    assert T.start_keys("gemm_ffn_up_chunk", F16, 1024, 384, [0, 124, 130], [False, True, True]) == {
        ("gemm_ffn_up_chunk", str(F16), False, True, True, True, False),
        ("gemm_ffn_up_chunk", str(F16), False, True, True, False, True),
        ("gemm_ffn_up_chunk", str(F16), False, True, False, True, True)}
    assert T.norm_key(F16, 2730, 2816, 0.1, True) == ("ffn_norm_fwd", str(F16), True, False, True, True)
    assert T.mid_key(BF16, 192, 256, True, 0.0, 2, True, True, False) == \
        ("ffn_mid_bwd", str(BF16), True, False, True, False, True, True, True, False)
    assert T.conv_step_key(BF16, 256, 256) == ("decode_conv_geglu", str(BF16), False)


def test_covered_set_holds_what_the_explicit_lists_cover():
    cov = T.covered_keys()
    # training shapes: the exact-width table and the backward without a bias gradient, both modes
    for det in (False, True):
        for null in (False, True):
            assert T.attn_key(3, 50, True, 50, det, null) in cov
            assert T.attn_key(8, 1024, True, 1024, det, null) in cov
            assert T.attn_key(16, 1024, True, 1024, det, null) in cov      # bench.py's cfg4 training step
    assert T.attn_key(16, 1024, True, 1024) in cov
    assert T.attn_key(8, 15, True, 15) in cov                          # the semantic stage's prefill in bench generation
    assert T.attn_key(1, 1, False, 41) in cov                          # CASES[0]
    assert T.attn_key(3, 257, True, 257 + 40) in cov                    # CASES (2, 257, 3, ...)
    assert T.attn_key(3, 3000, True, 3040) not in cov                   # no case runs N > 2048
    # the chunk tests: every head count, p0 = 0 chunks to the end, p0 > 0 off the 64-row grid where U < 64
    for h in (1, 2, 3, 6, 8, 16):
        assert ("attn_fwd_tc_chunk", h, False, False, False, True) in cov
        assert ("attn_fwd_tc_chunk", h, False, True, False, True) in cov
        assert (("attn_fwd_tc_chunk", h, False, True, True, True) in cov) == (call_forms.unit(h) < 64)
    for h in (1, 8, 12, 16):
        assert {("attn_fwd_tc_varlen", h, True), ("attn_fwd_tc_varlen", h, False)} <= cov
    for ragged in (False, True):
        for hm in (4, 8, 16):
            assert ("attn_decode_mqa", ragged, hm, True) in cov
    # the FFN files: the K tail and both act dtypes in the varlen and chunk tests, history rows, the null dgamma
    for adt in (BF16, F16):
        for entry in ("gemm_ffn_up_varlen", "gemm_ffn_up_chunk"):
            assert any(k[:3] == (entry, str(adt), True) for k in cov)
        assert ("gemm_ffn_up_chunk", str(adt), False, True, True, True, True) in cov
        assert T.mid_key(adt, 192, 256, True, 0.1, 2, True, True, False) in cov
        assert T.norm_key(adt, 192, 256, 0.0, False) in cov
    assert T.norm_key(F16, 192, 256, 0.1, True) in cov


def _brute_attention(q, kv, table, h, p0, n):
    """Rows p0 ... p0 + n - 1, one at a time: softmax over keys 0 ... position of 8 q.k + table[head, i - j]."""
    out = torch.zeros(n, h * 64, dtype=torch.float64)
    lse = torch.zeros(n, h, dtype=torch.float64)
    for r in range(n):
        i = p0 + r
        for hh in range(h):
            qv = q[i, hh * 64:(hh + 1) * 64].double()
            s = torch.stack([8.0 * qv @ kv[j, :64].double() + float(table[hh, i - j]) for j in range(i + 1)])
            p = torch.softmax(s, 0)
            out[r, hh * 64:(hh + 1) * 64] = p @ kv[:i + 1, 64:].double()
            lse[r, hh] = torch.logsumexp(s, 0) / math.log(2.0)
    return out, lse.reshape(-1)


def test_chunk_reference_slices_each_visible_prefix():
    g = torch.Generator().manual_seed(0)
    h, seqs = 3, [(0, 5), (7, 4), (2, 1)]
    q = [torch.randn(p0 + n + 1, h * 64, generator=g).bfloat16() for p0, n in seqs]
    kv = [torch.randn(p0 + n + 1, 128, generator=g).bfloat16() for p0, n in seqs]
    table = torch.randn(h, 20, generator=g)
    out, lse = T.chunk_reference(q, kv, table, h, seqs)
    bo, bl = zip(*[_brute_attention(qq, kk, table, h, p0, n) for (p0, n), qq, kk in zip(seqs, q, kv)])
    assert torch.allclose(out, torch.cat(bo), rtol=0, atol=1e-12)
    assert torch.allclose(lse, torch.cat(bl), rtol=0, atol=1e-12)
    # the shifted reference differs: the same queries one position later see other biases and one more key
    out1, _ = T.chunk_reference(q, kv, table, h, seqs, shift=1)
    assert float((out1 - out).abs().max()) > 1e-3


def test_packed_ffn_reference_slices_each_whole_sequence():
    g = torch.Generator().manual_seed(1)
    K, F = 8, 5
    c = dict(W1=torch.randn(2 * F, K, generator=g), cw=torch.randn(2 * F, 3, generator=g), gam=torch.randn(F, generator=g),
             adt=BF16)
    seqs = [(0, 3), (4, 2), (1, 1)]
    xs = [torch.randn(p0 + n, K, generator=g) for p0, n in seqs]
    ref, S, u_all = T.packed_ffn_reference(c, xs, seqs)
    rows = []
    for (p0, n), x in zip(seqs, xs):
        u = x.double() @ c["W1"].double().t()
        for t in range(p0, p0 + n):
            y = sum(c["cw"][:, k].double() * (u[t - 2 + k] if t - 2 + k >= 0 else 0.0) for k in range(3))
            hv = torch.nn.functional.gelu(y[F:]) * y[:F]
            rows.append((u[t], hv))
    assert torch.allclose(ref["u"], torch.stack([r[0] for r in rows]), rtol=0, atol=1e-12)
    assert torch.allclose(ref["h"], torch.stack([r[1] for r in rows]), rtol=0, atol=1e-12)
    assert torch.allclose(ref["s1"], ref["h"].sum(1)) and torch.allclose(ref["s2"], (ref["h"] ** 2).sum(1))
    assert all(u.shape[0] == p0 + n for u, (p0, n) in zip(u_all, seqs))
    assert bool((S["u"] >= ref["u"].abs()).all()) and bool((S["h"] >= ref["h"].abs() - 1e-12).all())
