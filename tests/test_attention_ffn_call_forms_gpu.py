"""The engine's attention and conv feed-forward calls, recorded over every phase of tests/call_forms.py (training
steps, eval_loss, generate, generation sessions with packed and chunked prefills) and replayed against float64.

The recorder wraps lib's attention entry points (attn_fwd_tc, attn_bwd_tc, attn_fwd_tc_varlen, attn_fwd_tc_chunk,
attn_decode, attn_decode_mqa) and conv feed-forward entry points (gemm_ffn_up, gemm_ffn_up_varlen, gemm_ffn_up_chunk,
ffn_norm_fwd, ffn_mid_bwd, decode_conv_geglu) and keeps each call's form: shapes, pitches, flags and, for the packed
and chunked kernels, the host plan of the session's packed prefill (session.PackedPrefill, taken when its arrays are
sent to the device): sequence lengths, p0 per chunk, kv_start, max_len / max_end.  Nothing reads device memory.

Each form is replayed at its shapes with fresh seeded inputs against the float64 references and bounds the families'
own files use (a conv feed-forward form of more than test_ffn_reference_gpu.REF_ROWS rows, as at bench.py's batches, is
launched whole and compared on its first, a middle and its last sequence, each alone) (test_attention_reference_gpu.py, test_generate_ragged_gpu.py, ffn_reference.py with the BOUNDS of
test_ffn_reference_gpu.py, test_sampling_gpu.py's conv step); outputs are poisoned and the rows past them guarded.  A
session issues a new plan at every boundary, so the packed and chunked kernels replay one form per coverage key.

Coverage keys name the properties that select a code path or a seam; the covered set comes from the explicit case
lists of the family files, and a key outside it fails the test (the fix is an explicit case in that file)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as nnf

sys.path.insert(0, os.path.dirname(__file__))
import call_forms  # noqa: E402
import ffn_reference as FR  # noqa: E402
import test_attention_reference_gpu as TA  # noqa: E402
import test_ffn_reference_gpu as TF  # noqa: E402
import test_generate_ragged_gpu as TR  # noqa: E402
import test_sampling_gpu as TS  # noqa: E402
import test_session_chunked_gpu as TC  # noqa: E402
import test_session_prefill_gpu as TP  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = 7.0
BF16, F16 = torch.bfloat16, torch.float16
ATTN = ("attn_fwd_tc", "attn_bwd_tc", "attn_fwd_tc_varlen", "attn_fwd_tc_chunk", "attn_decode", "attn_decode_mqa")
FFN = ("gemm_ffn_up", "gemm_ffn_up_varlen", "gemm_ffn_up_chunk", "ffn_norm_fwd", "ffn_mid_bwd", "decode_conv_geglu")


# ------------------------------------------------------------------------------------------------ coverage keys
def n_class(N):
    """The key tile seams of a sequence length: below one 64-row tile, on 64 and 128 boundaries, beyond 2048."""
    return (N < 64, N % 64 == 0, N % 128 == 0, N > 2048)


def attn_key(h, N, mask, table_ld, det=None, dtable_null=None):
    """attn_fwd_tc (det None) or attn_bwd_tc: heads (h does not divide 64: row tiles start mid-position), N's class,
    key mask, a table wider than N; the backward's mode and whether it forms the bias gradient."""
    k = (h, n_class(N), bool(mask), table_ld > N)
    return ("attn_fwd_tc",) + k if det is None else ("attn_bwd_tc",) + k + (bool(det), bool(dtable_null))


def varlen_keys(h, lens):
    """attn_fwd_tc_varlen: per sequence, whether it is shorter than one chunk unit U; per launch, whether it packs more
    than 16 sequences (as scoring does)."""
    return {("attn_fwd_tc_varlen", h, n < call_forms.unit(h)) for n in lens} | {("attn_fwd_tc_varlen", h, "sequences > 16", len(lens) > 16)}


def chunk_keys(h, seqs, kv_rows):
    """attn_fwd_tc_chunk, per chunk (p0, n, kv_start): shorter than U, p0 > 0, p0 off the 64-row grid, and whether
    the cache rows up to the next sequence's kv_start (or the cache's end) reach past the chunk's end."""
    starts = sorted(s for _, _, s in seqs)
    keys = set()
    for p0, n, s in seqs:
        nxt = next((t for t in starts if t > s), kv_rows)
        keys.add(("attn_fwd_tc_chunk", h, n < call_forms.unit(h), p0 > 0, p0 % 64 != 0, nxt - s > p0 + n))
    return keys


def decode_key(entry, h, ragged, crosses):
    """attn_decode(_mqa): entry, per-row positions, the mqa kernel's head instantiation HM (4, 8 or 16) and whether a
    position reaches past the first 128-key slice."""
    hm = None if entry == "attn_decode" else 4 if h <= 4 else 8 if h <= 8 else 16
    return (entry, bool(ragged), hm, bool(crosses))


def _near(s, m):
    return min(s % m, m - s % m) <= 2


def start_keys(entry, adt, K, Fp, starts, hist=()):
    """FFN up-projections, per sequence start row s of the launch: act dtype, K tail, odd channel-group count, and
    whether s lies within two rows of a 126-row tile seam or a 16-row slab edge; chunks: whether history rows feed it."""
    hist = list(hist) or [False] * len(starts)
    return {(entry, str(adt), K % 64 != 0, (Fp // 128) % 2 == 1, _near(s, 126), _near(s, 16), bool(c)) for s, c in zip(starts, hist)}


def up_keys(adt, K, F, Fp, conv, B, N):
    return {k + (F < Fp, bool(conv)) for k in start_keys("gemm_ffn_up", adt, K, Fp, [b * N for b in range(B)])}


def norm_key(adt, F, Fp, p, copy):
    return ("ffn_norm_fwd", str(adt), F < Fp, (Fp // 128) % 2 == 1, p > 0, bool(copy))


def mid_key(adt, F, Fp, conv, p, parts, det, dgamma_null, dconv_null):
    return ("ffn_mid_bwd", str(adt), F < Fp, (Fp // 128) % 2 == 1, bool(conv), p > 0, parts > 0, bool(det), bool(dgamma_null),
            bool(dconv_null))


def conv_step_key(adt, F, Fp):
    return ("decode_conv_geglu", str(adt), F < Fp)


def covered_keys():
    """Every key the explicit cases of the family files issue."""
    keys = set()
    for B, N, h, mask, _, _ in TA.CASES:
        keys.add(attn_key(h, N, mask, N + 40))
        if h <= 58:
            keys |= {attn_key(h, N, mask, N + 40, det, False) for det in (False, True)}
    for B, N, h, mask, _, _ in TA.EXACT_CASES:
        keys.add(attn_key(h, N, mask, N))
        keys |= {attn_key(h, N, mask, N, det, null) for det in (False, True) for null in (False, True)}
    for h, lens in list(TP.ATTN_LENS.items()) + list(TP.ATTN_LENS_MANY.items()):
        keys |= varlen_keys(h, lens)
    for h, N in TC.CHUNK_ATTN:
        chunks = TC.chunk_attn_chunks(h, N)
        keys |= chunk_keys(h, [(p0, n, s * (N + 8)) for s, (p0, n) in enumerate(chunks)], len(chunks) * (N + 8))
    for entry, B, h, n in TA.DECODE_CASES:
        keys.add(decode_key("attn_" + entry, h, False, n >= 128))
    for entry, B, h in TR.KCASES:
        seed = 31 * B + h
        pos = [TR.KPOS[(b * 5 + seed) % len(TR.KPOS)] for b in range(B)]
        keys.add(decode_key("attn_" + entry, h, True, max(pos) >= 128))
    for d, F, conv, B, N in TF.CASES.values():
        Fp = FR.padded(F)
        for adt in TF.ADT.values():
            keys |= up_keys(adt, d, F, Fp, conv, B, N)
            keys |= {norm_key(adt, F, Fp, p, copy and adt == F16) for p, copy in TF.norm_forms(adt)}
            for p in (0.0, 0.1, 0.5):
                for parts in ([0, Fp // 128] if Fp % 256 == 0 else [0]):
                    keys |= {mid_key(adt, F, Fp, conv, p, parts, det, null, not conv) for det in (False, True) for null in (False, True)}
    lens = TP._ffn_lens()
    starts = [sum(lens[:i]) for i in range(len(lens))]
    for K, Fp in [(192, 384)] + TP.VARLEN_FFN:
        for adt in (F16, BF16):
            keys |= start_keys("gemm_ffn_up_varlen", adt, K, Fp, starts)
    chunks = TC.chunk_ffn_chunks()
    cstarts = [sum(n for _, n in chunks[:i]) for i in range(len(chunks))]
    for K, Fp in TC.CHUNK_FFN:
        for adt in (F16, BF16):
            keys |= start_keys("gemm_ffn_up_chunk", adt, K, Fp, cstarts, [p0 > 0 for p0, _ in chunks])
    for F_, Fp in ((170, 256), (256, 256)):
        keys |= {conv_step_key(adt, F_, Fp) for adt in (BF16, F16)}
    return keys


# ------------------------------------------------------------------------------------------------ the recorder
class _Recorder:
    """Wraps the attention and conv feed-forward entry points of lib (the engine and the decode state look them up as
    module attributes at call time) and session.PackedPrefill.to_device (the host plan of the packed prefill that the
    varlen and chunk calls that follow run)."""

    def __init__(self, lib):
        from open_musiclm_b200 import session
        self.lib, self.session, self.forms, self.phase, self.seen, self.plan = lib, session, set(), None, set(), None
        self.orig = {n: getattr(lib, n) for n in ATTN + FFN}
        self.orig_to_device = session.PackedPrefill.to_device

    def _add(self, name, form):
        self.forms.add((name, form))
        self.seen.add((self.phase, name))

    def _seqs(self, M, n_work):
        p = self.plan
        assert p is not None and p.M == M and len(p.work) == n_work, "a packed call without the plan it runs"
        return p

    def __enter__(self):
        o, rec = self.orig, self

        def to_device(plan, dev):
            rec.plan = plan
            return rec.orig_to_device(plan, dev)

        def attn_fwd_tc(qn, kvn, table, key_mask, out, lse2, B, N, heads, scale=8.0):
            self._add("attn_fwd_tc", (B, N, heads, key_mask is not None, table.stride(0), float(scale)))
            return o["attn_fwd_tc"](qn, kvn, table, key_mask, out, lse2, B, N, heads, scale)

        def attn_bwd_tc(qn, kvn, d_o, out, lse2, table, key_mask, dsum, dqn, dkvn, dtable, B, N, heads, scale=8.0, det=None):
            self._add("attn_bwd_tc", (B, N, heads, key_mask is not None, table.stride(0), float(scale), det is not None, dtable is None))
            return o["attn_bwd_tc"](qn, kvn, d_o, out, lse2, table, key_mask, dsum, dqn, dkvn, dtable, B, N, heads, scale, det=det)

        def attn_fwd_tc_varlen(qn, kvn, table, work, seq_start, seq_len, max_len, out, lse2, heads, scale=8.0):
            p = self._seqs(qn.shape[0], work.shape[0])
            self._add("attn_fwd_tc_varlen", (heads, tuple(int(n) for n in p.P), max_len, table.stride(0)))
            return o["attn_fwd_tc_varlen"](qn, kvn, table, work, seq_start, seq_len, max_len, out, lse2, heads, scale)

        def attn_fwd_tc_chunk(qn, kv, table, work, seq_start, seq_len, q_off, kv_start, max_end, out, lse2, heads, scale=8.0):
            p = self._seqs(qn.shape[0], work.shape[0])
            assert max_end == p.max_end
            seqs = tuple((int(a), int(n), int(s)) for a, n, s in zip(p.p0, p.P, p.kv_start))
            self._add("attn_fwd_tc_chunk", (heads, seqs, max_end, table.stride(0), kv.numel() // 128))
            return o["attn_fwd_tc_chunk"](qn, kv, table, work, seq_start, seq_len, q_off, kv_start, max_end, out, lse2, heads, scale)

        def attn_decode(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, max_pos, out, heads, scale=8.0, ragged=False):
            self._add("attn_decode", (q_raw.shape[0], heads, max_pos, ragged, cache.stride(0), table.stride(0)))
            return o["attn_decode"](q_raw, kv_raw, q_scale, k_scale, cache, table, pos, max_pos, out, heads, scale=scale, ragged=ragged)

        def attn_decode_mqa(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, max_pos, out, heads, ws=None, scale=8.0, ragged=False):
            self._add("attn_decode_mqa", (q_raw.shape[0], heads, max_pos, ragged, cache.stride(0), table.stride(0)))
            return o["attn_decode_mqa"](q_raw, kv_raw, q_scale, k_scale, cache, table, pos, max_pos, out, heads, ws=ws, scale=scale,
                                        ragged=ragged)

        def gemm_ffn_up(xn, w1, conv, u, h, rowsum, Nseq, Fp, max_ctas=0):
            self._add("gemm_ffn_up", (xn.dtype, xn.shape[0], xn.shape[1], Nseq, Fp, max_ctas))
            return o["gemm_ffn_up"](xn, w1, conv, u, h, rowsum, Nseq, Fp, max_ctas=max_ctas)

        def gemm_ffn_up_varlen(xn, w1, conv, u, h, rowsum, row_pos, Fp, max_ctas=0):
            p = self._seqs(xn.shape[0], len(self.plan.work) if self.plan is not None else -1)
            assert not p.p0.any()
            self._add("gemm_ffn_up_varlen", (xn.dtype, xn.shape[1], Fp, tuple(int(n) for n in p.P), max_ctas))
            return o["gemm_ffn_up_varlen"](xn, w1, conv, u, h, rowsum, row_pos, Fp, max_ctas=max_ctas)

        def gemm_ffn_up_chunk(xn, w1, conv, u, h, rowsum, row_pos, hist, hist_idx, Fp, max_ctas=0):
            p = self._seqs(xn.shape[0], len(self.plan.work) if self.plan is not None else -1)
            chunks = tuple((int(a), int(n)) for a, n in zip(p.p0, p.P))
            self._add("gemm_ffn_up_chunk", (xn.dtype, xn.shape[1], Fp, chunks, hist.shape[0], max_ctas))
            return o["gemm_ffn_up_chunk"](xn, w1, conv, u, h, rowsum, row_pos, hist, hist_idx, Fp, max_ctas=max_ctas)

        def ffn_norm_fwd(h, rowsum, gamma, hn, stats, F, Fp, drop_p=0.0, seed=None, layer=0, keep_bits=None, hn_copy=None):
            self._add("ffn_norm_fwd", (h.dtype, h.shape[0], F, Fp, float(drop_p), keep_bits is not None, hn_copy is not None))
            return o["ffn_norm_fwd"](h, rowsum, gamma, hn, stats, F, Fp, drop_p, seed, layer, keep_bits=keep_bits, hn_copy=hn_copy)

        def ffn_mid_bwd(dhn, hn, u, stats, conv_w, gamma, rowstat, du, dgamma, dconv_w, B, N, F, Fp, drop_p=0.0, keep_bits=None,
                        rowstat_parts=0, part=None):
            self._add("ffn_mid_bwd", (u.dtype, B, N, F, Fp, float(drop_p), rowstat_parts, part is not None, dgamma is None, dconv_w is None))
            return o["ffn_mid_bwd"](dhn, hn, u, stats, conv_w, gamma, rowstat, du, dgamma, dconv_w, B, N, F, Fp, drop_p, keep_bits=keep_bits,
                                    rowstat_parts=rowstat_parts, part=part)

        def decode_conv_geglu(u_new, state, conv_w, h_out, rowsum):
            self._add("decode_conv_geglu", (u_new.dtype, u_new.shape[0], u_new.shape[1] // 2))
            return o["decode_conv_geglu"](u_new, state, conv_w, h_out, rowsum)

        for n in ATTN + FFN:
            setattr(self.lib, n, locals()[n])
        self.session.PackedPrefill.to_device = to_device
        return self

    def __exit__(self, *exc):
        for n, f in self.orig.items():
            setattr(self.lib, n, f)
        self.session.PackedPrefill.to_device = self.orig_to_device


def _record(act16, model, monkeypatch):
    from open_musiclm_b200 import lib
    with _Recorder(lib) as rec:
        call_forms.run(rec, model, act16, monkeypatch)
    if model in call_forms.SONGS_ONLY:
        expected = {("song session", n) for n in ("attn_decode_mqa", "decode_conv_geglu", "ffn_norm_fwd")} | \
            {("score songs", n) for n in ("attn_fwd_tc_varlen", "gemm_ffn_up_varlen", "ffn_norm_fwd")}
    elif model in call_forms.BENCH_MODELS:
        expected = {(p, n) for p in ("bench step", "bench deterministic step") for n in ("attn_fwd_tc", "attn_bwd_tc", "gemm_ffn_up",
                                                                                      "ffn_norm_fwd", "ffn_mid_bwd")} | \
            {("eval_loss", "attn_fwd_tc"), ("eval_loss", "gemm_ffn_up")}
        if model in call_forms.GENERATION_MODELS:
            expected |= {("bench generation", n) for n in ("attn_decode", "decode_conv_geglu", "gemm_ffn_up", "ffn_norm_fwd")}
    else:
        expected = {(p, "attn_fwd_tc_chunk") for p in call_forms.SESSION_PHASES} | \
            {(p, n) for p in call_forms.SESSION_PHASES for n in ("attn_decode_mqa", "decode_conv_geglu", "ffn_norm_fwd")} | \
            {("session join", "gemm_ffn_up_varlen"), ("session chunked", "gemm_ffn_up_chunk"), ("session logprobs", "gemm_ffn_up_chunk"),
             ("session sampling", "gemm_ffn_up_varlen")}
    if model in call_forms.SCORE_MODELS:
        expected |= {("score", n) for n in ("attn_fwd_tc_varlen", "gemm_ffn_up_varlen", "ffn_norm_fwd")}
    if model in call_forms.MODELS and model not in call_forms.SESSIONS_ONLY:
        expected |= {(p, n) for p, _, _ in call_forms.TRAIN_PHASES for n in ("attn_fwd_tc", "attn_bwd_tc", "gemm_ffn_up", "ffn_norm_fwd",
                                                                              "ffn_mid_bwd")} | \
            {("eval_loss", "attn_fwd_tc"), ("generate B=3", "attn_decode"), ("generate B=20", "attn_decode_mqa"),
             ("generate B=3", "decode_conv_geglu"), ("generate B=3", "gemm_ffn_up"), ("generate sampling", "attn_decode"),
             ("generate sampling", "attn_decode_mqa")}
    assert expected <= rec.seen, f"entry points the engine did not call through lib: {sorted(expected - rec.seen)}"
    return rec.forms


# ------------------------------------------------------------------------------------------------ attention replays
def _gd(g):
    """A device generator seeded from the host generator g (replays draw their seeds from one host stream)."""
    return torch.Generator(device=DEV).manual_seed(int(torch.randint(1 << 30, (1,), generator=g)))


def _qkv(M, h, g):
    """bf16 unit-norm queries [M, h*64] and keys (values random) [M, 128], as make_inputs draws them."""
    kv = torch.randn(M, 128, device=DEV, generator=g)
    kv[:, :64] = nnf.normalize(kv[:, :64], dim=-1)
    q = nnf.normalize(torch.randn(M, h, 64, device=DEV, generator=g), dim=-1)
    return q.reshape(M, h * 64).bfloat16(), kv.bfloat16()


def _table(h, ld, g):
    """make_inputs' "rand" bias (a random slope per head plus noise) over ld deltas."""
    d = torch.arange(ld, device=DEV, dtype=torch.float32)[None]
    return (0.05 * torch.randn(h, 1, device=DEV, generator=g) * d + 0.3 * torch.randn(h, ld, device=DEV, generator=g)).contiguous()


def _out_bufs(M, h):
    """(out [M, h*64] bf16, lse2 [M*h]) NaN, each the head of a buffer whose two rows past M hold SENT."""
    ob = torch.full((M + 2, h * 64), float("nan"), device=DEV, dtype=BF16)
    lb = torch.full(((M + 2) * h,), float("nan"), device=DEV)
    ob[M:], lb[M * h:] = SENT, SENT
    return ob, lb


def _guards(fails, what, ob, lb, M, h):
    if not (bool((ob[M:] == SENT).all()) and bool((lb[M * h:] == SENT).all())):
        fails.append(f"{what}: rows past M written")


def replay_attn(f, bwd, g):
    from open_musiclm_b200 import lib
    if bwd:
        B, N, h, mask, ld, scale, det, null = f
    else:
        B, N, h, mask, ld, scale = f
    assert scale == 8.0, f
    M = B * N
    qn, kvn, table, key_mask, d_o = TA.make_inputs(B, N, h, "rand" if mask else None, "rand", "rand", seed=int(torch.randint(1 << 30, (1,), generator=g)))
    gd = _gd(g)
    table = _table(h, ld, gd)
    tag = f"engine form {'attn_bwd_tc' if bwd else 'attn_fwd_tc'} {f}"
    ref = TA.reference(qn, kvn, table, key_mask, B, N, h, d_o if bwd else None)
    fails = []
    ob, lb = _out_bufs(M, h)
    lib.attn_fwd_tc(qn, kvn, table, key_mask, ob[:M], lb[:M * h].view(B, N * h), B, N, h)
    torch.cuda.synchronize()
    _guards(fails, tag, ob, lb, M, h)
    out, lse = ob[:M], lb[:M * h].view(B, N * h)
    if not bwd:
        TA.check(fails, "fwd_tc", "out", out, ref["out"].view(M, h * 64), B, N, h, tag)
        TA.check_lse2(fails, "fwd_tc", lse, ref["lse2"], tag)
        return fails, attn_key(h, N, mask, ld)
    ws = lib.AttnBwdDetWorkspace(DEV, B, N, h) if det else None
    dt0 = torch.randn(h, ld, device=DEV, generator=gd)
    dq = torch.full((M + 2, h * 64), float("nan"), device=DEV)
    dkv = torch.full((M + 2, 128), float("nan"), device=DEV)
    dq[M:], dkv[M:] = SENT, SENT
    dt = None if null else dt0.clone()
    lib.attn_bwd_tc(qn, kvn, d_o, out, lse, table, key_mask, torch.empty(M * h, device=DEV), dq[:M], dkv[:M], dt, B, N, h, det=ws)
    torch.cuda.synchronize()
    if not (bool((dq[M:] == SENT).all()) and bool((dkv[M:] == SENT).all())):
        fails.append(f"{tag}: gradient rows past M written")
    kernel = "bwd_tc_det" if det else "bwd_tc"
    peaked = N <= 2
    TA.check(fails, kernel, "dq", dq[:M], ref["dq"], B, N, h, tag, peaked)
    TA.check(fails, kernel, "dk", dkv[:M], ref["dkv"], B, N, h, tag, peaked)
    TA.check(fails, kernel, "dv", dkv[:M], ref["dkv"], B, N, h, tag, peaked)
    if not null:
        if not torch.equal(dt[:, N:], dt0[:, N:]):
            fails.append(f"{tag}: dtable written past N")
        TA.check(fails, kernel, "dtable", dt[:, :N] - dt0[:, :N], ref["dtable"], B, N, h, tag, peaked)
    if ws is not None:
        assert not ws.error()
    return fails, attn_key(h, N, mask, ld, det, null)


def chunk_reference(q_full, kv_full, table, h, seqs, shift=0):
    """Float64 out [sum n, h*64] and lse2 [sum n * h] of packed chunks: chunk (p0, n) of sequence b is the rows p0 ...
    p0 + n - 1 of the reference over its visible prefix, keys 0 ... p0 + n - 1 (q_full[b], kv_full[b]: at least p0 + n
    rows).  shift: the queries placed `shift` positions later (a kernel bug that misreads the query offset)."""
    outs, lses = [], []
    for (p0, n), q, kv in zip(seqs, q_full, kv_full):
        E = p0 + n + shift
        qq = torch.zeros(E, h * 64, device=q.device, dtype=q.dtype)
        qq[p0 + shift:E] = q[p0:p0 + n]
        r = TA.reference(qq, kv[:E], table, None, 1, E, h)
        outs.append(r["out"][0, p0 + shift:E])
        lses.append(r["lse2"][0].view(E, h)[p0 + shift:E].reshape(-1))
    return torch.cat(outs), torch.cat(lses)


def replay_packed_attn(h, seqs, ld, kv_rows, g, chunk=True, shift=0):
    """One attn_fwd_tc_chunk launch (seqs [(p0, n, kv_start)]; cache rows past each chunk's end NaN) or
    attn_fwd_tc_varlen (p0 = 0, kv packed) against float64 -> failures."""
    from open_musiclm_b200 import lib
    from open_musiclm_b200.session import lpt_work
    lens = [n for _, n, _ in seqs]
    M = sum(lens)
    gd = _gd(g)
    table = _table(h, ld, gd)
    full = [_qkv(p0 + n + 1, h, gd) for p0, n, _ in seqs]
    i32 = lambda v: torch.tensor(v, device=DEV, dtype=torch.int32)
    start = [sum(lens[:b]) for b in range(len(lens))]
    q = torch.cat([qf[p0:p0 + n] for (p0, n, _), (qf, _) in zip(seqs, full)])
    work = torch.from_numpy(lpt_work(lens, h, [p0 for p0, _, _ in seqs])).to(DEV).contiguous()
    ob, lb = _out_bufs(M, h)
    if chunk:
        cache = torch.full((kv_rows, 128), float("nan"), device=DEV, dtype=BF16)
        for (p0, n, s), (_, kf) in zip(seqs, full):
            cache[s:s + p0 + n] = kf[:p0 + n]
        cache0 = cache.clone()
        lib.attn_fwd_tc_chunk(q, cache, table, work, i32(start), i32(lens), i32([p0 for p0, _, _ in seqs]), i32([s for _, _, s in seqs]),
                              max(p0 + n for p0, n, _ in seqs), ob[:M], lb[:M * h], h)
    else:
        kv = torch.cat([kf[:n] for (_, n, _), (_, kf) in zip(seqs, full)])
        lib.attn_fwd_tc_varlen(q, kv, table, work, i32(start), i32(lens), max(lens), ob[:M], lb[:M * h], h)
    torch.cuda.synchronize()
    tag = f"{'chunk' if chunk else 'varlen'} h={h} seqs={list(seqs)[:6]}{'...' if len(seqs) > 6 else ''} shift={shift}"
    fails = []
    _guards(fails, tag, ob, lb, M, h)
    if chunk and not torch.equal(cache.view(torch.int16), cache0.view(torch.int16)):
        fails.append(f"{tag}: the cache was written")
    ro, rl = chunk_reference([qf for qf, _ in full], [kf for _, kf in full], table, h, [(p0, n) for p0, n, _ in seqs], shift)
    TA.check(fails, "fwd_tc", "out", ob[:M], ro, 1, M, h, tag)
    TA.check_lse2(fails, "fwd_tc", lb[:M * h].view(1, -1), rl.view(1, -1), tag)
    return fails


def replay_decode(entry, f, g):
    from open_musiclm_b200 import lib
    B, h, max_pos, ragged, cache_ld, table_ld = f
    assert cache_ld == max_pos * 128, f
    gd = _gd(g)
    k_scale = 0.5 + torch.rand(64, device=DEV, generator=gd)
    q_scale = 0.5 + torch.rand(64, device=DEV, generator=gd)
    k = nnf.normalize(torch.randn(B, max_pos, 64, device=DEV, generator=gd), dim=-1) * k_scale
    cache = torch.cat([k, torch.randn(B, max_pos, 64, device=DEV, generator=gd)], -1).bfloat16()
    q_raw = (2 * torch.randn(B, h * 64, device=DEV, generator=gd)).bfloat16()
    kv_raw = (2 * torch.randn(B, 128, device=DEV, generator=gd)).bfloat16()
    d = torch.arange(table_ld, device=DEV, dtype=torch.float32)[None]
    table = (0.5 * torch.randn(h, table_ld, device=DEV, generator=gd) - 0.01 * torch.rand(h, 1, device=DEV, generator=gd) * d).contiguous()
    edge = [0, 126, 127, 128, 129, max_pos - 1]
    if ragged:
        pos_l = [min(edge[b % len(edge)], max_pos - 1) if b < len(edge) else int(torch.randint(max_pos, (1,), generator=g)) for b in range(B)]
    else:
        pos_l = [max_pos - 1] * B
    for b in range(B):
        cache[b, pos_l[b]:] = float("nan")
    cache0 = cache.clone()
    pos = torch.tensor(pos_l if ragged else pos_l[:1], device=DEV, dtype=torch.int32)
    ob = torch.full((B + 1, h * 64), float("nan"), device=DEV, dtype=BF16)
    ob[B:] = SENT
    if entry == "attn_decode":
        lib.attn_decode(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, max_pos, ob[:B], h, ragged=ragged)
    else:
        ws = lib.DecodeWorkspace(DEV, B, [(1, 8)], max_pos=max_pos, heads=h)
        lib.attn_decode_mqa(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, max_pos, ob[:B], h, ws=ws, ragged=ragged)
    torch.cuda.synchronize()
    tag = f"engine form {entry} {f}"
    fails = [] if bool((ob[B:] == SENT).all()) else [f"{tag}: rows past B written"]
    row = torch.cat([(nnf.normalize(kv_raw[:, :64].float(), dim=-1) * k_scale).bfloat16(), kv_raw[:, 64:]], -1)
    for b in range(B):
        n = pos_l[b]
        if not (torch.equal(cache[b, :n], cache0[b, :n]) and bool(torch.isnan(cache[b, n + 1:].float()).all())):
            fails.append(f"{tag}: row {b}: cache rows other than {n} written")
    qn = (nnf.normalize(q_raw.float().view(B, h, 64), dim=-1) * q_scale).bfloat16()
    ref = TR.ragged_decode_reference(cache0, row, qn, table, pos_l)
    TA.check(fails, entry[5:], "out", ob[:B], ref, B, 1, h, tag)
    return fails, decode_key(entry, h, ragged, max_pos > 128)


# ------------------------------------------------------------------------------------------------ FFN replays
def _ffn_weights(K, F, adt, seed):
    """W1, conv weights and gamma of make_case at width K (its xn unused): (c dict)."""
    from open_musiclm_b200 import lib
    return TF.make_case(lib, (K, F, True, 1, 1), adt, seed=seed)


def packed_ffn_reference(c, xs, seqs):
    """Float64 (u, h, s1, s2) and componentwise scales of chunks (p0, n) packed back to back: sequence b's rows p0 ...
    p0 + n - 1 of FR.forward over its whole input xs[b] (>= p0 + n rows)."""
    R, S = [], []
    for (p0, n), x in zip(seqs, xs):
        E = p0 + n
        r = FR.forward(x[:E], c["W1"], c["cw"], c["gam"], E)
        m = FR.magnitude(x[:E], c["W1"], c["cw"], c["gam"], E, floor=TF.FLOOR_S[c["adt"]])
        R.append({k: r[k][p0:E] for k in ("u", "h", "s1", "s2")})
        S.append({k: m[k][p0:E] for k in ("u", "h", "s1", "s2")})
        R[-1]["u_all"] = r["u"]
    cat = lambda L, k: torch.cat([t[k] for t in L])
    return {k: cat(R, k) for k in ("u", "h", "s1", "s2")}, {k: cat(S, k) for k in ("u", "h", "s1", "s2")}, [t["u_all"] for t in R]


def replay_packed_ffn(adt, K, F, Fp, seqs, g, chunk, hist_shift=0, max_ctas=0):
    """One gemm_ffn_up_chunk (seqs [(p0, n)], history rows from the float64 u of the whole sequence, rounded to the
    act dtype; hist_shift = 1 takes them one row early) or gemm_ffn_up_varlen (p0 = 0) launch against float64."""
    from open_musiclm_b200 import lib
    c = _ffn_weights(K, F, adt, int(torch.randint(1 << 20, (1,), generator=g)))
    xs = [torch.randn(p0 + n, K, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7 * i + p0 + n)).to(adt)
          for i, (p0, n) in enumerate(seqs)]
    ref, S, u_all = packed_ffn_reference(c, xs, seqs)
    lens = [n for _, n in seqs]
    M = sum(lens)
    xp = torch.cat([x[p0:p0 + n] for (p0, n), x in zip(seqs, xs)])
    row_pos = torch.cat([torch.arange(p0, p0 + n, device=DEV, dtype=torch.int32) for p0, n in seqs])
    ub, u = TF.guarded(M, 2 * Fp, adt)
    hb, h = TF.guarded(M, Fp, adt)
    rb, rs = TF.guarded(M, Fp // 128 * 2, torch.float32)
    if chunk:
        hist = torch.zeros(2 * len(seqs) + 1, 2 * Fp, device=DEV, dtype=adt)
        hist_idx = torch.full((M,), -1, device=DEV, dtype=torch.int32)
        row = 0
        for b, (p0, n) in enumerate(seqs):
            for j in range(2):
                t = p0 - 2 + j - hist_shift
                if p0 > 0 and t >= 0:
                    hist[2 * b + j] = FR.to_kernel(u_all[b][t:t + 1], F)[0].to(adt)
            if p0 > 0:
                hist_idx[row] = b
            row += n
        lib.gemm_ffn_up_chunk(xp, c["w1p"], c["cwp"], u, h, rs.view(M, Fp // 128, 2), row_pos, hist, hist_idx, Fp, max_ctas=max_ctas)
    else:
        lib.gemm_ffn_up_varlen(xp, c["w1p"], c["cwp"], u, h, rs.view(M, Fp // 128, 2), row_pos, Fp, max_ctas=max_ctas)
    torch.cuda.synchronize()
    tag = f"{'chunk' if chunk else 'varlen'} {adt} K={K} F={F} seqs={list(seqs)[:6]}{'...' if len(seqs) > 6 else ''} hist_shift={hist_shift}"
    fails = []
    for name, buf in (("u", ub), ("h", hb), ("rowsum", rb)):
        TF.guard_ok(fails, f"{name} {tag}", buf, M)
    r = torch.arange(M, device=DEV)
    seq = torch.cat([torch.full((n,), b, device=DEV) for b, n in enumerate(lens)])
    t = torch.cat([torch.arange(n, device=DEV) for n in lens])
    nrow = torch.cat([torch.full((n,), n, device=DEV) for n in lens])
    keys = seq * (M // 126 + 2) + r // 126
    o6 = r % 126
    seams = (t < 2) | (o6 < 2) | (o6 >= 124) | (o6 % 16 >= 14) | (t >= nrow - 2)
    unit = TF.UNIT[adt]
    TF.check(fails, "u", u, FR.to_kernel(ref["u"], F), FR.to_kernel(2 * unit * S["u"], F), keys, seams, tag)
    TF.check(fails, "h chain", h, TF.pad_cols(ref["h"], Fp), TF.pad_cols(2 * unit * S["h"], Fp), keys, seams, tag)
    rsum = rs.view(M, Fp // 128, 2).double().sum(1)
    TF.check(fails, "rowsum chain", rsum, torch.stack([ref["s1"], ref["s2"]], 1), 2 * unit * torch.stack([S["s1"], S["s2"]], 1),
             keys, seams, tag, cb=1)
    return fails


# ------------------------------------------------------------------------------------------------ the test
def _one_per_key(items):
    """{key: first item} over (key, item) pairs in order."""
    out = {}
    for k, it in items:
        for kk in (k if isinstance(k, set) else {k}):
            out.setdefault(kk, it)
    return out


@pytest.mark.parametrize("model", call_forms.MODEL_KEYS)
@pytest.mark.parametrize("act16", ["fp16", "bf16"])
def test_engine_call_forms_replayed_and_covered(act16, model, monkeypatch):
    forms = sorted(_record(act16, model, monkeypatch), key=repr)
    g = torch.Generator().manual_seed(29)
    fails, keys = [], set()
    byname = {}
    for name, f in forms:
        byname.setdefault(name, []).append(f)
    Fmap = {f[3]: f[2] for f in byname.get("ffn_norm_fwd", [])}             # Fp -> F
    Kmap = {}
    for name in ("gemm_ffn_up", "gemm_ffn_up_varlen", "gemm_ffn_up_chunk"):
        for f in byname.get(name, []):
            Kmap[f[4] if name == "gemm_ffn_up" else f[2]] = f[2] if name == "gemm_ffn_up" else f[1]
    # attention
    for f in byname.get("attn_fwd_tc", []):
        fl, k = replay_attn(f, False, g)
        fails += fl
        keys.add(k)
    for f in byname.get("attn_bwd_tc", []):
        fl, k = replay_attn(f, True, g)
        fails += fl
        keys.add(k)
    for name in ("attn_decode", "attn_decode_mqa"):
        for f in byname.get(name, []):
            fl, k = replay_decode(name, f, g)
            fails += fl
            keys.add(k)
    sel = _one_per_key((varlen_keys(f[0], f[1]), f) for f in byname.get("attn_fwd_tc_varlen", []))
    for f in {repr(v): v for v in sel.values()}.values():
        h, lens, max_len, ld = f
        fails += replay_packed_attn(h, [(0, n, 0) for n in lens], ld, 0, g, chunk=False)
    keys |= set(sel)
    sel = _one_per_key((chunk_keys(f[0], f[1], f[4]), f) for f in byname.get("attn_fwd_tc_chunk", []))
    for f in {repr(v): v for v in sel.values()}.values():
        h, seqs, max_end, ld, kv_rows = f
        fails += replay_packed_attn(h, seqs, ld, kv_rows, g)
    keys |= set(sel)
    # conv feed-forward
    norms = byname.get("ffn_norm_fwd", [])
    done_norms = set()
    for f in byname.get("gemm_ffn_up", []):
        adt, M, K, Nseq, Fp, mc = f
        F = Fmap[Fp]
        mine = sorted({(n[4], n[6] or adt == BF16) for n in norms if (n[0], n[1], n[3]) == (adt, M, Fp)})
        done_norms |= {n for n in norms if (n[0], n[1], n[3]) == (adt, M, Fp)}
        c = TF.make_case(_lib(), (K, F, True, M // Nseq, Nseq), adt, seed=M)
        fails += TF.forward_checks(_lib(), c, f"engine form gemm_ffn_up {f}", (mc,), mine or [(0.0, True)],
                                   seqs=TF.check_seqs(M // Nseq, Nseq))
        keys |= up_keys(adt, K, F, Fp, True, M // Nseq, Nseq)
    for n in norms:
        adt, M, F, Fp, p, kb, copy = n
        keys.add(norm_key(adt, F, Fp, p, copy))
        if n not in done_norms:             # the packed prefill's: replayed over one sequence of M rows
            c = TF.make_case(_lib(), (Kmap[Fp], F, True, 1, M), adt, seed=M + 1)
            fails += TF.forward_checks(_lib(), c, f"engine form ffn_norm_fwd {n}", (0,), [(p, copy or adt == BF16)])
    for f in byname.get("ffn_mid_bwd", []):
        adt, B, N, F, Fp, p, parts, det, dg_null, dc_null = f
        c = TF.make_case(_lib(), (Kmap[Fp], F, True, B, N), adt, seed=B * N)
        fails += TF.backward_checks(_lib(), c, f"engine form ffn_mid_bwd {f}", (p,), dets=(det,), seqs=TF.check_seqs(B, N))
        keys.add(mid_key(adt, F, Fp, True, p, parts, det, dg_null, dc_null))
    for name, chunk in (("gemm_ffn_up_varlen", False), ("gemm_ffn_up_chunk", True)):
        items = []
        for f in byname.get(name, []):
            adt, K, Fp, seqs = f[0], f[1], f[2], f[3]
            seqs = [(0, n) for n in seqs] if not chunk else list(seqs)
            starts = [sum(n for _, n in seqs[:i]) for i in range(len(seqs))]
            items.append((start_keys(name, adt, K, Fp, starts, [p0 > 0 for p0, _ in seqs] if chunk else ()), (adt, K, Fp, tuple(seqs), f[-1])))
        sel = _one_per_key(items)
        for adt, K, Fp, seqs, mc in {repr(v): v for v in sel.values()}.values():
            fails += replay_packed_ffn(adt, K, Fmap[Fp], Fp, seqs, g, chunk, max_ctas=mc)
        keys |= set(sel)
    for f in byname.get("decode_conv_geglu", []):
        adt, B, Fp = f
        TS.conv_geglu_check(_lib(), adt, Fmap[Fp], Fp, B, 7, B + Fp)
        keys.add(conv_step_key(adt, Fmap[Fp], Fp))
    print(f"act16={act16} {model}: {len(keys)} keys issued by the engine")
    for fam, pick in (("attention", lambda k: k[0].startswith("attn")), ("conv feed-forward", lambda k: not k[0].startswith("attn"))):
        print(f"  {fam}:")
        for k in sorted(filter(pick, keys), key=repr):
            print("   ", k)
    assert not fails, "\n".join(fails)
    covered = covered_keys()
    missing = sorted((k for k in keys if k not in covered), key=repr)
    assert not missing, f"engine call forms without an explicit case: {missing}"


def _lib():
    from open_musiclm_b200 import lib
    return lib


# ------------------------------------------------------------------------------------------------ discrimination
CHUNK_FORM = (8, ((0, 40, 0), (48, 16, 512), (96, 37, 1024), (16, 5, 1536)), 2048)       # h, (p0, n, kv_start), kv rows


def test_chunk_replay_rejects_a_shifted_query_offset():
    """The chunk replay passes against the reference at the chunks' own offsets and fails its bounds against one whose
    queries sit one position later (a kernel that misreads q_off by one)."""
    h, seqs, kv_rows = CHUNK_FORM
    assert not replay_packed_attn(h, seqs, 600, kv_rows, torch.Generator().manual_seed(3))
    assert replay_packed_attn(h, seqs, 600, kv_rows, torch.Generator().manual_seed(3), shift=1)


@pytest.mark.parametrize("adt", [BF16, F16], ids=["bf16", "fp16"])
def test_chunk_ffn_replay_rejects_history_one_row_early(adt):
    """The chunk FFN-up replay passes with the history rows of positions p0 - 2, p0 - 1 and fails its bounds when they
    are taken one row early."""
    seqs = [(0, 20), (126, 30), (17, 5), (64, 64)]
    assert not replay_packed_ffn(adt, 72, 192, 256, seqs, torch.Generator().manual_seed(4), True)
    assert replay_packed_ffn(adt, 72, 192, 256, seqs, torch.Generator().manual_seed(4), True, hist_shift=1)
