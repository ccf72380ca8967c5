"""Prefixes of different lengths in one generate call (`generate(pred_lengths=...)`) on the H100 decode path: the
shared-position path untouched, the per-row decode kernels (omlm_attn_decode_ragged, omlm_attn_decode_mqa_ragged,
omlm_embed_gather_pos_ragged) against float64 and host references, every row of a ragged batch against the float
restatement of that row alone (tests/test_generate_ragged_cpu.py), seeded rows bit-identical to the row alone, the
absolute-position limits per row, and the shipped model widths."""
import dataclasses
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(__file__))
from test_attention_reference_gpu import check  # noqa: E402
from test_generate_ragged_cpu import ragged_reference  # noqa: E402
from test_stages_cpu import oracle_cfg  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
NEAR_TIE = 5e-2      # oracle top-2 gap below which 16-bit logits may legitimately sample the other token


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _model(stage="coarse", dim=128, depth=2, heads=2, cb=64, **kw):
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    args = dict(dim=dim, depth=depth, heads=heads, clap_codebook_size=cb, num_clap_quantizers=4, attn_dropout=0.0, ff_dropout=0.1, **kw)
    if stage == "coarse":
        m = O.create_coarse_transformer(semantic_codebook_size=cb, acoustic_codebook_size=cb, num_coarse_quantizers=3, **args)
    else:
        m = O.create_semantic_transformer(semantic_codebook_size=cb, **args)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m = m.cuda().eval()
    return m, O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False), sd, args


def _prompts(B, stage, steps, cb, g, n_cond=(4, 9)):
    q = 3 if stage == "coarse" else 1
    cond = [torch.randint(0, cb, (B, n_cond[0]), generator=g)]
    if stage == "coarse":
        cond.append(torch.randint(0, cb, (B, n_cond[1]), generator=g))
    pred = torch.randint(0, cb, (B, steps, q), generator=g) if q > 1 else torch.randint(0, cb, (B, steps), generator=g)
    return [t.cuda() for t in cond], pred.cuda(), q


def _alone(w, cond, pred, b, n, **kw):
    """Row b alone with its first n steps as the prefix."""
    return w.generate(conditioning_token_ids=[t[b:b + 1] for t in cond], pred_token_ids=pred[b:b + 1, :n] if n > 0 else None, **kw)


# ------------------------------------------------------------------------------------------------ 1. off means off
@pytest.mark.parametrize("seeded", [False, True])
@pytest.mark.parametrize("B", [3, 20])
def test_full_lengths_are_the_shared_position_path(B, seeded):
    """pred_lengths=[n] * B (n = the prefix's steps) is the call without pred_lengths, bit for bit: tokens and traced
    logits eagerly, tokens from CUDA graphs and from eager launches without a trace; SIMT (B = 3) and tensor-core
    (B = 20) decode, with the Engine.seed stream (reset before each call) or with per-row seeds."""
    m, w, _, _ = _model()
    eng = m.engine
    g = torch.Generator().manual_seed(B)
    cond, pred, _ = _prompts(B, "coarse", 3, 64, g)
    kw = dict(conditioning_token_ids=cond, pred_token_ids=pred, max_time_steps=7, temperature=0.8)
    if seeded:
        kw["seeds"] = [int(v) for v in torch.randint(0, 2 ** 62, (B,), generator=g)]
    s0 = eng.seed.clone()
    runs = {}
    for lengths in (None, [3] * B, torch.full((B,), 3, dtype=torch.int64)):
        key = "none" if lengths is None else "list" if isinstance(lengths, list) else "tensor"
        for mode in ("trace", "graph", "eager"):
            eng.seed.copy_(s0)
            tr = [] if mode == "trace" else None
            out = w.generate(pred_lengths=lengths, trace_logits=tr, use_cuda_graph=mode == "graph", **kw)
            runs[key, mode] = (out, tr)
    for key in ("list", "tensor"):
        for mode in ("trace", "graph", "eager"):
            assert torch.equal(runs[key, mode][0], runs["none", mode][0]), (key, mode)
        tr, tr0 = runs[key, "trace"][1], runs["none", "trace"][1]
        assert len(tr) == len(tr0) and all(torch.equal(a, b) for a, b in zip(tr, tr0))
    assert torch.equal(runs["none", "graph"][0], runs["none", "trace"][0])


# ------------------------------------------------------------------------------------------------ 2. kernels
MAX_POS = 300
KPOS = [0, 126, 127, 128, 129, 255, 256, MAX_POS - 1]       # key counts 1, 127, 128, 129, 130, ... 300


def _decode_inputs(B, h, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ld = MAX_POS + 8
    k_scale = 0.5 + torch.rand(64, device=DEV, generator=g)
    q_scale = 0.5 + torch.rand(64, device=DEV, generator=g)
    k = F.normalize(torch.randn(B, MAX_POS, 64, device=DEV, generator=g), dim=-1) * k_scale
    v = torch.randn(B, MAX_POS, 64, device=DEV, generator=g)
    cache = torch.cat([k, v], -1).bfloat16()
    q_raw = (2 * torch.randn(B, h * 64, device=DEV, generator=g)).bfloat16()
    kv_raw = (2 * torch.randn(B, 128, device=DEV, generator=g)).bfloat16()
    d = torch.arange(ld, device=DEV, dtype=torch.float32)[None]
    table = (0.5 * torch.randn(h, ld, device=DEV, generator=g) - 0.01 * torch.rand(h, 1, device=DEV, generator=g) * d).contiguous()
    pos = torch.tensor([KPOS[(b * 5 + seed) % len(KPOS)] for b in range(B)], device=DEV, dtype=torch.int32)
    for b in range(B):
        cache[b, int(pos[b]):] = float("nan")                 # a read past a row's own position shows as non-finite output
    return q_raw, kv_raw, q_scale, k_scale, cache, table, pos


def _run_decode(lib, kernel, q_raw, kv_raw, q_scale, k_scale, cache, table, pos, h):
    B = q_raw.shape[0]
    out = torch.full((B, h * 64), float("nan"), device=DEV, dtype=torch.bfloat16)
    if kernel == "decode":
        lib.attn_decode(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, MAX_POS, out, h, ragged=True)
        ws = None
    else:
        ws = lib.DecodeWorkspace(DEV, B, [(1, 8)], max_pos=MAX_POS, heads=h)
        lib.attn_decode_mqa(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, MAX_POS, out, h, ws=ws, ragged=True)
    torch.cuda.synchronize()
    if ws is not None:
        assert int(ws.counters.abs().sum()) == 0
    return out


def ragged_decode_reference(cache0, row, qn, table, pos):
    """Float64 output [B, h*64] of one ragged decode step: row b at position n_b = pos[b] attends to its cached keys
    0 .. n_b - 1 (cache0 [B, *, 128]) and its appended row n_b (row [B, 128]); qn [B, h, 64] the bf16 queries."""
    B, h = qn.shape[0], qn.shape[1]
    ref = torch.empty(B, h * 64, dtype=torch.float64, device=qn.device)
    for b in range(B):
        n = int(pos[b])
        keys = torch.cat([cache0[b, :n], row[b:b + 1]], 0).double()
        j = torch.arange(n + 1, device=qn.device)
        sim = 8.0 * qn[b].double() @ keys[:, :64].t() + table[:, n - j].double()
        ref[b] = (sim.softmax(-1) @ keys[:, 64:]).reshape(-1)
    return ref


KCASES = [(k, B, h) for k, Bs in (("decode", (1, 16)), ("decode_mqa", (1, 16, 17, 256))) for B in Bs for h in (1, 8, 16)]


@pytest.mark.parametrize("kernel,B,h", KCASES, ids=[f"{k}-B{B}-h{h}" for k, B, h in KCASES])
def test_ragged_decode_attention_against_float64(kernel, B, h):
    """Each row at its own position n_b (key counts 1 ... 300, across the 128-key slices): the appended row, the rows
    around it untouched, and the output against float64 over that row's keys 0..n_b with the bounds of
    test_attention_reference_gpu.py.  A ragged MQA row is bit-identical to the same row in a call with B = 1."""
    from open_musiclm_b200 import lib
    q_raw, kv_raw, q_scale, k_scale, cache, table, pos = _decode_inputs(B, h, 31 * B + h)
    cache0 = cache.clone()
    out = _run_decode(lib, kernel, q_raw, kv_raw, q_scale, k_scale, cache, table, pos, h)
    row = torch.cat([(F.normalize(kv_raw[:, :64].float(), dim=-1) * k_scale).bfloat16(), kv_raw[:, 64:]], -1)
    qn = (F.normalize(q_raw.float().view(B, h, 64), dim=-1) * q_scale).bfloat16()
    for b in range(B):
        n = int(pos[b])
        assert torch.equal(cache[b, :n], cache0[b, :n]) and torch.isnan(cache[b, n + 1:].float()).all(), b
        got = cache[b, n].float()
        assert ((got - row[b].float()).abs() <= row[b].float().abs() * 2.0 ** -7).all(), b
    ref = ragged_decode_reference(cache0, row, qn, table, pos)
    fails = []
    check(fails, kernel, "out", out, ref, B, 1, h, f"ragged B={B} h={h}")
    assert not fails, "\n".join(fails)
    if kernel == "decode_mqa" and B > 1:
        for b in sorted({0, 1, B // 2, B - 1}):
            c1 = cache0[b:b + 1].clone()
            o1 = _run_decode(lib, kernel, q_raw[b:b + 1], kv_raw[b:b + 1], q_scale, k_scale, c1, table, pos[b:b + 1].clone(), h)
            assert torch.equal(o1[0], out[b]), b
            assert torch.equal(c1[0].view(torch.int16), cache[b].view(torch.int16)), b       # bitwise: the NaN rows too


@pytest.mark.parametrize("B", [1, 17, 256])
def test_ragged_embed_gather_pos_matches_a_host_gather(B):
    """x[b] = table[next_row[b]] + table[row_base + pos[b] + offset] exactly, positions outside [0, pos_rows) adding
    nothing; eagerly and from a captured graph whose position array advances between replays."""
    from open_musiclm_b200 import lib
    D = 64
    g = torch.Generator(device=DEV).manual_seed(B)
    row_base, n_pos, off = 200, 90, -37
    table = torch.randn(row_base + n_pos + 10, D, device=DEV, generator=g)
    next_row = torch.randint(0, row_base, (B,), device=DEV, generator=g, dtype=torch.int32)
    pos = torch.randint(30, 37 + n_pos + 4, (B,), device=DEV, generator=g, dtype=torch.int32)
    x = torch.empty(B, D, device=DEV)

    def expect():
        e = table[next_row.long()].clone()
        for b in range(B):
            j = int(pos[b]) + off
            if 0 <= j < n_pos:
                e[b] += table[row_base + j]
        return e

    x.fill_(float("nan"))
    lib.embed_gather_pos(table, next_row, pos, off, row_base, n_pos, x, ragged=True)
    assert torch.equal(x, expect())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lib.embed_gather_pos(table, next_row, pos, off, row_base, n_pos, x, ragged=True)
    last = torch.full_like(pos, 37 + n_pos)
    pos0 = pos.clone()
    for _ in range(3):
        lib.decode_advance_pos(pos, last)
        x.fill_(float("nan"))
        graph.replay()
        assert torch.equal(x, expect())
    # a row advances by one per call while below its last position, and never moves from at or above it
    assert torch.equal(pos, torch.where(pos0 < last, torch.minimum(pos0 + 3, last), pos0))


# ------------------------------------------------------------------------------------------------ 3. against the oracle
def _compare_rows(name, out, trace, ref, otraces, lengths, q, T):
    """Row by row, the sampled tokens against the restatement of that row alone, up to a near tie (after which that row
    is not compared), with the logits along the shared trajectory within 1e-2; masked post-eos tokens match as -1."""
    exact = total = 0
    for b, n in enumerate(lengths):
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
                assert gap < NEAR_TIE, (name, b, s, int(mine[n * q + s]), int(gold[n * q + s]), gap)
                print(f"{name}: row {b} left the restatement's trajectory at token {s} (near tie, gap {gap:.3e})")
                break
            exact += 1
            lg, og = trace[s][b].cpu(), otraces[b][s][0][0]
            fin = torch.isfinite(og)
            assert rel(lg[fin], og[fin]) < 1e-2, (name, b, s, rel(lg[fin], og[fin]))
    print(f"{name}: {exact} of {total} sampled tokens identical to the restatement's")
    assert exact >= 0.8 * total


ORACLE_CASES = [(stage, B, abs_pos) for stage in ("coarse", "semantic") for B in (2, 20) for abs_pos in (False, True)]


@pytest.mark.parametrize("stage,B,abs_pos", ORACLE_CASES, ids=[f"{s}-B{B}-{'abspos' if a else 'relpos'}" for s, B, a in ORACLE_CASES])
def test_ragged_batch_matches_each_row_alone_in_the_restatement(stage, B, abs_pos):
    """A ragged batch under uniform_noise, with -1 padding, rows with no prefix, a full prefix and prefixes in between,
    against ragged_reference: each row is oracle generate of that row alone on the same weights.  SIMT decode at B = 2,
    tensor-core decode at B = 20; eager with trace and CUDA-graph runs agree."""
    steps, T = (4, 6) if stage == "coarse" else (9, 14)
    lim = 3 * T + 2 if stage == "coarse" else T + 2
    extra = dict(use_absolute_position_embeddings=True, max_absolute_position_embeddings=lim) if abs_pos else {}
    m, w, sd, args = _model(stage, **extra)
    g = torch.Generator().manual_seed(7 * B + abs_pos)
    cond, pred, q = _prompts(B, stage, steps, 64, g)
    lengths = [0, steps] if B == 2 else [(3 * b) % (steps + 1) for b in range(B)]
    for b, n in enumerate(lengths):
        pred[b, n:] = -1
    n_new = max((T - n) * q for n in lengths)
    C = 65
    uni = torch.rand(n_new, B, C, generator=g).clamp_(1e-6, 1 - 1e-6)
    kw = dict(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=lengths, max_time_steps=T, uniform_noise=uni,
              temperature=0.9, allow_eos_in_output=True)
    trace = []
    out = w.generate(trace_logits=trace, **kw)
    assert torch.equal(w.generate(**kw), out), "CUDA-graph replay and eager launches must sample the same tokens"
    assert out.shape == (B, T, q) and len(trace) == n_new
    cfg = oracle_cfg(stage, dict(args, num_coarse_quantizers=3))
    if abs_pos:
        cfg = dataclasses.replace(cfg, abs_pos=True, max_abs_pos=lim)
    ref, otraces = ragged_reference(cfg, sd, [t.cpu().numpy() for t in cond], uni, pred.cpu().numpy(), lengths, T, return_trace=True,
                                    temperature=0.9, allow_eos_in_output=True)
    _compare_rows(f"{stage} B={B}{' abspos' if abs_pos else ''}", out, trace, ref, otraces, lengths, q, T)


# ------------------------------------------------------------------------------------------------ 4. seeded independence
@pytest.mark.parametrize("top_p", [None, 0.8])
@pytest.mark.parametrize("B", [1, 17, 40])
def test_seeded_ragged_rows_equal_each_row_alone(B, top_p):
    """With seeds, every row of a ragged batch (rows that finish many steps before the others, empty and full prefixes)
    is bit-identical to that row alone with its real prefix: tokens and the traced logits of its own steps; the
    batch's eager and graph runs agree."""
    m, w, _, _ = _model(dim=256, heads=4)
    g = torch.Generator().manual_seed(B + (7 if top_p else 0))
    steps, T = 8, 10
    cond, pred, q = _prompts(B, "coarse", steps, 64, g)
    lengths = [steps - 1] if B == 1 else [[0, steps, 1, 9 % (steps + 1)][b] if b < 4 else int(v)
                                          for b, v in enumerate(torch.randint(0, steps + 1, (B,), generator=g))]
    seeds = [int(v) for v in torch.randint(0, 2 ** 62, (B,), generator=g)]
    kw = dict(max_time_steps=T, temperature=0.9, top_p=top_p)
    tr = []
    out = w.generate(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=lengths, seeds=seeds, trace_logits=tr, **kw)
    assert torch.equal(w.generate(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=lengths, seeds=seeds, **kw), out)
    for b, n in enumerate(lengths):
        atr = []
        alone = _alone(w, cond, pred, b, n, seeds=[seeds[b]], trace_logits=atr, **kw)
        width = alone.shape[1]
        assert torch.equal(out[b, :width], alone[0]), (B, b, n)
        assert bool((out[b, width:] == -1).all())
        assert len(atr) == max(0, (T - n) * q)
        for s, lg in enumerate(atr):
            assert torch.equal(tr[s][b], lg[0]), (B, b, n, s)


# ------------------------------------------------------------------------------------------------ 5. limits
def test_absolute_position_limit_is_checked_per_row_offsets(monkeypatch):
    """max_absolute_position_embeddings = T q - 1: every row that samples reaches exactly that many tokens and
    generates; a row whose prefix (garbage ids in its padding, and longer than max_time_steps) samples nothing is
    exempt.  One more step raises IndexError naming the first row that samples, before anything runs (Engine.seed
    unchanged).  No row's decode position passes its last position, which stays inside the table; the token-id error
    word stays clear, and every row equals the row alone."""
    from open_musiclm_b200 import decode as D
    T, q = 5, 3
    lim = T * q - 1
    m, w, _, _ = _model(use_absolute_position_embeddings=True, max_absolute_position_embeddings=lim)
    eng = m.engine
    g = torch.Generator().manual_seed(11)
    B, steps = 4, 7
    cond, pred, _ = _prompts(B, "coarse", steps, 64, g)
    lengths = [steps, 0, 4, 2]                               # row 0: 21 prefix tokens > lim, samples nothing
    pred[2, 4:] = 10 ** 6
    pred[3, 2:] = -1
    sessions = []
    orig = D.DecodeSession.__init__

    def record(self, *a, **k):
        orig(self, *a, **k)
        sessions.append(self)
    monkeypatch.setattr(D.DecodeSession, "__init__", record)
    seeds = [1, 2, 3, 4]
    out = w.generate(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=lengths, max_time_steps=T, seeds=seeds)
    torch.cuda.synchronize()
    assert int(eng.err_flag.item()) == 0
    assert out.shape == (B, steps, q) and torch.equal(out[0], pred[0])
    s = sessions[-1]
    pos, pos_last, pos_offset = s.pos.cpu(), s.pos_last.cpu(), s.pos_offset.cpu()
    assert bool((pos <= pos_last).all()) and int((pos_last + pos_offset).max()) < lim
    for b in range(1, B):
        alone = _alone(w, cond, pred, b, lengths[b], max_time_steps=T, seeds=[seeds[b]])
        assert torch.equal(out[b, :T], alone[0]) and bool((out[b, T:] == -1).all()), b
    seed = eng.seed.clone()
    n = len(sessions)
    with pytest.raises(IndexError, match=r"row 1 reaches 17 tokens"):
        w.generate(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=lengths, max_time_steps=T + 1)
    assert torch.equal(eng.seed, seed) and len(sessions) == n
    with pytest.raises(ValueError, match="pred_lengths"):
        w.generate(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=[1, 2, 3], max_time_steps=T)
    assert torch.equal(eng.seed, seed) and len(sessions) == n


# ------------------------------------------------------------------------------------------------ 6. shipped widths
@pytest.mark.parametrize("heads", [8, 16])
def test_ragged_coarse_at_model_width_equals_single_rows(heads):
    """Coarse stage at d = 1024, depth 2, h = 8 and h = 16: one seeded ragged call of 5 rows against each row alone."""
    m, w, _, _ = _model(dim=1024, depth=2, heads=heads, cb=1024)
    g = torch.Generator().manual_seed(heads)
    B, steps, T = 5, 6, 8
    cond, pred, q = _prompts(B, "coarse", steps, 1024, g, n_cond=(12, 40))
    lengths = [0, 6, 3, 1, 5]
    seeds = [int(v) for v in torch.randint(0, 2 ** 62, (B,), generator=g)]
    out = w.generate(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=lengths, max_time_steps=T, seeds=seeds)
    for b, n in enumerate(lengths):
        alone = _alone(w, cond, pred, b, n, max_time_steps=T, seeds=[seeds[b]])
        assert torch.equal(out[b], alone[0]), (heads, b, n)
