"""Generation sessions (continuous batching) on the H100: the per-row-index sampler against the float64 reference and
the seeded Philox replica, and bit for bit against omlm_sample_rows at each row's index; the per-row-offset position
gather against a host gather; every finished row of a random join schedule bit-identical to generate with that row
alone and its seed (tokens and traced logits), for slots 1, 17, 40 and 256, coarse and semantic, relative and absolute
positions, d = 1024 at 8 and 16 heads, and the three stages; slot reuse; a graph count that joins do not grow."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from test_generate_per_row_gpu import SENTINEL, _kernel_case, _launch, _rows  # noqa: E402
from test_generate_ragged_gpu import _model  # noqa: E402
from test_generate_seeded_cpu import seeded_uniforms  # noqa: E402
from test_sampling_nucleus_gpu import check_nucleus  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as L
    L.device_check()
    return L


# ------------------------------------------------------------------------------------------------ 1. the kernels
@pytest.mark.parametrize("nucleus", [False, True])
@pytest.mark.parametrize("C", [65, 1025, 16384])
def test_indexed_sampler_against_the_references(lib, C, nucleus):
    """30 rows at sample indices 0 ... 5, with rows at their last sample, past it, at a negative index and past the
    tokens' width: a row that samples writes tokens[b, t] and next_row[b] bit-identical to omlm_sample_rows with the
    shared counter at t (equal to the float64 reference under the seeded replica) and advances t; the others write
    nothing and keep t."""
    from open_musiclm_b200.decode import seeds_tensor
    x, ks, temps, tops, _, seeds, _ = _kernel_case(C, "per_sequence")
    B = x.shape[0]
    xd, seeds_t = x.to(DEV), seeds_tensor(seeds, B, DEV)
    row_tops = tops if nucleus else [None] * B
    rows = _rows(ks, temps, row_tops, nucleus)
    width = 6
    t0 = [b % width for b in range(B)]
    n = [t + 1 + b % 3 for b, t in enumerate(t0)]
    t0[3], n[3] = 4, 4                                    # has all its samples
    t0[4], n[4] = 5, 2                                    # past them
    t0[5] = -1                                            # a free slot's index
    t0[7], n[7] = width, width + 2                        # past the tokens' width
    for allow in (False, True):
        tokens = torch.full((B, width), SENTINEL, device=DEV, dtype=torch.int64)
        next_row = torch.full((B,), SENTINEL, device=DEV, dtype=torch.int32)
        t = torch.tensor(t0, device=DEV, dtype=torch.int32)
        lib.sample_rows_indexed(xd, C, allow, seeds_t, tokens, next_row, 5, t, torch.tensor(n, device=DEV, dtype=torch.int32),
                                rows["top_k_rows"], rows["temperature_rows"], rows["top_p_rows"])
        torch.cuda.synchronize()
        tokens, next_row, t = tokens.cpu(), next_row.cpu(), t.cpu()
        for b in range(B):
            samples = 0 <= t0[b] < min(n[b], width)
            assert int(t[b]) == t0[b] + samples, b
            if not samples:
                assert bool((tokens[b] == SENTINEL).all()) and int(next_row[b]) == SENTINEL, b
                continue
            others = [c for c in range(width) if c != t0[b]]
            assert bool((tokens[b, others] == SENTINEL).all()) and int(next_row[b]) == int(tokens[b, t0[b]]) + 5, b
            shared = _launch(lib, xd, C, "per_sequence", None, seeds_t, None, allow, rows=rows, step=t0[b]).cpu()
            assert int(tokens[b, t0[b]]) == int(shared[b]), (b, t0[b])
            u = torch.from_numpy(seeded_uniforms(seeds[b], t0[b], C))[None]
            top = None if row_tops[b] in (None, 1.0) else row_tops[b]
            check_nucleus(tokens[b:b + 1, t0[b]], x[b:b + 1], u, ks[b], float(np.float32(temps[b])), allow, top, (C, b))


def test_indexed_sampler_with_equal_indices_is_sample_rows(lib):
    """Every t_b equal: the whole launch is omlm_sample_rows with the shared counter at that index, bit for bit."""
    from open_musiclm_b200.decode import seeds_tensor
    C, B = 1025, 40
    x, ks, temps, tops, _, seeds, _ = _kernel_case(C, "per_sequence", B)
    xd, seeds_t, rows = x.to(DEV), seeds_tensor(seeds, B, DEV), _rows(ks, temps, tops)
    for step in (0, 3):
        tokens = torch.full((B, 8), SENTINEL, device=DEV, dtype=torch.int64)
        nr = torch.zeros(B, device=DEV, dtype=torch.int32)
        t = torch.full((B,), step, device=DEV, dtype=torch.int32)
        lib.sample_rows_indexed(xd, C, False, seeds_t, tokens, nr, 5, t, torch.full((B,), 8, device=DEV, dtype=torch.int32),
                                rows["top_k_rows"], rows["temperature_rows"], rows["top_p_rows"])
        shared = _launch(lib, xd, C, "per_sequence", None, seeds_t, None, False, rows=rows, step=step)
        assert torch.equal(tokens[:, step], shared) and bool((t == step + 1).all())


def test_per_row_offset_gather_against_a_host_gather(lib):
    g = torch.Generator().manual_seed(3)
    M, D, rows_tab, base, lim = 37, 64, 300, 200, 90
    table = torch.randn(rows_tab, D, generator=g).to(DEV)
    src = torch.randint(-1, 150, (M,), generator=g, dtype=torch.int32)
    pos = torch.randint(0, 120, (M,), generator=g, dtype=torch.int32)
    off = torch.randint(-60, 5, (M,), generator=g, dtype=torch.int32)
    x = torch.full((M, D), float("nan"), device=DEV)
    lib.embed_gather_pos_rows(table, src.to(DEV), pos.to(DEV), off.to(DEV), base, lim, x)
    tab = table.cpu()
    for m in range(M):
        want = tab[src[m]].clone() if src[m] >= 0 else torch.zeros(D)
        p = int(pos[m] + off[m])
        if 0 <= p < lim:
            want += tab[base + p]
        assert torch.equal(x[m].cpu(), want), m


# ------------------------------------------------------------------------------------------------ 2. the guarantee
def _request(g, stage_q, cb, cond_shapes, max_steps):
    """A random request: conditioning lengths, prefix length (0 ... 3 steps), seed and sampling arguments."""
    cond = [torch.randint(0, cb, (1, int(torch.randint(lo, hi + 1, (1,), generator=g))), generator=g) for lo, hi in cond_shapes]
    n_pre = int(torch.randint(0, 4, (1,), generator=g))
    pred = None
    if n_pre:
        pred = torch.randint(0, cb, (1, n_pre, stage_q), generator=g)
    T = int(torch.randint(max(n_pre, 1), max_steps + 1, (1,), generator=g))
    args = dict(seed=int(torch.randint(0, 2 ** 62, (1,), generator=g)), max_time_steps=T,
                temperature=round(0.3 + 1.7 * float(torch.rand(1, generator=g)), 4),
                filter_thres=(0.0, 0.5, 0.9, 0.8)[int(torch.randint(0, 4, (1,), generator=g))],
                top_p=(None, 0.9, 0.5, None)[int(torch.randint(0, 4, (1,), generator=g))])
    return dict(conditioning_token_ids=[c.cuda() for c in cond], pred_token_ids=pred.cuda() if pred is not None else None, **args)


def _alone(w, req, trace=None):
    r = dict(req)
    seed = r.pop("seed")
    return w.generate(seeds=[seed], trace_logits=trace, **r)


def _run_schedule(sess, reqs, g, traces=None, max_wait=3):
    """Adds the requests over time: a few at a time between steps, as room allows, until all have finished.
    traces (a dict, trace_logits sessions): receives each request's traced logits."""
    pending, handles, out = list(range(len(reqs))), {}, {}
    while pending or not sess.idle:
        for _ in range(int(torch.randint(0, max_wait + 1, (1,), generator=g)) if not sess.idle else 1):
            if not pending:
                break
            try:
                h = sess.add(**reqs[pending[0]])
            except ValueError:
                break                                      # no room: wait for a slot
            handles[h] = pending.pop(0)
        sess.step(int(torch.randint(1, 3, (1,), generator=g)))
        done = sess.finished()
        out.update(done)
        if traces is not None:
            traces.update({handles[h]: sess.traced_logits(h) for h in done})
    assert len(out) == len(reqs)
    return {handles[h]: v for h, v in out.items()}


GUARANTEE_CASES = [("coarse", 1, 128, 2, False, 3), ("coarse", 17, 128, 2, False, 40), ("semantic", 40, 128, 2, False, 70),
                   ("coarse", 256, 128, 2, False, 300), ("coarse", 17, 128, 2, True, 30), ("semantic", 17, 128, 4, True, 30),
                   ("coarse", 5, 1024, 8, False, 8), ("coarse", 5, 1024, 16, False, 8), ("semantic", 5, 1024, 8, False, 8),
                   ("semantic", 5, 1024, 16, False, 8)]


@pytest.mark.parametrize("stage,slots,dim,heads,abs_pos,n_req", GUARANTEE_CASES,
                         ids=[f"{s}-slots{n}-d{d}-h{h}-{'abspos' if a else 'relpos'}" for s, n, d, h, a, _ in GUARANTEE_CASES])
def test_every_row_equals_generate_alone(stage, slots, dim, heads, abs_pos, n_req):
    """A random schedule (rows joining at different boundaries, conditioning and prefix lengths that differ, per-row
    temperature, top-k, top-p and max_time_steps, slots reused after rows retire): every finished row is torch.equal
    to generate with that row alone and its seed; with trace_logits every logits row it sampled from is too."""
    import open_musiclm_b200 as O
    q = 3 if stage == "coarse" else 1
    max_steps = 6 if stage == "coarse" else 12
    extra = dict(use_absolute_position_embeddings=True, max_absolute_position_embeddings=max_steps * q + 1) if abs_pos else {}
    cb = 64 if dim == 128 else 1024
    m, w, _, _ = _model(stage, dim=dim, heads=heads, cb=cb, **extra)
    g = torch.Generator().manual_seed(slots * 7 + heads + abs_pos)
    shapes = [(2, 9)] + ([(3, 14)] if stage == "coarse" else [])
    reqs = [_request(g, q, cb, shapes, max_steps) for _ in range(n_req)]
    trace = dim == 1024 or (slots == 17 and not abs_pos)
    sess = O.GenerationSession(w, slots=slots, max_positions=64, max_queue=4, trace_logits=trace)
    traces = {} if trace else None
    got = _run_schedule(sess, reqs, g, traces)
    for i, r in enumerate(reqs):
        tr = [] if trace else None
        alone = _alone(w, r, tr)
        assert torch.equal(got[i], alone[0]), (i, r["max_time_steps"])
        if trace:
            assert traces[i].shape[0] == len(tr), i
            assert all(torch.equal(traces[i][s], tr[s][0]) for s in range(len(tr))), i


def test_slot_reuse_leaks_nothing():
    """A slot's second occupant is bit-identical whether the first was long, short or absent, and equals generate."""
    import open_musiclm_b200 as O
    m, w, _, _ = _model("coarse")
    g = torch.Generator().manual_seed(9)
    shapes = [(2, 9), (3, 14)]
    second = _request(g, 3, 64, shapes, 6)
    long_, short = _request(g, 3, 64, shapes, 6), _request(g, 3, 64, shapes, 6)
    long_.update(max_time_steps=6, pred_token_ids=None)
    short.update(max_time_steps=1, pred_token_ids=None)
    outs = []
    for first in (long_, short, None):
        sess = O.GenerationSession(w, slots=1, max_positions=64, max_queue=1)
        if first is not None:
            sess.add(**first)
        h = sess.add(**second)
        while not sess.idle:
            sess.step()
        outs.append(sess.finished()[h])
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    assert torch.equal(outs[0], _alone(w, second)[0])


@pytest.mark.parametrize("stage", ["coarse", "semantic"])
def test_graph_count_does_not_grow_with_joins(stage):
    """Graphs are captured once per (quantizer slot, kind, nucleus or not), at first need: 60 joins capture at most
    2 (q + 2), and none is captured twice."""
    import open_musiclm_b200 as O
    q = 3 if stage == "coarse" else 1
    m, w, _, _ = _model(stage)
    g = torch.Generator().manual_seed(4)
    shapes = [(2, 9)] + ([(3, 14)] if stage == "coarse" else [])
    sess = O.GenerationSession(w, slots=4, max_positions=64, max_queue=64)
    reqs = [_request(g, q, 64, shapes, 4) for _ in range(60)]
    counts = []
    for i, r in enumerate(reqs):
        sess.add(**r)
        sess.step()
        counts.append(sess.graph_count)
    while not sess.idle:
        sess.step()
    assert max(counts) <= sess.graph_count <= 2 * (q + 2) < len(reqs), counts
    assert counts == sorted(counts)                     # a key is captured once and kept


def test_three_stages_match_generate():
    """Semantic, coarse and fine wrappers, each through a session, against generate row by row."""
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
        shapes = [(4, 4)] + ([(6, 6)] if name == "coarse" else [(9, 9)] if name == "fine" else [])
        reqs = [_request(g, q, 64, shapes, 5) for _ in range(6)]
        if name == "fine":       # the coarse conditioning holds whole time steps of 3 quantizers
            for r in reqs:
                r["conditioning_token_ids"][1] = r["conditioning_token_ids"][1][:, :9]
        sess = O.GenerationSession(w, slots=3, max_positions=128, max_queue=8)
        got = _run_schedule(sess, reqs, g)
        for i, r in enumerate(reqs):
            assert torch.equal(got[i], _alone(w, r)[0]), (name, i)
