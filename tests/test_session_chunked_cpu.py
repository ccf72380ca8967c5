"""Chunked prefill in generation sessions, host side: GenerationSession's prefill_rows argument (ValueError before any
device work), the chunk schedule of SlotSchedule under random arrivals and budgets against the statements it must
hold, and PackedPrefill's arrays for chunks against direct statements."""
import random

import numpy as np
import pytest
import torch

import open_musiclm_b200 as O
from open_musiclm_b200.session import PackedPrefill, SlotSchedule, _Row, lpt_work


def _session(heads=2, **kw):
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=64, depth=1, heads=heads, clap_codebook_size=16, num_clap_quantizers=2, semantic_codebook_size=16,
                                    acoustic_codebook_size=16, num_coarse_quantizers=3)
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    return O.GenerationSession(w, slots=4, max_positions=60, **kw)


@pytest.mark.parametrize("heads,unit", [(1, 128), (2, 64), (6, 64), (8, 16), (16, 8)])
def test_prefill_rows_is_checked(heads, unit):
    for bad in (True, False, 16.0, "64", unit - 1, 0, -unit):
        with pytest.raises(ValueError, match="prefill_rows"):
            _session(heads=heads, prefill_rows=bad)
    for good in (None, unit, unit + 1, 10 ** 6, np.int64(unit)):
        sess = _session(heads=heads, prefill_rows=good)
        assert sess.dec is None and sess.sched.unit == unit and sess.prefill_rows == (None if good is None else int(good))


def _run(slots, q, budget, unit, arrivals, steps):
    """Drives a SlotSchedule with the given arrivals {step: [(P, n)]}; returns the per-request log of chunks
    (boundary, p0, length, slot), first sample boundary and the per-boundary row counts."""
    sched = SlotSchedule(slots, q, max_queue=10 ** 6, prefill_rows=budget, unit=unit)
    rows, log, first, per_boundary, submitted = {}, {}, {}, [], []
    h = 0
    for k in range(steps):
        for P, n in arrivals.get(k, []):
            r = _Row(h, P, n, pred_start=P - 3)
            rows[h] = r
            log[h] = []
            submitted.append(h)
            sched.submit(r)
            h += 1
        out = sched.admit()
        per_boundary.append(sum(r.chunk[1] for r in out))
        for r in out:
            log[r.handle].append((k, r.chunk[0], r.chunk[1], r.slot))
        for s, r in sched.rows.items():                       # every row in a slot holds it; a slot holds one row
            assert r.slot == s
        before = {r.handle: r.t for r in sched.rows.values()}
        active = dict(sched.rows)
        sched.advance()
        for r in active.values():
            if r.t > before[r.handle] and r.handle not in first:
                first[r.handle] = k
        assert all(not r.prefilled for r in sched.prefilling)
    return rows, log, first, per_boundary, submitted


@pytest.mark.parametrize("q,slots,unit", [(1, 1, 16), (3, 4, 16), (4, 17, 8), (3, 40, 64)])
@pytest.mark.parametrize("budget", [None, 1, 3, 10, 64])
def test_chunk_schedule_holds_its_statements(q, slots, unit, budget):
    budget = None if budget is None else budget * unit
    rnd = random.Random(q * 1000 + slots + (budget or 0))
    steps = 120
    arrivals = {k: [(rnd.choice((1, 2, unit - 1, unit, unit + 1, rnd.randint(3, 20 * unit))), q * rnd.randint(1, 6))
                    for _ in range(rnd.choice((0, 0, 1, 2, 5)))] for k in range(steps // 2)}
    rows, log, first, per_boundary, submitted = _run(slots, q, budget, unit, arrivals, steps)
    if budget is not None:
        assert max(per_boundary) <= budget                                        # rows per boundary <= prefill_rows
    started = []
    for h in submitted:
        r, chunks = rows[h], log[h]
        if not chunks:
            continue
        started.append((chunks[0][0], h))
        pos = 0
        for i, (k, p0, n, slot) in enumerate(chunks):
            assert p0 == pos and n >= 1                                           # every prompt row once, in order
            pos += n
            if i < len(chunks) - 1:
                assert n % unit == 0 and p0 % unit == 0                           # non-final chunks are whole units
                assert chunks[i + 1][0] == k + 1                                  # consecutive boundaries
            assert slot == chunks[0][3]                                           # the slot is held during prefill
        if budget is None:
            assert len(chunks) == 1
        if pos == r.P:
            assert first.get(h, chunks[-1][0]) == chunks[-1][0]                   # first sample at the last chunk's boundary
    # FIFO: requests start in submission order, and a request never gets a chunk at a boundary where an earlier one
    # still prefilling got none
    assert [h for _, h in sorted(started)] == sorted(h for _, h in started)
    for h in submitted:
        for k, *_ in log[h]:
            for e in submitted[:submitted.index(h)]:
                ke = [c[0] for c in log[e]]
                if ke and ke[0] <= k and sum(c[2] for c in log[e] if c[0] < k) < rows[e].P:
                    assert k in ke, (h, e, k)
    done = [h for h in submitted if log[h] and sum(c[2] for c in log[h]) == rows[h].P]
    assert len(done) > 0


def test_budget_is_shared_in_fifo_order():
    sched = SlotSchedule(4, 1, max_queue=10, prefill_rows=40, unit=16)
    rows = [_Row(h, P, 2, 0) for h, P in enumerate((70, 5, 20))]
    for r in rows:
        sched.submit(r)
    # row 0 takes the largest whole number of units, row 1 its whole prompt in the 8 rows left, row 2 needs 16
    assert [(r.handle, r.chunk) for r in sched.admit()] == [(0, (0, 32)), (1, (0, 5))]
    assert rows[2].slot is None and [r.slot for r in rows[:2]] == [0, 1]
    sched.advance()
    assert rows[0].t == 0 and rows[1].t == 1 and sched.prefilling == [rows[0]]     # prefilling rows sample nothing
    assert [(r.handle, r.chunk) for r in sched.admit()] == [(0, (32, 38))]          # 2 rows left: less than row 2's unit
    assert sched.prefilling == [] and rows[2].slot is None
    assert [r.handle for r in sched.advance()] == [1]
    assert rows[0].t == 1
    assert [(r.handle, r.chunk) for r in sched.admit()] == [(2, (0, 20))] and rows[2].slot == 1


# --------------------------------------------------------------------------------------------------- plan arrays
def test_chunk_plan_arrays():
    n_tok = [[3, 20, 5], [2, 4, 0], [1, 40, 2]]          # prompts of 31, 9 and 46 rows; prefixes of 5, 0 and 2 tokens
    full = [31, 9, 46]
    chunks = [(16, 15), (0, 9), (32, 8)]                 # final from 16; whole; middle chunk of the third
    slots, n_max, q, h = [5, 0, 2], 64, 2, 8
    base = [100, 300, 500]
    p = PackedPrefill(n_tok, slots, n_max, q, h, base, True, chunks)
    assert p.final.tolist() == [True, True, False] and p.k_final == 2
    assert p.start.tolist() == [0, 15, 24] and p.M == 32 and p.max_len == 15 and p.max_end == 40
    assert p.row_pos.tolist() == list(range(16, 31)) + list(range(9)) + list(range(32, 40))
    assert p.kv_dst.tolist() == [5 * 64 + i for i in range(16, 31)] + list(range(9)) + [2 * 64 + i for i in range(32, 40)]
    assert p.kv_start.tolist() == [320, 0, 128]
    whole = [np.concatenate([np.concatenate([[-1], base[s] + np.arange(n)]) for s, n in enumerate(t)]) for t in n_tok]
    assert p.src_row2.tolist() == whole[0][16:31].tolist() + whole[1].tolist() + whole[2][32:40].tolist()
    assert p.last_row.tolist() == [14, 23] and p.fin_slots.tolist() == [5, 0]
    # prefix token j of request 0 is scored at position 25 + j (packed row 9 + j); request 2's at 43 + j: not here
    assert p.prefix_span == [(0, 5), (0, 0), (0, 0)]
    assert p.prefix_rows[0].tolist() == [9, 11, 13] and p.prefix_rows[1].tolist() == [10, 12]
    assert p.label_idx.tolist() == [-1, -1, 0, 2, 4, 1, 3]
    assert p.groups == [(0, 0, 5), (1, 5, 2)]
    assert p.hist_idx.tolist() == [5] + [-1] * 23 + [2] + [-1] * 7
    assert p.hist_src.tolist() == [30, 31] and p.hist_dst.tolist() == [4, 5]
    assert p.conv_dst.tolist() == [10, 11, 0, 1] and p.conv_src.tolist() == [13, 14, 22, 23]
    assert len(p.conv_hdst) == 0 and len(p.conv_zero) == 0
    assert p.work.tolist() == lpt_work([15, 9, 8], h, [16, 0, 32]).tolist()
    # the last chunk of request 2 covers its prefix: span (0, 2), rows at positions 43, 44
    p2 = PackedPrefill([n_tok[2]], [2], n_max, q, h, None, True, [(40, 6)])
    assert p2.prefix_span == [(0, 2)] and p2.prefix_rows[0].tolist() == [3] and p2.prefix_rows[1].tolist() == [4]
    assert p2.last_row.tolist() == [5] and p2.label_idx.tolist() == [-1, 0, 1]
    # a chunk that splits a prefix scores the part inside it
    p3 = PackedPrefill([[1, 12, 6]], [0], n_max, 3, h, None, True, [(8, 8)])         # prefix tokens at positions 15 ... 20
    assert p3.prefix_span == [(0, 1)] and p3.prefix_rows[0].tolist() == [7] and p3.label_idx.tolist() == [0]
    p3 = PackedPrefill([[1, 12, 6]], [0], n_max, 3, h, None, True, [(16, 6)])
    assert p3.prefix_span == [(1, 6)] and [r.tolist() for r in p3.prefix_rows] == [[2], [0, 3], [1, 4]]
    assert p3.label_idx.tolist() == [-1, 3, 1, 4, 2, 5] and p3.last_row.tolist() == [5]
    assert full == [sum(n + 1 for n in t) for t in n_tok]


def test_final_chunk_of_one_row_takes_its_history_row():
    p = PackedPrefill([[3, 20, 5]], [3], 64, 1, 16, None, False, [(30, 1)])
    assert p.final.tolist() == [True] and p.row_pos.tolist() == [30] and p.last_row.tolist() == [0]
    assert p.hist_idx.tolist() == [3]                                            # its conv input from the history buffer
    assert p.conv_dst.tolist() == [6, 7] and p.conv_src.tolist()[1] == 0         # P - 1 from the chunk's row
    assert p.conv_hdst.tolist() == [6] and p.conv_hsrc.tolist() == [7]           # P - 2 = p0 - 1: history row 2 slot + 1
    assert len(p.hist_dst) == 0


def test_chunked_work_list_counts_key_tiles_from_position_zero():
    h = 8
    lens, p0 = [16, 160, 1, 300], [0, 128, 256, 512]
    w = lpt_work(lens, h, p0)
    got = [tuple(x) for x in w.tolist()]
    want = {(b, rb) for b, n in enumerate(lens) for rb in range(-(-n * h // 128))}
    assert len(got) == len(want) and set(got) == want
    cost = [min(p0[b] + lens[b] - 1, (p0[b] * h + rb * 128 + 127) // h) // 128 + 1 for b, rb in got]
    assert cost == sorted(cost, reverse=True)
    assert cost[0] == (512 + 299) // 128 + 1
    assert lpt_work(lens, h).tolist() == lpt_work(lens, h, [0] * 4).tolist()
