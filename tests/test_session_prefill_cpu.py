"""The host plan of a session's packed prefill, without device work: PackedPrefill's rows, positions, absolute-position
rows, output rows, head groups and install indices, the attention work list and the split of a boundary's joiners
over the packed workspace, each against a direct statement of what it must hold."""
import itertools

import numpy as np
import pytest

from open_musiclm_b200.session import PackedPrefill, lpt_work, split_joiners

# per joiner: token counts of its sequences (conditioning with eos, then the prefix), for q = 3 and q = 1 stages
CASES = [
    ([[5, 12, 0]], 3),
    ([[5, 12, 3], [2, 3, 9], [7, 1, 0], [1, 30, 6]], 3),
    ([[4, 1], [9, 2], [3, 0], [130, 3], [1, 1]], 1),
]


def _expected_rows(n_tok):
    """Per joiner: its first packed row, its prompt length and the packed row of each sequence's start token."""
    out, row = [], 0
    for t in n_tok:
        P = sum(n + 1 for n in t)
        starts = [row + sum(n + 1 for n in t[:s]) for s in range(len(t))]
        out.append((row, P, starts))
        row += P
    return out


@pytest.mark.parametrize("abs_pos", [False, True])
@pytest.mark.parametrize("logprob", [False, True])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_packing_plan(case, logprob, abs_pos):
    n_tok, q = CASES[case]
    k, n_max, h = len(n_tok), 200, 8
    slots = [7, 2, 5, 0, 3][:k]
    base = [100, 300, 500]
    p = PackedPrefill(n_tok, slots, n_max, q, h, base if abs_pos else None, logprob)
    rows = _expected_rows(n_tok)
    assert p.M == sum(P for _, P, _ in rows) and p.max_len == max(P for _, P, _ in rows)
    assert p.start.tolist() == [r for r, _, _ in rows] and p.P.tolist() == [P for _, P, _ in rows]
    for (r0, P, _), slot in zip(rows, slots):
        assert p.row_pos[r0:r0 + P].tolist() == list(range(P))                      # 0 at each start
        assert p.kv_dst[r0:r0 + P].tolist() == [slot * n_max + i for i in range(P)]
    if abs_pos:
        want = []
        for t in n_tok:
            for s, n in enumerate(t):
                want += [-1] + [base[s] + i for i in range(n)]                       # start token: no position row
        assert p.src_row2.tolist() == want
    else:
        assert p.src_row2 is None
    assert p.last_row.tolist() == [r0 + P - 1 for r0, P, _ in rows]
    # prefix rows of head qi: the row at the predicted sequence's start + j scores prefix token j (j % q == qi)
    for qi in range(q):
        want = [st[-1] + j for (_, _, st), t in zip(rows, n_tok) for j in range(t[-1]) if j % q == qi] if logprob else []
        assert p.prefix_rows[qi].tolist() == want
    out = [*p.last_row.tolist(), *itertools.chain.from_iterable(r.tolist() for r in p.prefix_rows)]
    assert p.head_rows == len(out) and len(set(out)) == len(out)
    assert [int(x) for x in np.flatnonzero(p.dest_row >= 0)] == sorted(out)
    assert all(p.dest_row[r] == i for i, r in enumerate(out))
    groups, b = [], 0
    for qi in range(q):
        cnt = len(p.prefix_rows[qi]) + (k if qi == 0 else 0)
        if cnt:
            groups.append((qi, b, cnt))
        b += cnt
    assert p.groups == groups
    tokens = [(i, j) for i, t in enumerate(n_tok) for j in range(t[-1] if logprob else 0)]
    off = np.cumsum([0] + [t[-1] if logprob else 0 for t in n_tok])[:-1]
    assert p.prefix_off.tolist() == off.tolist()
    want_idx = [-1] * k + [off[i] + j for qi in range(q) for i, j in tokens if j % q == qi]
    assert p.label_idx.tolist() == want_idx
    assert sorted(p.label_idx[k:].tolist()) == list(range(len(tokens)))              # every prefix token once
    for i, ((r0, P, _), slot) in enumerate(zip(rows, slots)):
        for j in range(2):
            assert p.conv_dst[2 * i + j] == slot * 2 + j
            assert p.conv_src[2 * i + j] == r0 + max(P - 2 + j, 0)
    assert p.conv_zero.tolist() == [2 * s + j for (_, P, _), s in zip(rows, slots) for j in range(2) if P - 2 + j < 0]


def test_conv_rows_before_a_short_prompt_are_zeroed():
    p = PackedPrefill([[0]], [4], 10, 1, 1)
    assert p.P.tolist() == [1] and p.conv_zero.tolist() == [8] and p.conv_src.tolist() == [0, 0]


@pytest.mark.parametrize("h", [1, 3, 8, 12, 16])
def test_attention_work_list(h):
    lens = [1, 2, 128 // h - 1 or 1, 128 // h + 1, 127, 128, 129, 700, 2048, 5]
    w = lpt_work(lens, h)
    assert w.dtype == np.int32 and w.shape[1] == 2
    want = {(b, rb) for b, n in enumerate(lens) for rb in range(-(-n * h // 128))}
    got = [tuple(x) for x in w.tolist()]
    assert len(got) == len(want) and set(got) == want                                # every unit exactly once
    cost = [min(lens[b] - 1, (rb * 128 + 127) // h) // 128 + 1 for b, rb in got]   # key tiles of the unit
    assert cost == sorted(cost, reverse=True)                                        # heaviest first


@pytest.mark.parametrize("lens,cap,want", [
    ([5, 5, 3, 8, 1], 10, [[0, 1], [2], [3, 4]]),
    ([10, 10], 10, [[0], [1]]),
    ([1] * 7, 3, [[0, 1, 2], [3, 4, 5], [6]]),
    ([4], 16384, [[0]]),
])
def test_split_in_admission_order(lens, cap, want):
    groups = split_joiners(lens, cap)
    assert groups == want
    assert [i for g in groups for i in g] == list(range(len(lens)))
    assert all(sum(lens[i] for i in g) <= cap for g in groups)
    # a group is closed only because the next joiner does not fit
    assert all(sum(lens[i] for i in a) + lens[b[0]] > cap for a, b in zip(groups, groups[1:]))
