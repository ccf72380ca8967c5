"""Generation sessions, host side: GenerationSession.add's argument checks (ValueError before any device work, on a
model that has never been on a GPU) and the slot schedule (allocation, reuse, queueing to the next boundary, and the
per-row sample index, position, last position and offset the device arrays hold) against a plain model of the
schedule that moves every row one sample at a time."""
import random

import pytest
import torch

import open_musiclm_b200 as O
from open_musiclm_b200.session import SlotSchedule, _Row


def _session(stage="coarse", slots=4, max_positions=60, heads=2, **kw):
    torch.manual_seed(0)
    args = dict(dim=64, depth=1, heads=heads, clap_codebook_size=16, num_clap_quantizers=2)
    if stage == "coarse":
        m = O.create_coarse_transformer(semantic_codebook_size=16, acoustic_codebook_size=16, num_coarse_quantizers=3, **args, **kw)
    else:
        m = O.create_semantic_transformer(semantic_codebook_size=16, **args, **kw)
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    return O.GenerationSession(w, slots=slots, max_positions=max_positions)


def _cond():
    return [torch.zeros(1, 2, dtype=torch.int64), torch.zeros(1, 5, dtype=torch.int64)]


def test_session_arguments_are_checked():
    for bad in (0, 257, True, 2.0):
        with pytest.raises(ValueError, match="slots"):
            _session(slots=bad)
    with pytest.raises(ValueError, match="at most 16 heads"):
        _session(heads=17)


@pytest.mark.parametrize("kw,match", [
    (dict(seed=None), "seed"), (dict(seed=1.5), "seed"), (dict(seed=True), "seed"), (dict(seed=[1, 2]), "seed"),
    (dict(seed=torch.tensor([1, 2])), "seed"), (dict(seed=torch.tensor([1.0])), "seed"),
    (dict(pred_token_ids=torch.zeros(1, 5, dtype=torch.int64)), "whole time steps"),
    (dict(pred_token_ids=torch.zeros(1, 2, 2, dtype=torch.int64)), "whole time steps"),
    (dict(pred_token_ids=torch.zeros(2, 2, 3, dtype=torch.int64)), "whole time steps"),
    (dict(temperature=0.0), "temperature"), (dict(temperature=float("nan")), "temperature"), (dict(temperature="1"), "temperature"),
    (dict(filter_thres=-1.0), "filter_thres"), (dict(filter_thres=float("inf")), "filter_thres"),
    (dict(top_p=0.0), "top_p"), (dict(top_p=1.5), "top_p"), (dict(top_p=True), "top_p"),
    (dict(max_time_steps=-1), "max_time_steps"), (dict(max_time_steps=2.5), "max_time_steps"),
    (dict(temperature=[1.0, 1.0]), "temperature"),
    (dict(max_time_steps=100), "max_positions"),
    (dict(conditioning_token_ids=[torch.zeros(1, 2, dtype=torch.int64)]), "conditioning_token_ids"),
    (dict(conditioning_token_ids=[torch.zeros(2, 2, dtype=torch.int64), torch.zeros(2, 5, dtype=torch.int64)]), "one row"),
])
def test_add_rejects_bad_arguments_before_device_work(kw, match):
    sess = _session()
    args = dict(conditioning_token_ids=_cond(), seed=1, max_time_steps=4)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        sess.add(**args)
    assert sess.dec is None and sess.idle          # nothing reached a device


def test_capacity_queue_and_absolute_position_limit():
    """The prompt (2+1+1 + 5+1+1 + 1 = 12 positions) plus 3 q per step must fit max_positions; a full session with a
    full queue rejects; the absolute-position limit raises IndexError as generate does."""
    sess = _session(slots=2, max_positions=12 + 12)
    sess.add(conditioning_token_ids=_cond(), seed=1, max_time_steps=4)
    with pytest.raises(ValueError, match="max_positions"):
        sess.add(conditioning_token_ids=_cond(), seed=1, max_time_steps=5)
    sess.add(conditioning_token_ids=_cond(), seed=2, max_time_steps=4)
    with pytest.raises(ValueError, match="slots are taken"):
        sess.add(conditioning_token_ids=_cond(), seed=3, max_time_steps=4)
    h = sess.add(conditioning_token_ids=_cond(), seed=3, max_time_steps=0)      # samples nothing: done at once, no slot
    assert sess.finished()[h].shape == (0, 3)
    sess = _session(use_absolute_position_embeddings=True, max_absolute_position_embeddings=8)
    with pytest.raises(IndexError, match="predicted sequence reaches 11"):
        sess.add(conditioning_token_ids=_cond(), seed=1, max_time_steps=4, pred_token_ids=torch.zeros(1, 1, 3, dtype=torch.int64))
    sess.add(conditioning_token_ids=_cond(), seed=1, max_time_steps=3, pred_token_ids=torch.zeros(1, 1, 3, dtype=torch.int64))


def test_finished_output_of_a_row_that_samples_nothing_is_generate_masking():
    sess = _session()
    pred = torch.tensor([[[1, 2, 3], [16, 4, 5]]])                  # 16 = eos of the coarse sequence
    h = sess.add(conditioning_token_ids=_cond(), seed=1, max_time_steps=2, pred_token_ids=pred)
    assert torch.equal(sess.finished()[h], torch.tensor([[1, 2, 3], [-1, -1, -1]]))


def _plain_model(q, slots, events, steps):
    """The schedule one sample at a time: events[k] = the requests (P, n) added before time step k.  Rows wait in
    order for the lowest free slot at a boundary, sample q tokens per time step and free their slot when done.
    Yields, after every time step, {handle: (slot, t, pos, pos_last)}."""
    free, rows, queue, handle = set(range(slots)), {}, [], 0
    for k in range(steps):
        for P, n in events.get(k, []):
            queue.append([handle, P, n])
            handle += 1
        while queue and free:
            h, P, n = queue.pop(0)
            s = min(free)
            free.discard(s)
            rows[s] = dict(h=h, t=0, n=n, pos=P - 1, last=P + max(n, 1) - 2)
        for _ in range(q):
            for r in rows.values():
                if r["t"] < r["n"]:
                    r["t"] += 1
                if r["pos"] < r["last"]:
                    r["pos"] += 1
        state = {r["h"]: (s, r["t"], r["pos"], r["last"]) for s, r in rows.items()}
        for s in [s for s, r in rows.items() if r["t"] >= r["n"]]:
            del rows[s]
            free.add(s)
        yield state


@pytest.mark.parametrize("q,slots", [(1, 1), (3, 4), (4, 17)])
def test_schedule_against_a_plain_model(q, slots):
    rnd = random.Random(q * 100 + slots)
    steps = 60
    events = {k: [(rnd.randint(5, 40), q * rnd.randint(1, 9)) for _ in range(rnd.choice((0, 0, 1, 2, 3)))] for k in range(steps)}
    sched = SlotSchedule(slots, q, max_queue=10 ** 6)
    handle, rows, reuse = 0, {}, 0
    for k, want in zip(range(steps), _plain_model(q, slots, events, steps)):
        for P, n in events.get(k, []):
            r = _Row(handle, P, n, pred_start=P - 3)
            rows[handle] = r
            sched.submit(r)
            handle += 1
        joined = sched.admit()
        reuse += sum(1 for r in joined if any(o.slot == r.slot and o is not r and o.join_step < k for o in rows.values()))
        active = dict(sched.rows)
        sched.advance()
        got = {}
        for s, r in active.items():
            st = r.device_state()
            assert st["pos_offset"] == -(r.P - 2)
            got[r.handle] = (s, st["t"], st["pos"], st["pos_last"])
        assert got == want, k
    assert reuse > 0                                    # slots were reused after rows retired


def test_queue_joins_at_the_next_boundary_in_order():
    sched = SlotSchedule(2, 3, max_queue=2)
    rows = [_Row(h, 10, 3 * (h + 1), 5) for h in range(4)]
    for r in rows:
        sched.submit(r)
    with pytest.raises(ValueError, match="slots are taken"):
        sched.submit(_Row(9, 10, 3, 5))
    assert [r.handle for r in sched.admit()] == [0, 1] and [r.slot for r in rows[:2]] == [0, 1]
    assert [r.handle for r in sched.advance()] == [0]
    assert [r.handle for r in sched.admit()] == [2] and rows[2].slot == 0 and rows[2].join_step == 1
    assert [r.handle for r in sched.advance()] == [1]
    assert [(r.handle, r.slot) for r in sched.admit()] == [(3, 1)]
