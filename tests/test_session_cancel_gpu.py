"""Cancel, suspend and resume in generation and song sessions on the H100: in random streams of add / cancel /
suspend / resume / step, every request that is not cancelled is bit for bit generate(..., seeds=[seed]) for that row
alone (tokens, and with return_logprobs both log-probabilities), at 1, 17, 40 and 256 slots, on the three stages,
with and without top_p, with absolute positions and with chunked prefill; rows suspended several times, for 0 steps,
at their last time step, and resumed into another slot or into an otherwise empty session; the same CUDA-graph count
as the session without suspensions; and song streams whose surviving songs equal generate_tokens alone."""
import os
import random
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from test_generate_ragged_gpu import _model  # noqa: E402
from test_generate_session_gpu import _request  # noqa: E402
from test_musiclm_prime_cpu import load  # noqa: E402
from test_musiclm_prime_gpu import h100_musiclm  # noqa: E402
from test_musiclm_session_gpu import FIX_WIN, song_args  # noqa: E402

pytestmark = pytest.mark.gpu


def _stage(name, abs_pos=False, max_steps=6):
    import open_musiclm_b200 as O
    if name != "fine":
        q = 3 if name == "coarse" else 1
        extra = dict(use_absolute_position_embeddings=True, max_absolute_position_embeddings=max_steps * q + 1) if abs_pos else {}
        return _model(name, **extra)[1], q, [(2, 9)] + ([(3, 14)] if name == "coarse" else [])
    torch.manual_seed(0)
    m = O.create_fine_transformer(dim=128, depth=2, heads=2, clap_codebook_size=64, num_clap_quantizers=4, attn_dropout=0.0,
                                  ff_dropout=0.0, acoustic_codebook_size=64, num_coarse_quantizers=3, num_fine_quantizers=4)
    return O.TokenConditionedTransformerWrapper(transformer=m.cuda().eval(), unique_consecutive=False), 4, [(4, 4), (9, 9)]


def _requests(name, q, shapes, n, g, max_steps, top_p=True):
    reqs = [_request(g, q, 64, shapes, max_steps) for _ in range(n)]
    for r in reqs:
        if name == "fine":        # the coarse conditioning holds whole time steps of 3 quantizers
            r["conditioning_token_ids"][1] = r["conditioning_token_ids"][1][:, :9]
        if not top_p:
            r["top_p"] = None
    return reqs


def _alone(w, req, logprobs):
    r = dict(req)
    seed = r.pop("seed")
    out = w.generate(seeds=[seed], return_logprobs=logprobs, **r)
    return tuple(t[0] for t in out) if logprobs else out[0]


def _equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b)) if isinstance(a, tuple) else torch.equal(a, b)


def _drive(sess, reqs, rng, ops=True, adds_at=None):
    """Adds the requests a few per step as room allows and, between steps, cancels (ops), suspends and resumes
    random requests: some suspended and resumed before the next step, some several times, rows just out of a chunked
    prefill preferably.  Returns ({request: output}, cancelled requests, counts, the step at which each was added)."""
    pending, handles, out, cancelled, held = list(range(len(reqs))), {}, {}, set(), set()
    counts = dict(cancel=0, suspend=0, zero=0, moved=0, multi=0)
    times, slot_at, step, added = {}, {}, 0, {}
    while pending or not sess.idle or held:
        n_add = len(adds_at.get(step, [])) if adds_at is not None else rng.randint(0, 3)
        for _ in range(n_add):
            if not pending:
                break
            try:
                h = sess.add(**reqs[pending[0]])
            except ValueError:
                break
            handles[h] = pending.pop(0)
            added.setdefault(step, []).append(handles[h])
        if ops:
            live = [h for h in handles if h not in cancelled and h not in held and sess.status(h) != "finished"]
            fresh = [h for h in live if sess.status(h) == "running" and sess.sched.live[h].t == sess.q]
            pick = rng.sample(live, min(len(live), rng.randint(0, 2))) + fresh[:1]
            for h in dict.fromkeys(pick):
                state, x = sess.status(h), rng.random()
                if x < 0.12 and h not in fresh:
                    assert sess.cancel(h) is True
                    cancelled.add(h)
                    counts["cancel"] += 1
                elif state in ("queued", "running"):
                    if state == "running":
                        slot_at[h] = sess.sched.live[h].slot
                    sess.suspend(h)
                    times[h] = times.get(h, 0) + 1
                    counts["suspend"] += 1
                    counts["multi"] += times[h] == 2
                    if x < 0.35:                                   # suspended for 0 steps
                        sess.resume(h)
                        counts["zero"] += 1
                    else:
                        held.add(h)
            for h in sorted(held):
                if rng.random() < 0.3 or sess.idle:
                    sess.resume(h)
                    held.discard(h)
        sess.step()
        step += 1
        for h, old in list(slot_at.items()):         # a row restored at this boundary: in which slot?
            row = sess.sched.live.get(h)
            if row is None or row.slot is not None:
                counts["moved"] += row is not None and row.slot != old
                del slot_at[h]
        for h, v in sess.finished().items():
            assert h not in cancelled and handles[h] not in out
            out[handles[h]] = v
    assert not set(out) & {handles[h] for h in cancelled}
    assert len(out) + len(cancelled) == len(reqs)
    return out, {handles[h] for h in cancelled}, counts, added


CASES = [("coarse", 1, True, False, False, 8), ("coarse", 17, True, True, False, 40), ("semantic", 40, False, False, False, 80),
         ("coarse", 256, True, False, False, 320), ("semantic", 17, True, True, True, 40), ("coarse", 17, False, False, True, 40),
         ("fine", 17, True, True, False, 40), ("fine", 1, False, False, False, 6), ("semantic", 256, False, True, False, 300)]


@pytest.mark.parametrize("stage,slots,top_p,logprobs,abs_pos,n_req", CASES,
                         ids=[f"{s}-slots{n}-{'top_p' if t else 'top_k'}-{'lp' if l else 'tok'}-{'abspos' if a else 'relpos'}"
                              for s, n, t, l, a, _ in CASES])
def test_every_surviving_row_equals_generate_alone(stage, slots, top_p, logprobs, abs_pos, n_req):
    import open_musiclm_b200 as O
    max_steps = 6 if stage != "semantic" else 12
    w, q, shapes = _stage(stage, abs_pos, max_steps)
    g = torch.Generator().manual_seed(slots * 5 + len(stage) + abs_pos)
    reqs = _requests(stage, q, shapes, n_req, g, max_steps, top_p)
    sess = O.GenerationSession(w, slots=slots, max_positions=64, max_queue=4, return_logprobs=logprobs)
    out, cancelled, counts, _ = _drive(sess, reqs, random.Random(slots + n_req))
    assert counts["suspend"] and counts["zero"] and (slots == 1 or counts["moved"]), counts
    assert n_req < 20 or (counts["cancel"] and counts["multi"]), counts
    for i, r in enumerate(reqs):
        if i not in cancelled:
            assert _equal(out[i], _alone(w, r, logprobs)), (i, counts)


@pytest.mark.parametrize("stage,budget", [("coarse", 64), ("semantic", 128)])
def test_chunked_prefill_with_cancel_and_suspend(stage, budget):
    """prefill_rows below the prompts' lengths: rows cancelled part-way through their prefill, rows suspended right
    after their last chunk (at their first sample); the others equal generate alone."""
    import open_musiclm_b200 as O
    w, q, _ = _stage(stage)
    g = torch.Generator().manual_seed(budget)
    shapes = [(2, 300)] + ([(3, 60)] if q == 3 else [])
    reqs = _requests(stage, q, shapes, 24, g, 5 if q == 3 else 10)
    sess = O.GenerationSession(w, slots=6, max_positions=512, max_queue=4, prefill_rows=budget)
    rng = random.Random(budget)
    pending, handles, out, cancelled, held, mid, fresh = list(range(len(reqs))), {}, {}, set(), set(), 0, 0
    while pending or not sess.idle or held:
        if pending and rng.random() < 0.5:
            try:
                h = sess.add(**reqs[pending[0]])
                handles[h] = pending.pop(0)
            except ValueError:
                pass
        for h in list(handles):
            if h in cancelled or h in held or sess.status(h) == "finished":
                continue
            row = sess.sched.live[h]
            if sess.status(h) == "prefilling":
                with pytest.raises(ValueError, match="prefilling"):
                    sess.suspend(h)
                if rng.random() < 0.15:
                    sess.cancel(h)
                    cancelled.add(h)
                    mid += 1
            elif sess.status(h) == "running" and row.t == q and row.P > budget:
                sess.suspend(h)
                held.add(h)
                fresh += 1
        for h in sorted(held):
            if rng.random() < 0.4 or sess.idle:
                sess.resume(h)
                held.discard(h)
        sess.step()
        for h, v in sess.finished().items():
            assert h not in cancelled
            out[handles[h]] = v
    assert mid and fresh, (mid, fresh)
    for i, r in enumerate(reqs):
        if i not in {handles[h] for h in cancelled}:
            assert torch.equal(out[i], _alone(w, r, False)), i


@pytest.mark.parametrize("stage", ["coarse", "semantic"])
def test_graph_count_equals_the_session_without_suspensions(stage):
    """The same requests added at the same steps, with and without random cancels and suspensions: the same number
    of captured graphs (restores are plain copies outside the graphs).  Every request has the same top_p, so which
    rows share a step does not change the nucleus part of a graph's key."""
    import open_musiclm_b200 as O
    w, q, shapes = _stage(stage)
    g = torch.Generator().manual_seed(11)
    reqs = _requests(stage, q, shapes, 60, g, 6 if q == 3 else 12)
    for r in reqs:
        r["top_p"] = 0.9
    plain = O.GenerationSession(w, slots=8, max_positions=64, max_queue=64)
    _, _, _, added = _drive(plain, reqs, random.Random(1), ops=False)
    sess = O.GenerationSession(w, slots=8, max_positions=64, max_queue=64)
    _, _, counts, _ = _drive(sess, reqs, random.Random(2), adds_at=added)
    assert counts["suspend"] and counts["cancel"], counts
    assert sess.graph_count == plain.graph_count <= q + 2


def test_last_time_step_and_empty_session_resume():
    """A row suspended with one time step left, resumed after every other row has finished (alone in the session,
    once with nothing else at that boundary and once beside a request that joins there), equals generate alone."""
    import open_musiclm_b200 as O
    w, q, shapes = _stage("coarse")
    g = torch.Generator().manual_seed(3)
    reqs = _requests("coarse", q, shapes, 6, g, 6)
    for r in reqs:                                    # four time steps to sample
        r["max_time_steps"] = (0 if r["pred_token_ids"] is None else r["pred_token_ids"].shape[1]) + 4
    for join in (False, True):
        sess = O.GenerationSession(w, slots=4, max_positions=64, max_queue=4, return_logprobs=True)
        a, b, c = (sess.add(**reqs[i]) for i in range(3))
        row = sess.sched.live[a]
        while row.t < row.n - q:
            sess.step()
        slot = row.slot
        sess.suspend(a)
        assert sess.status(a) == "suspended" and row.slot is None
        out = {}
        while not sess.idle:
            sess.step()
            out.update(sess.finished())
        assert set(out) == {b, c} and not sess.sched.rows
        sess.resume(a)
        d = sess.add(**reqs[3]) if join else None
        sess.step()                                   # restored into slot 0 (resumed rows go first) for its last time step
        assert row.slot == 0 and slot == 0 and sess.status(a) == "finished"
        out.update(sess.finished())
        while not sess.idle:
            sess.step()
            out.update(sess.finished())
        for h, i in ((a, 0), (b, 1), (c, 2)) + (((d, 3),) if join else ()):
            assert _equal(out[h], _alone(w, reqs[i], True)), (join, i)


# ------------------------------------------------------------------------------------------------ song sessions
def _song_stream(sess, songs, rng):
    res, pending, cancelled, held = {}, list(songs), set(), set()
    while pending or not sess.idle or held:
        for _ in range(rng.randint(0, 2)):
            if pending:
                kw = pending.pop(0)
                res[sess.add(**kw)] = dict(args=kw, rows=[])
        live = [h for h in res if h not in cancelled and h not in held and sess.status(h) != "finished"]
        if live and rng.random() < 0.35:
            h = rng.choice(live)
            if rng.random() < 0.25 and len(cancelled) < len(songs) // 3:
                assert sess.cancel(h) is True
                cancelled.add(h)
            else:
                sess.suspend(h)
                held.add(h)
        for h in sorted(held):
            if rng.random() < 0.3 or sess.idle:
                sess.resume(h)
                held.discard(h)
        sess.step()
        for h, r in sess.ready().items():
            assert h not in cancelled
            res[h]["rows"].append(r)
        for h, out in sess.finished().items():
            assert h not in cancelled
            res[h]["out"] = out
    return res, cancelled


def _check_songs(mlm, res, cancelled, win):
    assert cancelled and len(cancelled) < len(res)
    for h, r in res.items():
        if h in cancelled:
            assert "out" not in r
            continue
        kw = dict(r["args"])
        seed = kw.pop("seed")
        ref = mlm.generate_tokens(seeds=[seed], return_all=True, **kw, **win)
        if kw["coarse_only"]:
            assert torch.equal(r["out"], ref) and torch.equal(torch.cat(r["rows"], 1), ref), h
        else:
            assert all(torch.equal(a, b) for a, b in zip(r["out"], ref)) and torch.equal(torch.cat(r["rows"], 1), ref[0]), h


def test_song_stream_with_cancels_and_suspensions_on_a_side_stream():
    """At the fixture weights, 17 slots: the whole stream runs with a non-default current stream, and its outputs
    are compared there without a synchronize."""
    import open_musiclm_b200 as O
    _, win = load()
    mlm = h100_musiclm(win)
    rng, g = random.Random(21), torch.Generator().manual_seed(21)
    songs = song_args(rng, g, 14, 4, 64, 3, 5, [2, 3, 4.5], [(9, 7), (3, 2)])
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        sess = O.MusicLMSession(mlm, slots=17, max_songs=6, max_queue=len(songs), **FIX_WIN)
        res, cancelled = _song_stream(sess, songs, rng)
        _check_songs(mlm, res, cancelled, FIX_WIN)


def test_song_stream_with_cancels_and_suspensions_at_musiclm_small_dims():
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    mk = dict(dim=1024, depth=2, heads=8, attn_dropout=0.0, ff_dropout=0.1)
    mlm = O.MusicLM(semantic_transformer=O.create_semantic_transformer(**mk).cuda().eval(),
                    coarse_transformer=O.create_coarse_transformer(**mk, num_coarse_quantizers=3).cuda().eval(),
                    fine_transformer=O.create_fine_transformer(**mk, num_coarse_quantizers=3, num_fine_quantizers=5).cuda().eval())
    win = dict(semantic_window_seconds=4, coarse_window_seconds=2, fine_window_seconds=1)
    rng, g = random.Random(6), torch.Generator().manual_seed(6)
    songs = song_args(rng, g, 6, 12, 1024, 3, 5, [3, 5], [(120, 80)])
    sess = O.MusicLMSession(mlm, slots=(4, 4, 8), max_songs=4, max_queue=6, **win)
    res, cancelled = _song_stream(sess, songs, rng)
    _check_songs(mlm, res, cancelled, win)
