"""Cancel, suspend and resume in generation and song sessions, host side: SlotSchedule under random add, cancel,
suspend, resume and time-step sequences against a plain statement of its rules; every bad call to
GenerationSession.status / cancel / suspend / resume raises ValueError before any device work; and MusicLMSession's
cancel / suspend / resume over fake stage sessions: songs that survive equal generate_tokens alone, cancelled songs
submit nothing more and free their place, suspended songs submit nothing until resumed."""
import os
import random
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))

import open_musiclm_b200 as O  # noqa: E402
from open_musiclm_b200 import musiclm_session as MS  # noqa: E402
from open_musiclm_b200.session import SlotSchedule, _Row  # noqa: E402
from test_musiclm_session_cpu import Q_CLAP, SONG_WIN, hash_musiclm, rand_ids, random_songs  # noqa: E402


# ------------------------------------------------------------------------------------------------ 1. the schedule
class PlainSchedule:
    """The rules, stated directly: requests wait in a line (resumed requests first, in the order they were resumed,
    then the others in arrival order); at a boundary the budget goes first to the prompts part-way through, in
    admission order, then down the line; a row takes min(its remainder, the largest multiple of unit the budget left
    allows) and the first row that gets nothing stops the line; a row resumed with its prompt done takes a slot and
    no budget.  Every row that joins takes the lowest free slot.  Suspended rows are outside the line and the slots."""

    def __init__(self, slots, q, max_queue, budget, unit):
        self.slots, self.q, self.max_queue, self.budget, self.unit = slots, q, max_queue, budget, unit
        self.req = {}                        # handle -> dict(P, n, filled, t, slot)
        self.resumed, self.queue, self.suspended, self.prefilling = [], [], set(), []

    def room(self):
        slotted = sum(1 for r in self.req.values() if r["slot"] is not None)
        return slotted + len(self.resumed) + len(self.queue) < self.slots + self.max_queue

    def state(self, h):
        r = self.req[h]
        if h in self.suspended:
            return "suspended"
        if r["slot"] is None:
            return "queued"
        return "running" if r["filled"] == r["P"] else "prefilling"

    def leave(self, h):
        r = self.req[h]
        if h in self.suspended:
            self.suspended.discard(h)
        elif h in self.resumed:
            self.resumed.remove(h)
        elif h in self.queue:
            self.queue.remove(h)
        else:
            r["slot"] = None
            if h in self.prefilling:
                self.prefilling.remove(h)

    def boundary(self):
        left = float("inf") if self.budget is None else self.budget
        chunks, restored = [], []
        used = {r["slot"] for r in self.req.values() if r["slot"] is not None}
        free = sorted(set(range(self.slots)) - used)

        def chunk(h):
            nonlocal left
            r = self.req[h]
            rem = r["P"] - r["filled"]
            n = rem if rem <= left else int(left) // self.unit * self.unit
            if n:
                chunks.append((h, r["filled"], n))
                r["filled"] += n
                left -= n
            return n > 0

        stopped = False
        for h in list(self.prefilling):
            if not chunk(h):
                stopped = True
                break
        while free and (self.resumed or self.queue):
            line = self.resumed if self.resumed else self.queue
            h = line[0]
            r = self.req[h]
            if r["filled"] == r["P"]:
                restored.append(h)
            elif stopped or not chunk(h):
                break
            line.pop(0)
            r["slot"] = free.pop(0)
        self.prefilling = [h for h in self.prefilling if self.req[h]["filled"] < self.req[h]["P"]] + \
            [h for h, p0, n in chunks if p0 == 0 and self.req[h]["filled"] < self.req[h]["P"]]
        done = []
        for h, r in sorted(self.req.items(), key=lambda kv: -1 if kv[1]["slot"] is None else kv[1]["slot"]):
            if r["slot"] is not None and r["filled"] == r["P"] and h not in self.suspended:
                r["t"] += self.q
                if r["t"] >= r["n"]:
                    done.append(h)
        for h in done:
            self.req[h]["slot"] = None
        return chunks, restored, done


def _compare(sched, plain, rows):
    for h, r in plain.req.items():
        if h in sched.live:
            assert sched.status(rows[h]) == plain.state(h), h
            assert rows[h].slot == r["slot"] and rows[h].t == r["t"] and rows[h].filled == r["filled"], h
    assert set(sched.suspended) == plain.suspended
    assert [r.handle for r in sched.resumed] == plain.resumed and [r.handle for r in sched.queue] == plain.queue
    assert [r.handle for r in sched.prefilling] == plain.prefilling
    assert sorted(sched.free) == sorted(set(range(sched.slots)) - {r.slot for r in sched.rows.values()})


@pytest.mark.parametrize("q,slots,unit", [(1, 1, 16), (3, 4, 16), (4, 17, 8), (3, 40, 64), (1, 256, 1)])
@pytest.mark.parametrize("budget", [None, 1, 3, 10])
def test_schedule_with_cancel_suspend_resume_follows_its_rules(q, slots, unit, budget):
    budget = None if budget is None else budget * unit
    rnd = random.Random(q * 1000 + slots + (budget or 0))
    max_queue = rnd.choice((0, 2, 7))
    sched = SlotSchedule(slots, q, max_queue=max_queue, prefill_rows=budget, unit=unit)
    plain = PlainSchedule(slots, q, max_queue, budget, unit)
    rows, gone, n_ops = {}, set(), {"cancel": 0, "suspend": 0, "resume": 0, "restored": 0, "cancel_prefilling": 0}
    h = 0
    for step in range(300):
        for _ in range(rnd.choice((0, 1, 1, 2, 4))):
            op = rnd.choice(("add", "add", "cancel", "suspend", "resume"))
            live = [k for k in sched.live]
            if op == "add":
                P, n = rnd.choice((1, 2, unit, unit + 1, rnd.randint(3, 6 * unit))), q * rnd.randint(1, 6)
                ok = plain.room()
                row = _Row(h, P, n, pred_start=0)
                if not ok:
                    with pytest.raises(ValueError, match="slots are taken"):
                        sched.submit(row)
                    continue
                sched.submit(row)
                rows[h] = row
                plain.req[h] = dict(P=P, n=n, filled=0, t=0, slot=None)
                plain.queue.append(h)
                h += 1
            elif op == "cancel" and live:
                k = rnd.choice(live)
                n_ops["cancel_prefilling"] += plain.state(k) == "prefilling"
                sched.cancel(rows[k])
                plain.leave(k)
                del plain.req[k]
                gone.add(k)
                n_ops["cancel"] += 1
            elif op == "suspend":
                can = [k for k in live if plain.state(k) in ("queued", "running")]
                if can:
                    k = rnd.choice(can)
                    sched.suspend(rows[k])
                    plain.leave(k)
                    plain.suspended.add(k)
                    n_ops["suspend"] += 1
            elif op == "resume" and plain.suspended:
                k = rnd.choice(sorted(plain.suspended))
                sched.resume(rows[k])
                plain.suspended.discard(k)
                plain.resumed.append(k)
                n_ops["resume"] += 1
            _compare(sched, plain, rows)
        free_before = sorted(sched.free)
        out = sched.admit()
        restored = [r.handle for r in sched.restored]
        active = {r.handle: r.t for r in sched.rows.values()}
        done = [r.handle for r in sched.advance()]
        chunks, want_restored, want_done = plain.boundary()
        assert [(r.handle, *r.chunk) for r in out] == chunks
        assert restored == want_restored and sorted(done) == sorted(want_done)
        n_ops["restored"] += len(restored)
        joined = [r for r in out if r.chunk[0] == 0] + [rows[k] for k in restored]
        # the rows that joined took the lowest free slots; resumed ones were never behind queued ones
        assert sorted(r.slot for r in joined) == free_before[:len(joined)]
        if budget is not None:
            assert sum(r.chunk[1] for r in out) <= budget
        for k in done:
            assert active[k] + q >= rows[k].n and k not in sched.live
            del plain.req[k]
        _compare(sched, plain, rows)
        assert not gone & set(sched.live)
    assert n_ops["cancel"] and n_ops["suspend"] and n_ops["resume"] and n_ops["restored"], n_ops
    if budget is not None and budget <= 3 * unit:
        assert n_ops["cancel_prefilling"], n_ops


def test_suspended_rows_hold_no_slot_and_no_queue_place():
    sched = SlotSchedule(2, 1, max_queue=1)
    rows = [_Row(h, 5, 10, 0) for h in range(6)]
    for r in rows[:3]:
        sched.submit(r)
    sched.admit()
    sched.advance()
    sched.suspend(rows[0])                                   # running: frees slot 0
    sched.suspend(rows[2])                                   # queued: frees its queue place
    sched.submit(rows[3])
    sched.submit(rows[4])                                    # slot 0 and one queue place
    with pytest.raises(ValueError, match="slots are taken"):
        sched.submit(rows[5])
    sched.resume(rows[2])
    sched.resume(rows[0])                                    # over the limit: resume never refuses
    assert [r.handle for r in sched.resumed] == [2, 0] and [r.handle for r in sched.queue] == [3, 4]
    assert [r.handle for r in sched.admit()] == [2] and rows[2].slot == 0
    sched.advance()
    sched.cancel(rows[1])                                    # slot 1 free at once
    assert sched.admit() == [] and [r.handle for r in sched.restored] == [0] and rows[0].slot == 1
    assert rows[0].t == 1 and rows[0].filled == 5
    sched.advance()
    assert rows[0].t == 2


def test_cancelled_prefilling_row_releases_its_budget():
    sched = SlotSchedule(4, 1, max_queue=4, prefill_rows=40, unit=16)
    rows = [_Row(h, P, 2, 0) for h, P in enumerate((100, 30, 20, 5))]
    for r in rows:
        sched.submit(r)
    assert [(r.handle, r.chunk) for r in sched.admit()] == [(0, (0, 32))]
    sched.advance()
    assert sched.prefilling == [rows[0]] and rows[0].slot == 0
    sched.cancel(rows[0])                # the budget it would take goes to the rows behind it, in order
    assert sched.prefilling == [] and sched.rows == {} and rows[0].slot is None
    assert [(r.handle, r.chunk) for r in sched.admit()] == [(1, (0, 30))] and rows[1].slot == 0
    sched.advance()
    assert [(r.handle, r.chunk) for r in sched.admit()] == [(2, (0, 20)), (3, (0, 5))]
    assert [rows[2].slot, rows[3].slot] == [1, 2]


# ------------------------------------------------------------------------------------------------ 2. argument checks
def _session(**kw):
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=64, depth=1, heads=2, clap_codebook_size=16, num_clap_quantizers=2, semantic_codebook_size=16,
                                    acoustic_codebook_size=16, num_coarse_quantizers=3)
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    return O.GenerationSession(w, slots=2, max_positions=200, max_queue=4, **kw)


def _req(seed, steps=4, pred=None, clap=2, sem=6):
    g = torch.Generator().manual_seed(seed)
    return dict(conditioning_token_ids=[torch.randint(0, 16, (1, clap), generator=g), torch.randint(0, 16, (1, sem), generator=g)],
                pred_token_ids=pred, seed=seed, max_time_steps=steps)


def test_session_calls_are_checked_before_any_device_work():
    sess = _session()
    a, b, c = (sess.add(**_req(i)) for i in range(3))
    done = sess.add(**_req(3, steps=1, pred=torch.zeros(1, 1, 3, dtype=torch.int64)))    # nothing to sample: finished
    assert [sess.status(h) for h in (a, b, c, done)] == ["queued"] * 3 + ["finished"]
    for bad in (-1, 4, 99, True, 1.0, "0", None):
        for call in (sess.status, sess.cancel, sess.suspend, sess.resume):
            with pytest.raises(ValueError, match="not a handle"):
                call(bad)
    assert sess.cancel(done) is False and done in sess.finished()
    assert sess.status(done) == "finished" and sess.cancel(done) is False
    for call in (sess.suspend, sess.resume):
        with pytest.raises(ValueError, match="finished"):
            call(done)
    with pytest.raises(ValueError, match="not suspended"):
        sess.resume(a)
    assert sess.cancel(b) is True
    for call in (sess.status, sess.cancel, sess.suspend, sess.resume):
        with pytest.raises(ValueError, match="was cancelled"):
            call(b)
    sess.suspend(c)                                           # queued: host state only
    assert sess.status(c) == "suspended" and [r.handle for r in sess.sched.queue] == [a]
    with pytest.raises(ValueError, match="is suspended"):
        sess.suspend(c)
    sess.resume(c)
    assert sess.status(c) == "queued" and [r.handle for r in sess.sched.resumed] == [c]
    assert sess.dec is None and sess.eng is None


def test_suspend_mid_prefill_and_under_trace_logits_raise():
    sess = _session(prefill_rows=64)
    h = sess.add(**_req(0, sem=150))                          # a prompt of 157 rows: three chunks
    sess.sched.admit()                                        # host side of the boundary: its first chunk
    assert sess.status(h) == "prefilling"
    with pytest.raises(ValueError, match="prefilling"):
        sess.suspend(h)
    assert sess.status(h) == "prefilling" and sess.sched.prefilling and sess.dec is None
    assert sess.cancel(h) is True and not sess.sched.prefilling and sess.sched.free == [1, 0]
    tr = _session(trace_logits=True)
    h = tr.add(**_req(1))
    with pytest.raises(ValueError, match="trace_logits"):
        tr.suspend(h)
    assert tr.status(h) == "queued" and tr.cancel(h) is True and tr.idle and tr.dec is None


# ------------------------------------------------------------------------------------------------ 3. song sessions
class StageSession:
    """GenerationSession's surface over a HashWrapper, cancel / suspend / resume / status included: requests take one
    of `slots` rows (resumed ones first), and finish after a random number of time steps with generate's output for
    them alone; a suspended row keeps its remaining steps."""
    made = []

    def __init__(self, wrapper, slots, max_positions, max_queue=0):
        self.w, self.slots = wrapper, slots
        self.queue, self.resumed, self.rows, self.held, self.done, self.next = [], [], {}, {}, {}, 0
        self.rng = random.Random(len(StageSession.made))
        self.adds, self.gone = [], set()
        StageSession.made.append(self)

    def add(self, *, conditioning_token_ids, pred_token_ids=None, seed, max_time_steps, temperature=1.0, filter_thres=0.9, top_p=None):
        h = self.next
        self.next += 1
        args = dict(conditioning_token_ids=[t.clone() for t in conditioning_token_ids],
                    pred_token_ids=None if pred_token_ids is None else pred_token_ids.clone(), seeds=[seed],
                    max_time_steps=max_time_steps, temperature=temperature, filter_thres=filter_thres, top_p=top_p)
        self.adds.append(args)
        self.queue.append([h, self.rng.randint(1, 4), args])
        return h

    @property
    def idle(self):
        return not self.rows and not self.queue and not self.resumed

    def status(self, h):
        assert h not in self.gone
        if h in self.held:
            return "suspended"
        if h in self.rows:
            return "running"
        return "queued" if any(e[0] == h for e in self.queue + self.resumed) else "finished"

    def _find(self, h):
        for line in (self.resumed, self.queue):
            for e in line:
                if e[0] == h:
                    line.remove(e)
                    return e
        return [h] + self.rows.pop(h)

    def cancel(self, h):
        if self.status(h) == "finished":
            return False
        if self.held.pop(h, None) is None:
            self._find(h)
        self.gone.add(h)
        return True

    def suspend(self, h):
        assert self.status(h) in ("queued", "running")
        self.held[h] = self._find(h)

    def resume(self, h):
        self.resumed.append(self.held.pop(h))

    def step(self):
        while (self.resumed or self.queue) and len(self.rows) < self.slots:
            h, left, args = (self.resumed or self.queue).pop(0)
            self.rows[h] = [left, args]
        for h in list(self.rows):
            self.rows[h][0] -= 1
            if self.rows[h][0] == 0:
                self.done[h] = self.w.generate(**self.rows.pop(h)[1])[0]

    def finished(self):
        d, self.done = self.done, {}
        return d


@pytest.fixture
def stage_sessions(monkeypatch):
    StageSession.made = []
    monkeypatch.setattr(MS, "GenerationSession", StageSession)
    return StageSession.made


def _alone(kw, win):
    log = []
    kw = dict(kw)
    seed = kw.pop("seed")
    return hash_musiclm(log).generate_tokens(seeds=[seed], return_all=True, **kw, **win)


@pytest.mark.parametrize("slots,max_songs", [(1, 1), ((2, 3, 5), 4), (8, 64)])
def test_song_stream_with_cancels_and_suspensions(stage_sessions, slots, max_songs):
    """Random songs arriving over the steps, with random cancels, suspensions (of queued and admitted songs, for 0 or
    more steps, several times) and resumes: every song not cancelled equals generate_tokens alone and its ready()
    rows concatenate to its output; a cancelled song appears in neither ready() nor finished() after its cancel."""
    g = torch.Generator().manual_seed(slots if isinstance(slots, int) else 7)
    songs = random_songs(g, 16, SONG_WIN)
    sess = O.MusicLMSession(hash_musiclm([]), slots=slots, max_songs=max_songs, max_queue=len(songs), **SONG_WIN)
    rng = random.Random(max_songs)
    arrival, rows, done, cancelled, suspended = {}, {}, {}, set(), set()
    counts = {"cancel": 0, "suspend": 0, "resume": 0}
    pending = list(songs)
    while pending or not sess.idle or suspended:
        for _ in range(rng.randint(0, 2)):
            if pending:
                kw = pending.pop(0)
                arrival[sess.add(**kw)] = kw
        live = [h for h in arrival if h not in cancelled and sess.status(h) != "finished"]
        if live and rng.random() < 0.3:
            h = rng.choice(live)
            if rng.random() < 0.3:
                assert sess.cancel(h) is True
                cancelled.add(h)
                suspended.discard(h)
                counts["cancel"] += 1
            elif h in suspended:
                sess.resume(h)
                suspended.discard(h)
                counts["resume"] += 1
            else:
                sess.suspend(h)
                assert sess.status(h) == "suspended"
                suspended.add(h)
                counts["suspend"] += 1
        if suspended and (rng.random() < 0.3 or (sess.idle and not pending)):
            h = sorted(suspended)[0]
            sess.resume(h)
            suspended.discard(h)
            counts["resume"] += 1
        assert len(sess._songs) <= max_songs
        sess.step()
        for h, r in sess.ready().items():
            assert h not in cancelled
            rows.setdefault(h, []).append(r)
        for h, out in sess.finished().items():
            assert h not in cancelled and h not in done
            done[h] = out
    assert counts["cancel"] and counts["suspend"] and counts["resume"], counts
    assert sorted(done) == sorted(set(arrival) - cancelled)
    for h in done:
        ref = _alone(arrival[h], SONG_WIN)
        if arrival[h]["coarse_only"]:
            assert torch.equal(done[h], ref) and torch.equal(torch.cat(rows[h], 1), ref), h
        else:
            assert all(torch.equal(a, b) for a, b in zip(done[h], ref)) and torch.equal(torch.cat(rows[h], 1), ref[0]), h


def test_cancelled_song_submits_nothing_and_frees_its_place(stage_sessions):
    g = torch.Generator().manual_seed(4)
    sess = O.MusicLMSession(hash_musiclm([]), slots=4, max_songs=1, max_queue=1, **SONG_WIN)
    a = sess.add(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=1, output_seconds=4)
    b = sess.add(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=2, output_seconds=2)
    assert sess.status(a) == "waiting" and sess.status(b) == "queued"
    for _ in range(3):
        sess.step()
    assert sess.status(a) in ("running", "waiting")
    adds = [len(s.adds) for s in stage_sessions]
    seeds = {args["seeds"][0] for s in stage_sessions for args in s.adds}
    seeds_a = {j.seed for j in sess._songs[a].plan.jobs}
    assert sess.cancel(a) is True
    assert sess.status(b) in ("running", "waiting") and list(sess._songs) == [b]      # admitted at once
    with pytest.raises(ValueError, match="was cancelled"):
        sess.status(a)
    new_seeds = {args["seeds"][0] for s in stage_sessions for args in s.adds} - seeds
    while not sess.idle:
        sess.step()
        assert a not in sess.ready() and a not in sess.finished()
    later = {args["seeds"][0] for s in stage_sessions for args in s.adds} - seeds - new_seeds
    assert not seeds_a & (new_seeds | later)                 # no window of a was added after its cancel
    assert seeds_a - seeds                                    # and some never were
    assert sum(len(s.adds) for s in stage_sessions) > sum(adds)
    assert all(s.idle and not s.held for s in stage_sessions)


def test_suspended_song_submits_nothing_until_resumed(stage_sessions):
    g = torch.Generator().manual_seed(5)
    sess = O.MusicLMSession(hash_musiclm([]), slots=4, max_songs=2, **SONG_WIN)
    kw = dict(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=3, output_seconds=4)
    h = sess.add(**kw)
    for _ in range(4):
        sess.step()
    sess.suspend(h)
    assert sess.status(h) == "suspended" and sess.idle
    adds = [len(s.adds) for s in stage_sessions]
    ready = sess.ready()
    for _ in range(10):
        sess.step()
        assert not sess.ready() and not sess.finished()
    assert [len(s.adds) for s in stage_sessions] == adds and all(not s.rows for s in stage_sessions)
    with pytest.raises(ValueError, match="is suspended"):
        sess.suspend(h)
    sess.resume(h)
    with pytest.raises(ValueError, match="not suspended"):
        sess.resume(h)
    rows = [ready[h]] if h in ready else []
    while not sess.idle:
        sess.step()
        rows += list(sess.ready().values())
        out = sess.finished()
    assert sess.status(h) == "finished" and sess.cancel(h) is False
    ref = _alone(kw, SONG_WIN)
    assert all(torch.equal(a, b) for a, b in zip(out[h], ref)) and torch.equal(torch.cat(rows, 1), ref[0])


def test_song_calls_are_checked(stage_sessions):
    g = torch.Generator().manual_seed(6)
    sess = O.MusicLMSession(hash_musiclm([]), slots=4, max_songs=1, max_queue=1, **SONG_WIN)
    a = sess.add(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=1, output_seconds=2)
    b = sess.add(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=2, output_seconds=2)
    for bad in (-1, 2, True, "a", None, 0.0):
        for call in (sess.status, sess.cancel, sess.suspend, sess.resume):
            with pytest.raises(ValueError, match="not a song handle"):
                call(bad)
    with pytest.raises(ValueError, match="not suspended"):
        sess.resume(b)
    sess.suspend(b)                                           # queued: leaves the queue
    assert sess.status(b) == "suspended" and not sess._queue
    sess.add(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=3, output_seconds=2)     # its queue place is free
    sess.resume(b)
    assert [e[0] for e in sess._queue] == [b, 2]
    assert sess.cancel(b) is True and [e[0] for e in sess._queue] == [2]
    with pytest.raises(ValueError, match="was cancelled"):
        sess.resume(b)
    assert sess.status(a) == "waiting"
