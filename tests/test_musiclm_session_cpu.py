"""Song sessions (open_musiclm_b200/musiclm_session.py) and the song plan they share with MusicLM.generate_tokens
(stages.plan_song), without a GPU: stage wrappers whose tokens are a hash of everything a generate call is given log
every call, so a window that reads the wrong tokens, gets the wrong seed or runs in the wrong place changes the song.
1. the plan's jobs are, job for job, the generate calls of generate_tokens(seeds=[s]) over a grid of windowings,
   primes and coarse_only; 2. a MusicLMSession over stage sessions that finish each request after a random number of
   steps gives every song exactly its generate_tokens output, streams it through ready(), never submits a window
   before its inputs exist and keeps its admission and queue limits; 3. every argument check raises before anything
   runs."""
import hashlib
import itertools
import random
from types import SimpleNamespace

import pytest
import torch

import open_musiclm_b200 as O
from open_musiclm_b200 import musiclm_session as MS
from open_musiclm_b200.stages import COARSE, FINE, SEMANTIC, STREAMS, plan_song, window_seed

Q_CLAP, QC, QF, CB = 4, 3, 5, 64


class HashWrapper:
    """A stage wrapper whose generate returns the prefix followed by tokens drawn from a generator seeded by a hash of
    (stage, conditioning, prefix, seed, max_time_steps, temperature, filter_thres, top_p), row by row.  `log` keeps,
    per row, the call's stage, seed, conditioning (after the clap ids), prefix, arguments and output."""

    def __init__(self, stage, log):
        qs = ([Q_CLAP, 1], [Q_CLAP, 1, QC], [Q_CLAP, QC, QF])[stage]
        self.token_sequences = [SimpleNamespace(codebook_size=CB, num_quantizers=q) for q in qs]
        self.stage, self.log, self.device = stage, log, torch.device("cpu")

    def generate(self, *, conditioning_token_ids, pred_token_ids=None, max_time_steps, filter_thres=0.9, temperature=1.0,
                 include_eos_in_output=False, append_eos_to_conditioning_tokens=True, seeds=None, top_p=None):
        assert not include_eos_in_output and append_eos_to_conditioning_tokens
        q = self.token_sequences[-1].num_quantizers
        B = conditioning_token_ids[0].shape[0]
        T = 0 if pred_token_ids is None else pred_token_ids.shape[1]
        rows = []
        for b in range(B):
            cond = [c[b].reshape(-1).clone() for c in conditioning_token_ids]
            pre = None if pred_token_ids is None else pred_token_ids[b].reshape(T, q).clone()
            seed = None if seeds is None else int(seeds[b])
            args = (max_time_steps, float(temperature), float(filter_thres), top_p)
            h = hashlib.blake2b(repr((self.stage, [c.tolist() for c in cond], None if pre is None else pre.tolist(), seed, args)).encode(),
                                digest_size=8)
            g = torch.Generator().manual_seed(int.from_bytes(h.digest(), "little") >> 1)
            new = torch.randint(0, CB, (max(max_time_steps - T, 0), q), generator=g)
            rows.append(new if pre is None else torch.cat([pre, new]))
            self.log.append(dict(stage=self.stage, seed=seed, cond=cond[1:], prefix=pre, args=args, out=rows[-1]))
        return torch.stack(rows)


def hash_musiclm(log):
    wr = [HashWrapper(s, log) for s in (SEMANTIC, COARSE, FINE)]
    return O.MusicLM(stages=(O.SemanticStage(semantic_transformer=None, wrapper=wr[0]), O.CoarseStage(coarse_transformer=None, wrapper=wr[1]),
                             O.FineStage(fine_transformer=None, wrapper=wr[2])))


def rand_ids(g, *shape):
    return torch.randint(0, CB, shape, generator=g)


def make_primes(g, ts, ta):
    return dict(prime_semantic_token_ids=rand_ids(g, 1, ts), prime_coarse_token_ids=rand_ids(g, 1, ta, QC),
                prime_fine_token_ids=rand_ids(g, 1, ta, QF))


RATES = dict(semantic_steps_per_second=6, acoustic_steps_per_second=8)
WINDOWINGS = [dict(semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5),
              dict(semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5, fine_sliding_window_step_percent=0.5),
              dict(semantic_window_seconds=3, coarse_window_seconds=1.5, fine_window_seconds=1, semantic_sliding_window_step_percent=0.25,
                   coarse_sliding_window_step_percent=0.75),
              dict(semantic_window_seconds=2.5, coarse_window_seconds=1, fine_window_seconds=1, fine_sliding_window_step_percent=0.75)]


def grid():
    out = []
    for (wi, win), secs, prime, coarse_only in itertools.product(enumerate(WINDOWINGS), (1.5, 3, 5.5), (None, (2, 3), (20, 14)),
                                                                (False, True)):
        out.append(pytest.param(dict(win, **RATES), secs, prime, coarse_only, id=f"w{wi}-{secs}s-{prime}-{'coarse' if coarse_only else 'all'}"))
    return out


# ------------------------------------------------------------------------------------------------ 1. the plan
def reconstruct(plan, calls):
    """The generated streams rebuilt from the logged calls through the plan's dest and drop (whole length each)."""
    streams = {k: None for k in STREAMS}
    for job, call in zip(plan.jobs, calls):
        name = STREAMS[job.stage]
        out = call["out"][job.drop:]
        cur = streams[name]
        assert (0 if cur is None else cur.shape[0]) == job.dest
        streams[name] = out if cur is None else torch.cat([cur, out])
    return streams


@pytest.mark.parametrize("win,secs,prime,coarse_only", grid())
def test_plan_is_the_calls_of_generate_tokens(win, secs, prime, coarse_only):
    g = torch.Generator().manual_seed(5)
    log = []
    mlm = hash_musiclm(log)
    clap = rand_ids(g, 1, Q_CLAP)
    primes = make_primes(g, *prime) if prime else {}
    seed, top_p = 987654321, (None, 0.7, 0.9)
    kw = dict(output_seconds=secs, coarse_only=coarse_only, **win)
    lengths = (prime[0], prime[1], prime[1]) if prime else None
    try:
        plan = plan_song(prime_lengths=lengths, seed=seed, top_p=top_p, **kw)
    except ValueError as e:          # a song these arguments cannot make: generate_tokens refuses it before any call
        with pytest.raises(ValueError, match=str(e).split(":")[-1][:30]):
            mlm.generate_tokens(clap_token_ids=clap, seeds=[seed], return_all=True, top_p=top_p, **primes, **kw)
        assert not log
        return
    out = mlm.generate_tokens(clap_token_ids=clap, seeds=[seed], return_all=True, top_p=top_p, **primes, **kw)
    assert len(log) == len(plan.jobs)
    counts = {}
    for job, call in zip(plan.jobs, log):
        w = counts.get(job.stage, 0)
        counts[job.stage] = w + 1
        assert (call["stage"], job.window, call["seed"]) == (job.stage, w, window_seed(seed, job.stage, w))
        assert job.seed == call["seed"] and job.top_p == top_p[job.stage]
        assert call["args"] == (job.max_time_steps, job.temperature, 0.9, job.top_p)
        assert job.temperature == (1.0, 0.95, 0.4)[job.stage]
    # the calls' outputs, replayed through the plan, rebuild streams whose slices are every call's inputs
    streams = reconstruct(plan, log)
    src = dict(streams, prime_semantic=None, prime_coarse=None, prime_fine=None)
    if prime:
        src.update(prime_semantic=primes["prime_semantic_token_ids"][0, :, None], prime_coarse=primes["prime_coarse_token_ids"][0],
                   prime_fine=primes["prime_fine_token_ids"][0])
    have = {k: 0 for k in STREAMS}
    for job, call in zip(plan.jobs, log):
        for ref, got in ((job.cond, call["cond"][0] if call["cond"] else None), (job.prefix, call["prefix"])):
            assert (ref is None) == (got is None)
            if ref is None:
                continue
            name, a, b = ref
            assert torch.equal(src[name][a:b].reshape(-1), got.reshape(-1))
            if name in STREAMS:                       # it reads only tokens written before it, and its needs say so
                assert b <= have[name] and job.needs.get(name, 0) >= b
        for k, v in job.needs.items():
            assert v <= have[k]
        have[STREAMS[job.stage]] += max(job.steps - job.drop, 0)
    assert have == {k: plan.length[k] for k in STREAMS}
    expect = O.stages.song_output(plan, {k: v[None] for k, v in src.items() if v is not None}, True)
    if coarse_only:
        assert torch.equal(out, expect)
    else:
        assert all(torch.equal(a, b) for a, b in zip(out, expect))


# ------------------------------------------------------------------------------------------------ 2. the scheduler
class FakeSession:
    """GenerationSession's add / step / finished / idle surface over a HashWrapper: requests take one of `slots` rows
    first come, first served, and finish after a random number of time steps with generate's output for them alone."""
    made = []

    def __init__(self, wrapper, slots, max_positions, max_queue=0):
        self.w, self.slots, self.max_positions, self.max_queue = wrapper, slots, max_positions, max_queue
        self.queue, self.rows, self.done, self.next, self.steps = [], {}, {}, 0, 0
        self.rng = random.Random(len(FakeSession.made))
        self.adds = []
        FakeSession.made.append(self)

    def add(self, *, conditioning_token_ids, pred_token_ids=None, seed, max_time_steps, temperature=1.0, filter_thres=0.9, top_p=None):
        q = self.w.token_sequences[-1].num_quantizers
        T = 0 if pred_token_ids is None else pred_token_ids.shape[1]
        n = sum(t.numel() + 2 for t in conditioning_token_ids) + 1 + max(max_time_steps, T) * q
        assert n <= self.max_positions
        assert len(self.rows) + len(self.queue) < self.slots + self.max_queue
        h = self.next
        self.next += 1
        args = dict(conditioning_token_ids=[t.clone() for t in conditioning_token_ids],
                    pred_token_ids=None if pred_token_ids is None else pred_token_ids.clone(), seeds=[seed],
                    max_time_steps=max_time_steps, temperature=temperature, filter_thres=filter_thres, top_p=top_p)
        self.adds.append((self.steps, args))
        self.queue.append((h, args))
        return h

    @property
    def idle(self):
        return not self.rows and not self.queue

    def step(self):
        while self.queue and len(self.rows) < self.slots:
            h, args = self.queue.pop(0)
            self.rows[h] = [self.rng.randint(1, 4), args]
        assert len(self.rows) <= self.slots
        self.steps += 1
        for h in list(self.rows):
            self.rows[h][0] -= 1
            if self.rows[h][0] == 0:
                self.done[h] = self.w.generate(**self.rows.pop(h)[1])[0]

    def finished(self):
        d, self.done = self.done, {}
        return d


@pytest.fixture
def fake_sessions(monkeypatch):
    FakeSession.made = []
    monkeypatch.setattr(MS, "GenerationSession", FakeSession)
    return FakeSession.made


SONG_WIN = dict(semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5, **RATES)


def random_songs(g, n, win):
    songs = []
    rng = random.Random(3)
    for i in range(n):
        kw = dict(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=rng.getrandbits(64), output_seconds=rng.choice([2, 3, 4.5]),
                  top_p=rng.choice([None, 0.8, (None, 0.5, 0.9)]), coarse_only=rng.random() < 0.25)
        if rng.random() < 0.4:
            kw.update(make_primes(g, rng.choice([3, 9]), rng.choice([2, 7])))
        songs.append(kw)
    return songs


@pytest.mark.parametrize("fine_pct", [1, 0.5])
@pytest.mark.parametrize("slots,max_songs", [(1, 1), ((2, 3, 5), 4), (8, 64)])
def test_session_songs_equal_generate_tokens_alone(fake_sessions, slots, max_songs, fine_pct):
    g = torch.Generator().manual_seed(11)
    win = dict(SONG_WIN, fine_sliding_window_step_percent=fine_pct)
    songs = random_songs(g, 14, win)
    sess = O.MusicLMSession(hash_musiclm([]), slots=slots, max_songs=max_songs, max_queue=len(songs), **win)
    expect, rows, done, arrival, first_rows = {}, {}, {}, {}, {}
    pending = list(songs)
    step = 0
    while pending or not sess.idle:
        for _ in range(random.Random(step).randint(0, 3)):        # arrivals spread over the steps
            if pending:
                kw = pending.pop(0)
                h = sess.add(**kw)
                arrival[h] = kw
        assert len(sess._songs) <= max_songs
        sess.step()
        step += 1
        for h, r in sess.ready().items():
            first_rows.setdefault(h, step)
            rows.setdefault(h, []).append(r)
        for h, out in sess.finished().items():
            assert h not in done
            done[h] = (out, step)
    assert sorted(done) == sorted(arrival)
    log = []
    mlm = hash_musiclm(log)
    for h, kw in arrival.items():
        kw = dict(kw)
        seed = kw.pop("seed")
        ref = mlm.generate_tokens(seeds=[seed], return_all=True, **kw, **win)
        out, _ = done[h]
        if kw["coarse_only"]:
            assert torch.equal(out, ref)
            assert torch.equal(torch.cat(rows[h], 1), ref)
        else:
            assert all(torch.equal(a, b) for a, b in zip(out, ref))
            assert torch.equal(torch.cat(rows[h], 1), ref[0])
    # each stage session got, per window seed, exactly the inputs generate_tokens gave that window
    calls = {(c["stage"], c["seed"]): c for c in log}
    for st, fs in enumerate(fake_sessions):
        for _, args in fs.adds:
            c = calls[(st, args["seeds"][0])]
            assert all(torch.equal(a.reshape(-1), b) for a, b in zip(args["conditioning_token_ids"][1:], c["cond"]))
            got = args["pred_token_ids"]
            assert (got is None) == (c["prefix"] is None) and (got is None or torch.equal(got.reshape(c["prefix"].shape), c["prefix"]))


def test_session_pipelines_windows_and_streams_rows(fake_sessions):
    """One long song: coarse windows start before the semantic stream is complete, fine windows before the coarse
    stream is, several fine windows run at once, and rows come out before the song finishes."""
    g = torch.Generator().manual_seed(2)
    sess = O.MusicLMSession(hash_musiclm([]), slots=8, **SONG_WIN)
    h = sess.add(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=7, output_seconds=6)
    song = sess._songs[h]
    sem, coarse, fine = fake_sessions
    events = []
    step = 0
    while not sess.idle:
        sess.step()
        step += 1
        events.append((step, dict(song.done), len(fine.rows), bool(sess.ready()), bool(sess.finished())))
    sem_steps = [s for s, _ in sem.adds]
    coarse_steps = [s for s, _ in coarse.adds]
    fine_steps = [s for s, _ in fine.adds]
    assert len(sem_steps) >= 2 and len(coarse_steps) >= 3
    assert coarse_steps[0] < sem_steps[-1] and fine_steps[0] < coarse_steps[-1]
    assert max(n for _, _, n, _, _ in events) >= 2                                # independent fine windows side by side
    first_ready = min(s for s, _, _, r, _ in events if r)
    finished = min(s for s, _, _, _, f in events if f)
    assert first_ready < finished


def test_admission_and_queue_limits(fake_sessions):
    g = torch.Generator().manual_seed(4)
    sess = O.MusicLMSession(hash_musiclm([]), slots=4, max_songs=2, max_queue=1, **SONG_WIN)
    song = lambda i: dict(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=i, output_seconds=2)
    for i in range(3):
        sess.add(**song(i))
    assert len(sess._songs) == 2 and len(sess._queue) == 1
    with pytest.raises(ValueError, match="max_songs = 2"):
        sess.add(**song(3))
    n_adds = [len(f.adds) for f in fake_sessions]
    seen = 0
    while not sess.idle:
        sess.step()
        assert len(sess._songs) <= 2
        seen += len(sess.finished())
    assert seen == 3 and sum(len(f.adds) for f in fake_sessions) > sum(n_adds)
    sess.add(**song(4))                                     # room again


def test_prime_rows_are_ready_at_once(fake_sessions):
    g = torch.Generator().manual_seed(6)
    sess = O.MusicLMSession(hash_musiclm([]), slots=4, **SONG_WIN)
    primes = make_primes(g, 9, 7)
    h = sess.add(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=1, output_seconds=2, **primes)
    r = sess.ready()[h]
    assert torch.equal(r, torch.cat([primes["prime_coarse_token_ids"], primes["prime_fine_token_ids"]], -1))


# ------------------------------------------------------------------------------------------------ 3. argument checks
def test_every_check_raises_before_anything_runs(fake_sessions):
    g = torch.Generator().manual_seed(8)
    mlm = hash_musiclm([])
    for kw, match in [(dict(slots=0), "slots"), (dict(slots=(4, 4)), "three"), (dict(slots=1.5), "slots"), (dict(max_songs=0), "max_songs"),
                      (dict(max_queue=-1), "max_queue"), (dict(max_songs=True), "max_songs"), (dict(slots=(4, 4, 300)), "slots")]:
        with pytest.raises(ValueError, match=match):
            O.MusicLMSession(mlm, **dict(SONG_WIN, **kw))
    sess = O.MusicLMSession(mlm, slots=4, max_songs=1, **SONG_WIN)
    good = dict(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=3, output_seconds=2)
    primes = make_primes(g, 4, 4)
    bad = [(dict(seed=1.5), "seed"), (dict(seed=True), "seed"), (dict(seed=torch.tensor([1, 2])), "seed"),
           (dict(seed=torch.tensor([1], dtype=torch.int32)), "seed"), (dict(top_p=1.5), "top_p"), (dict(top_p=(0.5, 0.5)), "3 values"),
           (dict(output_seconds=0), "output_seconds"), (dict(output_seconds=-2), "output_seconds"), (dict(output_seconds=None), "output_seconds"),
           (dict(output_seconds=0.5), "coarse window"), (dict(clap_token_ids=rand_ids(g, 1, 5)), "clap length"),
           (dict(clap_token_ids=rand_ids(g, 2, Q_CLAP)), "clap length"),
           (dict(prime_semantic_token_ids=primes["prime_semantic_token_ids"]), "all three"),
           (dict(primes, prime_coarse_token_ids=rand_ids(g, 1, 4, QF)), r"\[1 or 1, T, 3\]"),
           (dict(primes, prime_fine_token_ids=rand_ids(g, 2, 4, QF)), r"\[1 or 1, T, 5\]"),
           (dict(primes, prime_semantic_token_ids=rand_ids(g, 1, 4, 2)), r"\[1 or 1, T, 1\]")]
    for kw, match in bad:
        with pytest.raises(ValueError, match=match):
            sess.add(**dict(good, **kw))
    with pytest.raises(TypeError):
        sess.add(**good, noise=O.NoiseStream(torch.rand(10, 1, 65)))
    assert sess.idle and all(not f.adds for f in fake_sessions)
    sess.add(**good)
    with pytest.raises(ValueError, match="max_songs"):                   # max_queue = 0: the second song is refused
        sess.add(**good)
    assert len(fake_sessions[0].adds) == 1


def test_context_beyond_a_window_is_refused(fake_sessions):
    """With a semantic step percent of 1 every semantic window is conditioned on the whole stream so far (as the
    reference does); a song long enough to outgrow the window is refused at add."""
    g = torch.Generator().manual_seed(9)
    sess = O.MusicLMSession(hash_musiclm([]), slots=4, **dict(SONG_WIN, semantic_sliding_window_step_percent=1))
    with pytest.raises(ValueError, match="positions"):
        sess.add(clap_token_ids=rand_ids(g, 1, Q_CLAP), seed=1, output_seconds=5)
    assert all(not f.adds for f in fake_sessions)
