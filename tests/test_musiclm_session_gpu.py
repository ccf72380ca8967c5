"""Song sessions (open_musiclm_b200/musiclm_session.py) on the H100 decode path: every song of a random stream, with
arrivals spread over the steps, mixed lengths, per-stage top_p, primes and coarse_only, is bit for bit
MusicLM.generate_tokens(seeds=[seed], return_all=True) for that song alone, and its ready() rows concatenate to its
output; at the musiclm_prime.pt weights and windowing with 1, 17 and 40 slots, and at musiclm_small dims.  Windows
of a song overlap across stages, rows stream out before the song finishes, and no stage session captures more CUDA
graphs as songs keep coming."""
import os
import random
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(__file__))

from test_musiclm_prime_cpu import load  # noqa: E402
from test_musiclm_prime_gpu import h100_musiclm  # noqa: E402

FIX_WIN = dict(semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5, semantic_steps_per_second=6,
               acoustic_steps_per_second=8)


@pytest.fixture(scope="module")
def fixture_musiclm():
    _, win = load()
    return h100_musiclm(win)


def song_args(rng, g, n, q_clap, codebook, qc, qf, seconds, prime_steps):
    songs = []
    for _ in range(n):
        kw = dict(clap_token_ids=torch.randint(0, codebook, (1, q_clap), generator=g).cuda(), seed=rng.getrandbits(64),
                  output_seconds=rng.choice(seconds), top_p=rng.choice([None, 0.9, (None, 0.8, 0.95), (0.7, None, None)]),
                  coarse_only=rng.random() < 0.2)
        if rng.random() < 0.35:
            ts, ta = rng.choice(prime_steps)
            kw.update(prime_semantic_token_ids=torch.randint(0, codebook, (1, ts), generator=g).cuda(),
                      prime_coarse_token_ids=torch.randint(0, codebook, (1, ta, qc), generator=g).cuda(),
                      prime_fine_token_ids=torch.randint(0, codebook, (1, ta, qf), generator=g).cuda())
        songs.append(kw)
    return songs


def run_stream(sess, songs, rng, max_arrivals=3):
    """Adds the songs a few per step and steps until idle: {handle: (args, output, ready rows, first ready step,
    finish step)}."""
    res, pending, step = {}, list(songs), 0
    while pending or not sess.idle:
        for _ in range(rng.randint(0, max_arrivals)):
            if pending:
                kw = pending.pop(0)
                res[sess.add(**kw)] = dict(args=kw, rows=[])
        sess.step()
        step += 1
        for h, r in sess.ready().items():
            res[h].setdefault("first_ready", step)
            res[h]["rows"].append(r)
        for h, out in sess.finished().items():
            res[h].update(out=out, done=step)
    return res


def check_alone(mlm, res, win):
    for h, r in res.items():
        kw = dict(r["args"])
        seed = kw.pop("seed")
        ref = mlm.generate_tokens(seeds=[seed], return_all=True, **kw, **win)
        out = r["out"]
        if kw["coarse_only"]:
            assert torch.equal(out, ref), h
            assert torch.equal(torch.cat(r["rows"], 1), ref), h
        else:
            assert len(out) == 4 and all(torch.equal(a, b) for a, b in zip(out, ref)), h
            assert torch.equal(torch.cat(r["rows"], 1), ref[0]), h


@pytest.mark.parametrize("fine_pct", [1, 0.5])
@pytest.mark.parametrize("slots", [1, 17, 40])
def test_song_stream_equals_generate_tokens_alone(fixture_musiclm, slots, fine_pct):
    import open_musiclm_b200 as O
    win = dict(FIX_WIN, fine_sliding_window_step_percent=fine_pct)
    rng, g = random.Random(slots * 10 + int(fine_pct * 2)), torch.Generator().manual_seed(slots)
    songs = song_args(rng, g, 12 if slots > 1 else 5, 4, 64, 3, 5, [2, 3, 4.5], [(9, 7), (3, 2)])
    sess = O.MusicLMSession(fixture_musiclm, slots=slots, max_songs=8, max_queue=len(songs), **win)
    res = run_stream(sess, songs, rng)
    assert all("out" in r for r in res.values())
    check_alone(fixture_musiclm, res, win)


def test_song_stream_at_musiclm_small_dims():
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    mk = dict(dim=1024, depth=2, heads=8, attn_dropout=0.0, ff_dropout=0.1)
    mlm = O.MusicLM(semantic_transformer=O.create_semantic_transformer(**mk).cuda().eval(),
                    coarse_transformer=O.create_coarse_transformer(**mk, num_coarse_quantizers=3).cuda().eval(),
                    fine_transformer=O.create_fine_transformer(**mk, num_coarse_quantizers=3, num_fine_quantizers=5).cuda().eval())
    win = dict(semantic_window_seconds=4, coarse_window_seconds=2, fine_window_seconds=1)
    rng, g = random.Random(5), torch.Generator().manual_seed(5)
    songs = song_args(rng, g, 4, 12, 1024, 3, 5, [3, 5], [(120, 80)])
    sess = O.MusicLMSession(mlm, slots=(4, 4, 8), max_songs=4, max_queue=4, **win)
    res = run_stream(sess, songs, rng, max_arrivals=2)
    check_alone(mlm, res, win)


def test_windows_pipeline_and_rows_stream(fixture_musiclm):
    """A 3 s song (7 coarse windows): its first fine window is added before its last coarse window finishes, several
    of its fine windows decode at once, and its first rows arrive before it finishes."""
    import open_musiclm_b200 as O
    from open_musiclm_b200.stages import COARSE, FINE
    sess = O.MusicLMSession(fixture_musiclm, slots=8, **FIX_WIN)
    h = sess.add(clap_token_ids=torch.randint(0, 64, (1, 4)).cuda(), seed=99, output_seconds=3)
    song = sess._songs[h]
    assert sum(j.stage == COARSE for j in song.plan.jobs) >= 3
    fine_add, coarse_done, fine_rows, first_ready, done, step = None, None, 0, None, None, 0
    while not sess.idle:
        sess.step()
        step += 1
        if fine_add is None and song.next[FINE] > 0:
            fine_add = step
        if coarse_done is None and song.done["coarse"] == song.plan.length["coarse"]:
            coarse_done = step
        fine_rows = max(fine_rows, len(sess.sessions[FINE].sched.rows))
        if sess.ready() and first_ready is None:
            first_ready = step
        if sess.finished():
            done = step
    assert fine_add < coarse_done and fine_rows >= 2 and first_ready < done


def test_graph_count_does_not_grow_with_songs(fixture_musiclm):
    """Each stage session captures at most 2 (q + 2) graphs (GenerationSession's bound), however many songs pass
    through it, and a second identical stream of songs captures none."""
    import open_musiclm_b200 as O
    sess = O.MusicLMSession(fixture_musiclm, slots=6, max_songs=4, max_queue=40, **FIX_WIN)
    stream = lambda n, seed: song_args(random.Random(seed), torch.Generator().manual_seed(seed), n, 4, 64, 3, 5, [2, 3, 4.5], [(9, 7)])
    run_stream(sess, stream(8, 1), random.Random(0))
    counts = [s.graph_count for s in sess.sessions]
    assert all(counts)
    run_stream(sess, stream(8, 1), random.Random(0))
    assert [s.graph_count for s in sess.sessions] == counts
    run_stream(sess, stream(24, 2), random.Random(3))
    assert all(s.graph_count <= 2 * (s.q + 2) for s in sess.sessions), [s.graph_count for s in sess.sessions]
