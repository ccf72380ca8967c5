"""Song sessions on three CUDA streams (open_musiclm_b200/musiclm_session.py): with the caller working on a stream of
its own, every song of a random stream is still bit for bit MusicLM.generate_tokens(seeds=[seed], return_all=True)
alone and its ready() rows concatenate to its output; the stages' decode kernels run on three streams, none of them
the caller's; once the stage sessions have their graphs, stepping a stream of songs to idle never synchronises with
the device; what finished() returns is read on the caller's stream right after step() without a synchronise; and
primed songs stay exact while the caller's stream lags far behind the stages."""
import json
import os
import random
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(__file__))

from test_musiclm_prime_cpu import load  # noqa: E402
from test_musiclm_prime_gpu import h100_musiclm  # noqa: E402
from test_musiclm_session_gpu import FIX_WIN, check_alone, run_stream, song_args  # noqa: E402


@pytest.fixture(scope="module")
def fixture_musiclm():
    _, win = load()
    return h100_musiclm(win)


def small_musiclm():
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    mk = dict(dim=1024, depth=2, heads=8, attn_dropout=0.0, ff_dropout=0.1)
    return O.MusicLM(semantic_transformer=O.create_semantic_transformer(**mk).cuda().eval(),
                     coarse_transformer=O.create_coarse_transformer(**mk, num_coarse_quantizers=3).cuda().eval(),
                     fine_transformer=O.create_fine_transformer(**mk, num_coarse_quantizers=3, num_fine_quantizers=5).cuda().eval())


def reseeded(songs, seed):
    """The same songs (lengths, top_p, primes' shapes, coarse_only) with other seeds and token values: the stage
    sessions run the same schedule, so they need the same graphs."""
    rng, g = random.Random(seed), torch.Generator().manual_seed(seed)
    out = []
    for kw in songs:
        kw = dict(kw, seed=rng.getrandbits(64))
        for k, v in kw.items():
            if isinstance(v, torch.Tensor):
                kw[k] = torch.randint(0, 64, v.shape, generator=g).cuda()
        out.append(kw)
    return out


@pytest.mark.parametrize("slots", [1, 17, 40])
def test_songs_on_a_caller_stream_equal_generate_tokens_alone(fixture_musiclm, slots):
    import open_musiclm_b200 as O
    rng, g = random.Random(slots * 7 + 1), torch.Generator().manual_seed(slots + 100)
    songs = song_args(rng, g, 12 if slots > 1 else 5, 4, 64, 3, 5, [2, 3, 4.5], [(9, 7), (3, 2)])
    caller = torch.cuda.Stream()
    with torch.cuda.stream(caller):
        sess = O.MusicLMSession(fixture_musiclm, slots=slots, max_songs=8, max_queue=len(songs), **FIX_WIN)
        assert len({s.cuda_stream for s in sess.streams} | {caller.cuda_stream}) == 4
        res = run_stream(sess, songs, rng)
        assert all("out" in r for r in res.values())
        check_alone(fixture_musiclm, res, FIX_WIN)


def test_songs_on_a_caller_stream_at_musiclm_small_dims():
    import open_musiclm_b200 as O
    mlm = small_musiclm()
    win = dict(semantic_window_seconds=4, coarse_window_seconds=2, fine_window_seconds=1)
    rng, g = random.Random(6), torch.Generator().manual_seed(6)
    songs = song_args(rng, g, 5, 12, 1024, 3, 5, [3, 5], [(120, 80)])
    caller = torch.cuda.Stream()
    with torch.cuda.stream(caller):
        sess = O.MusicLMSession(mlm, slots=(4, 4, 8), max_songs=4, max_queue=5, **win)
        res = run_stream(sess, songs, rng, max_arrivals=2)
        check_alone(mlm, res, win)


def test_stage_kernels_run_on_three_streams(fixture_musiclm, tmp_path):
    """A torch.profiler trace of a short stream: the decode GEMMs of the three stages run on three CUDA streams, and the
    caller's marker kernel on a fourth."""
    import open_musiclm_b200 as O
    from torch.profiler import ProfilerActivity, profile
    rng, g = random.Random(11), torch.Generator().manual_seed(11)
    songs = song_args(rng, g, 4, 4, 64, 3, 5, [3], [(9, 7)])
    for kw in songs:
        kw["coarse_only"] = False
    sess = O.MusicLMSession(fixture_musiclm, slots=8, max_songs=4, max_queue=4, **FIX_WIN)
    run_stream(sess, reseeded(songs, 1), random.Random(0))                 # first launches and graph capture
    caller = torch.cuda.Stream()
    marker = torch.zeros(1 << 20, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(caller), profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        marker.fill_(1.0)
        run_stream(sess, songs, random.Random(0))
        torch.cuda.synchronize()
    path = tmp_path / "trace.json"
    prof.export_chrome_trace(str(path))
    kernels = sorted((e for e in json.loads(path.read_text())["traceEvents"] if e.get("cat") == "kernel"),
                     key=lambda e: e["args"]["correlation"])                # launch order: the marker first
    decode = {e["args"]["stream"] for e in kernels if "decode_gemm" in e["name"]}
    fills = [e["args"]["stream"] for e in kernels if "FillFunctor" in e["name"]]
    assert len(decode) == 3, decode
    assert fills and fills[0] not in decode, (fills[:1], decode)


def test_no_sync_once_graphs_exist_and_outputs_read_on_the_caller_stream(fixture_musiclm):
    """After a warm-up stream has captured every graph, a second stream of songs (other seeds and tokens, the same
    schedule) is stepped to idle under sync debug mode "error".  finished() outputs are read (copied) on the caller's
    stream right after step(), without a synchronise, and equal generate_tokens alone."""
    import open_musiclm_b200 as O
    rng, g = random.Random(21), torch.Generator().manual_seed(21)
    warm = song_args(rng, g, 10, 4, 64, 3, 5, [2, 3, 4.5], [(9, 7), (3, 2)])
    sess = O.MusicLMSession(fixture_musiclm, slots=6, max_songs=4, max_queue=len(warm), **FIX_WIN)
    for _ in range(2):
        run_stream(sess, warm, random.Random(5))
    counts = [s.graph_count for s in sess.sessions]
    assert all(0 < c <= 2 * (s.q + 2) for c, s in zip(counts, sess.sessions)), counts
    songs = reseeded(warm, 22)
    caller = torch.cuda.Stream()
    res, pending, arrivals, step = {}, list(songs), random.Random(5), 0
    with torch.cuda.stream(caller):
        torch.cuda.set_sync_debug_mode("error")
        try:
            while pending or not sess.idle:
                for _ in range(arrivals.randint(0, 3)):
                    if pending:
                        kw = pending.pop(0)
                        res[sess.add(**kw)] = dict(args=kw, rows=[])
                sess.step()
                step += 1
                for h, r in sess.ready().items():
                    res[h]["rows"].append(r)
                for h, out in sess.finished().items():                 # read on the caller's stream at once
                    res[h].update(out=tuple(t.clone() for t in out) if isinstance(out, tuple) else out.clone(), done=step)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert [s.graph_count for s in sess.sessions] == counts
        assert all("out" in r for r in res.values())
        check_alone(fixture_musiclm, res, FIX_WIN)


def test_primed_songs_exact_while_the_caller_stream_lags(fixture_musiclm):
    """The caller's stream runs far behind the stages (a sleep kernel before every ready() and finished()), so the
    concatenations those calls make there read the songs' coarse and fine streams long after the host has dropped the
    finished songs.  Meanwhile queued songs are admitted and stepped, allocating on the stage streams.  Every primed
    song's output and rows, kept as returned (no copy), still equal generate_tokens alone."""
    import open_musiclm_b200 as O
    rng, g = random.Random(31), torch.Generator().manual_seed(31)
    songs = song_args(rng, g, 10, 4, 64, 3, 5, [2, 3, 4.5], [(9, 7), (3, 2)])
    for i, kw in enumerate(songs):
        kw["coarse_only"] = False
        if "prime_semantic_token_ids" not in kw:
            ts, ta = ((9, 7), (3, 2))[i % 2]
            kw.update(prime_semantic_token_ids=torch.randint(0, 64, (1, ts), generator=g).cuda(),
                      prime_coarse_token_ids=torch.randint(0, 64, (1, ta, 3), generator=g).cuda(),
                      prime_fine_token_ids=torch.randint(0, 64, (1, ta, 5), generator=g).cuda())
    caller = torch.cuda.Stream()
    with torch.cuda.stream(caller):
        sess = O.MusicLMSession(fixture_musiclm, slots=6, max_songs=3, max_queue=len(songs), **FIX_WIN)
        res = {sess.add(**kw): dict(args=kw, rows=[]) for kw in songs}       # all queued now: later admissions wait on nothing new
        while not sess.idle:
            sess.step()
            torch.cuda._sleep(2_000_000)
            for h, r in sess.ready().items():
                res[h]["rows"].append(r)
            torch.cuda._sleep(2_000_000)
            for h, out in sess.finished().items():
                res[h]["out"] = out
        torch.cuda.synchronize()
        assert all("out" in r for r in res.values())
        check_alone(fixture_musiclm, res, FIX_WIN)
