"""Teacher-forced scoring (open_musiclm_b200/score.py), host side: the rows MusicLM.score_tokens scores, over the grid of
windowings, primes and coarse_only of tests/test_musiclm_session_cpu.py, against the generate calls of
generate_tokens(seeds=[s]) logged by hash stage wrappers (every sampled token scored once, no prime token scored, each
window's prompt the tokens its call was given and returned); the packing plan; and every argument check raising
before the engine is touched.  tests/test_score_gpu.py runs the scores themselves."""
import os
import random
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import open_musiclm_b200 as O  # noqa: E402
from open_musiclm_b200 import score as SC  # noqa: E402
from open_musiclm_b200.stages import STREAMS, plan_song, song_output  # noqa: E402
from test_musiclm_session_cpu import CB, Q_CLAP, QC, QF, grid, hash_musiclm, make_primes, rand_ids, reconstruct  # noqa: E402


class Recorder:
    """Stands in for score.score_rows: keeps every row's conditioning and predicted tokens (cut from the sources) and
    adds 1 at each scored position, so the returned scores count how often each token was scored."""

    def __init__(self):
        self.rows = [[], [], []]
        self.max_rows = []

    def __call__(self, wrapper, cond_src, pred_src, rows, out, max_rows=SC.MAX_ROWS):
        stage = wrapper.stage
        for r in rows:
            self.rows[stage].append(dict(cond=[c[torch.from_numpy(i)] for c, i in zip(cond_src, r.cond)],
                                         pred=pred_src[torch.from_numpy(r.pred)], first=r.first))
            out.index_add_(0, torch.from_numpy(r.out), torch.ones(len(r.out)))
        self.max_rows.append(max_rows)


def sampled_masks(plan, log):
    """Per generated stream, which steps a window sampled (not copied from its prefix), rebuilt from the logged calls
    through each job's drop: a bool [T, q] stream."""
    masks = {}
    for job, call in zip(plan.jobs, log):
        plen = 0 if call["prefix"] is None else call["prefix"].shape[0]
        m = torch.arange(call["out"].shape[0])[:, None].expand_as(call["out"]) >= plen
        name = STREAMS[job.stage]
        masks[name] = m[job.drop:] if name not in masks else torch.cat([masks[name], m[job.drop:]])
    return masks


@pytest.mark.parametrize("win,secs,prime,coarse_only", grid())
def test_rows_are_the_windows_of_generate_tokens(monkeypatch, win, secs, prime, coarse_only):
    g = torch.Generator().manual_seed(7)
    log = []
    mlm = hash_musiclm(log)
    clap = rand_ids(g, 1, Q_CLAP)
    primes = make_primes(g, *prime) if prime else {}
    kw = dict(output_seconds=secs, **win)
    lengths = (prime[0], prime[1], prime[1]) if prime else None
    try:
        plan = plan_song(prime_lengths=lengths, coarse_only=coarse_only, **kw)
    except ValueError:
        return
    out = mlm.generate_tokens(clap_token_ids=clap, seeds=[3], return_all=True, coarse_only=coarse_only, **primes, **kw)
    calls = list(log)
    assert len(calls) == len(plan.jobs)
    if coarse_only:         # the coarse stream as it is returned; the semantic stream as return_all returns it
        coarse, fine = out, None
        sem = reconstruct(plan, calls)["semantic"][None, plan.sem_lo:]
    else:
        sem, coarse, fine = out[1:]
    rec = Recorder()
    monkeypatch.setattr(SC, "score_rows", rec)
    args = dict(clap_token_ids=clap, semantic_token_ids=sem, coarse_token_ids=coarse, fine_token_ids=None if coarse_only else fine,
                coarse_only=coarse_only, max_rows=999, **primes, **kw)
    try:
        got = mlm.score_tokens(**args)
    except ValueError as e:
        # a prime shorter than the crop generate_tokens makes: the output lacks generated tokens
        assert "shorter than" in str(e) and prime
        with pytest.raises(ValueError, match="shorter than"):         # from the plan alone
            SC.song_layouts(plan, lengths, (1, QC, QF))
        return
    assert rec.max_rows and set(rec.max_rows) == {999}
    # every sampled token scored once, nothing else
    masks = sampled_masks(plan, calls)
    src = {name: masks[name][None].long() for name in masks}
    if prime:
        src.update(prime_semantic=torch.zeros(1, prime[0], 1, dtype=torch.long), prime_coarse=torch.zeros(1, prime[1], QC, dtype=torch.long),
                   prime_fine=torch.zeros(1, prime[1], QF, dtype=torch.long))
    want = song_output(plan, src, True)
    want = (want[1], want[2], want[3]) if not coarse_only else (None, want, None)
    assert got[2] is None if coarse_only else got[2].shape == fine.shape
    for st, (lp, tok) in enumerate(zip(got, (sem, coarse, fine))):
        if lp is None:
            continue
        assert lp.shape == tok.shape and lp.dtype == torch.float32
        if want[st] is not None:
            assert torch.equal(lp.reshape(want[st].shape), want[st].float()), STREAMS[st]
    # each row is its window's call: clap ids, the call's cond slice, its prefix, then the tokens it sampled and kept
    rows = [iter(r) for r in rec.rows]
    for job, call in zip(plan.jobs, calls):
        plen = 0 if call["prefix"] is None else call["prefix"].shape[0]
        kept = call["out"][max(plen, job.drop):]
        if kept.shape[0] == 0:
            continue
        r = next(rows[job.stage])
        assert torch.equal(r["cond"][0], clap.reshape(-1))
        assert len(r["cond"]) == 1 + len(call["cond"])
        if call["cond"]:
            assert torch.equal(r["cond"][1], call["cond"][0].reshape(-1))
        pre = torch.zeros(0, dtype=torch.long) if call["prefix"] is None else call["prefix"].reshape(-1)
        assert torch.equal(r["pred"], torch.cat([pre, kept.reshape(-1)]))
        assert r["first"] == pre.numel()
    assert all(next(it, None) is None for it in rows)


def test_songs_as_lists_and_tensors(monkeypatch):
    """Songs of different lengths in a list, with and without a prime, score as each song alone; a tensor batch of
    equal songs scores as the list of its rows."""
    g = torch.Generator().manual_seed(2)
    win = dict(semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5, semantic_steps_per_second=6,
               acoustic_steps_per_second=8)
    mlm = hash_musiclm([])
    songs = []
    for i, secs in enumerate((1.5, 3, 5.5, 3)):
        clap = rand_ids(g, 1, Q_CLAP)
        primes = make_primes(g, 20, 14) if i == 1 else {}
        _, sem, coarse, fine = mlm.generate_tokens(clap_token_ids=clap, seeds=[i], return_all=True, output_seconds=secs, **primes, **win)
        songs.append(dict(clap=clap, secs=secs, primes=primes, sem=sem, coarse=coarse, fine=fine))
    rec = Recorder()
    monkeypatch.setattr(SC, "score_rows", rec)
    alone = [mlm.score_tokens(clap_token_ids=s["clap"], semantic_token_ids=s["sem"], coarse_token_ids=s["coarse"], fine_token_ids=s["fine"],
                              output_seconds=s["secs"], **s["primes"], **win) for s in songs]
    n_alone = [len(r) for r in rec.rows]
    pr = lambda k: [s["primes"].get(k) for s in songs]
    got = mlm.score_tokens(clap_token_ids=[s["clap"] for s in songs], semantic_token_ids=[s["sem"] for s in songs],
                           coarse_token_ids=[s["coarse"] for s in songs], fine_token_ids=[s["fine"] for s in songs],
                           output_seconds=[s["secs"] for s in songs], prime_semantic_token_ids=pr("prime_semantic_token_ids"),
                           prime_coarse_token_ids=pr("prime_coarse_token_ids"), prime_fine_token_ids=pr("prime_fine_token_ids"), **win)
    assert [len(r) for r in rec.rows] == [2 * n for n in n_alone]
    for st in range(3):
        assert len(got[st]) == len(songs)
        for a, b in zip(got[st], alone):
            assert torch.equal(a, b[st])
        for a, b in zip(rec.rows[st][:n_alone[st]], rec.rows[st][n_alone[st]:]):
            assert torch.equal(a["pred"], b["pred"]) and a["first"] == b["first"]
            assert all(torch.equal(x, y) for x, y in zip(a["cond"], b["cond"]))
    same = [songs[0], songs[0]]
    batch = mlm.score_tokens(clap_token_ids=torch.cat([s["clap"] for s in same]), semantic_token_ids=torch.cat([s["sem"] for s in same]),
                             coarse_token_ids=torch.cat([s["coarse"] for s in same]), fine_token_ids=torch.cat([s["fine"] for s in same]),
                             output_seconds=1.5, **win)
    for st in range(3):
        assert torch.equal(batch[st], torch.cat([alone[0][st]] * 2))


# ------------------------------------------------------------------------------------------------ packing
@pytest.mark.parametrize("max_rows", [1, 50, 300, 1000, 16384])
def test_pack_groups(max_rows):
    rng = random.Random(max_rows)
    for _ in range(20):
        lengths = [rng.choice([1, 7, 49, 50, 51, 299, 300, 700, 2000]) for _ in range(rng.randint(1, 60))]
        groups = SC.pack_groups(lengths, max_rows)
        flat = sorted(i for g in groups for i in g)
        assert flat == list(range(len(lengths)))
        for g in groups:
            total = sum(lengths[i] for i in g)
            assert total <= max_rows or len(g) == 1
            assert g == sorted(g)
        # first fit decreasing: no two groups could be merged into one forward
        sums = sorted(sum(lengths[i] for i in g) for g in groups)
        assert len(sums) < 2 or sums[0] + sums[1] > max_rows


def test_song_windows_pack_within_max_rows(monkeypatch):
    """The window rows of a stage across songs go to score_rows whole; their packing keeps every group within max_rows."""
    g = torch.Generator().manual_seed(4)
    win = dict(semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5, semantic_steps_per_second=6,
               acoustic_steps_per_second=8)
    mlm = hash_musiclm([])
    outs = [mlm.generate_tokens(clap_token_ids=rand_ids(g, 1, Q_CLAP), seeds=[i], return_all=True, output_seconds=s, **win)
            for i, s in enumerate((3, 5.5, 5.5))]
    rec = Recorder()
    monkeypatch.setattr(SC, "score_rows", rec)
    mlm.score_tokens(clap_token_ids=[rand_ids(g, 1, Q_CLAP) for _ in outs], semantic_token_ids=[o[1] for o in outs],
                     coarse_token_ids=[o[2] for o in outs], fine_token_ids=[o[3] for o in outs], output_seconds=[3, 5.5, 5.5], **win)
    assert len(rec.max_rows) == 3
    for st in range(3):
        lens = [sum(c.numel() + 2 for c in r["cond"]) + r["pred"].numel() + 1 for r in rec.rows[st]]
        for max_rows in (1, 40, 100, max(lens)):
            groups = SC.pack_groups(lens, max_rows)
            assert sorted(i for gr in groups for i in gr) == list(range(len(lens)))
            assert all(sum(lens[i] for i in gr) <= max_rows or len(gr) == 1 for gr in groups)


# ------------------------------------------------------------------------------------------------ argument checks
def _cpu_wrapper(**kw):
    m = O.create_coarse_transformer(dim=64, depth=1, heads=2, clap_codebook_size=16, semantic_codebook_size=16,
                                    acoustic_codebook_size=16, num_clap_quantizers=2, num_coarse_quantizers=3, **kw)
    return m, O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)


def test_score_checks_raise_before_the_engine():
    """Every bad argument raises ValueError (IndexError for the absolute-position limit) before the engine exists; good
    arguments reach the engine (on this CPU-only model its first use raises OmlmError)."""
    m, w = _cpu_wrapper()
    z = lambda *s: torch.zeros(*s, dtype=torch.int64)
    good = dict(conditioning_token_ids=[z(3, 2), z(3, 4)], pred_token_ids=z(3, 5, 3))
    bad_x = z(3, 5, 3)
    bad_x[1, 4, 2] = 16
    bad_c = z(3, 4)
    bad_c[2, 0] = -1
    ragged_bad = z(3, 5, 3)
    ragged_bad[0, 4, 0] = -1                       # past row 0's length: never read
    cases = [(dict(conditioning_token_ids=[z(3, 2)]), "2 tensors"), (dict(conditioning_token_ids=[z(3, 2), z(2, 4)]), "3 rows"),
             (dict(pred_token_ids=z(3, 5, 2)), r"\[b, t, 3\]"), (dict(pred_token_ids=z(3, 15)), r"\[b, t, 3\]"),
             (dict(pred_token_ids=[[0, 0, 0]]), r"\[b, t, 3\]"), (dict(pred_token_ids=bad_x), "codebook"),
             (dict(conditioning_token_ids=[z(3, 2), bad_c]), "conditioning sequence 1"), (dict(max_rows=0), "max_rows"),
             (dict(max_rows=True), "max_rows"), (dict(max_rows=2.0), "max_rows"), (dict(pred_lengths=[1, 2]), "pred_lengths"),
             (dict(pred_lengths=[1, 2, 6]), "pred_lengths"), (dict(pred_lengths=[1, True, 2]), "pred_lengths"),
             (dict(pred_token_ids=ragged_bad, pred_lengths=[5, 5, 5]), "codebook")]
    for kw, match in cases:
        with pytest.raises(ValueError, match=match):
            w.score(**dict(good, **kw))
    assert m._engine is None
    with pytest.raises(O.lib.OmlmError):
        w.score(**dict(good, pred_token_ids=ragged_bad, pred_lengths=[4, 5, 0]))
    m, w = _cpu_wrapper(use_absolute_position_embeddings=True, max_absolute_position_embeddings=12)
    with pytest.raises(IndexError, match="row 1"):
        w.score(**dict(good, pred_lengths=[4, 5, 0]))
    with pytest.raises(IndexError, match="conditioning sequence 1"):
        w.score(conditioning_token_ids=[z(3, 2), z(3, 12)], pred_token_ids=z(3, 1, 3))
    assert m._engine is None
    with pytest.raises(O.lib.OmlmError):
        w.score(**dict(good, pred_lengths=[4, 3, 0]))


def test_score_tokens_checks_raise_before_anything_runs(monkeypatch):
    g = torch.Generator().manual_seed(3)
    win = dict(semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5, semantic_steps_per_second=6,
               acoustic_steps_per_second=8)
    mlm = hash_musiclm([])
    clap = rand_ids(g, 1, Q_CLAP)
    primes = make_primes(g, 20, 14)
    _, sem, coarse, fine = mlm.generate_tokens(clap_token_ids=clap, seeds=[1], return_all=True, output_seconds=3, **primes, **win)
    calls = []
    monkeypatch.setattr(SC, "score_rows", lambda *a, **k: calls.append(a))
    good = dict(clap_token_ids=clap, semantic_token_ids=sem, coarse_token_ids=coarse, fine_token_ids=fine, output_seconds=3, **primes, **win)
    mlm.score_tokens(**good)
    assert len(calls) == 3
    calls.clear()
    bad_fine = fine.clone()
    bad_fine[0, -1, 0] = CB
    short = make_primes(g, 2, 3)
    cases = [(dict(semantic_token_ids=sem[:, 1:]), "semantic stream has"), (dict(coarse_token_ids=coarse[:, :-1]), "coarse stream has"),
             (dict(fine_token_ids=fine[:, :-2]), "fine stream has"), (dict(output_seconds=5.5), "stream has"),
             (dict(fine_token_ids=None), "fine_token_ids"), (dict(coarse_only=True), "fine_token_ids"),
             (dict(coarse_only=1), "coarse_only"), (dict(max_rows=0), "max_rows"), (dict(max_rows=False), "max_rows"),
             (dict(fine_token_ids=bad_fine), "codebook"), (dict(prime_fine_token_ids=None), "all three"),
             (dict(short), "shorter than"), (dict(output_seconds=0.5), "coarse window"), (dict(output_seconds=True), "output_seconds"),
             (dict(output_seconds=[3, 3]), "output_seconds"), (dict(clap_token_ids=clap.repeat(2, 1)), "clap_token_ids"),
             (dict(coarse_token_ids=coarse[..., :2]), r"\[1, T, 3\]"), (dict(semantic_token_ids=[sem, sem]), "list of 2 tensors"),
             (dict(prime_coarse_token_ids=rand_ids(g, 1, 14, QF)), r"\[1 or 1, T, 3\]")]
    for kw, match in cases:
        with pytest.raises(ValueError, match=match):
            mlm.score_tokens(**dict(good, **kw))
    assert not calls
