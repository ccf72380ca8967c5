"""Teacher-forced song scoring (MusicLM.score_tokens) against a loop of per-window teacher-forced generate calls, at
the stages of bench.py's cfg5: musiclm_small dims (d = 1024, L = 6, h = 8, coarse q 3, fine q 5), random init,
synthetic clap ids, the default windowing of MusicLM.forward.

N songs (default 24) with output_seconds uniform in 4 ... 20 (whole seconds) and seeds 0 ... N - 1, as in
tools/time_musiclm_session.py, are generated once (generate_tokens over groups of equal length, return_all) and then
scored by
  score_tokens  one call over the whole list, at each --max-rows value (default 4096, 16384, 65536);
  windows       every window of every song alone: stage.generate(conditioning, pred_token_ids=<prefix + its tokens>,
                max_time_steps=<their length>, return_logprobs=True), the call a user would write today (the windows'
                inputs are cut before the clock starts).
The variants are alternated --runs times after a warm-up of each; the windows' values are checked bit for bit equal
to score_tokens.  Reported per variant: wall time (host clock around the whole list, ending in a synchronise) and
scored tokens per second (the generated tokens of the three streams, each scored once).  The card (name, power
limit, max SM clock) is read in the same run.

    python tools/time_score_songs.py [--songs 24] [--runs 3] [--max-rows 4096,16384,65536] [--out DIR]
"""
import argparse
import json
import os
import random
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_generate_batch import card, stat  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--songs", type=int, default=24)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--max-rows", default="4096,16384,65536")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_score_songs: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    from open_musiclm_b200.stages import STREAMS, plan_song
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    torch.manual_seed(0)
    mk = dict(dim=1024, attn_dropout=0.0, ff_dropout=0.1, grad_shrink_alpha=0.1, depth=6, heads=8)
    mlm = O.MusicLM(semantic_transformer=O.create_semantic_transformer(**mk).cuda().eval(),
                    coarse_transformer=O.create_coarse_transformer(**mk, num_coarse_quantizers=3).cuda().eval(),
                    fine_transformer=O.create_fine_transformer(**mk, num_coarse_quantizers=3, num_fine_quantizers=5).cuda().eval())
    N = args.songs
    g, rng = torch.Generator().manual_seed(1234), random.Random(1234)
    clap = torch.randint(0, 1024, (N, 12), generator=g).cuda()
    seconds = [rng.randint(4, 20) for _ in range(N)]
    songs = [None] * N
    groups = {}
    for i, s in enumerate(seconds):
        groups.setdefault(s, []).append(i)
    for s, idx in sorted(groups.items()):
        res = mlm.generate_tokens(clap_token_ids=clap[idx], seeds=idx, output_seconds=s, return_all=True)
        for k, i in enumerate(idx):
            songs[i] = tuple(t[k:k + 1] for t in res[1:])
    torch.cuda.synchronize()
    tokens = sum(t.numel() for s in songs for t in s)
    print(f"{N} songs, {sum(seconds)} s of audio, {tokens} generated tokens", flush=True)
    song_args = dict(clap_token_ids=[clap[i:i + 1] for i in range(N)], semantic_token_ids=[s[0] for s in songs],
                     coarse_token_ids=[s[1] for s in songs], fine_token_ids=[s[2] for s in songs], output_seconds=seconds)
    # every window's teacher-forced call (without a prime the outputs are the whole streams the windows read)
    stages = (mlm.semantic, mlm.coarse, mlm.fine)
    calls = []
    for i, s in enumerate(songs):
        streams = dict(zip(STREAMS, s))
        part = lambda ref: None if ref is None else streams[ref[0]][:, ref[1]:ref[2]]
        for job in plan_song(output_seconds=seconds[i]).jobs:
            pre = part(job.prefix)
            plen = 0 if pre is None else pre.shape[1]
            a, b = job.dest + max(plen - job.drop, 0), job.dest + job.steps - job.drop
            if b <= a:
                continue
            x = streams[STREAMS[job.stage]][:, a:b]
            x = x if pre is None else torch.cat([pre, x], 1)
            cond = [clap[i:i + 1]] + ([] if job.cond is None else [part(job.cond)])
            calls.append((job.stage, i, plen, (a, b), dict(conditioning_token_ids=cond, pred_token_ids=x, max_time_steps=x.shape[1])))
    print(f"{len(calls)} windows", flush=True)

    def windows_run():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = [stages[st].transformer_wrapper.generate(return_logprobs=True, **kw)[1] for st, _, _, _, kw in calls]
        torch.cuda.synchronize()
        return out, (time.perf_counter() - t0) * 1e3

    def score_run(max_rows):
        def run():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = mlm.score_tokens(max_rows=max_rows, **song_args)
            torch.cuda.synchronize()
            return out, (time.perf_counter() - t0) * 1e3
        return run

    variants = {"windows": windows_run}
    for r in (int(v) for v in args.max_rows.split(",")):
        variants[f"score_tokens max_rows={r}"] = score_run(r)
    for fn in variants.values():                    # first launches, workspaces
        fn()
    walls = {k: [] for k in variants}
    outs = {}
    for _ in range(args.runs):
        for k, fn in variants.items():
            outs[k], w = fn()
            walls[k].append(w)
            print(f"{k}: {w:.0f} ms", flush=True)
    ref = outs[next(k for k in variants if k != "windows")]
    for k in variants:                              # every packing gives the same bits
        if k != "windows":
            assert all(torch.equal(a, b) for st in range(3) for a, b in zip(outs[k][st], ref[st])), k
    for (st, i, plen, (a, b), _), lp in zip(calls, outs["windows"]):
        assert torch.equal(ref[st][i][:, a:b], lp[:, plen:]), (st, i, a)
    res = dict(card=info, songs=N, output_seconds=seconds, audio_seconds=sum(seconds), window_calls=len(calls), tokens=tokens)
    for k, w in walls.items():
        res[k] = dict(wall_ms=stat(w), tokens_per_s=tokens / (stat(w)[0] / 1e3))
        print(f"{k}: wall {stat(w)[0]:.0f} ms (spread {stat(w)[1]:.0f}), {res[k]['tokens_per_s']:.0f} scored tokens/s", flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_score_songs.json"), "w") as f:
            json.dump(res, f, indent=1, default=str)


if __name__ == "__main__":
    main()
