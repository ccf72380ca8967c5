"""Song sessions (MusicLMSession) against generate_tokens on a stream of songs, at the stages of bench.py's cfg5:
musiclm_small dims (d = 1024, L = 6, h = 8, coarse q 3, fine q 5), random init, synthetic clap ids, the default
windowing of MusicLM.forward.

N songs (default 24) with output_seconds uniform in 4 ... 20 (whole seconds) and seeds 0 ... N - 1, all queued at
once, through
  session  one MusicLMSession (slots per stage --slots, max_songs N), stepped until idle;
  alone    generate_tokens(seeds=[seed]) one song at a time;
  grouped  generate_tokens over static batches of the songs with equal output_seconds, one call per group.
The three are alternated --runs times after a warm-up of each (graph capture), and their outputs are checked equal
song by song.  Reported per variant: wall time (host clock around the whole stream, ending in a synchronise),
generated tokens per second over the three streams (the tokens of generate_tokens' semantic, coarse and fine
outputs), per-song latency p50 / p90 (CUDA events from the start of the stream to the song's output) and the time
to each song's first output rows (the session's first ready() rows; for the others, the song's output).  The card
(name, power limit, max SM clock) is read in the same run.

    python tools/time_musiclm_session.py [--songs 24] [--runs 1] [--slots 32,64,128] [--out DIR]
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


def pct(v, p):
    v = sorted(v)
    return v[min(len(v) - 1, int(round(p * (len(v) - 1))))]


class Clock:
    """CUDA events against one start event: mark(key) records an event now; ms() -> {key: ms since start}."""

    def __init__(self):
        self.start = torch.cuda.Event(enable_timing=True)
        self.start.record()
        self.events = {}

    def mark(self, key):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.events[key] = e

    def ms(self):
        torch.cuda.synchronize()
        return {k: self.start.elapsed_time(e) for k, e in self.events.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--songs", type=int, default=24)
    ap.add_argument("--runs", type=int, default=1)
    ap.add_argument("--slots", default="32,64,128", help="slots of the semantic, coarse and fine sessions")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_musiclm_session: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    torch.manual_seed(0)
    mk = dict(dim=1024, attn_dropout=0.0, ff_dropout=0.1, grad_shrink_alpha=0.1, depth=6, heads=8)
    mlm = O.MusicLM(semantic_transformer=O.create_semantic_transformer(**mk).cuda().eval(),
                    coarse_transformer=O.create_coarse_transformer(**mk, num_coarse_quantizers=3).cuda().eval(),
                    fine_transformer=O.create_fine_transformer(**mk, num_coarse_quantizers=3, num_fine_quantizers=5).cuda().eval())
    N, slots = args.songs, tuple(int(s) for s in args.slots.split(","))
    g, rng = torch.Generator().manual_seed(1234), random.Random(1234)
    clap = torch.randint(0, 1024, (N, 12), generator=g).cuda()
    seconds = [rng.randint(4, 20) for _ in range(N)]

    sess = O.MusicLMSession(mlm, slots=slots, max_songs=N)         # one session for every run, as a server keeps one

    def session_run(songs):
        torch.cuda.synchronize()
        t0, clock = time.perf_counter(), Clock()
        handles = {sess.add(clap_token_ids=clap[i:i + 1], seed=i, output_seconds=seconds[i]): i for i in songs}
        out = {}
        while not sess.idle:
            sess.step()
            for h in sess.ready():
                if ("first", handles[h]) not in clock.events:
                    clock.mark(("first", handles[h]))
            for h, o in sess.finished().items():
                out[handles[h]] = o
                clock.mark(("done", handles[h]))
        torch.cuda.synchronize()
        return out, (time.perf_counter() - t0) * 1e3, clock.ms()

    def alone_run(songs):
        torch.cuda.synchronize()
        t0, clock, out = time.perf_counter(), Clock(), {}
        for i in songs:
            out[i] = mlm.generate_tokens(clap_token_ids=clap[i:i + 1], seeds=[i], output_seconds=seconds[i], return_all=True)
            clock.mark(("done", i))
        torch.cuda.synchronize()
        return out, (time.perf_counter() - t0) * 1e3, clock.ms()

    def grouped_run(songs):
        groups = {}
        for i in songs:
            groups.setdefault(seconds[i], []).append(i)
        torch.cuda.synchronize()
        t0, clock, out = time.perf_counter(), Clock(), {}
        for s, idx in sorted(groups.items()):
            res = mlm.generate_tokens(clap_token_ids=clap[idx], seeds=idx, output_seconds=s, return_all=True)
            for k, i in enumerate(idx):
                out[i] = tuple(t[k:k + 1] for t in res)
                clock.mark(("done", i))
        torch.cuda.synchronize()
        return out, (time.perf_counter() - t0) * 1e3, clock.ms()

    variants = dict(session=session_run, alone=alone_run, grouped=grouped_run)
    warm = [int(min(range(N), key=lambda i: seconds[i]))]
    for fn in variants.values():                                    # graph capture and first-launch costs
        fn(warm)
    runs = {k: [] for k in variants}
    for _ in range(args.runs):
        for k, fn in variants.items():
            runs[k].append(fn(list(range(N))))
            print(f"{k}: {runs[k][-1][1]:.0f} ms", flush=True)
    outs = {k: r[-1][0] for k, r in runs.items()}
    for i in range(N):                      # the three schedules give the same songs
        ref = outs["alone"][i]
        for k in ("session", "grouped"):
            assert all(torch.equal(a, b) for a, b in zip(outs[k][i], ref)), (k, i)
    tokens = sum(t.numel() for i in range(N) for t in outs["alone"][i][1:])
    res = dict(card=info, songs=N, output_seconds=seconds, audio_seconds=sum(seconds), slots=slots, tokens=tokens)
    for k, r in runs.items():
        walls = [w for _, w, _ in r]
        ev = r[-1][2]
        done = [ev[("done", i)] for i in range(N)]
        first = [ev.get(("first", i), ev[("done", i)]) for i in range(N)]
        res[k] = dict(wall_ms=stat(walls), tokens_per_s=tokens / (stat(walls)[0] / 1e3),
                      latency_ms_p50=pct(done, 0.5), latency_ms_p90=pct(done, 0.9),
                      first_rows_ms_p50=pct(first, 0.5), first_rows_ms_min=min(first))
        print(f"{k}: wall {stat(walls)[0]:.0f} ms (spread {stat(walls)[1]:.0f}), {res[k]['tokens_per_s']:.0f} tokens/s, "
              f"latency p50 {res[k]['latency_ms_p50']:.0f} / p90 {res[k]['latency_ms_p90']:.0f} ms, first rows p50 "
              f"{res[k]['first_rows_ms_p50']:.0f} ms (earliest {res[k]['first_rows_ms_min']:.0f})", flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_musiclm_session.json"), "w") as f:
            json.dump(res, f, indent=1, default=str)


if __name__ == "__main__":
    main()
