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
(name, power limit, max SM clock) is read in the same run.  --variants picks which of the three run; --root imports
the package from another checkout of this repository (built).

The session's host side, without a profiler (last run): time inside step() per call, the step loop's time, and the
time the final synchronise waits for the device after the loop (the work the host had enqueued ahead of the GPU).

--profile: after the runs, one more session run under torch.profiler; its trace goes to DIR/trace_session.json
(--out).  Reported per stage (its kernels are those on its session stream): kernel time, kernel time per step and
the time from a step's first to its last kernel of that stage (mean over the steps in which the stage ran); for the
session: host time per step() call, the fraction of the run's GPU span with any stage kernel in flight, and with
kernels of two or more stages in flight.  Profiling slows the host, so these are shares, not end-to-end times.

--ab PARENT: the session stream on the checkout PARENT (the parent build) and on this one, alternated --runs times,
each run a fresh process (warm-up, then one timed stream); wall time and tokens/s per build, median and spread.

    python tools/time_musiclm_session.py [--songs 24] [--runs 1] [--slots 32,64,128] [--out DIR] [--profile]
                                         [--variants session,alone,grouped] [--root DIR] [--ab PARENT]
"""
import argparse
import json
import os
import random
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_generate_batch import card, stat  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if "--root" in sys.argv:                  # the package of another checkout (time_generate_batch put this one first)
    ROOT = os.path.abspath(sys.argv[sys.argv.index("--root") + 1])
sys.path.insert(0, ROOT)


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
    ap.add_argument("--variants", default="session,alone,grouped")
    ap.add_argument("--root", default=None, help="checkout whose package is imported (default: this one)")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--ab", default=None, metavar="PARENT", help="alternate the session stream with the checkout PARENT")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_musiclm_session: needs a CUDA device (nothing is measured without one)")
    if args.profile and not args.out:
        raise SystemExit("time_musiclm_session: --profile writes its trace under --out")
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    if args.ab:
        return ab_main(args, info)
    import open_musiclm_b200 as O
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
    host = {}                                                      # the last session run's host timings

    def session_run(songs):
        torch.cuda.synchronize()
        t0, clock = time.perf_counter(), Clock()
        handles = {sess.add(clap_token_ids=clap[i:i + 1], seed=i, output_seconds=seconds[i]): i for i in songs}
        out, n_steps, in_step = {}, 0, 0.0
        while not sess.idle:
            t = time.perf_counter()
            sess.step()
            in_step += time.perf_counter() - t
            n_steps += 1
            for h in sess.ready():
                if ("first", handles[h]) not in clock.events:
                    clock.mark(("first", handles[h]))
            for h, o in sess.finished().items():
                out[handles[h]] = o
                clock.mark(("done", handles[h]))
        t = time.perf_counter()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        host.update(steps=n_steps, step_ms=in_step * 1e3 / n_steps, loop_ms=(t - t0) * 1e3, drain_ms=(t1 - t) * 1e3)
        return out, (t1 - t0) * 1e3, clock.ms()

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

    variants = {k: v for k, v in dict(session=session_run, alone=alone_run, grouped=grouped_run).items()
                if k in args.variants.split(",")}
    warm = [int(min(range(N), key=lambda i: seconds[i]))]
    for fn in variants.values():                                    # graph capture and first-launch costs
        fn(warm)
    runs = {k: [] for k in variants}
    for _ in range(args.runs):
        for k, fn in variants.items():
            runs[k].append(fn(list(range(N))))
            print(f"{k}: {runs[k][-1][1]:.0f} ms", flush=True)
    outs = {k: r[-1][0] for k, r in runs.items()}
    base = next(iter(outs))
    for i in range(N):                      # the schedules give the same songs
        ref = outs[base][i]
        for k in outs:
            assert all(torch.equal(a, b) for a, b in zip(outs[k][i], ref)), (k, i)
    tokens = sum(t.numel() for i in range(N) for t in outs[base][i][1:])
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
    if "session" in res:
        res["session"]["host"] = dict(host)
        print(f"session host: {host['steps']} steps, {host['step_ms']:.3f} ms per step() call, step loop "
              f"{host['loop_ms']:.0f} ms, then {host['drain_ms']:.1f} ms until the device was done", flush=True)
    if args.profile:
        res["profile"] = profile_session(sess, session_run, N, args.out)
    print(json.dumps(res, default=str))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_musiclm_session.json"), "w") as f:
            json.dump(res, f, indent=1, default=str)


def profile_session(sess, session_run, N, out_dir):
    """One session run under torch.profiler (trace: out_dir/trace_session.json): per-stage kernel time and per-step
    spans, host time per step, and the shares of the GPU span with one or more, and two or more, stages in flight."""
    from torch.profiler import ProfilerActivity, profile, record_function
    os.makedirs(out_dir, exist_ok=True)
    step = sess.step

    def traced_step():
        with record_function("song_step"):
            step()
    sess.step = traced_step
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for st in sess.streams:           # one marker kernel per stage stream, in stage order: the trace's stream ids
            with torch.cuda.stream(st):
                torch.full((1,), 0, device="cuda")
        session_run(list(range(N)))
    del sess.step
    path = os.path.join(out_dir, "trace_session.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    kernels = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["args"]["correlation"])
    stage_of = {}
    for e in kernels:
        if "FillFunctor" in e["name"] and e["args"]["stream"] not in stage_of:
            stage_of[e["args"]["stream"]] = len(stage_of)
            if len(stage_of) == 3:
                break
    steps = sorted((e["ts"], e["ts"] + e["dur"]) for e in ev if e.get("cat") == "user_annotation" and e["name"] == "song_step")
    launches = sorted((e["ts"], e["args"]["correlation"]) for e in ev if e.get("cat") == "cuda_runtime" and "correlation" in e.get("args", {}))
    step_of_corr, j = {}, 0
    for i, (a, b) in enumerate(steps):
        while j < len(launches) and launches[j][0] < a:
            j += 1
        while j < len(launches) and launches[j][0] <= b:
            step_of_corr[launches[j][1]] = i
            j += 1
    staged = [(stage_of[e["args"]["stream"]], e["ts"], e["ts"] + e["dur"], step_of_corr.get(e["args"]["correlation"]))
              for e in kernels if e["args"]["stream"] in stage_of]
    lo, hi = min(k[1] for k in staged), max(k[2] for k in staged)
    per_step = {}
    for s, a, b, i in staged:
        if i is not None:
            d = per_step.setdefault((s, i), [0.0, a, b])
            d[0] += b - a
            d[1], d[2] = min(d[1], a), max(d[2], b)
    marks = sorted([(a, 1, s) for s, a, _, _ in staged] + [(b, -1, s) for s, _, b, _ in staged])
    active, busy, overlap, prev = [0, 0, 0], 0.0, 0.0, lo
    for t, d, s in marks:
        n = sum(1 for c in active if c > 0)
        busy += (t - prev) if n >= 1 else 0.0
        overlap += (t - prev) if n >= 2 else 0.0
        active[s] += d
        prev = t
    names = ("semantic", "coarse", "fine")
    out = dict(trace=path, steps=len(steps), gpu_span_ms=(hi - lo) / 1e3, host_ms_per_step=sum(b - a for a, b in steps) / len(steps) / 1e3,
               busy_fraction=busy / (hi - lo), overlap_fraction=overlap / (hi - lo), stages={})
    for s, name in enumerate(names):
        mine = [v for (t, _), v in per_step.items() if t == s]
        out["stages"][name] = dict(kernel_ms=sum(b - a for t, a, b, _ in staged if t == s) / 1e3, steps=len(mine),
                                   kernel_ms_per_step=sum(v[0] for v in mine) / max(len(mine), 1) / 1e3,
                                   span_ms_per_step=sum(v[2] - v[1] for v in mine) / max(len(mine), 1) / 1e3)
    print("profile:", json.dumps(out), flush=True)
    return out


def ab_main(args, info):
    """--ab: the session stream in fresh processes, alternating the checkout args.ab and this one."""
    import subprocess
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    builds = dict(parent=os.path.abspath(args.ab), this=here)
    walls, tps = {k: [] for k in builds}, {k: [] for k in builds}
    for r in range(args.runs):
        for k, root in builds.items():
            cmd = [sys.executable, os.path.abspath(__file__), "--root", root, "--variants", "session", "--runs", "1",
                   "--songs", str(args.songs), "--slots", args.slots]
            p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            if p.returncode != 0:
                sys.stdout.write(p.stdout)
                raise SystemExit(f"time_musiclm_session --ab: the {k} run failed")
            res = json.loads(p.stdout.strip().splitlines()[-1])
            walls[k].append(res["session"]["wall_ms"][0])
            tps[k].append(res["session"]["tokens_per_s"])
            print(f"run {r} {k}: wall {walls[k][-1]:.0f} ms, {tps[k][-1]:.0f} tokens/s", flush=True)
    res = dict(card=info, songs=args.songs, slots=args.slots, runs=args.runs,
               **{k: dict(wall_ms=walls[k], wall_ms_median_spread=stat(walls[k]), tokens_per_s=tps[k],
                          tokens_per_s_median=stat(tps[k])[0]) for k in builds})
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_musiclm_session_ab.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
