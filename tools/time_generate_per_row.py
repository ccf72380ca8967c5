"""Sampling arguments per row (`generate(temperature=[...], filter_thres=[...], top_p=[...], max_time_steps=[...])`):
what the per-row sampler costs, and what one per-row call saves against one call per setting.

1. The sampler alone: omlm_sample_rows with every row at the same arguments (k = 0.1 C, T = 0.95; top_p None or 0.9)
   against omlm_sample / omlm_sample_nucleus with those arguments as scalars, randn * 3 logits, Philox noise, B in
   {40, 256} x C in {1025, 16384}: a CUDA graph of --inner launches replayed --reps times, CUDA events, variants
   alternated run by run.
2. One decode step + sample of the musiclm_small coarse stage (d = 1024, L = 6, h = 8) at B = 40 and a context of
   --context positions, replayed from a CUDA graph as tools/time_sample_nucleus.py does, with per-row arguments (40
   temperatures 0.5 ... 1.5, k = 0.1 C, top_p 0.9 in every other row).  DESIGN section 6 keeps the comparison with the
   single-value session this package no longer has.
3. A settings sweep: 5 prompts (12 clap + 40 semantic tokens, no prefix, max_time_steps 30) at 8 settings (temperature
   x top_p in {0.7, 1.0} x {None, 0.8, 0.9, 0.95}) as one per-row call of 40 rows against 8 single-value calls of 5
   rows; host clock around each, ending in a device synchronise, alternated, median of --runs after one warm-up.
Every table gives the median and the spread (max - min) of the runs and the card (name, power limit, max SM clock),
read in the same run.

    python tools/time_generate_per_row.py [--runs 5] [--context 1000] [--out DIR]
"""
import argparse
import itertools
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_generate_batch import card, stat  # noqa: E402
from time_generate_seeded import graph_of, ms_per_replay  # noqa: E402


def alternate(graphs, reps, runs, per=1):
    ms = {v: [] for v in graphs}
    for _ in range(runs):
        for v, g in graphs.items():
            ms[v].append(ms_per_replay(g, reps) / per)
    return {v: (*stat(x), x) for v, x in ms.items()}


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--context", type=int, default=1000)
    ap.add_argument("--inner", type=int, default=50)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_generate_per_row: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    from open_musiclm_b200 import lib
    from open_musiclm_b200.decode import DecodeSession, row_arrays
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    dev = "cuda"
    seed = torch.tensor([12345], device=dev, dtype=torch.int64)

    # ---- 1. the sampler alone, equal arguments
    sampler = []
    for C, B in itertools.product((1025, 16384), (40, 256)):
        k, T = max(int(0.1 * C), 1), 0.95
        g = torch.Generator(device=dev).manual_seed(C + B)
        logits = torch.randn(B, C, device=dev, generator=g) * 3
        tokens = torch.zeros(B, args.inner, device=dev, dtype=torch.int64)
        next_row = torch.zeros(B, device=dev, dtype=torch.int32)
        counters = torch.zeros(2, device=dev, dtype=torch.int32)
        k_rows = torch.full((B,), k, device=dev, dtype=torch.int32)
        t_rows = torch.full((B,), T, device=dev, dtype=torch.float32)
        p_rows = torch.full((B,), 0.9, device=dev, dtype=torch.float32)

        def body(tp, per_row):
            counters.zero_()
            rows = dict(top_k_rows=k_rows, temperature_rows=t_rows, top_p_rows=None if tp is None else p_rows) if per_row else {}
            for _ in range(args.inner):
                lib.sample(logits, C, k, T, False, None, seed, tokens, next_row, 0, counters, None, B,
                           top_p=None if per_row else tp, **rows)
        for tp in (None, 0.9):
            graphs = {v: graph_of(lambda pr=pr: body(tp, pr)) for v, pr in (("single", False), ("rows", True))}
            res = alternate(graphs, args.reps, args.runs, per=args.inner)
            r = dict(C=C, B=B, top_p=tp, **{v: dict(us_per_launch=1e3 * res[v][0], spread_us=1e3 * res[v][1]) for v in graphs})
            sampler.append(r)
            print(json.dumps(r), flush=True)
            del graphs

    # ---- 2. one decode step + sample at B = 40
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    eng = m.engine
    n, C, B = args.context, 1025, 40
    k = max(int(0.1 * C), 1)
    temps = [0.5 + b / (B - 1) for b in range(B)]
    tops = [0.9 if b % 2 else None for b in range(B)]
    s = DecodeSession(eng, B, n + 8, 8, row_arrays(dev, B, pos=n, pos_last=n, pos_offset=0, top_k=k, temperature=temps, top_p=tops))
    g = torch.Generator(device=dev).manual_seed(B)
    for c in s.cache:
        c.copy_(torch.randn(c.shape, device=dev, generator=g) * 0.3)
    for c in s.conv:
        c.zero_()

    def step():
        s.step(0)
        s.counters.zero_()
        s.sample(0, False, None, eng.seed, advance=False)
    graphs = {"rows": graph_of(step)}
    res = alternate(graphs, 100, args.runs)
    decode = dict(B=B, context=n, **{v: dict(ms_per_step=res[v][0], spread_ms=res[v][1], runs_ms=res[v][2]) for v in graphs})
    print(json.dumps(decode), flush=True)
    del graphs, s
    torch.cuda.empty_cache()

    # ---- 3. a sweep of 8 settings x 5 prompts
    P, T = 5, 30
    settings = list(itertools.product((0.7, 1.0), (None, 0.8, 0.9, 0.95)))
    g = torch.Generator().manual_seed(1)
    cond = [torch.randint(0, 1024, (P, 12), generator=g).cuda(), torch.randint(0, 1024, (P, 40), generator=g).cuda()]
    rep = [t.repeat(len(settings), 1) for t in cond]
    row_t = [t for t, _ in settings for _ in range(P)]
    row_p = [p for _, p in settings for _ in range(P)]

    def per_row():
        return w.generate(conditioning_token_ids=rep, max_time_steps=T, temperature=row_t, top_p=row_p)

    def per_setting():
        for t, p in settings:
            w.generate(conditioning_token_ids=cond, max_time_steps=T, temperature=t, top_p=p)

    calls = dict(per_row=per_row, per_setting=per_setting)
    for f in calls.values():
        f()
    times = {c: [] for c in calls}
    for _ in range(args.runs):
        for c, f in calls.items():
            times[c].append(wall(f) * 1e3)
    sweep = {c: dict(zip(("median_ms", "spread_ms"), stat(v)), runs_ms=v) for c, v in times.items()}
    for c, r in sweep.items():
        print(json.dumps(dict(call=c, **r)), flush=True)

    print()
    print(f"{info}; sampler alone, equal arguments: CUDA graph of {args.inner} launches, median of {args.runs} runs (spread), us per launch")
    print(f"{'C':>6} {'B':>4} {'top_p':>6} {'single value':>18} {'per row':>18}")
    for r in sampler:
        a, b = r["single"], r["rows"]
        print(f"{r['C']:>6} {r['B']:>4} {str(r['top_p']):>6} {a['us_per_launch']:>8.2f} ({a['spread_us']:.2f}) "
              f"{b['us_per_launch']:>8.2f} ({b['spread_us']:.2f})")
    b = decode["rows"]
    print(f"\nmusiclm_small coarse, B = {B}, context {n}: decode step + sample from a CUDA graph, per-row arguments, ms "
          f"{b['ms_per_step']:.4f} ({b['spread_ms']:.4f})")
    print(f"\nsweep of {len(settings)} settings x {P} prompts, max_time_steps {T}, median of {args.runs} (spread)")
    for c, r in sweep.items():
        print(f"  {c:<12} {r['median_ms']:9.1f} ms ({r['spread_ms']:.1f})")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_generate_per_row.json"), "w") as f:
            json.dump(dict(card=info, sampler=sampler, decode=decode, sweep=sweep), f, indent=1)


if __name__ == "__main__":
    main()
