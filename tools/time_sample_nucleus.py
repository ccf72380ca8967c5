"""Cost of nucleus (top-p) sampling: the sampler alone and one decode step with its sample, top_p None against 0.9.

1. omlm_sample (top_p None) and omlm_sample_nucleus (top_p 0.9) alone on random logits (randn * 3, Philox noise,
   top-k 0.1 C, temperature 0.95) for C in {1025, 2049, 16384} x B in {1, 64, 256}: a CUDA graph of --inner launches,
   replayed --reps times and timed with CUDA events; the two variants alternated, --runs runs each.
2. The musiclm_small coarse stage (d = 1024, L = 6, h = 8) at a context of --context positions: one decode step (all
   layers + logit head) and the sample of its token, replayed from a CUDA graph as tools/time_generate_seeded.py
   does (every replay processes the same position; the sample counter is reset inside the graph), B in {1, 64}.
The table gives the median and the spread (max - min) of the runs, and the card it ran on (name, power limit, max SM
clock), read in the same run.

    python tools/time_sample_nucleus.py [--out DIR]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_generate_batch import card, stat  # noqa: E402
from time_generate_seeded import graph_of, ms_per_replay  # noqa: E402

VARIANTS = (("none", None), ("top_p=0.9", 0.9))


def alternate(graphs, reps, runs, per=1):
    """{variant: (median, spread, runs)} in ms per replay / per, the variants alternated run by run."""
    ms = {v: [] for v in graphs}
    for _ in range(runs):
        for v, g in graphs.items():
            ms[v].append(ms_per_replay(g, reps) / per)
    return {v: (*stat(x), x) for v, x in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--classes", default="1025,2049,16384")
    ap.add_argument("--batches", default="1,64,256")
    ap.add_argument("--step-batches", default="1,64")
    ap.add_argument("--context", type=int, default=1000)
    ap.add_argument("--inner", type=int, default=50)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sample_nucleus: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    from open_musiclm_b200 import lib
    from open_musiclm_b200.decode import DecodeSession, row_arrays
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    dev = "cuda"
    seed = torch.tensor([12345], device=dev, dtype=torch.int64)

    # ---- 1. the sampler alone
    sampler = []
    for C in [int(c) for c in args.classes.split(",")]:
        k = max(int(0.1 * C), 1)
        for B in [int(b) for b in args.batches.split(",")]:
            g = torch.Generator(device=dev).manual_seed(C + B)
            logits = torch.randn(B, C, device=dev, generator=g) * 3
            tokens = torch.zeros(B, args.inner, device=dev, dtype=torch.int64)
            next_row = torch.zeros(B, device=dev, dtype=torch.int32)
            counters = torch.zeros(2, device=dev, dtype=torch.int32)

            def body(tp):
                counters.zero_()
                for _ in range(args.inner):
                    lib.sample(logits, C, k, 0.95, False, None, seed, tokens, next_row, 0, counters, None, B, top_p=tp)
            graphs = {name: graph_of(lambda tp=tp: body(tp)) for name, tp in VARIANTS}
            res = alternate(graphs, args.reps, args.runs, per=args.inner)
            r = dict(C=C, B=B, k=k, **{name: dict(us_per_launch=1e3 * res[name][0], spread_us=1e3 * res[name][1]) for name in graphs})
            sampler.append(r)
            print(json.dumps(r), flush=True)
            del graphs

    # ---- 2. one decode step + sample of the musiclm_small coarse stage
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    eng = m.engine
    n, C = args.context, 1025
    steps = []
    for B in [int(b) for b in args.step_batches.split(",")]:
        s = DecodeSession(eng, B, n + 8, 8, row_arrays(dev, B, pos=n, pos_last=n, pos_offset=0, top_k=max(int(0.1 * C), 1), temperature=0.95))
        top_p_rows = {tp: None if tp is None else torch.full((B,), tp, device=dev) for _, tp in VARIANTS}
        g = torch.Generator(device=dev).manual_seed(B)
        for c in s.cache:
            c.copy_(torch.randn(c.shape, device=dev, generator=g) * 0.3)
        for c in s.conv:
            c.zero_()
        s.pos.fill_(n)                    # every replay processes position n: keys 0..n

        def step(tp, s=s):
            s.step(0)
            s.counters.zero_()            # the token goes to column 0 on every replay
            s.top_p = top_p_rows[tp]          # read when the graph is captured
            s.sample(0, False, None, eng.seed, advance=False)
        graphs = {name: graph_of(lambda tp=tp: step(tp)) for name, tp in VARIANTS}
        res = alternate(graphs, 100, args.runs)
        r = dict(B=B, path="tensor-core" if s.batched else "simt",
                 **{name: dict(ms_per_step=res[name][0], spread_ms=res[name][1], runs_ms=res[name][2]) for name in graphs})
        steps.append(r)
        print(json.dumps(r), flush=True)
        del s, graphs
        torch.cuda.empty_cache()

    print()
    print(f"{info}; sampler alone: CUDA graph of {args.inner} launches, median of {args.runs} runs (spread), us per launch")
    print(f"{'C':>6} {'B':>4} {'top_p None':>18} {'top_p 0.9':>18} {'extra':>8}")
    for r in sampler:
        a, b = r["none"], r["top_p=0.9"]
        print(f"{r['C']:>6} {r['B']:>4} {a['us_per_launch']:>8.2f} ({a['spread_us']:.2f}) {b['us_per_launch']:>8.2f} ({b['spread_us']:.2f}) "
              f"{b['us_per_launch'] - a['us_per_launch']:>8.2f}")
    print(f"\nmusiclm_small coarse stage, context {n}: one decode step + sample from a CUDA graph, median of {args.runs} runs (spread), ms")
    print(f"{'B':>4} {'path':>12} {'top_p None':>18} {'top_p 0.9':>18} {'ratio':>6}")
    for r in steps:
        a, b = r["none"], r["top_p=0.9"]
        print(f"{r['B']:>4} {r['path']:>12} {a['ms_per_step']:>8.4f} ({a['spread_ms']:.4f}) {b['ms_per_step']:>8.4f} ({b['spread_ms']:.4f}) "
              f"{b['ms_per_step'] / a['ms_per_step']:>6.3f}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_sample_nucleus.json"), "w") as f:
            json.dump(dict(card=info, context=n, sampler=sampler, steps=steps), f, indent=1)


if __name__ == "__main__":
    main()
