"""Decode-step time of seeded generation against the default path: the musiclm_small coarse stage (d = 1024, L = 6,
h = 8) at a context of about 1000 positions, one incremental step (all layers + logit head) replayed from a CUDA graph
and timed with CUDA events, as tools/time_generate_batch.py does.

Per batch size, a default session (SIMT kernels up to 16 rows, tensor-core GEMM with the batch-dependent K split
above) and a seeded one (tensor-core GEMM with the K split of a 64-row batch at every B): the two are timed
alternately, three runs each; the table gives the median and the spread (max - min) and the card it ran on.

    python tools/time_generate_seeded.py [--batches 1,8,16,17,64,256] [--context 1000] [--out DIR]
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


def graph_of(fn):
    fn()                                  # once eagerly (lazy kernel attributes)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(10):
        g.replay()
    return g


def ms_per_replay(g, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        g.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,16,17,64,256")
    ap.add_argument("--context", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_generate_seeded: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    from open_musiclm_b200.decode import DecodeSession, row_arrays
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    eng = m.engine
    n = args.context
    rows = []
    for B in [int(b) for b in args.batches.split(",")]:
        sess, graphs = {}, {}
        for mode in ("default", "seeded"):
            s = DecodeSession(eng, B, n + 8, 8, row_arrays("cuda", B, pos=n, pos_last=n, pos_offset=0, top_k=1, temperature=1.0), seeded=mode == "seeded")
            g = torch.Generator(device="cuda").manual_seed(B)
            for c in s.cache:
                c.copy_(torch.randn(c.shape, device="cuda", generator=g) * 0.3)
            for c in s.conv:
                c.zero_()
            s.pos.fill_(n)                # every replay processes position n: keys 0..n
            sess[mode] = s
            graphs[mode] = graph_of(lambda s=s: s.step(0))
        ms = {mode: [] for mode in graphs}
        for _ in range(args.runs):       # the two modes alternated, so that clock drift hits both alike
            for mode in ("default", "seeded"):
                ms[mode].append(ms_per_replay(graphs[mode], args.reps))
        r = dict(B=B, default_path="tensor-core" if sess["default"].batched else "simt")
        for mode in ms:
            med, spread = stat(ms[mode])
            r[mode] = dict(ms_per_step=med, spread_ms=spread, runs_ms=ms[mode])
        r["seeded_over_default"] = r["seeded"]["ms_per_step"] / r["default"]["ms_per_step"]
        rows.append(r)
        print(json.dumps(r), flush=True)
        del sess, graphs
        torch.cuda.empty_cache()
    print()
    print(f"{info}; musiclm_small coarse stage, context {n}, one decode step from a CUDA graph, median of {args.runs} runs (spread)")
    print(f"{'B':>4} {'default path':>12} {'default ms':>18} {'seeded ms':>18} {'ratio':>6}")
    for r in rows:
        d, s = r["default"], r["seeded"]
        print(f"{r['B']:>4} {r['default_path']:>12} {d['ms_per_step']:>8.4f} ({d['spread_ms']:.4f}) {s['ms_per_step']:>8.4f} ({s['spread_ms']:.4f}) "
              f"{r['seeded_over_default']:>6.3f}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_generate_seeded.json"), "w") as f:
            json.dump(dict(card=info, context=n, steps=rows), f, indent=1)


if __name__ == "__main__":
    main()
