"""Generation from prefixes of different lengths (`generate(pred_lengths=...)`): what one ragged call saves against one
call per distinct length, and what the per-row positions cost in the decode step.

The musiclm_small coarse stage (d = 1024, L = 6, h = 8), B = 40 rows whose real prefixes are 0 ... 20 time steps
(row b: b mod 21 steps), conditioning of 12 clap + 40 semantic tokens, max_time_steps = 30, Philox noise.  Timed
end to end (host clock around generate, ending in a device synchronise; prefill, graph capture and every decode step
included), alternating, median of --runs after one warm-up of each:
  ragged     one call with pred_lengths: 90 decode steps for all 40 rows
  per_length one call per distinct length (21 calls of 1 or 2 rows: the SIMT path)
  uniform    one call of the same 40 rows with no prefix (90 steps)
Then the decode step alone from a CUDA graph (CUDA events), per-row positions spread over the last 60 positions before
--context, at B = 8 (SIMT) and 40 (tensor cores).  DESIGN section 6 keeps the comparison with the shared-position step
this package no longer has.

    python tools/time_generate_ragged.py [--runs 5] [--context 1000] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else f"{torch.cuda.get_device_name()} (nvidia-smi unavailable)"


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def time_graph(fn, reps, runs=3, warm=10):
    """fn once eagerly (lazy kernel attributes), then a CUDA graph of fn; ms per fn over `reps` replays, `runs` times."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(warm):
        g.replay()
    out = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            g.replay()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) / reps)
    return out


def stat(v):
    v = sorted(v)
    return v[len(v) // 2], v[-1] - v[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--context", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_generate_ragged: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    from open_musiclm_b200.decode import DecodeSession, row_arrays
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    eng = m.engine
    B, T, P = 40, 30, 20
    g = torch.Generator().manual_seed(1)
    cond = [torch.randint(0, 1024, (B, 12), generator=g).cuda(), torch.randint(0, 1024, (B, 40), generator=g).cuda()]
    pred = torch.randint(0, 1024, (B, P, 3), generator=g).cuda()
    lengths = [b % (P + 1) for b in range(B)]
    groups = {}
    for b, n in enumerate(lengths):
        groups.setdefault(n, []).append(b)

    def ragged():
        return w.generate(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=lengths, max_time_steps=T)

    def per_length():
        for n, rows in groups.items():
            idx = torch.tensor(rows, device="cuda")
            w.generate(conditioning_token_ids=[t[idx] for t in cond], pred_token_ids=pred[idx, :n] if n else None, max_time_steps=T)

    def uniform():
        return w.generate(conditioning_token_ids=cond, max_time_steps=T)

    calls = dict(ragged=ragged, per_length=per_length, uniform=uniform)
    for f in calls.values():
        f()
    times = {k: [] for k in calls}
    for _ in range(args.runs):
        for k, f in calls.items():
            times[k].append(wall(f) * 1e3)
    res = {k: dict(zip(("median_ms", "spread_ms"), stat(v)), runs_ms=v) for k, v in times.items()}
    for k, r in res.items():
        print(json.dumps(dict(call=k, **r)), flush=True)
    # the decode step alone, per-row positions
    n = args.context
    steps = []
    for Bs in (8, 40):
        pos = [n - (60 * b) // Bs for b in range(Bs)]
        sess = DecodeSession(eng, Bs, n + 8, 8, row_arrays("cuda", Bs, pos=pos, pos_last=n + 8, pos_offset=0, top_k=1, temperature=1.0))
        gen = torch.Generator(device="cuda").manual_seed(Bs)
        for c in sess.cache:
            c.copy_(torch.randn(c.shape, device="cuda", generator=gen) * 0.3)
        for c in sess.conv:
            c.zero_()
        ms = time_graph(lambda: sess.step(0), args.reps)
        med, spread = stat(ms)
        r = dict(B=Bs, positions="per-row", ms_per_step=med, spread_ms=spread, runs_ms=ms, path="tensor-core" if sess.batched else "simt")
        steps.append(r)
        print(json.dumps(r), flush=True)
        del sess
        torch.cuda.empty_cache()
    print()
    print(f"{info}; musiclm_small coarse stage, B = {B}, prefixes 0..{P} steps, max_time_steps {T}; median of {args.runs} (spread)")
    for k, r in res.items():
        print(f"  {k:<11} {r['median_ms']:9.1f} ms ({r['spread_ms']:.1f})")
    print(f"decode step from a CUDA graph at a context of about {n}, median of 3 (spread)")
    for r in steps:
        print(f"  B={r['B']:>3} {r['path']:>11} {r['positions']:>8} positions: {r['ms_per_step']:.4f} ms ({r['spread_ms']:.4f})")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_generate_ragged.json"), "w") as f:
            json.dump(dict(card=info, B=B, max_time_steps=T, lengths=lengths, calls=res, steps=steps), f, indent=1)


if __name__ == "__main__":
    main()
