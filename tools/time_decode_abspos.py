"""Cost of absolute position embeddings in the decode step: the musiclm_small coarse stage (d = 1024, L = 6, h = 8) at a
context of about 1000 positions, one incremental step (all layers + logit head) replayed from a CUDA graph and timed with
CUDA events, with and without use_absolute_position_embeddings, at B = 1, 16 and 64.  With absolute positions the step's
input gather is omlm_embed_gather_pos (one more table row, read at the position the device-side counter gives) instead of
omlm_embed_gather; every other launch is the same.  Also the two gathers alone.

The two models are timed alternately, three runs each; the table gives the median and the spread (max - min).

    python tools/time_decode_abspos.py [--batches 1,16,64] [--context 1000] [--reps 200] [--out DIR]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from time_generate_batch import card, stat, time_graph  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,16,64")
    ap.add_argument("--context", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_decode_abspos: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    from open_musiclm_b200 import lib
    from open_musiclm_b200.decode import DecodeSession, row_arrays
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    n = args.context
    j = 200                     # token index of the processed position within the predicted sequence
    engines = {}
    for abs_pos in (False, True):
        torch.manual_seed(0)
        m = O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1,
                                        use_absolute_position_embeddings=abs_pos).cuda().eval()
        engines[abs_pos] = (m, m.engine)
        assert not abs_pos or j < m.engine.max_abs_pos
    rows = []
    for B in [int(b) for b in args.batches.split(",")]:
        sess = {}
        for abs_pos, (_, eng) in engines.items():
            s = DecodeSession(eng, B, n + 8, 8, row_arrays("cuda", B, pos=n, pos_last=n, pos_offset=j - n, top_k=1, temperature=1.0))
            g = torch.Generator(device="cuda").manual_seed(B)
            for c in s.cache:
                c.copy_(torch.randn(c.shape, device="cuda", generator=g) * 0.3)
            for c in s.conv:
                c.zero_()
            s.pos.fill_(n)               # every replay processes position n: keys 0..n
            sess[abs_pos] = s
        ms = {False: [], True: []}
        for _ in range(3):               # alternate the two models
            for abs_pos in (False, True):
                ms[abs_pos] += time_graph(lambda: sess[abs_pos].step(0), args.reps, runs=1)
        r = dict(B=B, path="tensor-core" if sess[False].batched else "simt")
        for abs_pos, key in ((False, "plain"), (True, "abspos")):
            med, spread = stat(ms[abs_pos])
            r[key] = dict(ms_per_step=med, spread_ms=spread, runs_ms=ms[abs_pos])
        r["extra_us"] = (r["abspos"]["ms_per_step"] - r["plain"]["ms_per_step"]) * 1e3
        # the two gathers alone, 20 launches per replay
        s = sess[True]
        eng = engines[True][1]
        x = s.x[0]
        plain = lambda: [lib.embed_gather(eng.table, s.next_row, x) for _ in range(20)]
        with_pos = lambda: [lib.embed_gather_pos_rows(eng.table, s.next_row, s.pos, s.pos_offset, eng.abs_row_base[-1], eng.max_abs_pos, x)
                            for _ in range(20)]
        for key, f in (("embed_gather_us", plain), ("embed_gather_pos_us", with_pos)):
            med, spread = stat([t / 20 * 1e3 for t in time_graph(f, max(args.reps // 4, 10))])
            r[key] = dict(median=med, spread=spread)
        rows.append(r)
        print(json.dumps(r), flush=True)
        del sess, s
        torch.cuda.empty_cache()
    print()
    print(f"{info}; musiclm_small coarse stage, context {n}, one decode step from a CUDA graph, median of 3 alternated runs (spread)")
    print(f"{'B':>4} {'path':>11} {'plain ms':>18} {'abspos ms':>18} {'extra us':>9} {'gather us':>16} {'gather_pos us':>16}")
    for r in rows:
        p, a, g0, g1 = r["plain"], r["abspos"], r["embed_gather_us"], r["embed_gather_pos_us"]
        print(f"{r['B']:>4} {r['path']:>11} {p['ms_per_step']:>9.4f} ({p['spread_ms']:.4f}) {a['ms_per_step']:>9.4f} ({a['spread_ms']:.4f}) "
              f"{r['extra_us']:>9.2f} {g0['median']:>8.2f} ({g0['spread']:.2f}) {g1['median']:>8.2f} ({g1['spread']:.2f})")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_decode_abspos.json"), "w") as f:
            json.dump(dict(card=info, context=n, steps=rows), f, indent=1)


if __name__ == "__main__":
    main()
