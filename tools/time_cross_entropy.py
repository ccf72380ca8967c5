"""Cross-entropy call time across class counts, and the training step at three semantic codebook sizes.

1. The fused CE call (loss + dlogits, omlm_cross_entropy) at the musiclm_small semantic-stage shape: B = 16 sequences of
   500 labelled positions = 8000 rows, fp32 logits [rows, Cp] and bf16 dlogits [rows, Cp] as the trainer lays them out.
   C = 1025 takes the register-cached kernel, larger C the streaming one.  Each call is timed with CUDA events over
   `--reps` launches after warm-up, three runs; the table gives the median, the spread, the bytes the call must move
   (logits read once + dlogits written, from shapes) and that traffic over the time as a share of the H100 SXM
   data-sheet 3.35 TB/s.
2. One graph-replayed HotPathTrainer.train_step of the musiclm_small semantic stage (d = 1024, L = 6, h = 8, clap
   1024 x 12, B = 16, 499 semantic tokens) with semantic codebooks of 1024, 2048 and 4096 entries.

The card's name, power limit and max SM clock are read in the same run.

    python tools/time_cross_entropy.py [--reps 200] [--steps 20] [--out DIR]
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

HBM_BYTES_PER_S = 3.35e12


def time_ce(C, rows, reps, runs):
    from open_musiclm_b200 import lib
    Cp = (C + 63) // 64 * 64
    g = torch.Generator(device="cuda").manual_seed(C)
    logits = torch.randn(rows, Cp, device="cuda", generator=g) * 4
    labels = torch.randint(0, C, (rows,), device="cuda", generator=g, dtype=torch.int32)
    dl = torch.empty(rows, Cp, device="cuda", dtype=torch.bfloat16)
    acc = torch.zeros(2, device="cuda")
    call = lambda: lib.cross_entropy(logits, labels, C, acc, grad_scale=1.0 / rows, dlogits=dl, loss_scale=1.0 / rows)
    for _ in range(20):
        call()
    torch.cuda.synchronize()
    ms = []
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(runs):
        a.record()
        for _ in range(reps):
            call()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b) / reps)
    med, spread = stat(ms)
    nbytes = rows * C * 4 + rows * Cp * 2 + rows * 4
    return dict(C=C, Cp=Cp, rows=rows, kernel="register-cached" if C <= 1280 and Cp <= 1280 else "streaming",
                us_per_call=med * 1e3, spread_us=spread * 1e3, runs_us=[x * 1e3 for x in ms], bytes=nbytes,
                share_of_hbm=nbytes / (med * 1e-3) / HBM_BYTES_PER_S)


def time_step(codebook, steps, runs):
    import open_musiclm_b200 as O
    torch.manual_seed(0)
    m = O.create_semantic_transformer(dim=1024, depth=6, heads=8, semantic_codebook_size=codebook, attn_dropout=0.0,
                                      ff_dropout=0.1).cuda()
    tr = O.HotPathTrainer(m, cross_entropy_loss_weights=[0.0, 1.0], lr=3e-4, lr_warmup=10, wd=0.01)
    g = torch.Generator().manual_seed(1)
    batch = [torch.randint(0, 1024, (16, 12), generator=g).cuda(), torch.randint(0, codebook, (16, 499), generator=g).cuda()]
    for _ in range(5):                   # eager steps, the capture, replays
        tr.train_step([batch])
    torch.cuda.synchronize()
    assert tr._graphs, "the step was not captured"
    ms = []
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(runs):
        a.record()
        for _ in range(steps):
            tr.train_step([batch])
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b) / steps)
    loss = float(tr.train_step([batch]))
    med, spread = stat(ms)
    del tr, m
    torch.cuda.empty_cache()
    return dict(codebook=codebook, C=codebook + 1, ms_per_step=med, spread_ms=spread, runs_ms=ms, last_loss=loss)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--classes", default="1025,1281,2049,4097,16385")
    ap.add_argument("--rows", type=int, default=8000)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--codebooks", default="1024,2048,4096")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_cross_entropy: needs a CUDA device (nothing is measured without one)")
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    ce = [time_ce(int(c), args.rows, args.reps, args.runs) for c in args.classes.split(",")]
    for r in ce:
        print(json.dumps(r), flush=True)
    step = [time_step(int(c), args.steps, args.runs) for c in args.codebooks.split(",")] if args.steps > 0 else []
    for r in step:
        print(json.dumps(r), flush=True)
    print()
    print(f"{info}; cross-entropy call (loss + dlogits), {args.rows} rows, median of {args.runs} runs of {args.reps} launches (spread)")
    print(f"{'C':>6} {'Cp':>6} {'kernel':>16} {'us':>16} {'MB moved':>9} {'of 3.35 TB/s':>12}")
    for r in ce:
        print(f"{r['C']:>6} {r['Cp']:>6} {r['kernel']:>16} {r['us_per_call']:>8.1f} ({r['spread_us']:.1f}) {r['bytes'] / 1e6:>9.1f} "
              f"{100 * r['share_of_hbm']:>11.1f}%")
    if step:
        print(f"\nmusiclm_small semantic stage, B = 16, graph-replayed train_step, median of {args.runs} runs of {args.steps} steps (spread)")
        for r in step:
            print(f"codebook {r['codebook']:>5} (C = {r['C']:>5}): {r['ms_per_step']:8.2f} ms ({r['spread_ms']:.2f})")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_cross_entropy.json"), "w") as f:
            json.dump(dict(card=info, cross_entropy=ce, train_step=step), f, indent=1)


if __name__ == "__main__":
    main()
