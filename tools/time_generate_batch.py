"""Decode-step time against the batch size: the musiclm_small coarse stage (d = 1024, L = 6, h = 8) at a context of about
1000 positions, one incremental step (all layers + logit head) replayed from a CUDA graph and timed with CUDA events.

Per batch size: ms per step, tokens/s (B tokens per step), the bytes one step must move (16-bit weights + the K/V cache
rows, from shapes) and the achieved GB/s against the H100 SXM data-sheet 3.35 TB/s.  Also times skinny_gemm against
decode_gemm alone at B = 8 and 16 on the FFN shapes (w1, w2), for the placement of the 16-row cutover.  Three runs of
everything; the table gives the median and the spread (max - min).

    python tools/time_generate_batch.py [--batches 1,8,16,...] [--context 1000] [--out DIR] [--profile 64,256]

--profile: for those batch sizes also the device time per step of each kernel (torch.profiler over eager steps, in a
pass of its own after the timed ones).
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35      # H100 SXM data sheet, not measured


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else f"{torch.cuda.get_device_name()} (nvidia-smi unavailable)"


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
    ap.add_argument("--batches", default="1,8,16,17,32,64,128,256")
    ap.add_argument("--context", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default="", help="comma-separated batch sizes whose step is broken down by kernel")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_generate_batch: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    from open_musiclm_b200 import lib
    from open_musiclm_b200.decode import DecodeSession
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    eng = m.engine
    d, HD, Fp, L = eng.d, eng.HD, eng.Fp, eng.L
    S = len(eng.seqs) - 1
    w_bytes = 2 * (L * (HD * d + 128 * d + d * HD + 2 * Fp * d + d * Fp) + eng.Cp[S] * d)
    n = args.context
    rows = []
    for B in [int(b) for b in args.batches.split(",")]:
        sess = DecodeSession(eng, B, n, 8)
        g = torch.Generator(device="cuda").manual_seed(B)
        for c in sess.cache:
            c.copy_(torch.randn(c.shape, device="cuda", generator=g) * 0.3)
        for c in sess.conv:
            c.zero_()
        sess.pos.fill_(n)                    # every replay processes position n: keys 0..n
        ms = time_graph(lambda: sess.step_ops(0), args.reps)
        med, spread = stat(ms)
        kv_bytes = L * B * (n + 1) * 128 * 2
        byts = w_bytes + kv_bytes
        r = dict(B=B, ms_per_step=med, spread_ms=spread, runs_ms=ms, tokens_per_s=B / med * 1e3, bytes_per_step=byts,
                 weight_bytes=w_bytes, kv_bytes=kv_bytes, gb_per_s=byts / med / 1e6, share_of_3_35_tbs=byts / med / 1e6 / (HBM_TBS * 1e3),
                 path="tensor-core" if sess.batched else "simt")
        rows.append(r)
        print(json.dumps(r), flush=True)
        del sess
        torch.cuda.empty_cache()
    # the two FFN GEMMs alone at the cutover batch sizes
    gemms = []
    for B in (8, 16):
        for name, (N, K, prologue) in dict(w1=(2 * Fp, d, 2), w2=(d, Fp, 3)).items():
            W = eng.pk[0][name]
            gen = torch.Generator(device="cuda").manual_seed(N + B)
            A = torch.randn(B, K, device="cuda", generator=gen) if prologue == 2 else torch.randn(B, K, device="cuda", generator=gen).to(W.dtype)
            gamma = torch.ones(K, device="cuda")
            rowsum = torch.ones(B, K // 128, 2, device="cuda") if prologue == 3 else None
            out = torch.empty(B, N, device="cuda", dtype=W.dtype)
            ws = lib.DecodeWorkspace("cuda", B, [(N, K)])
            kw = dict(prologue=prologue, gamma=gamma, rowsum=rowsum, n_real=K - 64 if prologue == 3 else 0)
            res = {}
            for kern in ("skinny_gemm", "decode_gemm"):
                f = (lambda: [lib.skinny_gemm(A, W, out, **kw) for _ in range(20)]) if kern == "skinny_gemm" else \
                    (lambda: [lib.decode_gemm(A, W, out, ws=ws, **kw) for _ in range(20)])
                med, spread = stat([t / 20 for t in time_graph(f, max(args.reps // 4, 10))])
                res[kern] = dict(us=med * 1e3, spread_us=spread * 1e3, gb_per_s=N * K * 2 / med / 1e6)
            gemms.append(dict(B=B, matrix=name, N=N, K=K, **res))
            print(json.dumps(gemms[-1]), flush=True)
    print()
    print(f"{info}; musiclm_small coarse stage, context {n}, one decode step from a CUDA graph, median of 3 runs (spread)")
    print(f"{'B':>4} {'path':>11} {'ms/step':>16} {'tokens/s':>10} {'MB/step':>8} {'GB/s':>7} {'of 3.35 TB/s':>12}")
    for r in rows:
        print(f"{r['B']:>4} {r['path']:>11} {r['ms_per_step']:>8.4f} ({r['spread_ms']:.4f}) {r['tokens_per_s']:>10.0f} "
              f"{r['bytes_per_step'] / 1e6:>8.1f} {r['gb_per_s']:>7.0f} {100 * r['share_of_3_35_tbs']:>11.1f}%")
    for gm in gemms:
        print(f"B={gm['B']:>2} {gm['matrix']} [{gm['N']}x{gm['K']}]: skinny_gemm {gm['skinny_gemm']['us']:.1f} us "
              f"({gm['skinny_gemm']['spread_us']:.1f}), decode_gemm {gm['decode_gemm']['us']:.1f} us ({gm['decode_gemm']['spread_us']:.1f})")
    for B in [int(b) for b in args.profile.split(",") if b]:
        sess = DecodeSession(eng, B, n, 8)
        for c in sess.cache + sess.conv:
            c.zero_()
        sess.pos.fill_(n)
        sess.step_ops(0)
        torch.cuda.synchronize()
        steps = 5
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                sess.step_ops(0)
            torch.cuda.synchronize()
        per = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                k = e.name.split("(")[0].replace("void ", "").replace("omlm::", "")
                t = per.setdefault(k, [0.0, 0])
                t[0] += e.device_time_total
                t[1] += 1
        print(f"B={B}: device time per step by kernel (eager, {steps} steps)")
        for k, (us, cnt) in sorted(per.items(), key=lambda kv: -kv[1][0]):
            print(f"  {k:<50} {us / steps:9.1f} us  ({cnt // steps} launches)")
        del sess
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_generate_batch.json"), "w") as f:
            json.dump(dict(card=info, context=n, steps=rows, gemms=gemms), f, indent=1)


if __name__ == "__main__":
    main()
