"""Chunked prefill in a generation session on the musiclm_small coarse stage (d = 1024, L = 6, h = 8, 1024-entry
codebooks): how long the running rows stall while a mass join prefills, and what the budget costs a request stream.

1. Stall: B slots (64, 256), B - k running rows (12 clap + 500 semantic tokens), then k requests of 12 clap + 960
   semantic tokens join at once (k = 16 at 64 slots, 16 and 64 at 256).  Every time step from that boundary until the
   last joiner has finished prefilling is timed (host clock around a synchronised `step(1)`); reported: the longest
   of them, their number, and a steady time step before the join.  For prefill_rows None, 8192, 4096, 2048, 1024.
   Median (min ... max spread) over --runs joins.
2. Stream: 256 requests (12 clap + 50 ... 960 semantic tokens, max_time_steps uniform in 50 ... 400, top_p 0.9, seeds
   0 ... 255, all queued at once) through a 64-slot session per budget: total ms and tokens/s; every budget's tokens
   equal the unbudgeted session's.
3. --parent-lib PATH (a build of the library without chunks): omlm_attn_fwd_tc_varlen and omlm_gemm_ffn_up_varlen at
   p0 = 0 on equal-length packings, alternated between this build and PATH in one process (CUDA events, 50 launches).
The card (name, power limit, max SM clock) is read in the same run.

    python tools/time_session_chunked.py [--runs 3] [--parent-lib PATH] [--only-kernels]
"""
import argparse
import ctypes
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_generate_batch import card, stat  # noqa: E402

BUDGETS = (None, 8192, 4096, 2048, 1024)


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def events(fn, n=50):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n * 1e3          # us per launch


def kernels(lib, parent_path, runs):
    """Item 3: the p0 = 0 varlen kernels of this build against the parent build, alternated."""
    from open_musiclm_b200.session import lpt_work
    mine = lib.load()
    parent = ctypes.CDLL(parent_path)
    parent.omlm_last_error.restype = ctypes.c_char_p
    h, d = 8, 1024
    Fp = (int(d * 2 * 4 / 3) + 127) // 128 * 128
    for B, N in ((8, 1024), (16, 500), (64, 128)):
        M = B * N
        qn = torch.nn.functional.normalize(torch.randn(M, h, 64, device="cuda"), dim=-1).reshape(M, h * 64).bfloat16()
        kvn = torch.randn(M, 128, device="cuda").bfloat16()
        table = 0.1 * torch.randn(h, N, device="cuda")
        out, lse = torch.empty(M, h * 64, device="cuda", dtype=torch.bfloat16), torch.empty(M * h, device="cuda")
        i32 = lambda v: torch.tensor(v, device="cuda", dtype=torch.int32)
        start, lens, work = i32([b * N for b in range(B)]), i32([N] * B), torch.from_numpy(lpt_work([N] * B, h)).cuda().contiguous()
        xn = torch.randn(M, d, device="cuda").half()
        w1 = (torch.randn(2 * Fp, d, device="cuda") / 32).half()
        conv = torch.randn(2 * Fp, 3, device="cuda")
        u, hh, rs = torch.empty(M, 2 * Fp, device="cuda").half(), torch.empty(M, Fp, device="cuda").half(), torch.empty(M, Fp // 128, 2, device="cuda")
        row_pos = torch.arange(N, device="cuda", dtype=torch.int32).repeat(B)
        results = {}
        for which, handle in (("this", mine), ("parent", parent)):
            lib._lib = handle
            lib.attn_fwd_tc_varlen(qn, kvn, table, work, start, lens, N, out, lse, h)
            lib.gemm_ffn_up_varlen(xn, w1, conv, u, hh, rs, row_pos, Fp)
            torch.cuda.synchronize()
            results[which] = (out.clone(), lse.clone(), u.clone(), hh.clone(), rs.clone())
        same = all(torch.equal(a, b) for a, b in zip(results["this"], results["parent"]))
        fns = {}
        for which, handle in (("this", mine), ("parent", parent)):
            def attn(handle=handle):
                lib._lib = handle
                lib.attn_fwd_tc_varlen(qn, kvn, table, work, start, lens, N, out, lse, h)

            def ffn(handle=handle):
                lib._lib = handle
                lib.gemm_ffn_up_varlen(xn, w1, conv, u, hh, rs, row_pos, Fp)
            fns[f"attn_varlen[{which}]"] = attn
            fns[f"ffn_up_varlen[{which}]"] = ffn
        t = {k: [] for k in fns}
        for _ in range(runs):
            for k, fn in fns.items():
                t[k].append(events(fn))
        lib._lib = mine
        print(f"kernels B = {B}, N = {N}, h = {h} (outputs equal to the parent's: {same}): " +
              ", ".join(f"{k} {stat(v)} us" for k, v in t.items()), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--only-kernels", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_session_chunked: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    from open_musiclm_b200 import lib
    print("card (name, power limit, max SM clock):", card(), flush=True)
    if args.parent_lib:
        kernels(lib, args.parent_lib, max(args.runs, 3))
    if args.only_kernels:
        return
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    g = torch.Generator().manual_seed(1)
    req = lambda n_sem, seed, T: dict(conditioning_token_ids=[torch.randint(0, 1024, (1, 12), generator=g).cuda(),
                                                              torch.randint(0, 1024, (1, n_sem), generator=g).cuda()],
                                      seed=seed, max_time_steps=T, top_p=0.9)

    # ---- 1. stalls
    for B, ks in ((64, (16,)), (256, (16, 64))):
        for rows in BUDGETS:
            T_run = 400
            sess = O.GenerationSession(w, slots=B, max_positions=14 + 962 + 3 * T_run, max_queue=64, prefill_rows=rows)
            for b in range(B - max(ks)):
                sess.add(**req(500, b, T_run))
            sess.step(2)
            for _ in range(max(ks)):                       # warm the join path and the workspace
                sess.add(**req(960, 10 ** 6, 1))
            while sess.sched.prefilling or sess.sched.queue:
                sess.step(1)
            sess.step(2)
            for k in ks:
                worst, n_steps, steady = [], [], []
                for r in range(args.runs):
                    steady.append(wall(lambda: sess.step(1)))
                    for i in range(k):
                        sess.add(**req(960, 10 ** 7 + 100 * r + i, 1))
                    ts = [wall(lambda: sess.step(1))]
                    while sess.sched.prefilling or sess.sched.queue:
                        ts.append(wall(lambda: sess.step(1)))
                    worst.append(max(ts))
                    n_steps.append(len(ts))
                    sess.step(1)                           # the joiners leave
                print(f"B = {B}, k = {k} joiners of 972 tokens, prefill_rows = {rows}: longest time step {stat(worst)} ms over "
                      f"{stat(n_steps)[0]} time steps of prefill; steady time step {stat(steady)} ms; packed workspace "
                      f"{sess._pack_rows} rows", flush=True)
            del sess
            torch.cuda.empty_cache()

    # ---- 2. a request stream
    Nr, slots = 256, 64
    sem_len = [int(v) for v in torch.randint(50, 961, (Nr,), generator=g)]
    steps = [int(v) for v in torch.randint(50, 401, (Nr,), generator=g)]
    clap = torch.randint(0, 1024, (Nr, 12), generator=g).cuda()
    sem = [torch.randint(0, 1024, (1, n), generator=g).cuda() for n in sem_len]
    tokens = 3 * sum(steps)

    def session_run(rows):
        sess = O.GenerationSession(w, slots=slots, max_positions=14 + 962 + 3 * 400, max_queue=Nr, prefill_rows=rows)
        for i in range(Nr):
            sess.add(conditioning_token_ids=[clap[i:i + 1], sem[i]], seed=i, max_time_steps=steps[i], top_p=0.9)
        while not sess.idle:
            sess.step(1)
        out = sess.finished()
        assert len(out) == Nr
        return out

    ref = session_run(None)
    for rows in BUDGETS[1:]:
        out = session_run(rows)
        assert all(torch.equal(ref[h], out[h]) for h in ref), rows
    t = {rows: [] for rows in BUDGETS}
    for _ in range(args.runs):
        for rows in BUDGETS:
            t[rows].append(wall(lambda: session_run(rows)))
    print(f"stream of {Nr} requests, {slots} slots, semantic 50 ... 960, 50 ... 400 time steps ({tokens} tokens; every budget's "
          "tokens equal the unbudgeted session's): " +
          ", ".join(f"prefill_rows {k}: {stat(v)} ms ({tokens / (sorted(v)[len(v) // 2] / 1e3) / 1e3:.1f}k tokens/s)" for k, v in t.items()),
          flush=True)


if __name__ == "__main__":
    main()
