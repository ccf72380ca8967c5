"""Generation sessions (continuous batching) on the musiclm_small coarse stage (d = 1024, L = 6, h = 8, 1024-entry
codebooks): what a session costs per step and per join, and what it gains on a stream of requests.

1. Steady state: B slots (B in {40, 256}; B - 1 rows decoding, every slot computed) with prompts of 12 clap + 960 semantic tokens (977 positions, so the context
   runs from about 980 to 1040), all in their slots; ms per decode step of `sess.step(K)` (host clock around K time
   steps of 3 decode steps, ending in a synchronise) against generate's seeded step at the same B, the difference of
   two generate calls that differ by K time steps over 3K.  Variants alternated, median of --runs (spread).
2. One join: a time step with one row joining (prefill alone + install) minus a steady time step, against generate
   for that prompt alone with one time step (prefill, its decode-session set-up and 2 eager steps).
3. A request stream: 256 requests (12 clap + 100 semantic tokens, max_time_steps uniform in 50 ... 400, top_p 0.9,
   seeds 0 ... 255) through a 64-slot session (all queued at once, stepped until idle) against static batches: 4
   generate calls of 64 rows with per-row max_time_steps, each running until its longest row.  Total time, generated
   tokens per second and the session's mean occupancy.
The card (name, power limit, max SM clock) is read in the same run.

    python tools/time_generate_session.py [--runs 3] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_generate_batch import card, stat  # noqa: E402


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=12, help="K, time steps per steady-state sample")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_generate_session: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    g = torch.Generator().manual_seed(1)
    K, res = args.steps, {"card": info}

    # ---- 1. steady state and 2. one join
    for B in (40, 256):
        clap = torch.randint(0, 1024, (B, 12), generator=g).cuda()
        sem = torch.randint(0, 1024, (B, 960), generator=g).cuda()
        seeds = list(range(B))
        T = 2 + args.runs * (K + 2) + 2
        sess = O.GenerationSession(w, slots=B, max_positions=977 + 3 * T, max_queue=1)
        for b in range(B - 1):                             # one slot stays free for the joins below
            sess.add(conditioning_token_ids=[clap[b:b + 1], sem[b:b + 1]], seed=b, max_time_steps=T, top_p=0.9)
        sess.step(2)                                       # joins, warm-up and graph capture
        gen = lambda t: w.generate(conditioning_token_ids=[clap, sem], seeds=seeds, max_time_steps=t, top_p=0.9)
        gen(2)
        ms = {"session": [], "generate": []}
        for _ in range(args.runs):
            ms["session"].append(wall(lambda: sess.step(K)) / (3 * K))
            ms["generate"].append((wall(lambda: gen(2 + K)) - wall(lambda: gen(2))) / (3 * K))
        # one join: a row of one time step takes the free slot (and leaves it at the end of that step)
        join, steady, alone = [], [], []
        for r in range(args.runs):
            steady.append(wall(lambda: sess.step(1)))
            row = dict(conditioning_token_ids=[clap[B - 1:B], sem[B - 1:B]], seed=10 ** 6 + r, max_time_steps=1, top_p=0.9)
            sess.add(**row)
            join.append(wall(lambda: sess.step(1)))
            alone.append(wall(lambda: w.generate(seeds=[row["seed"]], conditioning_token_ids=row["conditioning_token_ids"],
                                                 max_time_steps=1, top_p=0.9)))
        res[f"steady_B{B}"] = {v: (*stat(x), x) for v, x in ms.items()}
        res[f"join_B{B}"] = dict(join_step=stat(join), steady_step=stat(steady), generate_alone_one_step=stat(alone),
                                 graphs=sess.graph_count)
        print(f"B = {B}, context ~1000: ms per decode step, session {stat(ms['session'])}, generate {stat(ms['generate'])}; "
              f"time step with one join {stat(join)} ms, steady time step {stat(steady)} ms, generate alone with one time step "
              f"{stat(alone)} ms; {sess.graph_count} graphs", flush=True)
        del sess

    # ---- 3. a request stream
    N, slots = 256, 64
    clap = torch.randint(0, 1024, (N, 12), generator=g).cuda()
    sem = torch.randint(0, 1024, (N, 100), generator=g).cuda()
    steps = [int(v) for v in torch.randint(50, 401, (N,), generator=g)]
    tokens = 3 * sum(steps)

    def session_run():
        sess = O.GenerationSession(w, slots=slots, max_positions=117 + 3 * 400, max_queue=N)
        for i in range(N):
            sess.add(conditioning_token_ids=[clap[i:i + 1], sem[i:i + 1]], seed=i, max_time_steps=steps[i], top_p=0.9)
        n_steps = 0
        while not sess.idle:
            sess.step(1)
            n_steps += 1
        out = sess.finished()
        assert len(out) == N
        return n_steps, out

    def static_run():
        out = []
        for c in range(0, N, slots):
            out.append(w.generate(conditioning_token_ids=[clap[c:c + slots], sem[c:c + slots]], seeds=list(range(c, c + slots)),
                                  max_time_steps=steps[c:c + slots], top_p=0.9))
        return out

    session_run()
    static_run()
    t_sess, t_static = [], []
    for _ in range(max(2, args.runs - 1)):
        box = {}
        t_sess.append(wall(lambda: box.update(s=session_run())))
        t_static.append(wall(lambda: box.update(t=static_run())))
    n_steps, out = box["s"]
    static = box["t"]
    for i in range(N):           # the two schedules give the same tokens (every row is its generate row alone)
        c = i // slots * slots
        assert torch.equal(out[i], static[i // slots][i - c, :steps[i]]), i
    occupancy = sum(steps) / (n_steps * slots)
    res["stream"] = dict(session_ms=stat(t_sess), static_ms=stat(t_static), tokens=tokens, session_time_steps=n_steps,
                         occupancy=occupancy, session_tok_s=tokens / (stat(t_sess)[0] / 1e3), static_tok_s=tokens / (stat(t_static)[0] / 1e3))
    print(f"stream of {N} requests, max_time_steps 50 ... 400, {slots} slots: session {stat(t_sess)} ms "
          f"({res['stream']['session_tok_s']:.0f} tokens/s, {n_steps} time steps, occupancy {occupancy:.3f}); static batches "
          f"{stat(t_static)} ms ({res['stream']['static_tok_s']:.0f} tokens/s)", flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_generate_session.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
