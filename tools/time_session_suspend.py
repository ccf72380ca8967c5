"""Suspend and resume in a generation session on the musiclm_small coarse stage (d = 1024, L = 6, h = 8, 1024-entry
codebooks), 64 slots: what moving a row's decode state out of its slot and back costs.

Each case is a session of 64 slots with 47 rows of 12 clap + 500 semantic tokens decoding (top_p 0.9) and k target
rows (k = 1 at about 100, 500 and 1400 positions; k = 16 at about 500), after warm-up and graph capture.  Per run:
1. a steady time step (`sess.step(1)`);
2. `suspend` of the k target rows: the snapshot copies (host clock around the calls, ending in a synchronise);
3. a time step without them, then `resume` of the k rows and the time step in which they are restored into their
   (new) slots; the restore cost is that step minus the steady one.
Host clock around work that ends in a device synchronise, median (max - min) of --runs.  The snapshot's size is
L x pos x 256 B of K/V (one 128-wide bf16 row per layer and position) plus L x 2 x 2Fp x 2 B of conv history and the
row's tokens.  The target rows then run to their end and are checked bit for bit against generate alone.  The card
(name, power limit, max SM clock) is read in the same run.

    python tools/time_session_suspend.py [--runs 5] [--out DIR]
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
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_session_suspend: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    g = torch.Generator().manual_seed(1)
    res = {"card": info}
    R, bg = args.runs, 47
    T_target = 3 * R + 6                                        # time steps of a target row: it runs through every run
    clap = torch.randint(0, 1024, (bg + 16, 12), generator=g).cuda()
    sem_bg = torch.randint(0, 1024, (bg, 500), generator=g).cuda()

    for k, sem_len in ((1, 80), (1, 480), (1, 1340), (16, 480)):
        sess = O.GenerationSession(w, slots=64, max_positions=1500, max_queue=0)
        for b in range(bg):
            sess.add(conditioning_token_ids=[clap[b:b + 1], sem_bg[b:b + 1]], seed=b, max_time_steps=300, top_p=0.9)
        sem = torch.randint(0, 1024, (k, sem_len), generator=g).cuda()
        reqs = [dict(conditioning_token_ids=[clap[bg + i:bg + i + 1], sem[i:i + 1]], seed=1000 + i, max_time_steps=T_target, top_p=0.9)
                for i in range(k)]
        hs = [sess.add(**r) for r in reqs]
        sess.step(3)                                            # joins, warm-up and graph capture
        steady, susp, restore, pos = [], [], [], []
        for _ in range(R):
            steady.append(wall(lambda: sess.step(1)))
            rows = [sess.sched.live[h] for h in hs]
            pos.append(sum(r.P - 1 + r.t for r in rows) / k)
            susp.append(wall(lambda: [sess.suspend(h) for h in hs]))
            sess.step(1)
            for h in hs:
                sess.resume(h)
            restore.append(wall(lambda: sess.step(1)))
        out = {}
        while not all(h in out for h in hs):
            sess.step(1)
            out.update(sess.finished())
        for h, r in zip(hs, reqs):                              # bit for bit the row alone
            r = dict(r)
            seed = r.pop("seed")
            assert torch.equal(out[h], w.generate(seeds=[seed], **r)[0]), h
        eng = m.engine
        p = sum(pos) / len(pos)
        nbytes = k * (eng.L * p * 128 * 2 + eng.L * 2 * 2 * eng.Fp * 2)
        key = f"k{k}_pos{round(p)}"
        cost = [a - b for a, b in zip(restore, steady)]
        res[key] = dict(rows=k, mean_pos=p, snapshot_MB=nbytes / 1e6, steady_step_ms=stat(steady), suspend_ms=stat(susp),
                        restore_step_ms=stat(restore), restore_minus_steady_ms=stat(cost), graphs=sess.graph_count,
                        raw=dict(steady=steady, suspend=susp, restore=restore))
        print(f"{k} row(s) at ~{p:.0f} positions ({nbytes / 1e6:.2f} MB of snapshot): suspend {stat(susp)} ms; "
              f"steady time step {stat(steady)} ms; time step with the restore {stat(restore)} ms "
              f"(difference {stat(cost)} ms); {sess.graph_count} graphs", flush=True)
        del sess
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_session_suspend.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
