"""Packed prefill of a generation session's joiners on the musiclm_small coarse stage (d = 1024, L = 6, h = 8,
1024-entry codebooks): what a boundary with k joiners costs, what a request stream gains, and the varlen kernels against
the fixed-length ones.

1. Boundary cost: B slots (64, 256), B - k running rows (12 clap + 500 semantic tokens), k joiners of 12 clap + 50 ...
   960 semantic tokens (one time step each); a time step with those joins minus a steady time step, the packed
   prefill against the one-row-at-a-time install it replaces (each joiner's decode.prefill with its capture into its
   slot), alternated in the same session.  Median (min ... max) of --runs.
2. A request stream: 256 requests (12 clap + 50 ... 960 semantic tokens, max_time_steps uniform in 50 ... 400, top_p
   0.9, seeds 0 ... 255) through a 64-slot session (all queued at once) with the packed and with the one-row install,
   against static batches (4 generate calls of 64 rows, each until its longest row): total ms, tokens/s, mean occupancy.
3. Kernels: attn_fwd_tc_varlen and gemm_ffn_up_varlen on equal-length packings against attn_fwd_tc and gemm_ffn_up at
   the same B x N (CUDA events over 50 launches, alternated).
4. --profile DIR: a torch.profiler trace of one boundary with 16 joiners (packed), its kernel table and totals.
The card (name, power limit, max SM clock) is read in the same run.

    python tools/time_session_prefill.py [--runs 5] [--profile DIR] [--only-kernels]
"""
import argparse
import os
import sys
import time
import types

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


def one_row_install(sess, rows):
    """The install this change replaces: each joiner prefilled alone (decode.prefill) and captured into its slot."""
    from open_musiclm_b200.decode import prefill
    for row in rows:
        a = row.payload
        prefill(sess.w, a["ids"][:-1], a["prefix"], False, sess.dec, slice(row.slot, row.slot + 1),
                torch.full((1,), row.P, device=sess.eng.dev))


def set_install(sess, packed):
    if packed:
        sess.__dict__.pop("_prefill_packed", None)
    else:
        sess._prefill_packed = types.MethodType(one_row_install, sess)


def events(fn, n=50):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n * 1e3          # us per launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--profile", default=None)
    ap.add_argument("--only-kernels", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_session_prefill: needs a CUDA device (nothing is measured without one)")
    import open_musiclm_b200 as O
    from open_musiclm_b200 import lib
    from open_musiclm_b200.session import lpt_work
    print("card (name, power limit, max SM clock):", card(), flush=True)
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    g = torch.Generator().manual_seed(1)
    req = lambda n_sem, seed, T: dict(conditioning_token_ids=[torch.randint(0, 1024, (1, 12), generator=g).cuda(),
                                                              torch.randint(0, 1024, (1, n_sem), generator=g).cuda()],
                                      seed=seed, max_time_steps=T, top_p=0.9)

    # ---- 1. boundary cost
    for B in (() if args.only_kernels else (64, 256)):
        ks = [k for k in (1, 4, 16, 64) if k < B]
        T_run = 2 + len(ks) * 2 * args.runs * 2 + 4
        sess = O.GenerationSession(w, slots=B, max_positions=14 + 962 + 3 * max(T_run, 2), max_queue=64)
        for b in range(B - max(ks)):
            sess.add(**req(500, b, T_run))
        sess.step(2)
        for packed in (True, False):                       # warm both installs and every shape of the eager prefill path
            set_install(sess, packed)
            for _ in range(max(ks)):
                sess.add(**req(int(torch.randint(50, 961, (1,), generator=g)), 10 ** 6, 1))
            sess.step(1)
        for k in ks:
            res = {True: [], False: []}
            for r in range(args.runs):
                for packed in (True, False):
                    set_install(sess, packed)
                    steady = wall(lambda: sess.step(1))
                    for i in range(k):
                        sess.add(**req(int(torch.randint(50, 961, (1,), generator=g)), 10 ** 7 + 100 * r + i, 1))
                    res[packed].append(wall(lambda: sess.step(1)) - steady)
            print(f"B = {B}, k = {k} joiners: boundary cost (join step - steady step) packed {stat(res[True])} ms, "
                  f"one row at a time {stat(res[False])} ms", flush=True)
        set_install(sess, True)
        ws = [t for v in sess._pack_ws.values() for t in (v if isinstance(v, list) else [v])]
        print(f"B = {B}: packed workspace {sess._pack_rows} rows, {sum(t.numel() * t.element_size() for t in ws) / 2 ** 20:.1f} MiB",
              flush=True)
        if args.profile and B == 64:
            os.makedirs(args.profile, exist_ok=True)
            from torch.profiler import ProfilerActivity, profile
            sess.step(1)
            for i in range(16):
                sess.add(**req(int(torch.randint(50, 961, (1,), generator=g)), 10 ** 8 + i, 1))
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                t = wall(lambda: sess.step(1))
            prof.export_chrome_trace(os.path.join(args.profile, "join16_B64.json"))
            table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=40)
            with open(os.path.join(args.profile, "join16_B64.txt"), "w") as f:
                f.write(f"wall {t:.3f} ms (profiled)\n{table}\n")
            kern = sum(e.device_time_total for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA)
            print(f"profile: one join step with 16 joiners at B = 64 (profiled wall {t:.2f} ms), device time {kern / 1e3:.2f} ms",
                  flush=True)
        del sess

    # ---- 3. kernels at equal-length packings
    h, d = 8, 1024
    Fp = (int(d * 2 * 4 / 3) + 127) // 128 * 128            # the conv feed-forward width of d = 1024, padded
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
        fns = dict(attn=lambda: lib.attn_fwd_tc(qn, kvn, table, None, out, lse, B, N, h),
                   attn_varlen=lambda: lib.attn_fwd_tc_varlen(qn, kvn, table, work, start, lens, N, out, lse, h),
                   ffn_up=lambda: lib.gemm_ffn_up(xn, w1, conv, u, hh, rs, N, Fp),
                   ffn_up_varlen=lambda: lib.gemm_ffn_up_varlen(xn, w1, conv, u, hh, rs, row_pos, Fp))
        t = {k: [] for k in fns}
        for _ in range(args.runs):
            for k, fn in fns.items():
                t[k].append(events(fn))
        print(f"kernels B = {B}, N = {N}, h = {h}: " + ", ".join(f"{k} {stat(v)} us" for k, v in t.items()), flush=True)

    if args.only_kernels:
        return
    # ---- 2. a request stream
    Nr, slots = 256, 64
    sem_len = [int(v) for v in torch.randint(50, 961, (Nr,), generator=g)]
    steps = [int(v) for v in torch.randint(50, 401, (Nr,), generator=g)]
    clap = torch.randint(0, 1024, (Nr, 12), generator=g).cuda()
    sem = [torch.randint(0, 1024, (1, n), generator=g).cuda() for n in sem_len]
    tokens = 3 * sum(steps)

    def session_run(packed):
        sess = O.GenerationSession(w, slots=slots, max_positions=14 + 962 + 3 * 400, max_queue=Nr)
        set_install(sess, packed)
        for i in range(Nr):
            sess.add(conditioning_token_ids=[clap[i:i + 1], sem[i]], seed=i, max_time_steps=steps[i], top_p=0.9)
        occ = []
        while not sess.idle:
            sess.step(1)
            occ.append(len(sess.sched.rows))
        out = sess.finished()
        assert len(out) == Nr
        return out, occ

    def static_run():
        for c in range(0, Nr, slots):
            n = max(sem_len[c:c + slots])
            # static batches share a conditioning length: each row's semantic prompt right-aligned would change its
            # tokens, so the batch runs at the longest prompt (the cost a static server pays)
            s = torch.cat([torch.nn.functional.pad(x, (0, n - x.shape[1])) for x in sem[c:c + slots]])
            w.generate(conditioning_token_ids=[clap[c:c + slots], s], seeds=list(range(c, c + slots)),
                       max_time_steps=steps[c:c + slots], top_p=0.9)

    a, _ = session_run(True)
    b, occ = session_run(False)
    assert all(torch.equal(a[h], b[h]) for h in a)
    static_run()
    t = {"packed": [], "one_row": [], "static": []}
    for _ in range(max(2, args.runs - 2)):
        t["packed"].append(wall(lambda: session_run(True)))
        t["one_row"].append(wall(lambda: session_run(False)))
        t["static"].append(wall(static_run))
    occ_mean = sum(occ) / (len(occ) * slots)
    print(f"stream of {Nr} requests, {slots} slots, semantic 50 ... 960, 50 ... 400 time steps ({tokens} tokens): " +
          ", ".join(f"{k} {stat(v)} ms ({tokens / (sorted(v)[len(v) // 2] / 1e3) / 1e3:.1f}k tokens/s)" for k, v in t.items()) +
          f"; session mean occupancy {occ_mean:.3f} over {len(occ)} time steps", flush=True)


if __name__ == "__main__":
    main()
