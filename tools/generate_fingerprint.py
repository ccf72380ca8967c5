"""Fingerprint of KV-cache generation: a fixed seeded matrix of generate calls, a GenerationSession stream and one seeded
MusicLM.generate_tokens on small random-init models, with every output saved, so that two versions of the package can
be compared bit for bit on one GPU.  The script uses only the public API, so it runs unchanged against any tree.

Matrix: stages coarse (q = 3), semantic (q = 1) and a coarse stage with absolute position embeddings; B in {1, 5, 16,
17, 40}; noise from the Engine.seed Philox stream, uniform_noise or seeds; top_p None or 0.9.  Each case also takes
one prefix kind in turn (none, a full prefix, ragged pred_lengths, the prefix flattened to [B, n] at q > 1), per-row
temperature, top_p and max_time_steps on every third case, and one flag in turn (return_logprobs, trace_logits,
use_cuda_graph=False, allow_eos_in_output, include_eos_in_output).  A few cases raise on purpose (absolute-position
limit, bad pred_lengths).  Saved per case: every output tensor, Engine.seed after the case, the exception type, the
number of synchronising calls torch.cuda.set_sync_debug_mode("warn") reports in the first call, and with --times the
wall time of the fastest of three further calls (host clock ending in a device synchronise).

    python tools/generate_fingerprint.py --root TREE --out FILE [--times]
    python tools/generate_fingerprint.py --compare PARENT.pt BRANCH.pt [PARENT2.pt BRANCH2.pt ...]

--compare checks the first pair for equal tensors (torch.equal), Engine.seed values, graph counts and exception types,
and sync counts no higher in the branch, then prints each case's fastest time per file.
"""
import argparse
import os
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def models(O, torch):
    torch.manual_seed(0)
    kw = dict(dim=128, depth=2, heads=2, clap_codebook_size=64, num_clap_quantizers=4, attn_dropout=0.0, ff_dropout=0.0)
    out = {}
    for name, extra in (("coarse", {}), ("abspos", dict(use_absolute_position_embeddings=True, max_absolute_position_embeddings=80))):
        m = O.create_coarse_transformer(semantic_codebook_size=64, acoustic_codebook_size=64, num_coarse_quantizers=3, **kw, **extra)
        out[name] = O.TokenConditionedTransformerWrapper(transformer=m.cuda().eval(), unique_consecutive=False)
    m = O.create_semantic_transformer(semantic_codebook_size=64, **kw)
    out["semantic"] = O.TokenConditionedTransformerWrapper(transformer=m.cuda().eval(), unique_consecutive=False)
    return out


PREFIXES = ("none", "full", "ragged", "flat")
FLAGS = ({}, dict(return_logprobs=True), dict(trace_logits=True), dict(use_cuda_graph=False), dict(allow_eos_in_output=True),
         dict(include_eos_in_output=True))


def generate_cases(torch):
    """(name, stage, kwargs builder) of the generate matrix; the builder returns generate's keyword arguments."""
    cases, i = [], 0
    for stage in ("coarse", "semantic", "abspos"):
        for B in (1, 5, 16, 17, 40):
            for noise in ("philox", "uniform", "seeds"):
                for top_p in (None, 0.9):
                    i += 1
                    prefix = PREFIXES[i % 4]
                    if prefix == "flat" and stage == "semantic":
                        prefix = "full"
                    cases.append((f"{stage}-B{B}-{noise}-p{top_p}-{prefix}-{i}", stage,
                                  dict(B=B, noise=noise, top_p=top_p, prefix=prefix, per_row=i % 3 == 0, flags=FLAGS[i % len(FLAGS)], i=i)))
    cases.append(("abspos-limit", "abspos", dict(B=5, noise="philox", top_p=None, prefix="ragged", per_row=False, flags={}, i=0, T=40)))
    cases.append(("abspos-limit-uniform", "abspos", dict(B=5, noise="philox", top_p=None, prefix="full", per_row=False, flags={}, i=0, T=40)))
    cases.append(("bad-pred-lengths", "coarse", dict(B=5, noise="philox", top_p=None, prefix="ragged", per_row=False, flags={}, i=0,
                                                     lengths=[1, 2])))
    return cases


def generate_args(w, torch, c):
    info, eos = w.token_sequences[-1], w.eos_ids[-1]
    q, C = info.num_quantizers, info.codebook_size + 1
    B, i = c["B"], c["i"]
    g = torch.Generator().manual_seed(1000 + i)
    cond = [torch.randint(0, 64, (B, 4 * 3), generator=g).cuda(), torch.randint(0, 64, (B, 9), generator=g).cuda()]
    if len(w.token_sequences) == 2:
        cond = cond[:1]
    T = c.get("T", 8)
    kw = dict(conditioning_token_ids=cond, max_time_steps=T, **c["flags"])
    lengths = [T // 2] * B
    if c["prefix"] != "none":
        pre = torch.randint(0, 64, (B, T // 2, q), generator=g)
        if c["flags"].get("allow_eos_in_output") or c["flags"].get("include_eos_in_output"):
            pre[0, 1, q - 1] = eos
        # flat: the first 6 tokens as [B, 6]; generate counts its 6 columns as time steps
        kw["pred_token_ids"] = pre.cuda().reshape(B, -1)[:, :6] if c["prefix"] == "flat" else pre.cuda()
        if c["prefix"] == "ragged":
            lengths = c.get("lengths", [(b * 3) % (T // 2 + 1) for b in range(B)])
            kw["pred_lengths"] = lengths
    else:
        lengths = [0] * B
    steps = [T] * B
    if c["per_row"]:
        kw["temperature"] = [0.5 + b / max(B, 2) for b in range(B)]
        if c["top_p"] is not None:
            kw["top_p"] = [c["top_p"] if b % 2 else None for b in range(B)]
        if c["prefix"] != "flat":
            steps = [T - (b % 3) for b in range(B)]
            kw["max_time_steps"] = steps
    elif c["top_p"] is not None:
        kw["top_p"] = c["top_p"]
    if c["noise"] == "seeds":
        kw["seeds"] = [(b * 7919 + i) * 2654435761 for b in range(B)]
    elif c["noise"] == "uniform":
        flat = c["prefix"] == "flat"
        n_new = max(max(0, (t - (6 if flat else n)) * q) for t, n in zip(steps, lengths))
        kw["uniform_noise"] = torch.rand(max(n_new, 1), B, C, generator=g).clamp(1e-6, 1 - 1e-6)[:n_new].cuda()
    return kw


def run(fn, torch, times):
    """fn() once under the sync debug mode (outputs, exception type, syncs), then (times) three timed calls."""
    rec = dict(exc=None, syncs=0, tensors={}, ms=None)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            rec["tensors"] = fn()
        except Exception as e:           # a case that raises on purpose: its type is the fingerprint
            rec["exc"] = type(e).__name__
            print(f"  raised {type(e).__name__}: {e}", flush=True)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    rec["syncs"] = sum(1 for w in caught if "synchroniz" in str(w.message))
    torch.cuda.synchronize()
    if times and rec["exc"] is None:
        best = []
        for _ in range(3):
            torch.cuda.synchronize()
            t = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            best.append((time.perf_counter() - t) * 1e3)
        rec["ms"] = min(best)
    rec["tensors"] = {k: v.detach().cpu() for k, v in rec["tensors"].items()}
    return rec


def fingerprint(out_path, times):
    import torch
    import open_musiclm_b200 as O
    torch.cuda.set_device(0)
    ws = models(O, torch)
    res = {}
    for name, stage, c in generate_cases(torch):
        w = ws[stage]
        kw = generate_args(w, torch, c)

        def call(w=w, kw=kw):
            trace = [] if kw.get("trace_logits") else None
            out = w.generate(**dict(kw, trace_logits=trace))
            out = out if isinstance(out, tuple) else (out,)
            t = {f"out{j}": o for j, o in enumerate(out)}
            if trace:
                t["trace"] = torch.stack(trace)
            return t
        rec = run(call, torch, times)
        rec["seed"] = int(w.transformer.engine.seed.item())
        res[name] = rec
        print(name, rec["exc"], rec["syncs"], rec["ms"], flush=True)
    # a GenerationSession stream: joins at different steps, log-probabilities, and a traced variant
    for traced in (False, True):
        def session(traced=traced):
            w = ws["coarse"]
            s = O.GenerationSession(w, slots=4, max_positions=120, max_queue=8, return_logprobs=not traced, trace_logits=traced)
            g = torch.Generator().manual_seed(7)
            handles, out = [], {}
            for step in range(14):
                if step in (0, 2, 5, 6, 9):
                    for r in range(1 + step % 3):
                        pre = torch.randint(0, 64, (1, r, 3), generator=g).cuda() if r else None
                        handles.append(s.add(conditioning_token_ids=[torch.randint(0, 64, (1, 12), generator=g).cuda(),
                                                                     torch.randint(0, 64, (1, 9), generator=g).cuda()],
                                             pred_token_ids=pre, seed=100 * step + r, max_time_steps=3 + (step + r) % 5,
                                             temperature=0.7 + 0.1 * r, top_p=0.9 if r % 2 else None))
                s.step(1)
                for h, v in s.finished().items():
                    for j, t in enumerate(v if isinstance(v, tuple) else (v,)):
                        out[f"h{h}-{j}"] = t
                    if traced:
                        out[f"h{h}-trace"] = s.traced_logits(h)
            while not s.idle:
                s.step(1)
                for h, v in s.finished().items():
                    for j, t in enumerate(v if isinstance(v, tuple) else (v,)):
                        out[f"h{h}-{j}"] = t
                    if traced:
                        out[f"h{h}-trace"] = s.traced_logits(h)
            out["graph_count"] = torch.tensor(s.graph_count)
            return out
        rec = run(session, torch, times)
        rec["seed"] = int(ws["coarse"].transformer.engine.seed.item())
        res[f"session-traced{traced}"] = rec
        print(f"session-traced{traced}", rec["exc"], rec["syncs"], rec["ms"], flush=True)
    # one seeded MusicLM.generate_tokens
    torch.manual_seed(1)
    kw = dict(dim=128, depth=2, heads=2, clap_codebook_size=64, num_clap_quantizers=4, attn_dropout=0.0, ff_dropout=0.0)
    mlm = O.MusicLM(semantic_transformer=O.create_semantic_transformer(semantic_codebook_size=64, **kw).cuda().eval(),
                    coarse_transformer=O.create_coarse_transformer(semantic_codebook_size=64, acoustic_codebook_size=64,
                                                                   num_coarse_quantizers=3, **kw).cuda().eval(),
                    fine_transformer=O.create_fine_transformer(acoustic_codebook_size=64, num_coarse_quantizers=3, num_fine_quantizers=2,
                                                               **kw).cuda().eval())
    clap = torch.randint(0, 64, (2, 4), generator=torch.Generator().manual_seed(3)).cuda()

    def musiclm():
        a, s_, c_, f_ = mlm.generate_tokens(clap_token_ids=clap, output_seconds=3, semantic_window_seconds=2, coarse_window_seconds=1,
                                            fine_window_seconds=0.5, semantic_steps_per_second=6, acoustic_steps_per_second=8,
                                            seeds=[11, 12], return_all=True, top_p=0.9)
        return dict(acoustic=a, semantic=s_, coarse=c_, fine=f_)
    res["musiclm"] = run(musiclm, torch, times)
    res["musiclm"]["seed"] = int(mlm.semantic.transformer_wrapper.transformer.engine.seed.item())
    print("musiclm", res["musiclm"]["exc"], res["musiclm"]["syncs"], res["musiclm"]["ms"], flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    torch.save(res, out_path)


def compare(paths):
    import torch
    a, b = torch.load(paths[0]), torch.load(paths[1])
    bad = []
    assert a.keys() == b.keys(), set(a) ^ set(b)
    for k in a:
        x, y = a[k], b[k]
        if x["exc"] != y["exc"] or x["seed"] != y["seed"] or x["tensors"].keys() != y["tensors"].keys():
            bad.append((k, "exc/seed/keys", x["exc"], y["exc"], x["seed"], y["seed"]))
            continue
        diff = [t for t in x["tensors"] if not torch.equal(x["tensors"][t], y["tensors"][t])]
        if diff:
            bad.append((k, "tensors", diff))
        if y["syncs"] > x["syncs"]:
            bad.append((k, "syncs", x["syncs"], y["syncs"]))
    print(f"{len(a)} cases, {sum(len(v['tensors']) for v in a.values())} tensors; mismatches: {len(bad)}")
    for m in bad:
        print("  MISMATCH", m)
    print("syncs parent -> branch, per case where nonzero:",
          {k: (a[k]["syncs"], b[k]["syncs"]) for k in a if a[k]["syncs"] or b[k]["syncs"]})
    runs = [torch.load(p) for p in paths]
    if all(r[k]["ms"] is not None for r in runs for k in runs[0] if runs[0][k]["exc"] is None):
        print("fastest-of-three ms per case, files in the order given (parent, branch alternating)")
        slower = []
        for k in runs[0]:
            if runs[0][k]["exc"] is not None:
                continue
            v = [r[k]["ms"] for r in runs]
            pa, br = v[0::2], v[1::2]
            flag = "" if min(br) <= max(pa) else "  <- branch above the parent's range"
            if flag:
                slower.append(k)
            print(f"  {k:<40} parent {min(pa):8.2f}-{max(pa):8.2f}  branch {min(br):8.2f}-{max(br):8.2f}{flag}")
        tot = [sum(r[k]["ms"] for k in r if r[k]["ms"] is not None) for r in runs]
        print("total ms per file:", [round(t, 1) for t in tot], "cases above the parent's range:", len(slower))
    return not bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--out")
    ap.add_argument("--times", action="store_true")
    ap.add_argument("--compare", nargs="+")
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(args.compare) else 1)
    sys.path.insert(0, os.path.abspath(args.root))
    fingerprint(args.out, args.times)


if __name__ == "__main__":
    main()
