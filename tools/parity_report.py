#!/usr/bin/env python
"""GPU-side parity report (test tooling): the CUDA path against the fp32 CPU oracle at the BASELINE.json shapes —
logits, loss and every parameter gradient — for each 16-bit operand mode.  Writes parity_report.json (under the temporary directory unless --out is given).

    python tools/parity_report.py [--cases cfg1,cfg2,cfg3,cfg4] [--modes fp16,bf16] [--no-grads cfg4]
"""
import argparse
import json
import os
import tempfile
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def cos(a, b):
    a, b = a.double().cpu().reshape(-1), b.double().cpu().reshape(-1)
    return float((a @ b) / (a.norm() * b.norm()).clamp_min(1e-30))


def cases():
    import open_musiclm_b200 as O
    from oracle import restatement as R
    g = lambda: torch.Generator().manual_seed(1234)
    common = dict(attn_dropout=0.0, ff_dropout=0.1)
    out = {}
    gg = g()
    out["cfg1"] = dict(make=lambda: O.create_semantic_transformer(dim=1024, depth=6, heads=8, **common),
                       cfg=R.semantic_cfg(ce_weights=[0.0, 1.0]), ce=[0.0, 1.0],
                       toks=[torch.randint(0, 1024, (2, 12), generator=gg), torch.randint(0, 1024, (2, 241), generator=gg)],
                       what="configs[0]: semantic L=6 h=8, B=2, N=256")
    gg = g()
    out["cfg2"] = dict(make=lambda: O.create_coarse_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, **common),
                       cfg=R.coarse_cfg(ce_weights=[0.0, 0.0, 1.0]), ce=[0.0, 0.0, 1.0],
                       toks=[torch.randint(0, 1024, (2, 12), generator=gg), torch.randint(0, 1024, (2, 197), generator=gg),
                             torch.randint(0, 1024, (2, 270, 3), generator=gg)],
                       what="configs[1] shape: coarse L=6 h=8, N=1024, B=2 of 16")
    gg = g()
    out["cfg3"] = dict(make=lambda: O.create_fine_transformer(dim=1024, depth=6, heads=8, num_coarse_quantizers=3, num_fine_quantizers=5, **common),
                       cfg=R.fine_cfg(ce_weights=[0.0, 0.0, 1.0]), ce=[0.0, 0.0, 1.0],
                       toks=[torch.randint(0, 1024, (1, 12), generator=gg), torch.randint(0, 1024, (1, 254, 3), generator=gg),
                             torch.randint(0, 1024, (1, 1269), generator=gg)],
                       what="configs[2] shape: fine L=6 h=8, N=2048 (remainder heads), B=1 of 8")
    gg = g()
    out["cfg4"] = dict(make=lambda: O.create_coarse_transformer(dim=1024, depth=24, heads=16, num_coarse_quantizers=3, **common),
                       cfg=R.coarse_cfg(depth=24, heads=16, ce_weights=[0.0, 0.0, 1.0]), ce=[0.0, 0.0, 1.0],
                       toks=[torch.randint(0, 1024, (1, 12), generator=gg), torch.randint(0, 1024, (1, 197), generator=gg),
                             torch.randint(0, 1024, (1, 270, 3), generator=gg)],
                       what="configs[3] architecture: musiclm_large coarse L=24 h=16, N=1024, B=1 of 16/GPU")
    return out


def oracle(case, want_grads):
    from oracle import restatement as R
    torch.manual_seed(0)
    m = case["make"]()
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    names = [k for k, _ in m.named_parameters()]
    t0 = time.time()
    toks = [t.numpy() for t in case["toks"]]
    if want_grads:
        sd_g = {k: (v.clone().requires_grad_(True) if k in names else v) for k, v in sd.items()}
        loss, logits, labels, ids, mask = R.loss_and_logits(case["cfg"], sd_g, toks)
        loss.backward()
        grads = {k: (sd_g[k].grad if sd_g[k].grad is not None else torch.zeros_like(sd[k])) for k in names}
        logits = [l.detach() for l in logits]
    else:
        with torch.no_grad():
            loss, logits, labels, ids, mask = R.loss_and_logits(case["cfg"], sd, toks)
        grads = None
    return dict(sd=sd, names=names, loss=float(loss), logits=logits, ids=ids, mask=mask, grads=grads, secs=time.time() - t0)


def gpu(case, ref, mode):
    import open_musiclm_b200 as O
    os.environ["OMLM_ACT16"] = mode
    torch.manual_seed(0)
    m = case["make"]()
    m.load_state_dict(ref["sd"], strict=True)
    m = m.cuda().eval()
    tr = O.HotPathTrainer(m, cross_entropy_loss_weights=case["ce"], use_cuda_graph=False)
    toks = [t.cuda() for t in case["toks"]]
    loss = float(tr.eval_loss(toks))
    with torch.no_grad():
        logits = m(all_token_ids=[torch.from_numpy(i).cuda() for i in ref["ids"]], self_attn_mask=torch.from_numpy(ref["mask"]).cuda())
    res = dict(loss=loss, loss_ref=ref["loss"], loss_rel=abs(loss - ref["loss"]) / abs(ref["loss"]),
               logits_rel=[rel(a, b) for a, b in zip(logits, ref["logits"])])
    if ref["grads"] is not None:
        tr.eng.arena_g.zero_()
        tr._micro_batch(toks, False, 0, True)
        torch.cuda.synchronize()
        rows = []
        for k in ref["names"]:
            g_ref = ref["grads"][k]
            if float(g_ref.norm()) < 1e-9 or k.endswith("rel_pos_bias.net.3.bias"):     # analytically zero gradient
                continue
            mine = tr.eng.gview[k]
            rows.append((k, cos(mine, g_ref), rel(mine, g_ref), g_ref.numel()))
        res["grad_worst_cos"] = min(rows, key=lambda r: r[1])[:3]
        res["grad_worst_rel"] = max(rows, key=lambda r: r[2])[:3]
        res["grad_over_2e-2"] = [(k, round(c, 5), round(r, 5)) for k, c, r, n in rows if r > 2e-2 or c < 0.999]
        res["grad_median_rel"] = sorted(r for _, _, r, _ in rows)[len(rows) // 2]
        res["grad_relpos"] = [(k, round(c, 6), round(r, 5)) for k, c, r, n in rows if "rel_pos_bias" in k]
        kb, kw = "transformer.rel_pos_bias.net.3.bias", "transformer.rel_pos_bias.net.3.weight"
        res["net3_bias_norms"] = dict(mine=float(tr.eng.gview[kb].double().norm()), ref=float(ref["grads"][kb].double().norm()),
                                      ref_net3_weight=float(ref["grads"][kw].double().norm()))
        tr.eng.arena_g.zero_()
    del tr, m
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="cfg1,cfg2,cfg3,cfg4")
    ap.add_argument("--modes", default="fp16,bf16")
    ap.add_argument("--no-grads", default="")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "parity_report.json"))
    args = ap.parse_args()
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    allc = cases()
    report = {}
    for name in args.cases.split(","):
        case = allc[name]
        ref = oracle(case, name not in args.no_grads.split(","))
        report[name] = dict(what=case["what"], oracle_secs=round(ref["secs"], 1))
        for mode in args.modes.split(","):
            try:
                report[name][mode] = gpu(case, ref, mode)
            except Exception as e:  # keep going: the report is a diagnostic
                report[name][mode] = dict(error=repr(e))
            print(name, mode, json.dumps(report[name][mode]), flush=True)
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
