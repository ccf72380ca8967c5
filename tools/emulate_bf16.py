"""CPU experiment (test tooling, not product): the oracle forward with bf16 rounding inserted at exactly the
places where the CUDA path rounds (GEMM operands and the bf16 activations it stores), each site switchable,
to see which roundings dominate the logits distance to the fp32 oracle at depth."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.nn.functional as F
from oracle import restatement as R


def rb(t):
    return t.bfloat16().float()


def rh(t):
    return t.half().float()


def forward(cfg, sd, ids, key_mask, sites, f16=frozenset()):
    """sites: where a 16-bit rounding happens; f16: the subset of those that round to fp16 instead of bf16."""
    on = lambda s: (rh if s in f16 else rb) if s in sites else (lambda t: t)
    x = R.embed(cfg, sd, ids)
    B, N, _ = x.shape
    table = R.rel_pos_table(sd, N)
    km = None if key_mask is None else torch.from_numpy(key_mask)
    h, dh = cfg.heads, cfg.dim_head
    i = torch.arange(N)
    delta = i[:, None] - i[None, :]
    neg = -torch.finfo(torch.float32).max
    for l in range(cfg.depth):
        p = f"transformer.layers.{l}.0."
        xn = R.layer_norm(x, sd[p + "norm.gamma"])
        q = on("qkv_in")(xn) @ on("w")(sd[p + "to_q.weight"]).t()
        kv = on("qkv_in")(x) @ on("w")(sd[p + "to_kv.weight"]).t()
        q, kv = on("qkv_out")(q), on("qkv_out")(kv)
        k, v = kv[..., :dh], kv[..., dh:]
        q = q.view(B, N, h, dh).permute(0, 2, 1, 3)
        q = on("qkn")(q / q.norm(dim=-1, keepdim=True).clamp_min(1e-12) * sd[p + "q_scale"])
        k = on("qkn")(k / k.norm(dim=-1, keepdim=True).clamp_min(1e-12) * sd[p + "k_scale"])
        v = on("qkn")(v)
        sim = torch.einsum("bhid,bjd->bhij", q, k) * cfg.attn_scale + table[:, delta.clamp_min(0)][None]
        if km is not None:
            sim = sim.masked_fill(~km[:, None, None, :], neg)
        sim = sim.masked_fill((delta < 0)[None, None], neg)
        m = sim.amax(-1, keepdim=True)
        pexp = torch.exp(sim - m)
        l_ = pexp.sum(-1, keepdim=True)
        o = torch.einsum("bhij,bjd->bhid", on("p")(pexp), v) / l_
        o = on("o")(o.permute(0, 2, 1, 3).reshape(B, N, h * dh))
        x = o @ on("w")(sd[p + "to_out.0.weight"]).t() + x
        p = f"transformer.layers.{l}.2."
        Fi = cfg.ff_inner
        xn = R.layer_norm(x, sd[p + "0.gamma"])
        u = on("u")(on("ffn_in")(xn) @ on("w")(sd[p + "1.weight"]).t())
        w = sd[p + "2.ds_conv.weight"][:, 0, :]
        up = F.pad(u, (0, 0, 2, 0))
        y = up[:, 0:-2] * w[:, 0] + up[:, 1:-1] * w[:, 1] + up[:, 2:] * w[:, 2]
        a, g = y[..., :Fi], y[..., Fi:]
        hm = on("h")(F.gelu(g) * a)
        hn = on("hn")(R.layer_norm(hm, sd[p + "4.gamma"]))
        x = hn @ on("w")(sd[p + "6.weight"]).t() + x
    hid = R.layer_norm(x, sd["transformer.norm.gamma"])
    sd2 = dict(sd)
    for s in range(len(cfg.seqs)):
        sd2[f"logit_weights.{s}"] = on("head")(sd[f"logit_weights.{s}"])
    return R.logits_from_hidden(cfg, sd2, on("head")(hid), [t.shape[1] for t in ids])


ALL = {"qkv_in", "w", "qkv_out", "qkn", "p", "o", "ffn_in", "u", "h", "hn", "head"}


def main():
    depth = int(sys.argv[1]) if len(sys.argv) > 1 else 6
    heads = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    S = int(sys.argv[3]) if len(sys.argv) > 3 else 60
    T = int(sys.argv[4]) if len(sys.argv) > 4 else 60
    torch.manual_seed(0)
    cfg = R.coarse_cfg(depth=depth, heads=heads, ce_weights=[0., 0., 1.])
    sd = R.init_state(cfg, seed=0)
    g = torch.Generator().manual_seed(1234)
    toks = [torch.randint(0, 1024, (1, 12), generator=g).numpy(), torch.randint(0, 1024, (1, S), generator=g).numpy(),
            torch.randint(0, 1024, (1, T, 3), generator=g).numpy()]
    ids, mask, labels = R.prepare_ids(cfg, toks, True, None)
    with torch.no_grad():
        t0 = time.time()
        ref = forward(cfg, sd, ids, mask, set())
        print("N", sum(t.shape[1] + 1 for t in ids), "fp32 fwd s", time.time() - t0)
        def dist(sites):
            out = forward(cfg, sd, ids, mask, sites)
            return float((out[-1] - ref[-1]).norm() / ref[-1].norm())
        print("all sites        ", dist(ALL))
        for s in sorted(ALL):
            print(f"without {s:8s} ", dist(ALL - {s}), "   only", dist({s}))
        print("without head,u,h  ", dist(ALL - {"head", "u", "h"}))
        print("without head,u,h,o,qkv_out", dist(ALL - {"head", "u", "h", "o", "qkv_out"}))
        for name, f16 in [("fp16: w, ffn_in, hn, head", {"w", "ffn_in", "hn", "head"}),
                          ("fp16: + u, h", {"w", "ffn_in", "hn", "head", "u", "h"}),
                          ("fp16: + qkv_in", {"w", "ffn_in", "hn", "head", "u", "h", "qkv_in"}),
                          ("fp16: everything", set(ALL))]:
            out = forward(cfg, sd, ids, mask, ALL, f16)
            print(name, float((out[-1] - ref[-1]).norm() / ref[-1].norm()))


if __name__ == "__main__":
    main()
