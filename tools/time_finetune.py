"""Training-step time of a fine-tune with frozen parameters, and the attention backward with and without the bias
gradient, at the cfg2 and cfg4 shapes of bench.py (CUDA events; the card's name and power limit are printed with the
numbers).

  full       every parameter trains
  relpos     the relative-position MLP is frozen: the attention backward runs without the bias gradient
  top4/top1  only the top 4 / 1 layers, the final norm and the logit heads train: the backward stops below them
"""
import argparse
import gc
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402
import open_musiclm_b200 as O  # noqa: E402
from open_musiclm_b200 import lib  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else torch.cuda.get_device_name()


def frozen_names(m, kind, depth):
    names = [n for n, _ in m.named_parameters()]
    if kind == "full":
        return set()
    if kind == "relpos":
        return {n for n in names if n.startswith("transformer.rel_pos_bias.")}
    k = int(kind[3:])
    keep = tuple(f"transformer.layers.{l}." for l in range(depth - k, depth)) + ("transformer.norm.", "logit_weights.")
    return {n for n in names if not n.startswith(keep)}


def time_steps(wl, kind, steps, warmup):
    torch.manual_seed(0)
    m = bench.make_model(wl)
    frozen = frozen_names(m, kind, wl["model"]["depth"])
    for n, p in m.named_parameters():
        p.requires_grad_(n not in frozen)
    m = m.cuda()
    tr = O.HotPathTrainer(m, cross_entropy_loss_weights=[0.0, 0.0, 1.0], lr=3e-4, wd=1e-2, max_grad_norm=0.5)
    gen = torch.Generator().manual_seed(1)
    batches = [[t.cuda() for t in bench.synth_batch(wl["batch"], gen, wl["shapes"])] for _ in range(4)]
    for i in range(warmup):
        tr.train_step([batches[i % 4]])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        tr.train_step([batches[i % 4]])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    del tr, m
    gc.collect()                # the module and its engine refer to each other
    torch.cuda.empty_cache()
    return ms


def time_attn_bwd(B, N, h, det, reps=20):
    M = B * N
    torch.manual_seed(0)
    qn = F.normalize(torch.randn(M, h, 64, device="cuda"), dim=-1).reshape(M, h * 64).bfloat16()
    kvn = torch.randn(M, 128, device="cuda").bfloat16()
    kvn[:, :64] = F.normalize(kvn[:, :64].float(), dim=-1).bfloat16()
    table = (torch.randn(h, 1, device="cuda") * 0.05 * torch.arange(N, device="cuda")[None]).contiguous()
    km = (torch.rand(B, N, device="cuda") > 0.15).to(torch.uint8)
    km[:, 0] = 1
    out = torch.empty(M, h * 64, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(M * h, device="cuda")
    lib.attn_fwd_tc(qn, kvn, table, km, out, lse, B, N, h)
    d_o = torch.randn(M, h * 64, device="cuda").bfloat16()
    dqn, dkvn = torch.empty(M, h * 64, device="cuda"), torch.empty(M, 128, device="cuda")
    dtab, dsum = torch.zeros_like(table), torch.empty(M * h, device="cuda")
    ws = lib.AttnBwdDetWorkspace("cuda", B, N, h) if det else None
    res = {}
    for tag, dt in (("with table", dtab), ("without", None)):
        fn = lambda: lib.attn_bwd_tc(qn, kvn, d_o, out, lse, table, km, dsum, dqn, dkvn, dt, B, N, h, det=ws)
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res[tag] = e0.elapsed_time(e1) / reps * 1e3
    if ws is not None:
        assert not ws.error()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--configs", default="cfg2,cfg4")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_finetune.py needs an H100")
    print(f"card: {card()}", flush=True)
    for cfg in args.configs.split(","):
        wl = bench.WORKLOADS[cfg]
        h = wl["model"]["heads"]
        for det in (False, True):
            r = time_attn_bwd(wl["batch"], wl["N"], h, det)
            print(f"{cfg} attention backward per layer ({'deterministic' if det else 'default'}): with the bias gradient "
                  f"{r['with table']:.1f} us, without {r['without']:.1f} us ({r['with table'] / r['without']:.2f}x)", flush=True)
        full = None
        for kind in ("full", "relpos", "top4", "top1"):
            ms = time_steps(wl, kind, args.steps, args.warmup)
            full = full or ms
            print(f"{cfg} step {kind:6s}: {ms:.2f} ms ({ms / full:.2f} of full)", flush=True)


if __name__ == "__main__":
    main()
