"""Per-kernel breakdown of one coarse-stage training step.
  python tools/profile_step.py            -> CUDA-event time per C-ABI entry point (aggregated over one step)
  ncu --profile-from-start off ... python tools/profile_step.py --ncu   -> brackets one step with cudaProfilerStart/Stop
"""
import argparse
import collections
import json
import os
import tempfile
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
import open_musiclm_b200 as O  # noqa: E402
from open_musiclm_b200 import lib  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ncu", action="store_true")
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--config", default="cfg2")
    ap.add_argument("--depth", type=int, default=None, help="override the layer count (1 keeps an ncu --set full capture short)")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "step_breakdown.json"))
    args = ap.parse_args()
    torch.manual_seed(0)
    wl = bench.WORKLOADS[args.config]
    cfg = dict(bench.COMMON, **wl["model"])
    if args.depth is not None:
        cfg["depth"] = args.depth
    fn = {"coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}[wl["stage"]]
    model = fn(**cfg).cuda()
    tr = O.HotPathTrainer(model, cross_entropy_loss_weights=bench.TRAIN["ce_weights"], lr=3e-4, lr_warmup=6000, wd=0.01, use_cuda_graph=False)
    gen = torch.Generator().manual_seed(1234)
    batch = [t.cuda() for t in bench.synth_batch(args.batch or wl["batch"], gen, wl["shapes"])]
    for _ in range(3):
        tr.train_step([batch])
    torch.cuda.synchronize()
    if args.ncu:
        torch.cuda.cudart().cudaProfilerStart()
        tr.train_step([batch])
        torch.cuda.synchronize()
        torch.cuda.cudart().cudaProfilerStop()
        return
    log = []
    orig = lib.call

    def call(name, *a):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); r = orig(name, *a); e1.record()
        log.append((name, e0, e1))
        return r
    lib.call = call
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record(); tr.train_step([batch]); s1.record()
    torch.cuda.synchronize()
    lib.call = orig
    agg = collections.OrderedDict()
    for name, e0, e1 in log:
        d = agg.setdefault(name, [0, 0.0])
        d[0] += 1; d[1] += e0.elapsed_time(e1)
    total = s0.elapsed_time(s1)
    rows = sorted(agg.items(), key=lambda kv: -kv[1][1])
    print(f"step total {total:.3f} ms; sum of kernels {sum(v[1] for v in agg.values()):.3f} ms")
    for k, (n, ms) in rows:
        print(f"{k:28s} n={n:4d}  {ms:8.3f} ms  {100 * ms / total:5.1f}%")
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({"step_ms": total, "kernels": {k: {"launches": n, "ms": ms} for k, (n, ms) in rows}}, f, indent=1)


if __name__ == "__main__":
    main()
