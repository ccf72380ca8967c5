"""Deterministic mode (torch.use_deterministic_algorithms(True)) on the bench workloads.

  1. Reproducibility: for each of cfg2, cfg3, cfg4, two separate processes each build the workload's trainer from the same
     seed, take --steps training steps on the same batches with the switch on, and write bench.dump_outputs' files
     (loss, gradient norm, parameter sample); the files of the two processes are compared bit for bit.
  2. Cost: ms per step with the switch off and on, alternated in one process (--rounds x --time-steps steps each), and a
     torch.profiler breakdown of one eager step per mode by kernel.
Prints the card's name and power limit.  Writes only under --out (default: a temporary directory).

    python tools/check_deterministic.py [--configs cfg2,cfg3,cfg4] [--steps 5] [--rounds 3] [--time-steps 20]
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _trainer(cfg):
    import torch
    import bench
    import open_musiclm_b200 as O
    wl = bench.WORKLOADS[cfg]
    torch.manual_seed(0)
    m = bench.make_model(wl).cuda()
    t = bench.TRAIN
    tr = O.HotPathTrainer(m, cross_entropy_loss_weights=t["ce_weights"], lr=t["lr"], lr_warmup=t["lr_warmup"], wd=t["wd"],
                          max_grad_norm=t["max_grad_norm"])
    gen = torch.Generator().manual_seed(1)
    batches = [[x.cuda() for x in bench.synth_batch(wl["batch"], gen, wl["shapes"])] for _ in range(4)]
    return tr, batches


def child(cfg, steps, out):
    import torch
    import bench
    torch.use_deterministic_algorithms(True)
    tr, batches = _trainer(cfg)
    loss = None
    for i in range(steps):
        loss = tr.train_step([batches[i % len(batches)]])
    bench.dump_outputs(out, tr, loss)


def _step_ms(tr, batches, n):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(n):
        tr.train_step([batches[i % len(batches)]])
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def _kernel_times(tr, batches):
    """us per kernel name over one eager step (the profiler sees every launch)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    graph = tr.use_cuda_graph
    tr.use_cuda_graph = False
    tr.train_step([batches[0]])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        tr.train_step([batches[1]])
        torch.cuda.synchronize()
    tr.use_cuda_graph = graph
    out = collections.Counter()
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            out[e.key[:90]] += e.self_device_time_total
    return out


def timing(cfg, rounds, n):
    import torch
    tr, batches = _trainer(cfg)
    res = {"off": [], "on": []}
    for mode in ("off", "on"):               # warm-up: eager steps and the graph capture of each mode
        torch.use_deterministic_algorithms(mode == "on")
        _step_ms(tr, batches, 4)
    for _ in range(rounds):
        for mode in ("off", "on"):
            torch.use_deterministic_algorithms(mode == "on")
            res[mode].append(_step_ms(tr, batches, n))
    prof = {}
    for mode in ("off", "on"):
        torch.use_deterministic_algorithms(mode == "on")
        prof[mode] = _kernel_times(tr, batches)
    torch.use_deterministic_algorithms(False)
    del tr
    torch.cuda.empty_cache()
    return res, prof


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg2,cfg3,cfg4")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--time-steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.child, args.steps, args.out)
        return
    import bench
    out = args.out or tempfile.mkdtemp(prefix="omlm_det_")
    print("card:", json.dumps(bench.gpu_info()))
    for cfg in args.configs.split(","):
        dirs = [os.path.join(out, cfg, f"run{i}") for i in range(2)]
        for d in dirs:
            subprocess.run([sys.executable, os.path.abspath(__file__), "--child", cfg, "--steps", str(args.steps), "--out", d], check=True)
        same = {f: np.array_equal(np.load(os.path.join(dirs[0], f)), np.load(os.path.join(dirs[1], f)), equal_nan=False)
                for f in ("loss.npy", "grad_norm.npy", "params.npy")}
        loss = float(np.load(os.path.join(dirs[0], "loss.npy"))[0])
        print(f"{cfg}: two processes, {args.steps} steps with the switch on: bit-identical {same} (loss {loss:.6f})")
        res, prof = timing(cfg, args.rounds, args.time_steps)
        off, on = np.median(res["off"]), np.median(res["on"])
        print(f"{cfg}: ms/step off {['%.2f' % x for x in res['off']]} on {['%.2f' % x for x in res['on']]}; "
              f"median {off:.2f} -> {on:.2f} ({100 * (on / off - 1):+.1f} %)")
        keys = set(prof["off"]) | set(prof["on"])
        rows = sorted(keys, key=lambda k: -(prof["on"][k] - prof["off"][k]))
        tot_off, tot_on = sum(prof["off"].values()), sum(prof["on"].values())
        print(f"{cfg}: eager-step kernel time {tot_off / 1e3:.2f} -> {tot_on / 1e3:.2f} ms; largest differences (us, off -> on):")
        for k in rows[:12]:
            print(f"    {prof['off'][k]:9.0f} -> {prof['on'][k]:9.0f}  {k}")


if __name__ == "__main__":
    main()
