"""Cost of return_logprobs on the H100: the sampler alone at C = 1025 and 16384 (B = 16 and 256), and whole generate
calls of a coarse stage (d = 1024, 12 layers, 16 heads, codebook 1024, a prompt of ~1000 positions, 24 sampled tokens)
at B = 1, 16, 17, 64, 256, with and without it, alternated.  Prints the card and its power limit first."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import open_musiclm_b200 as O  # noqa: E402
from open_musiclm_b200 import lib  # noqa: E402


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    dev = "cuda"
    for C in (1025, 16384):
        for B in (16, 256):
            x = torch.randn(B, C, device=dev) * 3
            nr = torch.zeros(B, device=dev, dtype=torch.int32)
            seeds = torch.arange(B, device=dev, dtype=torch.int64)
            tok, lp, slp = lib.logprob_buffers(B, 1, dev)
            cnt = torch.zeros(2, device=dev, dtype=torch.int32)

            def run(with_lp, top_p):
                cnt.zero_()
                lib.sample(x, C, max(1, C // 10), 1.0, False, None, None, tok, nr, 0, cnt, None, B, seeds=seeds, top_p=top_p,
                           logprobs=lp if with_lp else None, sample_logprobs=slp if with_lp else None)
            for top_p in (None, 0.9):
                t = [[], []]
                for _ in range(7):
                    for f in (0, 1):
                        t[f].append(timed(lambda: run(bool(f), top_p), 200) * 1e3)
                print(f"sampler C={C} B={B} top_p={top_p}: plain {min(t[0]):.2f} (max {max(t[0]):.2f}) us, with logprobs "
                      f"{min(t[1]):.2f} (max {max(t[1]):.2f}) us over 7 alternated rounds", flush=True)
    torch.manual_seed(0)
    m = O.create_coarse_transformer(dim=1024, depth=12, heads=16, clap_codebook_size=1024, semantic_codebook_size=1024,
                                    acoustic_codebook_size=1024, num_clap_quantizers=12, num_coarse_quantizers=3,
                                    attn_dropout=0.0, ff_dropout=0.0).cuda().eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    for B in (1, 16, 17, 64, 256):
        g = torch.Generator().manual_seed(B)
        cond = [torch.randint(0, 1024, (B, 24), generator=g).to(dev), torch.randint(0, 1024, (B, 500), generator=g).to(dev)]
        pred = torch.randint(0, 1024, (B, 150, 3), generator=g).to(dev)
        kw = dict(conditioning_token_ids=cond, pred_token_ids=pred, max_time_steps=158, seeds=list(range(B)))
        t = [[], []]
        for _ in range(3):
            for f in (0, 1):
                t[f].append(timed(lambda: w.generate(return_logprobs=bool(f), **kw), 2))
        n_new = 8 * 3
        print(f"generate B={B} (prompt ~1000 positions, {n_new} sampled): {min(t[0]):.2f} (max {max(t[0]):.2f}) ms plain, "
              f"{min(t[1]):.2f} (max {max(t[1]):.2f}) ms with logprobs ({(min(t[1]) - min(t[0])) / n_new * 1e3:.1f} us per sampled token incl. prefix scoring)", flush=True)


if __name__ == "__main__":
    main()
