"""Records what the REAL reference computes for the CPU tests that compare against it (tests/golden/reference_live.pt):

  forgetful_mask   utils.generate_mask_with_prob under a fixed torch seed            (tests/test_oracle_cpu.py)
  restatement      loss and a seeded sample of the logits of the reference wrapper,
                   plus the SHA-256 of the state dict it ran on, per stage              (tests/test_oracle_cpu.py)
  crops            PreprocessedDataset.__getitem__ crops of a synthetic database       (tests/test_data_cpu.py)
  init_sha         SHA-256 of every tensor of the reference's init under seed 0       (tests/test_boundary_cpu.py)

Needs a reference checkout:   OMLM_REFERENCE_ROOT=<checkout> python oracle/make_golden_live.py
"""
import hashlib
import os
import random
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_harness  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference_live.pt")
LOGIT_SAMPLE = 2048

# shared with the tests
LIVE_COMMON = dict(attn_dropout=0.0, ff_dropout=0.1, grad_shrink_alpha=0.1, non_causal_prefix_size=0,
                   relative_position_bias_type="continuous", use_memory_efficient_attention=False)
LIVE_STAGES = {
    "semantic": (dict(dim=192, depth=2, heads=3), [(2, 12), (2, 40)]),
    "coarse": (dict(dim=192, depth=2, heads=3, num_coarse_quantizers=3), [(2, 12), (2, 20), (2, 9, 3)]),
    "fine": (dict(dim=192, depth=2, heads=3, num_coarse_quantizers=3, num_fine_quantizers=5), [(2, 12), (2, 5, 3), (2, 5, 5)]),
}
INIT_BASE = dict(dim=128, depth=2, heads=2, attn_dropout=0.0, ff_dropout=0.1)
INIT_VARIANTS = [dict(), dict(use_conv_ff=False, relative_position_bias_type="t5"),
                 dict(relative_position_bias_type="none", use_absolute_position_embeddings=True)]


def sha(t: torch.Tensor) -> str:
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def state_sha(sd) -> str:
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(v.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def logit_sample_index(n: int, i: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(1000 + i)
    return torch.randperm(n, generator=g)[:min(n, LOGIT_SAMPLE)]


def live_tokens(shapes):
    g = torch.Generator().manual_seed(99)
    return [torch.randint(0, 1024, s, generator=g) for s in shapes]


def main():
    ref = ref_harness.import_reference()
    utils = sys.modules["open_musiclm.utils"]
    out = {}
    torch.manual_seed(11)
    out["forgetful_mask"] = utils.generate_mask_with_prob((4, 50), 0.15, device="cpu").clone()

    out["restatement"] = {}
    for stage, (kw, shapes) in LIVE_STAGES.items():
        torch.manual_seed(5)
        model = getattr(ref, f"create_{stage}_transformer")(**kw, **LIVE_COMMON)
        ce = [0.0, 1.0] if stage == "semantic" else [0.0, 0.0, 1.0]
        wrapper = ref.TokenConditionedTransformerWrapper(transformer=model, unique_consecutive=False,
                                                         cross_entropy_loss_weights=ce).eval()
        toks = live_tokens(shapes)
        with torch.no_grad():
            loss, logits, _ = wrapper(all_token_ids=[t.clone() for t in toks], return_loss=True)
        samples = []
        for i, lg in enumerate(logits):
            flat = lg.permute(0, 2, 1).reshape(-1)        # the restatement's [b, n, C] order
            samples.append(flat[logit_sample_index(flat.numel(), i)].clone())
        out["restatement"][stage] = dict(loss=float(loss), logit_numel=[int(lg.numel()) for lg in logits], logits=samples,
                                         state_sha=state_sha(model.state_dict()))

    import importlib
    import test_data_cpu as T
    ref_data = importlib.import_module("open_musiclm.data")
    from open_musiclm_b200 import data as D
    out["crops"] = {}
    for stage in ["semantic", "coarse", "fine"]:
        items = T.synth_items(5, seed=3)
        with tempfile.TemporaryDirectory() as d:
            D.write_sqlite(d, items)
            ds = ref_data.PreprocessedDataset(d, stage)
            crops = []
            for idx in range(len(ds)):
                random.seed(100 + idx)
                crops.append([t.clone() for t in ds[idx]])
        out["crops"][stage] = crops

    out["init_sha"] = {}
    for vi, extra in enumerate(INIT_VARIANTS):
        for stage in ["semantic", "coarse", "fine"]:
            torch.manual_seed(0)
            sd = getattr(ref, f"create_{stage}_transformer")(**dict(INIT_BASE, **extra)).state_dict()
            out["init_sha"][(vi, stage)] = {k: sha(v) for k, v in sd.items()}
    torch.save(out, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
