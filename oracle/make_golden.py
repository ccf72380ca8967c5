"""ORACLE — test infrastructure only.  Generates tests/golden/*.pt from the REAL reference.

Needs a reference checkout:   OMLM_REFERENCE_ROOT=<checkout> python oracle/make_golden.py
The fixtures pin oracle/restatement.py (tests/test_oracle_cpu.py) and give the GPU parity tests
(tests/test_parity_gpu.py) reference outputs that the GPU tests compare against.

Each fixture holds: hyper-parameters, the reference model's state_dict, the input token ids, and —
computed by the reference's own TokenConditionedTransformerWrapper on CPU fp32 in eval mode
(ff dropout and the forgetful mask off, SURVEY.md §8d) — ids after pre-processing, the key mask,
labels, every logits tensor, the loss, and the gradient of the loss w.r.t. every parameter.
A second fixture family holds two optimiser steps of the reference's get_optimizer/clip recipe.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")

CASES = {
    # name: (stage, transformer kwargs, token shapes, ce weights, batch)
    "tiny_semantic": ("semantic", dict(dim=64, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=64,
                                       num_clap_quantizers=4), [(2, 4), (2, 27)], [0.0, 1.0]),
    "tiny_coarse": ("coarse", dict(dim=128, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=64,
                                   acoustic_codebook_size=64, num_clap_quantizers=4, num_coarse_quantizers=3),
                    [(2, 4), (2, 11), (2, 10, 3)], [0.0, 0.0, 1.0]),
    # fine passed 2-D flattened with a remainder (exercises open_musiclm.py:177-182) and all-ones CE weights
    "tiny_fine": ("fine", dict(dim=64, depth=1, heads=3, clap_codebook_size=64, acoustic_codebook_size=64,
                               num_clap_quantizers=4, num_coarse_quantizers=3, num_fine_quantizers=5),
                  [(2, 4), (2, 6, 3), (2, 23)], [1.0, 1.0, 1.0]),
    # configuration variants (SURVEY 8f rank 3): plain GEGLU FeedForward (transformer.py:152-161) + T5 bias (69-117);
    # no relative bias + per-sequence absolute position embeddings (open_musiclm.py:81-82,134-136)
    "tiny_plainff_t5": ("coarse", dict(dim=64, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=64,
                                       acoustic_codebook_size=64, num_clap_quantizers=4, num_coarse_quantizers=3,
                                       use_conv_ff=False, relative_position_bias_type="t5"),
                        [(2, 4), (2, 9), (2, 7, 3)], [0.0, 0.0, 1.0]),
    "tiny_nobias_abspos": ("semantic", dict(dim=64, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=64,
                                            num_clap_quantizers=4, relative_position_bias_type="none",
                                            use_absolute_position_embeddings=True),
                           [(2, 4), (2, 27)], [1.0, 1.0]),
}
COMMON = dict(attn_dropout=0.0, ff_dropout=0.1, grad_shrink_alpha=0.1, non_causal_prefix_size=0,
              relative_position_bias_type="continuous", use_memory_efficient_attention=False)


def build(ref, stage, kw):
    fn = {"semantic": ref.create_semantic_transformer, "coarse": ref.create_coarse_transformer,
          "fine": ref.create_fine_transformer}[stage]
    return fn(**dict(COMMON, **kw))


def main():
    ref = ref_harness.import_reference()
    os.makedirs(GOLD, exist_ok=True)
    only = set(sys.argv[1:])
    for name, (stage, kw, shapes, cew) in CASES.items():
        if only and name not in only:
            continue
        torch.manual_seed(0)
        model = build(ref, stage, kw)
        # perturb the unit-initialised parameters so that parity tests see non-trivial gammas / scales
        g0 = torch.Generator().manual_seed(7)
        with torch.no_grad():
            for k, p in model.named_parameters():
                if k.endswith("gamma") or k.endswith("q_scale") or k.endswith("k_scale"):
                    p.mul_(1.0 + 0.2 * torch.randn(p.shape, generator=g0))
        wrapper = ref.TokenConditionedTransformerWrapper(transformer=model, unique_consecutive=False,
                                                         cross_entropy_loss_weights=cew, mask_prob=0.15)
        wrapper.eval()
        g = torch.Generator().manual_seed(1234)
        cb = kw.get("clap_codebook_size", 64)
        tokens = [torch.randint(0, cb, s, generator=g) for s in shapes]
        loss, logits, labels = wrapper(all_token_ids=[t.clone() for t in tokens], return_loss=True)
        loss.backward()
        # the pre-processed ids / mask the transformer actually saw (recomputed the reference's way)
        ids = [t.clone().reshape(t.shape[0], -1) for t in tokens]
        utils = sys.modules["open_musiclm.utils"]
        ids = [utils.append_eos_id(t, e) for t, e in zip(ids, model.eos_ids)]
        ids[-1] = ids[-1][:, :-1]
        masks = []
        for t, e in zip(ids[:-1], model.eos_ids[:-1]):
            m = (t != -1) & (t != e)
            t.masked_fill_(~m, 0)
            masks.append(torch.nn.functional.pad(m, (1, 0), value=True))
        masks.append(torch.ones(ids[-1].shape[0], ids[-1].shape[1] + 1, dtype=torch.bool))
        fx = {
            "stage": stage, "kwargs": dict(COMMON, **kw), "ce_weights": cew,
            "state_dict": {k: v.detach().clone() for k, v in model.state_dict().items()},
            "tokens": tokens, "ids": ids, "key_mask": torch.cat(masks, 1),
            "labels": labels, "logits": [l.detach().permute(0, 2, 1).contiguous() for l in logits],  # back to [b, n, c]
            "loss": loss.detach(),
            "grads": {k: (p.grad.detach().clone() if p.grad is not None else None) for k, p in model.named_parameters()},
        }
        # two optimiser steps, the reference's recipe (optimizer.py + trainer.py:443-449)
        import importlib
        opt_mod = importlib.import_module("open_musiclm.optimizer")
        optim = opt_mod.get_optimizer(model.parameters(), lr=3e-4, wd=1e-2)
        sched = opt_mod.get_linear_scheduler(optim, total_iters=10)
        steps = []
        for it in range(2 if name == "tiny_coarse" else 0):
            if it > 0:
                optim.zero_grad()
                loss, _, _ = wrapper(all_token_ids=[t.clone() for t in tokens], return_loss=True)
                loss.backward()
            norm = torch.nn.utils.clip_grad_norm_(model.parameters(), 0.5)
            optim.step()
            sched.step()
            steps.append({"grad_norm": norm.detach().clone(), "loss": loss.detach().clone(),
                          "params": ({k: p.detach().clone() for k, p in model.named_parameters()} if it == 1 else None)})
        fx["opt_steps"] = steps
        path = os.path.join(GOLD, f"{name}.pt")
        torch.save(fx, path)
        print(name, "loss", float(fx["loss"]), "->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
