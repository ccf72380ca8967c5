"""ORACLE — test infrastructure only.  Golden token sequences of the REAL reference's autoregressive generate
(TokenConditionedTransformerWrapper.generate, open_musiclm.py:253-326) under a FIXED Gumbel noise stream.

Needs a reference checkout:   OMLM_REFERENCE_ROOT=<checkout> python oracle/make_golden_generate.py
The reference draws its Gumbel noise as torch.zeros_like(logits).uniform_(0, 1) from torch's default CPU generator
(utils.py:71-73): seeding that generator right before generate() fixes the stream, and the fixture stores the very
same draws (re-generated with the same seed and shapes) so that the oracle restatement and the CUDA sampler can consume
them.  Fixture: state_dict, conditioning / prefix tokens, uniforms [steps, B, C], the reference's output tokens.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402
from oracle.make_golden import COMMON, GOLD, build  # noqa: E402

CASES = {
    # name: (stage, kwargs, conditioning shapes, prefix shape or None, max_time_steps, temperature, allow_eos)
    "gen_semantic": ("semantic", dict(dim=64, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=64, num_clap_quantizers=4),
                     [(2, 4)], None, 24, 1.0, False),
    "gen_coarse": ("coarse", dict(dim=128, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=64,
                                  acoustic_codebook_size=64, num_clap_quantizers=4, num_coarse_quantizers=3),
                   [(2, 4), (2, 11)], (2, 2, 3), 10, 0.95, False),
    "gen_fine_eos": ("fine", dict(dim=64, depth=1, heads=3, clap_codebook_size=64, acoustic_codebook_size=64,
                                  num_clap_quantizers=4, num_coarse_quantizers=3, num_fine_quantizers=5),
                     [(2, 4), (2, 6, 3)], None, 6, 1.0, True),
}
SEED = 4321


def main():
    ref = ref_harness.import_reference()
    for name, (stage, kw, cshapes, pshape, steps, temp, allow_eos) in CASES.items():
        torch.manual_seed(0)
        model = build(ref, stage, kw)
        g0 = torch.Generator().manual_seed(7)
        with torch.no_grad():
            for k, p in model.named_parameters():
                if k.endswith("gamma") or k.endswith("q_scale") or k.endswith("k_scale"):
                    p.mul_(1.0 + 0.2 * torch.randn(p.shape, generator=g0))
        wrapper = ref.TokenConditionedTransformerWrapper(transformer=model, unique_consecutive=False)
        g = torch.Generator().manual_seed(99)
        cb = kw.get("clap_codebook_size", 64)
        cond = [torch.randint(0, cb, s, generator=g) for s in cshapes]
        prefix = torch.randint(0, cb, pshape, generator=g) if pshape is not None else None
        q = model.token_sequences[-1].num_quantizers
        n_new = (steps - (pshape[1] if pshape is not None else 0)) * q
        B, C = cshapes[0][0], cb + 1
        torch.manual_seed(SEED)
        out = wrapper.generate(conditioning_token_ids=[t.clone() for t in cond], pred_token_ids=None if prefix is None else prefix.clone(),
                               max_time_steps=steps, temperature=temp, allow_eos_in_output=allow_eos, include_eos_in_output=allow_eos)
        torch.manual_seed(SEED)
        uniforms = torch.stack([torch.zeros(B, C).uniform_(0, 1) for _ in range(n_new)])
        fx = {"stage": stage, "kwargs": dict(kw, **COMMON), "state_dict": {k: v.detach().clone() for k, v in model.state_dict().items()},
              "cond": cond, "prefix": prefix, "max_time_steps": steps, "temperature": temp, "filter_thres": 0.9,
              "allow_eos_in_output": allow_eos, "include_eos_in_output": allow_eos, "uniforms": uniforms, "out": out}
        path = os.path.join(GOLD, f"{name}.pt")
        torch.save(fx, path)
        print(name, tuple(out.shape), "->", path, os.path.getsize(path) // 1024, "KiB", out[0].reshape(-1)[:12].tolist())


if __name__ == "__main__":
    main()
