"""Records tests/golden/cbsize_*.pt: the REAL reference with codebooks of different sizes in different sequences, and
with a semantic codebook above 1280 entries: C = 1501 logit classes, padded to Cp = 1536, which takes the streaming
cross-entropy kernel and leaves a 35-column zero tail in every gradient row.  Every sequence's tokens are drawn from its
own codebook, so ids >= 1024 reach the embedding rows, the offsets and the labels.

The recipes are oracle/make_golden.py's (training: logits, loss, every gradient, two optimiser steps of the reference's
get_optimizer / clip recipe) and oracle/make_golden_generate.py's (generate under a seeded Gumbel-noise stream) -- same
seeds, same perturbed gammas / scales -- with per-sequence codebooks for the token draws.  The files are kept small in
the form tests/codebook_fixtures.py describes: no weights (the tests rebuild them with this package's factory under
the same seed, pinned by the SHA-256 of the reference's state dict), seeded samples of the large tensors with their
norms, and the seed and SHA-256 of the noise draws instead of the draws.

Needs a reference checkout:   OMLM_REFERENCE_ROOT=<checkout> python tools/make_golden_codebooks.py
"""
import importlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402
from oracle.make_golden import COMMON, GOLD, build  # noqa: E402
from oracle.make_golden_generate import SEED  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import codebook_fixtures as CF  # noqa: E402

TRAIN = {
    # name: (stage, transformer kwargs, token shapes, per-sequence codebook sizes, ce weights, optimiser steps)
    "cbsize_semantic": ("semantic", dict(dim=64, depth=1, heads=2, clap_codebook_size=64, semantic_codebook_size=1500,
                                         num_clap_quantizers=4), [(2, 4), (2, 27)], [64, 1500], [0.0, 1.0], 2),
    # a 1500-entry conditioning sequence (its eos id 1500 is masked out of the keys) ahead of a 64-entry predicted one
    "cbsize_coarse": ("coarse", dict(dim=64, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=1500,
                                     acoustic_codebook_size=64, num_clap_quantizers=4, num_coarse_quantizers=3),
                      [(2, 4), (2, 11), (2, 10, 3)], [64, 1500, 64], [0.0, 0.0, 1.0], 0),
}
GEN = {
    # name: (stage, kwargs, conditioning shapes, conditioning codebooks, max_time_steps, temperature)
    "cbsize_gen_semantic": ("semantic", dict(dim=64, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=1500,
                                             num_clap_quantizers=4), [(2, 4)], [64], 24, 1.0),
    # 20 sequences: the tensor-core decode path (more than the 16 rows the SIMT kernels serve)
    "cbsize_gen_semantic_b20": ("semantic", dict(dim=64, depth=1, heads=2, clap_codebook_size=64, semantic_codebook_size=1500,
                                                 num_clap_quantizers=4), [(20, 4)], [64], 8, 0.95),
}


def perturbed(ref, stage, kw):
    torch.manual_seed(0)
    model = build(ref, stage, kw)
    g0 = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for k, p in model.named_parameters():
            if k.endswith("gamma") or k.endswith("q_scale") or k.endswith("k_scale"):
                p.mul_(1.0 + 0.2 * torch.randn(p.shape, generator=g0))
    return model


def draw(shapes, cbs, g):
    """Tokens of sequence s uniform in [0, cbs[s]), with the last id of each codebook placed once."""
    toks = [torch.randint(0, cb, s, generator=g) for s, cb in zip(shapes, cbs)]
    for t, cb in zip(toks, cbs):
        t.view(-1)[-1] = cb - 1
    return toks


def record_training(ref, name, stage, kw, shapes, cbs, cew, n_steps):
    model = perturbed(ref, stage, kw)
    wrapper = ref.TokenConditionedTransformerWrapper(transformer=model, unique_consecutive=False,
                                                     cross_entropy_loss_weights=cew, mask_prob=0.15)
    wrapper.eval()
    tokens = draw(shapes, cbs, torch.Generator().manual_seed(1234))
    state = CF.state_sha(model.state_dict())
    loss, logits, labels = wrapper(all_token_ids=[t.clone() for t in tokens], return_loss=True)
    loss.backward()
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
        "stage": stage, "kwargs": dict(COMMON, **kw), "ce_weights": cew, "codebooks": cbs, "state_sha": state,
        "tokens": tokens, "ids": ids, "key_mask": torch.cat(masks, 1), "labels": labels,
        "logits": [CF.sample(l.detach().permute(0, 2, 1), seed=i) for i, l in enumerate(logits)],   # [b, n, c] order
        "loss": loss.detach(),
        "grads": {k: (CF.sample(p.grad, seed=i) if p.grad is not None else None) for i, (k, p) in enumerate(model.named_parameters())},
    }
    opt_mod = importlib.import_module("open_musiclm.optimizer")
    optim = opt_mod.get_optimizer(model.parameters(), lr=3e-4, wd=1e-2)
    sched = opt_mod.get_linear_scheduler(optim, total_iters=10)
    steps = []
    for it in range(n_steps):
        if it > 0:
            optim.zero_grad()
            loss, _, _ = wrapper(all_token_ids=[t.clone() for t in tokens], return_loss=True)
            loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(model.parameters(), 0.5)
        optim.step()
        sched.step()
        steps.append({"grad_norm": norm.detach().clone(), "loss": loss.detach().clone(),
                      "params": ({k: CF.sample(p, seed=i) for i, (k, p) in enumerate(model.named_parameters())}
                                 if it == n_steps - 1 else None)})
    fx["opt_steps"] = steps
    return fx


def record_generate(ref, name, stage, kw, cshapes, ccbs, steps, temp):
    model = perturbed(ref, stage, kw)
    wrapper = ref.TokenConditionedTransformerWrapper(transformer=model, unique_consecutive=False)
    cond = draw(cshapes, ccbs, torch.Generator().manual_seed(99))
    info = model.token_sequences[-1]
    n_new = steps * info.num_quantizers
    B, C = cshapes[0][0], info.codebook_size + 1
    torch.manual_seed(SEED)
    out = wrapper.generate(conditioning_token_ids=[t.clone() for t in cond], max_time_steps=steps, temperature=temp)
    torch.manual_seed(SEED)
    noise = torch.stack([torch.zeros(B, C).uniform_(0, 1) for _ in range(n_new)])     # the draws generate consumed
    fx = {"stage": stage, "kwargs": dict(kw, **COMMON), "codebooks": ccbs + [info.codebook_size],
          "state_sha": CF.state_sha(model.state_dict()), "cond": cond, "prefix": None, "max_time_steps": steps,
          "temperature": temp, "filter_thres": 0.9, "allow_eos_in_output": False, "include_eos_in_output": False,
          "noise_seed": SEED, "noise_shape": tuple(noise.shape), "noise_sha": CF.tensor_sha(noise), "out": out}
    assert torch.equal(CF.uniforms(fx), noise)
    return fx


def check_rebuild(fx):
    """The tests rebuild the weights with this package's factory: make sure that gives the reference's."""
    CF.model_of(fx)


def main():
    ref = ref_harness.import_reference()
    only = set(sys.argv[1:])
    jobs = [(n, record_training, a) for n, a in TRAIN.items()] + [(n, record_generate, a) for n, a in GEN.items()]
    for name, fn, args in jobs:
        if only and name not in only:
            continue
        fx = fn(ref, name, *args)
        check_rebuild(fx)
        path = os.path.join(GOLD, f"{name}.pt")
        torch.save(fx, path)
        print(name, "->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
