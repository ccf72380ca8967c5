"""ORACLE — test infrastructure only.  Records a training-mode step of the REAL reference (tests/golden/train_mode.pt).

The eval fixtures (oracle/make_golden.py) run the reference wrapper with FFN dropout and the forgetful causal mask off.
This one runs it in `.train()`, as a training step does, and records the masks the reference itself drew:
  forget   [B, N] bool   the output of utils.generate_mask_with_prob (wrapped where open_musiclm.py calls it)
  keeps    per layer [B, N, F] bool   where the FFN nn.Dropout let its input through (a forward hook: out != 0;
           the hook asserts that the input holds no exact zero, so out == 0 means dropped)
together with the loss, every logits tensor ([b, n, c], as in the eval fixtures) and the gradient of the loss w.r.t.
every parameter.  A gradient is kept as its norm and a seeded sample of GRAD_SAMPLE entries (all of them when it has
fewer; positions from grad_sample_index), which keeps the file small.  Given those masks,
oracle/restatement.loss_and_logits(..., forget_mask=, drop_keeps=) must reproduce the step (tests/test_train_mode_cpu.py).

Cases: the weights and tokens of tests/golden/tiny_coarse.pt (conv FFN, F = 341) and tiny_plainff_t5.pt (plain FFN,
F = 256), each at ff_dropout 0.1 and 0.5, under a fixed torch seed.  The weights are not copied: each case names its
eval fixture and the SHA-256 of the state dict it ran on.

Needs a reference checkout:   OMLM_REFERENCE_ROOT=<checkout> python oracle/make_golden_train.py
"""
import hashlib
import os
import sys
import zlib

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
OUT = os.path.join(GOLD, "train_mode.pt")
SOURCES = ("tiny_coarse", "tiny_plainff_t5")
DROPOUTS = (0.1, 0.5)
MASK_PROB = 0.15
GRAD_SAMPLE = 1024


def grad_sample_index(numel: int, name: str) -> torch.Tensor:
    """The positions of the flattened gradient of parameter `name` that the fixture keeps (seeded by the name)."""
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    return torch.randperm(numel, generator=g)[:min(numel, GRAD_SAMPLE)]


def grad_record(name, grad):
    """None (no gradient), or the gradient's float64 norm and its entries at grad_sample_index."""
    if grad is None:
        return None
    flat = grad.detach().reshape(-1)
    return dict(norm=float(flat.double().norm()), sample=flat[grad_sample_index(flat.numel(), name)].clone())


def state_sha(sd) -> str:
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def record_case(ref, fx, ff_dropout, seed):
    mod = sys.modules["open_musiclm.open_musiclm"]
    kw = dict(fx["kwargs"], ff_dropout=ff_dropout)
    model = {"semantic": ref.create_semantic_transformer, "coarse": ref.create_coarse_transformer,
             "fine": ref.create_fine_transformer}[fx["stage"]](**kw)
    model.load_state_dict(fx["state_dict"], strict=True)
    wrapper = ref.TokenConditionedTransformerWrapper(transformer=model, unique_consecutive=False,
                                                     cross_entropy_loss_weights=fx["ce_weights"], mask_prob=MASK_PROB).train()
    forget = []
    orig = mod.generate_mask_with_prob

    def recording_mask(*a, **k):
        m = orig(*a, **k)
        forget.append(m.clone())
        return m

    keeps = {}
    hooks = []
    for l, layer in enumerate(model.transformer.layers):
        drops = [m for m in layer[2] if isinstance(m, torch.nn.Dropout)]
        assert len(drops) == 1 and drops[0].p == ff_dropout

        def hook(module, inp, out, l=l):
            assert bool((inp[0] != 0).all()), "an exact zero in the dropout input would read as dropped"
            keeps[l] = (out != 0).clone()
        hooks.append(drops[0].register_forward_hook(hook))
    mod.generate_mask_with_prob = recording_mask
    try:
        torch.manual_seed(seed)
        loss, logits, _ = wrapper(all_token_ids=[t.clone() for t in fx["tokens"]], return_loss=True)
        loss.backward()
    finally:
        mod.generate_mask_with_prob = orig
        for h in hooks:
            h.remove()
    assert len(forget) == 1 and len(keeps) == len(model.transformer.layers)
    grads = {k: grad_record(k, p.grad) for k, p in model.named_parameters()}
    return dict(ff_dropout=ff_dropout, mask_prob=MASK_PROB, seed=seed, forget=forget[0],
                keeps=[keeps[l] for l in range(len(keeps))], loss=float(loss.detach()),
                logits=[lg.detach().permute(0, 2, 1).contiguous() for lg in logits], grads=grads)   # [b, n, c]


def main():
    ref = ref_harness.import_reference()
    out = {}
    for i, name in enumerate(SOURCES):
        fx = torch.load(os.path.join(GOLD, f"{name}.pt"), weights_only=False)
        for j, p in enumerate(DROPOUTS):
            case = record_case(ref, fx, p, seed=100 + 10 * i + j)
            case.update(source=name, state_sha=state_sha(fx["state_dict"]))
            out[f"{name}_p{p}"] = case
            print(f"{name} p={p}: train loss {case['loss']:.6f} (eval {float(fx['loss']):.6f}), "
                  f"dropped per row {(~case['forget']).sum(1).tolist()}, kept {float(case['keeps'][0].float().mean()):.3f}")
    torch.save(out, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
