"""ORACLE — test infrastructure only.  Golden token log-probabilities of the REAL reference's generate
(TokenConditionedTransformerWrapper.generate, open_musiclm.py:253-326) on the gen_* cases of make_golden_generate.py,
under the same fixed Gumbel noise stream.

Needs a reference checkout:   OMLM_REFERENCE_ROOT=<checkout> python oracle/make_golden_logprobs.py
The reference's transformer is wrapped so that every call's final-sequence logits are recorded: the first call's rows
give the prefix tokens' log-softmax (row i predicts token i of the predicted sequence), and every call's last row,
before the eos masking, is the raw row of one sampled token.  The sampled token is recovered from the recorded uniforms
with the reference's own top_k (utils.py:78-84) and Gumbel argmax (utils.py:71-76).  Fixture tests/golden/logprobs_<case>.pt:
the gen_* fixture's inputs and output (its state_dict stays in tests/golden/<case>.pt, named by "weights") plus
  rows [n_new, B, C]            raw logits rows of the sampled tokens,
  sampled [n_new, B]            the sampled tokens (before the after-eos masking),
  logprobs [n_new, B]           log_softmax(row)[token],
  sample_logprobs [n_new, B]    log_softmax(top_k(masked row, thres) / T)[token],
  prefix_rows [B, n_prefix, C]  the first call's rows of the prefix positions (row i predicts prefix token i),
  prefix_logprobs [B, n_prefix] log_softmax of those rows at the prefix tokens (None without a prefix).
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402
from oracle.make_golden import COMMON, GOLD, build  # noqa: E402
from oracle.make_golden_generate import CASES, SEED  # noqa: E402


def main():
    ref = ref_harness.import_reference()
    utils = sys.modules[ref.__name__.rsplit(".", 1)[0] + ".utils"]
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
        calls = []
        forward = model.forward

        def recording(*a, **k):
            out = forward(*a, **k)
            calls.append(out[-1].detach().clone())
            return out
        model.forward = recording
        torch.manual_seed(SEED)
        out = wrapper.generate(conditioning_token_ids=[t.clone() for t in cond], pred_token_ids=None if prefix is None else prefix.clone(),
                               max_time_steps=steps, temperature=temp, allow_eos_in_output=allow_eos, include_eos_in_output=allow_eos)
        model.forward = forward
        torch.manual_seed(SEED)
        uniforms = torch.stack([torch.zeros(B, C).uniform_(0, 1) for _ in range(n_new)])
        assert len(calls) == n_new
        rows = torch.stack([c[:, -1] for c in calls])
        n_pre = 0 if prefix is None else prefix[0].numel()
        sampled, lp, slp = [], [], []
        for s in range(n_new):
            masked = rows[s].clone()
            if not allow_eos or (n_pre + s) % q != q - 1:
                masked[:, -1] = float("-inf")
            filt = utils.top_k(masked, thres=0.9)
            tok = (filt / temp + (-torch.log(-torch.log(uniforms[s])))).argmax(-1)
            sampled.append(tok)
            lp.append(torch.log_softmax(rows[s].double(), -1).gather(1, tok[:, None])[:, 0])
            slp.append(torch.log_softmax(filt.double() / temp, -1).gather(1, tok[:, None])[:, 0])
        sampled = torch.stack(sampled)
        flat = torch.cat([prefix.reshape(B, -1) if prefix is not None else torch.empty(B, 0, dtype=torch.long), sampled.t()], 1)
        gen = torch.load(os.path.join(GOLD, f"{name}.pt"), weights_only=False)      # the same weights: stored there once
        assert all(torch.equal(v, gen["state_dict"][k]) for k, v in model.state_dict().items())
        fx = {"stage": stage, "kwargs": dict(kw, **COMMON), "weights": f"{name}.pt",
              "cond": cond, "prefix": prefix, "max_time_steps": steps, "temperature": temp, "filter_thres": 0.9,
              "allow_eos_in_output": allow_eos, "include_eos_in_output": allow_eos, "uniforms": uniforms, "out": out,
              "rows": rows, "sampled": sampled, "logprobs": torch.stack(lp), "sample_logprobs": torch.stack(slp),
              "prefix_rows": None if prefix is None else calls[0][:, :n_pre].clone(),
              "prefix_logprobs": None if prefix is None else
              torch.log_softmax(calls[0][:, :n_pre].double(), -1).gather(2, flat[:, :n_pre, None])[..., 0]}
        path = os.path.join(GOLD, name.replace("gen_", "logprobs_") + ".pt")
        torch.save(fx, path)
        print(name, "->", path, os.path.getsize(path) // 1024, "KiB", fx["logprobs"][:3, 0].tolist())


if __name__ == "__main__":
    main()
