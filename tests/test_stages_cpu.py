"""The stage wrappers and the three-stage sliding-window generation (open_musiclm_b200/stages.py) against the token
output of the REAL reference's MusicLM.forward (tests/golden/musiclm_windows.pt, oracle/make_golden_musiclm.py).
The window bookkeeping is host logic: here it runs on CPU with the oracle's generate() standing in for the CUDA
wrapper, so the comparison is bit-exact; tests/test_decode_gpu.py runs the same fixture through the H100 decode path."""
import os
from types import SimpleNamespace

import pytest
import torch

from oracle import restatement as R
import open_musiclm_b200 as O

FX = os.path.join(os.path.dirname(__file__), "golden", "musiclm_windows.pt")


def oracle_cfg(stage, kw):
    base = dict(dim=kw["dim"], depth=kw["depth"], heads=kw["heads"], codebook=kw["clap_codebook_size"], n_clap_q=kw["num_clap_quantizers"])
    if stage == "semantic":
        return R.semantic_cfg(**base)
    if stage == "coarse":
        return R.coarse_cfg(n_coarse_q=kw["num_coarse_quantizers"], **base)
    return R.fine_cfg(n_coarse_q=kw["num_coarse_quantizers"], n_fine_q=kw["num_fine_quantizers"], **base)


class OracleWrapper:
    """Same generate() contract as TokenConditionedTransformerWrapper, computed by the CPU oracle."""

    def __init__(self, cfg, sd):
        self.cfg, self.sd = cfg, sd
        self.token_sequences = [SimpleNamespace(codebook_size=s.codebook_size, num_quantizers=s.num_quantizers) for s in cfg.seqs]
        self.device = torch.device("cpu")
        self.min_gap = float("inf")

    def generate(self, *, conditioning_token_ids, pred_token_ids=None, max_time_steps, filter_thres=0.9, temperature=1.0,
                 include_eos_in_output=False, append_eos_to_conditioning_tokens=True, uniform_noise=None):
        assert append_eos_to_conditioning_tokens
        out, trace = R.generate(self.cfg, self.sd, [t.numpy() for t in conditioning_token_ids], lambda s, shape: uniform_noise[s],
                                pred_token_ids=None if pred_token_ids is None else pred_token_ids.numpy(), max_time_steps=max_time_steps,
                                filter_thres=filter_thres, temperature=temperature, include_eos_in_output=include_eos_in_output,
                                return_trace=True)
        for _, gap in trace:
            self.min_gap = min(self.min_gap, float(gap.min()))
        return out


def test_three_stage_windowing_reproduces_reference_tokens():
    fx = torch.load(FX, weights_only=False)
    wr = {k: OracleWrapper(oracle_cfg(k, fx["kwargs"][k]), fx["state_dicts"][k]) for k in ("semantic", "coarse", "fine")}
    stages = (O.SemanticStage(semantic_transformer=None, wrapper=wr["semantic"]), O.CoarseStage(coarse_transformer=None, wrapper=wr["coarse"]),
              O.FineStage(fine_transformer=None, wrapper=wr["fine"]))
    mlm = O.MusicLM(stages=stages)
    noise = O.NoiseStream(fx["uniforms"])
    out, sem, coarse, fine = mlm.generate_tokens(clap_token_ids=fx["clap_ids"], noise=noise, return_all=True, **fx["args"])
    assert noise.at == fx["uniforms"].shape[0]                       # exactly the reference's number of sampled tokens
    assert out.shape == fx["out"].shape and torch.equal(out, fx["out"])
    assert coarse.shape[-1] == 3 and fine.shape[-1] == 5 and sem.shape[-1] == 1
    print("smallest top-2 gap along the trajectory:", min(w.min_gap for w in wr.values()))


def test_window_helper_matches_unfold():
    from open_musiclm_b200.stages import _windows
    t = torch.arange(2 * 23 * 3).view(2, 23, 3)
    for size, step in [(5, 2), (7, 7), (23, 4), (4, 1)]:
        ref = t.unfold(1, size, step).permute(1, 0, 3, 2)           # 'b n q w -> n b w q'
        got = _windows(t, size, step)
        assert len(got) == ref.shape[0] and all(torch.equal(a, b) for a, b in zip(got, ref))
