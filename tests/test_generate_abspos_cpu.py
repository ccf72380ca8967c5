"""Pins the oracle restatement's generate with absolute position embeddings (oracle/restatement.py, Cfg.abs_pos)
against the token sequences the REAL reference's generate produced under a fixed Gumbel noise stream
(tests/golden/abspos_gen_*.pt, tools/make_golden_generate_abspos.py).  The GPU decode path is compared against the
same fixtures in tests/test_generate_abspos_gpu.py."""
import dataclasses
import glob
import os

import pytest
import torch

from oracle import restatement as R

ABS_GEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "abspos_gen_*.pt")))


def abspos_cfg(fx):
    """The oracle configuration of an abspos_gen_*.pt fixture."""
    kw = fx["kwargs"]
    base = dict(dim=kw["dim"], depth=kw["depth"], heads=kw["heads"], codebook=kw["clap_codebook_size"],
                n_clap_q=kw["num_clap_quantizers"], abs_pos=True, max_abs_pos=kw["max_absolute_position_embeddings"])
    if fx["stage"] == "semantic":
        return R.semantic_cfg(**base)
    if fx["stage"] == "coarse":
        return R.coarse_cfg(n_coarse_q=kw["num_coarse_quantizers"], **base)
    return R.fine_cfg(n_coarse_q=kw["num_coarse_quantizers"], n_fine_q=kw["num_fine_quantizers"], **base)


def test_abspos_fixtures_exist():
    names = {os.path.basename(p) for p in ABS_GEN}
    assert {"abspos_gen_coarse.pt", "abspos_gen_fine_eos.pt", "abspos_gen_coarse_b20.pt"} <= names


@pytest.mark.parametrize("path", ABS_GEN, ids=[os.path.basename(p) for p in ABS_GEN])
def test_generate_restatement_with_absolute_positions_reproduces_reference_tokens(path):
    """oracle.generate with abs_pos=True against the reference's tokens: bit-exact."""
    fx = torch.load(path, weights_only=False)
    cfg = abspos_cfg(fx)
    assert fx["kwargs"]["use_absolute_position_embeddings"]
    uni = fx["uniforms"]
    out = R.generate(cfg, fx["state_dict"], [t.numpy() for t in fx["cond"]], lambda step, shape: uni[step],
                     pred_token_ids=None if fx["prefix"] is None else fx["prefix"].numpy(), max_time_steps=fx["max_time_steps"],
                     filter_thres=fx["filter_thres"], temperature=fx["temperature"],
                     include_eos_in_output=fx["include_eos_in_output"], allow_eos_in_output=fx["allow_eos_in_output"])
    assert out.shape == fx["out"].shape and torch.equal(out, fx["out"])
    # without the position rows the restatement leaves the reference's trajectory
    plain = R.generate(dataclasses.replace(cfg, abs_pos=False), fx["state_dict"], [t.numpy() for t in fx["cond"]],
                       lambda step, shape: uni[step], pred_token_ids=None if fx["prefix"] is None else fx["prefix"].numpy(),
                       max_time_steps=fx["max_time_steps"], filter_thres=fx["filter_thres"], temperature=fx["temperature"],
                       include_eos_in_output=fx["include_eos_in_output"], allow_eos_in_output=fx["allow_eos_in_output"])
    assert not torch.equal(plain, fx["out"])


def test_fixture_position_tables_are_just_large_enough():
    """Each fixture's max_absolute_position_embeddings equals the longest sequence its generate feeds through the
    model: a conditioning sequence with its eos, or prefix + n_new - 1 predicted tokens."""
    for path in ABS_GEN:
        fx = torch.load(path, weights_only=False)
        B = fx["cond"][0].shape[0]
        q = fx["out"].shape[2]
        n_cond = [t.reshape(B, -1).shape[1] + 1 for t in fx["cond"]]
        init = 0 if fx["prefix"] is None else fx["prefix"].shape[1]
        n_pred = init * q + (fx["max_time_steps"] - init) * q - 1
        assert fx["kwargs"]["max_absolute_position_embeddings"] == max(n_cond + [n_pred]), os.path.basename(path)
