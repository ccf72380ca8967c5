"""Audio continuation (MusicLM.forward(prime_wave=...)), the coarse-only wave (return_coarse_generated_wave) and best-of-N
sampling (MusicLM.generate_top_match) of open_musiclm_b200/stages.py against what the REAL reference computed with the
same weights, stub tokenizers and noise stream (tests/golden/musiclm_prime.pt, oracle/make_golden_musiclm_prime.py).
As in tests/test_stages_cpu.py the oracle's generate() stands in for the CUDA wrapper, so the comparison is bit-exact;
tests/test_musiclm_prime_gpu.py runs the same fixture through the H100 decode path.  The last test runs the
reference's two inference scripts against this package's MusicLM where a reference checkout is present."""
import os
import runpy
import sys
import types
from types import SimpleNamespace

import pytest
import torch

from oracle import ref_harness
from oracle import restatement as R
import open_musiclm_b200 as O

sys.path.insert(0, os.path.dirname(__file__))
import musiclm_stubs as stubs  # noqa: E402
from test_stages_cpu import OracleWrapper, oracle_cfg  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden")
FX = os.path.join(GOLD, "musiclm_prime.pt")
STAGES = ("semantic", "coarse", "fine")


def load():
    fx = torch.load(FX, weights_only=False)
    win = torch.load(os.path.join(GOLD, fx["weights"]), weights_only=False)
    return fx, win


def make_stubs(fx, case):
    """The stubs the reference ran with (oracle/make_golden_musiclm_prime.py)."""
    r = fx["rates"]
    clap = stubs.Clap(64, 4, torch.randn(8, 6, generator=torch.Generator().manual_seed(77)), r["clap"])
    if case["kind"] == "top_match":
        return None, stubs.Codec(torch.zeros(1, 1, 8, dtype=torch.long), r["codec"]), clap
    return stubs.Wav2Vec(case["sem_ids"], r["wav2vec"]), stubs.Codec(case["acoustic_ids"], r["codec"]), clap


def oracle_musiclm(win, w2v=None, codec=None, clap=None, wrappers=None):
    wr = wrappers or {k: OracleWrapper(oracle_cfg(k, win["kwargs"][k]), win["state_dicts"][k]) for k in STAGES}
    return O.MusicLM(stages=(O.SemanticStage(semantic_transformer=None, wrapper=wr["semantic"]),
                             O.CoarseStage(coarse_transformer=None, wrapper=wr["coarse"]),
                             O.FineStage(fine_transformer=None, wrapper=wr["fine"])), wav2vec=w2v, clap=clap, neural_codec=codec)


def expected_wave(fx, case):
    """The reference's wave; where it could not join its streams (fine condition length > 0), the streams it had,
    with the coarse stream's copy of the fine-conditioning prime tokens dropped (MusicLM.generate_tokens)."""
    if "out" in case:
        return case["out"]
    a = case["args"]
    ta = case["acoustic_ids"].shape[1]
    cond_fine = int(a["acoustic_steps_per_second"] * a["fine_window_seconds"] * (1 - a["fine_sliding_window_step_percent"]))
    assert cond_fine > 0 and "join_error" in case
    coarse = torch.cat([case["coarse"][:, :ta], case["coarse"][:, ta + cond_fine:]], 1)
    assert coarse.shape == case["fine"].shape[:2] + (3,)
    return torch.cat([coarse, case["fine"]], -1).reshape(coarse.shape[0], -1).float()


@pytest.mark.parametrize("name", ["long_prime", "short_prime_fine_cond", "coarse_wave"])
def test_prime_wave_continuation_reproduces_reference(name):
    fx, win = load()
    case = fx["cases"][name]
    w2v, codec, clap = make_stubs(fx, case)
    mlm = oracle_musiclm(win, w2v, codec, clap)
    noise = O.NoiseStream(case["uniforms"])
    out = mlm(text=case["prompts"], prime_wave=fx["prime_wave"], prime_wave_sample_hz=fx["prime_hz"], noise=noise, **case["args"])
    assert noise.at == case["uniforms"].shape[0]                      # the reference's number of sampled tokens
    # the waves handed to the tokenizers: prepare_audio at each tokenizer's rate, bit for bit
    assert len(w2v.seen) == len(codec.seen) == 1
    assert torch.equal(w2v.seen[0], case["wav2vec_seen"][0]) and torch.equal(codec.seen[0], case["codec_seen"][0])
    ref = expected_wave(fx, case)
    assert out.shape == ref.shape and torch.equal(out, ref)


def test_short_prime_with_fine_condition_keeps_every_reference_token():
    """Where the reference fails to join its streams, every token it generated is still in the output, and the output
    starts with the full prime streams."""
    fx, win = load()
    case = fx["cases"]["short_prime_fine_cond"]
    w2v, codec, clap = make_stubs(fx, case)
    mlm = oracle_musiclm(win, w2v, codec, clap)
    prime = mlm.prime_token_ids(fx["prime_wave"], fx["prime_hz"], case["args"]["semantic_window_seconds"])
    acoustic = mlm.generate_tokens(clap_token_ids=clap(text_input=case["prompts"]), noise=O.NoiseStream(case["uniforms"]),
                                   **prime, **case["args"])
    ta = case["acoustic_ids"].shape[1]
    assert torch.equal(acoustic[:, :ta], case["acoustic_ids"])
    assert torch.equal(acoustic[..., 3:], case["fine"])
    assert torch.equal(acoustic[:, ta:, :3], case["coarse"][:, -(acoustic.shape[1] - ta):])


def test_generate_top_match_reproduces_reference():
    fx, win = load()
    case = fx["cases"]["top_match"]
    _, codec, clap = make_stubs(fx, case)
    mlm = oracle_musiclm(win, None, codec, clap)
    batches = []
    for st in (mlm.semantic, mlm.coarse, mlm.fine):
        orig = st.transformer_wrapper.generate

        def shim(orig=orig, **kw):
            batches.append(kw["conditioning_token_ids"][0].shape[0])
            return orig(**kw)
        st.transformer_wrapper.generate = shim
    noise = O.NoiseStream(case["uniforms"])
    waves, sims = mlm.generate_top_match(text=case["prompts"], num_samples=case["num_samples"],
                                         num_top_matches=case["num_top_matches"], noise=noise, **case["args"])
    assert noise.at == case["uniforms"].shape[0]
    assert set(batches) == {case["num_samples"]}                      # one batch of num_samples per prompt
    assert len(clap.seen) == len(case["clap_seen"]) and all(torch.equal(a, b) for a, b in zip(clap.seen, case["clap_seen"]))
    assert len(waves) == len(sims) == len(case["prompts"])
    for w, s, rw, rs in zip(waves, sims, case["waves"], case["sims"]):
        assert torch.equal(w, rw)
        assert s.device.type == "cpu" and s.dtype == torch.float32 and torch.equal(s, rs)


@pytest.mark.parametrize("setting", ["normalized", "plain"])
def test_prepare_audio_matches_reference(setting):
    p = torch.load(FX, weights_only=False)["prepare_audio"]
    got = O.prepare_audio(p["wave"], p["sample_hz"], p["target_hz"], normalize=setting == "normalized",
                          target_length_seconds=p["target_length_seconds"])
    assert got.shape == p[setting].shape and torch.equal(got, p[setting])


def test_continuation_needs_the_tokenizers():
    fx, win = load()
    case = fx["cases"]["long_prime"]
    w2v, codec, clap = make_stubs(fx, case)
    kw = dict(text=case["prompts"], prime_wave=fx["prime_wave"], prime_wave_sample_hz=fx["prime_hz"], **case["args"])
    with pytest.raises(ValueError, match="wav2vec"):
        oracle_musiclm(win, None, codec, clap)(**kw)
    with pytest.raises(ValueError, match="neural_codec"):
        oracle_musiclm(win, w2v, None, clap)(**kw)
    with pytest.raises(ValueError, match="prime_wave_sample_hz"):
        oracle_musiclm(win, w2v, codec, clap)(**dict(kw, prime_wave_sample_hz=None))
    with pytest.raises(ValueError, match="clap and neural_codec"):
        oracle_musiclm(win, w2v, None, clap).generate_top_match(text=["x"], num_samples=2)
    assert not w2v.seen and not codec.seen                            # nothing was tokenized, nothing generated


def test_prime_token_shapes_are_checked():
    fx, win = load()
    mlm = oracle_musiclm(win)
    clap_ids = torch.zeros(2, 4, dtype=torch.long)
    good = dict(prime_semantic_token_ids=torch.zeros(1, 5, 1, dtype=torch.long), prime_coarse_token_ids=torch.zeros(1, 4, 3, dtype=torch.long),
                prime_fine_token_ids=torch.zeros(1, 4, 5, dtype=torch.long))
    with pytest.raises(ValueError, match="all three"):
        mlm.generate_tokens(clap_token_ids=clap_ids, prime_semantic_token_ids=good["prime_semantic_token_ids"])
    with pytest.raises(ValueError, match=r"\[1 or 2, T, 3\]"):
        mlm.generate_tokens(clap_token_ids=clap_ids, **dict(good, prime_coarse_token_ids=torch.zeros(3, 4, 3, dtype=torch.long)))
    with pytest.raises(ValueError, match=r"\[1 or 2, T, 5\]"):
        mlm.generate_tokens(clap_token_ids=clap_ids, **dict(good, prime_fine_token_ids=torch.zeros(1, 4, 8, dtype=torch.long)))


# ------------------------------------------------------------------------------------ the reference's inference scripts
class _SampledOracle(OracleWrapper):
    """The oracle wrapper drawing its Gumbel noise from torch's default generator, as the reference does."""

    def generate(self, *, conditioning_token_ids, pred_token_ids=None, max_time_steps, filter_thres=0.9, temperature=1.0,
                 include_eos_in_output=False, append_eos_to_conditioning_tokens=True, uniform_noise=None):
        return R.generate(self.cfg, self.sd, [t.numpy() for t in conditioning_token_ids], lambda s, shape: torch.rand(shape),
                          pred_token_ids=None if pred_token_ids is None else pred_token_ids.numpy(), max_time_steps=max_time_steps,
                          filter_thres=filter_thres, temperature=temperature, include_eos_in_output=include_eos_in_output)


SCRIPT_RUNS = [("infer.py", []), ("infer.py", ["--return_coarse_wave"]),
               ("infer_top_match.py", ["a song", "--num_samples", "2", "--input_audio", "prime.wav"]),
               ("infer_top_match.py", ["a song", "--num_samples", "2", "--input_audio", "prime.wav", "--return_coarse_wave"])]


@pytest.mark.skipif(not ref_harness.available(), reason="needs a reference checkout (OMLM_REFERENCE_ROOT)")
@pytest.mark.parametrize("script,extra", SCRIPT_RUNS, ids=["infer", "infer-coarse", "top_match-prime", "top_match-prime-coarse"])
def test_reference_inference_scripts_run_on_this_musiclm(script, extra, tmp_path, monkeypatch):
    """The reference's scripts/infer.py and scripts/infer_top_match.py, unchanged, with create_musiclm_from_config
    returning this package's MusicLM over tiny random-weight oracle-backed stages and the stub tokenizers.  Audio
    files are read and written through stand-ins for torchaudio.load / torchaudio.save."""
    import torchaudio
    win = torch.load(os.path.join(GOLD, "musiclm_windows.pt"), weights_only=False)
    wr = {k: _SampledOracle(oracle_cfg(k, win["kwargs"][k]), R.init_state(oracle_cfg(k, win["kwargs"][k]), seed=i))
          for i, k in enumerate(STAGES)}
    g = torch.Generator().manual_seed(1)
    w2v = stubs.Wav2Vec(torch.randint(0, 64, (1, 9), generator=g), 60)
    codec = stubs.Codec(torch.randint(0, 64, (1, 7, 8), generator=g), 80)
    clap = stubs.Clap(64, 4, torch.randn(8, 6, generator=g), 50)
    mlm = oracle_musiclm(win, w2v, codec, clap, wrappers=wr)
    cfg = SimpleNamespace(global_cfg=SimpleNamespace(semantic_audio_length_seconds=2, coarse_audio_length_seconds=1,
                                                     fine_audio_length_seconds=0.5),
                          hubert_kmeans_cfg=SimpleNamespace(output_hz=6), encodec_cfg=SimpleNamespace(output_hz=8))
    config = types.ModuleType("open_musiclm.config")
    config.load_model_config = lambda path: cfg
    config.create_musiclm_from_config = lambda **kw: mlm
    pkg = types.ModuleType("open_musiclm")
    pkg.__path__ = []
    monkeypatch.setitem(sys.modules, "open_musiclm", pkg)
    monkeypatch.setitem(sys.modules, "open_musiclm.config", config)
    saved = []
    monkeypatch.setattr(torchaudio, "save", lambda path, wave, rate: saved.append((str(path), tuple(wave.shape), rate)))
    monkeypatch.setattr(torchaudio, "load", lambda path: (torch.randn(2, 250, generator=torch.Generator().manual_seed(2)), 100))
    monkeypatch.chdir(tmp_path)
    (tmp_path / "results").mkdir()
    monkeypatch.setattr(sys, "argv", [script, "--semantic_path", "s.pt", "--coarse_path", "c.pt", "--fine_path", "f.pt",
                                      "--duration", "3"] + extra)
    runpy.run_path(os.path.join(ref_harness.REF_ROOT, "scripts", script), run_name="__main__")
    # 3 s at 6 semantic / 8 acoustic steps per second through 2 s / 1 s / 0.5 s windows: 7 coarse windows, 32 acoustic
    # steps.  Continuing a prime, the semantic stream loses 3 steps (6 coarse windows: 28 coarse steps), the coarse
    # stream 4 more, and the 7-step prime goes in front: 31 steps.
    steps = (28 if "--return_coarse_wave" in extra else 31) if "--input_audio" in extra else 32
    q = 3 if "--return_coarse_wave" in extra else 8
    assert {s for _, s, _ in saved} == {(1, steps * q)} and all(r == 80 for _, _, r in saved)
    if script == "infer.py":
        assert len(saved) == 12                                          # 3 batches of 4 prompts
    else:
        assert len(saved) == 1 and len(w2v.seen) == len(codec.seen) == 1
