"""Audio continuation, the coarse-only wave and best-of-N sampling (open_musiclm_b200/stages.py) on the H100 prefill +
KV-cache decode path: the reference's tokens of tests/golden/musiclm_prime.pt (oracle/make_golden_musiclm_prime.py),
a batch-1 prime broadcast to many prompts under per-prompt seeds, and generate_top_match as one batch per prompt."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(__file__))

from test_musiclm_prime_cpu import expected_wave, load, make_stubs, oracle_musiclm  # noqa: E402


def h100_musiclm(win, w2v=None, codec=None, clap=None):
    import open_musiclm_b200 as O
    fns = {"semantic": O.create_semantic_transformer, "coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer}
    models = {}
    for k, fn in fns.items():
        m = fn(**win["kwargs"][k]); m.load_state_dict(win["state_dicts"][k], strict=True); models[k] = m.cuda().eval()
    return O.MusicLM(semantic_transformer=models["semantic"], coarse_transformer=models["coarse"], fine_transformer=models["fine"],
                     wav2vec=w2v, clap=clap, neural_codec=codec)


def log_generate(mlm, log, gaps=None):
    """Record the new tokens of every generate call ([b, n_new]); for the oracle-backed chain also the gap between the
    best and second-best noisy score of each of them."""
    from oracle import restatement as R
    for st in (mlm.semantic, mlm.coarse, mlm.fine):
        w = st.transformer_wrapper
        orig = w.generate

        def shim(orig=orig, w=w, **kw):
            if gaps is None:
                out = orig(**kw)
            else:
                out, trace = R.generate(w.cfg, w.sd, [t.numpy() for t in kw["conditioning_token_ids"]],
                                        lambda s, shape: kw["uniform_noise"][s],
                                        pred_token_ids=None if kw.get("pred_token_ids") is None else kw["pred_token_ids"].numpy(),
                                        max_time_steps=kw["max_time_steps"], filter_thres=kw.get("filter_thres", 0.9),
                                        temperature=kw.get("temperature", 1.0), return_trace=True)
                gaps.append(torch.stack([g for _, g in trace], 1) if trace else None)
            init = 0 if kw.get("pred_token_ids") is None else kw["pred_token_ids"].shape[1]
            log.append(out[:, init:].reshape(out.shape[0], -1).cpu())
            return out
        w.generate = shim


def run_case(mlm, fx, case, noise):
    if case["kind"] == "forward":
        return mlm(text=case["prompts"], prime_wave=fx["prime_wave"].cuda(), prime_wave_sample_hz=fx["prime_hz"], noise=noise,
                   **case["args"])
    return mlm.generate_top_match(text=case["prompts"], num_samples=case["num_samples"], num_top_matches=case["num_top_matches"],
                                  noise=noise, **case["args"])


@pytest.mark.parametrize("name", ["long_prime", "short_prime_fine_cond", "coarse_wave", "top_match"])
def test_prime_fixtures_on_the_decode_path(name):
    """The reference's tokens under its noise stream, up to the first draw where the oracle's best and second-best noisy
    scores are within 5e-2 (from there the cascaded streams legitimately differ), as in
    tests/test_decode_gpu.py::test_three_stage_windowed_generation_on_the_decode_path."""
    import open_musiclm_b200 as O
    fx, win = load()
    case = fx["cases"][name]
    mlm = h100_musiclm(win, *make_stubs(fx, case))
    log = []
    log_generate(mlm, log)
    noise = O.NoiseStream(case["uniforms"])
    out = run_case(mlm, fx, case, noise)
    assert noise.at == case["uniforms"].shape[0]
    if case["kind"] == "forward":
        same = torch.equal(out.cpu(), expected_wave(fx, case))
    else:
        waves, sims = out
        same = all(torch.equal(w.cpu(), r) for w, r in zip(waves, case["waves"]))
        if same:
            for s, r in zip(sims, case["sims"]):
                assert s.device.type == "cpu" and torch.allclose(s, r, rtol=1e-4, atol=1e-5), (s, r)
    if same:
        print(name, ": all tokens identical to the reference's")
        return
    olog, gaps = [], []
    ref_chain = oracle_musiclm(win, *make_stubs(fx, case))
    log_generate(ref_chain, olog, gaps)
    if case["kind"] == "forward":
        ref_chain(text=case["prompts"], prime_wave=fx["prime_wave"], prime_wave_sample_hz=fx["prime_hz"],
                  noise=O.NoiseStream(case["uniforms"]), **case["args"])
    else:
        ref_chain.generate_top_match(text=case["prompts"], num_samples=case["num_samples"], num_top_matches=case["num_top_matches"],
                                     noise=O.NoiseStream(case["uniforms"]), **case["args"])
    for call, (mine, ref, gap) in enumerate(zip(log, olog, gaps)):
        if torch.equal(mine, ref):
            continue
        diff = (mine != ref).nonzero()
        b, s = (int(v) for v in diff[diff[:, 1].argmin()])
        assert float(gap[b, s]) < 5e-2, ("generate call", call, "sequence", b, "token", s, "gap", float(gap[b, s]))
        print(f"{name}: left the reference trajectory in generate call {call} at a near tie (gap {float(gap[b, s]):.3e})")
        return
    raise AssertionError("outputs differ but every generate call matched the oracle's")


@pytest.mark.parametrize("b", [3, 20])
def test_seeded_prime_broadcast_equals_single_prompt_runs(b):
    """A batch-1 prime continued by b prompts in one batch: the streams of prompt i are, bit for bit, those of prompt i
    continuing the same prime alone with seeds[i]."""
    fx, win = load()
    case = fx["cases"]["long_prime"]
    w2v, codec, clap = make_stubs(fx, case)
    mlm = h100_musiclm(win, w2v, codec, clap)
    prime = mlm.prime_token_ids(fx["prime_wave"].cuda(), fx["prime_hz"], case["args"]["semantic_window_seconds"])
    assert prime["prime_semantic_token_ids"].shape[0] == 1
    clap_ids = torch.randint(0, 64, (b, 4), generator=torch.Generator().manual_seed(b)).cuda()
    seeds = [1000003 * i + 7 for i in range(b)]
    batch = mlm.generate_tokens(clap_token_ids=clap_ids, seeds=seeds, return_all=True, **prime, **case["args"])
    ta = case["acoustic_ids"].shape[1]
    assert torch.equal(batch[0][:, :ta].cpu(), case["acoustic_ids"].expand(b, -1, -1))    # the prime comes first
    for i in range(b):
        one = mlm.generate_tokens(clap_token_ids=clap_ids[i:i + 1], seeds=[seeds[i]], return_all=True, **prime, **case["args"])
        for a, r in zip(batch, one):
            assert torch.equal(a[i:i + 1], r), i
    assert not torch.equal(batch[0][0, ta:], batch[0][1, ta:])


def test_generate_top_match_runs_one_batch_per_prompt():
    """generate_top_match(num_samples=4) with a prime and seeds: every generate call holds the 4 samples of one prompt,
    the scores come back sorted on the CPU, and the same seeds give the same result."""
    fx, win = load()
    case = fx["cases"]["long_prime"]
    w2v, codec, clap = make_stubs(fx, case)
    mlm = h100_musiclm(win, w2v, codec, clap)
    batches = []
    for st in (mlm.semantic, mlm.coarse, mlm.fine):
        orig = st.transformer_wrapper.generate

        def shim(orig=orig, **kw):
            batches.append(kw["conditioning_token_ids"][0].shape[0])
            return orig(**kw)
        st.transformer_wrapper.generate = shim
    prompts = ["song with synths and flute", "beethoven piano sonata"]
    kw = dict(text=prompts, num_samples=4, num_top_matches=3, prime_wave=fx["prime_wave"].cuda(), prime_wave_sample_hz=fx["prime_hz"],
              seeds=[11, 12, 13, 14], **case["args"])
    waves, sims = mlm.generate_top_match(**kw)
    per_prompt = len(batches) // len(prompts)
    assert set(batches) == {4} and per_prompt * len(prompts) == len(batches)
    assert per_prompt == 2 + 6 + 6                                   # semantic, coarse and fine windows of one song
    assert len(waves) == len(sims) == 2
    for w, s in zip(waves, sims):
        assert w.shape[0] == 3 and s.shape == (3,) and s.device.type == "cpu" and bool((s[:-1] >= s[1:]).all())
    again = mlm.generate_top_match(**kw)
    assert all(torch.equal(a, b) for a, b in zip(waves, again[0])) and all(torch.equal(a, b) for a, b in zip(sims, again[1]))
