"""Seeded generation without a GPU: the host replica of the seeded sampler stream (csrc/decode.cu sample_kernel with
per-sequence seeds), the splitmix64 window-seed derivation of MusicLM.generate_tokens (open_musiclm_b200/stages.py),
and the seeds every generate call of a batched song receives against the seeds of single-prompt songs.
tests/test_generate_seeded_gpu.py checks the kernels and the decode path against these on an H100."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from test_philox_cpu import _key, philox4x32, sampler_uniforms  # noqa: E402

import open_musiclm_b200 as O  # noqa: E402
from open_musiclm_b200.stages import COARSE, FINE, SEMANTIC, splitmix64, window_seed  # noqa: E402


def seeded_uniforms(seed, step, C):
    """float32 [C]: the uniform behind the Gumbel noise of class c at sample index `step` of a sequence with seed `seed`
    (csrc/decode.cu, omlm_sample_seeded): word x0 of the counter (c, step, 0, 0x5eed) under the key seed (low word
    first), u = (x0 >> 8) / 2^24.  The row of the sequence and the batch size do not enter."""
    x0 = philox4x32(np.arange(C), step, 0, 0x5EED, *_key(seed))[0]
    return ((x0 >> np.uint32(8)).astype(np.float64) / 2.0 ** 24).astype(np.float32)


def test_seeded_stream_is_24_bit_uniform_and_keyed_by_every_argument():
    u = np.stack([seeded_uniforms(12345, t, 1025) for t in range(64)])
    assert u.dtype == np.float32 and u.min() >= 0.0 and u.max() < 1.0
    assert np.array_equal(u * np.float32(2 ** 24), np.floor(u * np.float32(2 ** 24)))
    assert abs(float(u.mean()) - 0.5) < 0.01 and abs(float(u.var()) - 1 / 12) < 0.005
    base = seeded_uniforms(3, 5, 256)
    for other in (seeded_uniforms(4, 5, 256), seeded_uniforms(3 + (1 << 32), 5, 256), seeded_uniforms(3, 6, 256)):
        assert (other != base).mean() > 0.99
    assert (base[:-1] != base[1:]).mean() > 0.99
    # the counter's last words differ from the default stream's (c, b, step, 0x5a17): a seed equal to Engine.seed
    # does not replay the unseeded noise of any row
    for b in range(4):
        assert (sampler_uniforms(3, 5, 4, 256)[b] != base).mean() > 0.99


def test_splitmix64_known_answers():
    """The first outputs of the splitmix64 generator seeded with 0: state += 0x9E3779B97F4A7C15, output = mix(state)."""
    golden = 0x9E3779B97F4A7C15
    assert [splitmix64(i * golden % (1 << 64)) for i in range(3)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]


def test_window_seed_formula_and_spread():
    m = (1 << 64) - 1
    for seed in (0, 1, 2 ** 63 + 5, m):
        for stage in (SEMANTIC, COARSE, FINE):
            for w in (0, 1, 7):
                assert window_seed(seed, stage, w) == splitmix64(seed ^ splitmix64((stage << 32) | w))
    # negative ints are taken modulo 2^64
    assert window_seed(-1, FINE, 3) == window_seed(m, FINE, 3)
    vals = {window_seed(s, st, w) for s in range(8) for st in range(3) for w in range(8)}
    assert len(vals) == 8 * 3 * 8 and all(0 <= v <= m for v in vals)


def test_seeds_tensor_reads_raw_64_bit_patterns():
    from open_musiclm_b200.decode import seeds_tensor
    t = seeds_tensor([0, 1, 2 ** 64 - 1, 2 ** 63, -2], 5, "cpu")
    assert t.dtype == torch.int64 and t.tolist() == [0, 1, -1, -(2 ** 63), -2]
    raw = torch.tensor([-5, 7, 2 ** 62], dtype=torch.int64)
    assert torch.equal(seeds_tensor(raw, 3, "cpu"), raw)
    with pytest.raises(ValueError, match="2 seeds for 3"):
        seeds_tensor([1, 2], 3, "cpu")
    with pytest.raises(ValueError, match="int64"):
        seeds_tensor(torch.tensor([1.0, 2.0, 3.0]), 3, "cpu")


# ------------------------------------------------------------------------------------------------ MusicLM seed plumbing
class RecordingWrapper:
    """generate() of a stage wrapper that records the seeds it is handed and returns tokens that depend only on each
    row's own inputs and seed (so the windowing of a batch and of its single rows follows the same token streams)."""

    def __init__(self, q, codebook, log, name):
        self.q, self.cb, self.log, self.name = q, codebook, log, name
        self.token_sequences = [SimpleNamespace(codebook_size=codebook, num_quantizers=q)] * 3
        self.device = torch.device("cpu")

    def generate(self, *, conditioning_token_ids, pred_token_ids=None, max_time_steps, seeds=None, **kw):
        B = conditioning_token_ids[0].shape[0]
        assert seeds is not None and len(seeds) == B
        self.log.append((self.name, list(seeds)))
        init = 0 if pred_token_ids is None else pred_token_ids.shape[1]
        rows = []
        for b in range(B):
            h = seeds[b]
            for c in conditioning_token_ids:
                for v in c[b].reshape(-1).tolist():
                    h = splitmix64(h ^ (v & 0xFFFFFFFF))
            g = torch.Generator().manual_seed(h & 0x7FFFFFFFFFFFFFFF)
            new = torch.randint(0, self.cb, (max_time_steps - init, self.q), generator=g)
            rows.append(new if pred_token_ids is None else torch.cat([pred_token_ids[b], new], 0))
        return torch.stack(rows, 0)


def _mlm(log):
    wr = dict(semantic=RecordingWrapper(1, 64, log, "semantic"), coarse=RecordingWrapper(3, 64, log, "coarse"),
              fine=RecordingWrapper(5, 64, log, "fine"))
    return O.MusicLM(stages=(O.SemanticStage(semantic_transformer=None, wrapper=wr["semantic"]),
                             O.CoarseStage(coarse_transformer=None, wrapper=wr["coarse"]),
                             O.FineStage(fine_transformer=None, wrapper=wr["fine"])))


ARGS = dict(output_seconds=3, semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5,
            semantic_steps_per_second=6, acoustic_steps_per_second=8)


def test_batched_song_hands_every_call_the_single_prompt_seeds():
    clap = torch.randint(0, 64, (3, 4), generator=torch.Generator().manual_seed(3))
    seeds = [11, 2 ** 64 - 3, 12345678901234567]
    log3 = []
    out3 = _mlm(log3).generate_tokens(clap_token_ids=clap, seeds=seeds, return_all=True, **ARGS)
    singles = []
    for b in range(3):
        log1 = []
        out1 = _mlm(log1).generate_tokens(clap_token_ids=clap[b:b + 1], seeds=torch.tensor([seeds[b]]) if seeds[b] < 2 ** 63 else [seeds[b]],
                                          return_all=True, **ARGS)
        singles.append((log1, out1))
        assert len(log1) == len(log3)
        for (name3, s3), (name1, s1) in zip(log3, log1):
            assert name3 == name1 and s1 == [s3[b]]
        for a, r in zip(out3, out1):
            assert torch.equal(a[b:b + 1], r)
    # the seeds follow window_seed(seed, stage, window index) with one window counter per stage
    counts = {}
    for name, s in log3:
        stage = dict(semantic=SEMANTIC, coarse=COARSE, fine=FINE)[name]
        w = counts.get(stage, 0)
        counts[stage] = w + 1
        assert s == [window_seed(x, stage, w) for x in seeds]
    assert counts[SEMANTIC] >= 2 and counts[COARSE] >= 2 and counts[FINE] >= 2, counts
    # another seed: other calls' seeds and (with this fake) other tokens
    log_other = []
    other = _mlm(log_other).generate_tokens(clap_token_ids=clap[:1], seeds=[12], return_all=True, **ARGS)
    assert all(s != [x[0]] for (_, s), (_, x) in zip(log_other, singles[0][0]))
    assert not torch.equal(other[0], singles[0][1][0])


def test_seeds_argument_errors():
    clap = torch.zeros(2, 4, dtype=torch.int64)
    with pytest.raises(ValueError, match="1 seeds for 2"):
        _mlm([]).generate_tokens(clap_token_ids=clap, seeds=[1], **ARGS)
    with pytest.raises(ValueError, match="exclude"):
        _mlm([]).generate_tokens(clap_token_ids=clap, seeds=[1, 2], noise=O.NoiseStream(torch.rand(10, 2, 65)), **ARGS)
