"""ORACLE — test infrastructure only.  Golden token output of the REAL reference's three-stage windowed generation
(MusicLM.forward, open_musiclm.py:860-1035: semantic -> coarse -> fine with sliding windows) on tiny random-weight
stage transformers, under a fixed Gumbel noise stream.

Needs a reference checkout:   OMLM_REFERENCE_ROOT=<checkout> python oracle/make_golden_musiclm.py
CLAP and the neural codec do not exist here (SURVEY 8c); they are replaced by stubs that (a) return fixed clap token ids
for the text and (b) "decode" by returning the acoustic token ids themselves, so the fixture's output is the [b, T, 8]
token tensor the reference hands to the codec.  The fixture stores the three state_dicts, the clap ids, the windowing
arguments, the uniform draws behind every sampled token (in order) and the reference's output.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402
from oracle.make_golden import COMMON, GOLD  # noqa: E402

KW = dict(dim=64, depth=1, heads=2, clap_codebook_size=64, num_clap_quantizers=4)
STAGES = {
    "semantic": dict(KW, semantic_codebook_size=64),
    "coarse": dict(KW, semantic_codebook_size=64, acoustic_codebook_size=64, num_coarse_quantizers=3),
    "fine": dict(KW, acoustic_codebook_size=64, num_coarse_quantizers=3, num_fine_quantizers=5),
}
# tiny "sample rates": 6 semantic and 8 acoustic steps per second, 3 s of output through 2 s / 1 s / 0.5 s windows
ARGS = dict(output_seconds=3, semantic_window_seconds=2, coarse_window_seconds=1, fine_window_seconds=0.5,
            semantic_steps_per_second=6, acoustic_steps_per_second=8)


class _Clap:
    def __init__(self, ids):
        self.ids = ids

    def __call__(self, text_input=None, audio_input=None, **kw):
        return self.ids.clone()


class _Codec:
    def decode_from_codebook_indices(self, ids):
        return ids.reshape(ids.shape[0], 1, -1).float()


def main():
    ref = ref_harness.import_reference()
    utils = sys.modules["open_musiclm.utils"]
    models = {}
    torch.manual_seed(0)
    for name, kw in STAGES.items():
        fn = {"semantic": ref.create_semantic_transformer, "coarse": ref.create_coarse_transformer, "fine": ref.create_fine_transformer}[name]
        models[name] = fn(**dict(COMMON, **kw))
    B = 2
    clap_ids = torch.randint(0, 64, (B, 4), generator=torch.Generator().manual_seed(5))
    mlm = ref.MusicLM(wav2vec=None, clap=_Clap(clap_ids), neural_codec=_Codec(), semantic_transformer=models["semantic"],
                      coarse_transformer=models["coarse"], fine_transformer=models["fine"])
    # count the draws: wrap gumbel_noise (every sampled token calls it once with the [b, 65] logits)
    draws = []
    orig = utils.gumbel_noise

    def counting(t):
        draws.append(tuple(t.shape))
        return orig(t)
    om = sys.modules["open_musiclm.open_musiclm"]
    # pick, among a few seeds, the noise stream whose trajectory has the widest smallest gap between the best and the
    # second-best noisy score (measured with the oracle-backed stages): a 16-bit replay then samples the same tokens
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import open_musiclm_b200 as O
    from test_stages_cpu import OracleWrapper, oracle_cfg
    best = None
    for seed in range(100, 124):
        draws.clear()
        utils.gumbel_noise = counting
        om.gumbel_sample.__globals__["gumbel_noise"] = counting
        torch.manual_seed(seed)
        wave = mlm(text=["x"] * B, **ARGS)
        utils.gumbel_noise = orig
        om.gumbel_sample.__globals__["gumbel_noise"] = orig
        assert all(d == (B, 65) for d in draws)
        torch.manual_seed(seed)
        uniforms = torch.stack([torch.zeros(B, 65).uniform_(0, 1) for _ in range(len(draws))])
        wr = {k: OracleWrapper(oracle_cfg(k, dict(COMMON, **STAGES[k])), {n: v.detach() for n, v in models[k].state_dict().items()})
              for k in STAGES}
        mine = O.MusicLM(stages=(O.SemanticStage(semantic_transformer=None, wrapper=wr["semantic"]),
                                 O.CoarseStage(coarse_transformer=None, wrapper=wr["coarse"]),
                                 O.FineStage(fine_transformer=None, wrapper=wr["fine"])))
        out = mine.generate_tokens(clap_token_ids=clap_ids, noise=O.NoiseStream(uniforms), **ARGS)
        assert torch.equal(out, wave.long().view(B, -1, 8))
        gap = min(w.min_gap for w in wr.values())
        print("seed", seed, "draws", len(draws), "smallest gap", round(gap, 4))
        if best is None or gap > best[3]:
            best = (seed, wave.clone(), uniforms, gap)
    seed, wave, uniforms = best[:3]
    out = wave.long().view(B, -1, 8)
    fx = {"kwargs": {k: dict(COMMON, **kw) for k, kw in STAGES.items()},
          "state_dicts": {k: {n: v.detach().clone() for n, v in m.state_dict().items()} for k, m in models.items()},
          "clap_ids": clap_ids, "args": ARGS, "uniforms": uniforms, "out": out, "seed": seed}
    path = os.path.join(GOLD, "musiclm_windows.pt")
    torch.save(fx, path)
    print("musiclm_windows", tuple(out.shape), "draws", len(uniforms), "->", path, os.path.getsize(path) // 1024, "KiB")
    print(out[0, :4].tolist())


if __name__ == "__main__":
    main()
