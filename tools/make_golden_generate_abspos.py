"""Records tests/golden/abspos_gen_*.pt: the REAL reference's generate on models trained with per-sequence absolute
position embeddings (use_absolute_position_embeddings=True, open_musiclm.py:134-136), so that the KV-cache decode step's
position rows are pinned against it.  The recipe is oracle/make_golden_generate.py's -- same seeds, same perturbed
gammas / scales, same recorded Gumbel-noise stream -- run on these cases only, so that the existing gen_*.pt fixtures are
not rewritten.  The files are named abspos_gen_* rather than gen_*: the tests that glob gen_*.pt build their oracle
configuration without absolute positions.

max_absolute_position_embeddings is set just large enough for each case: the largest of every conditioning sequence's
length with its eos and prefix + n_new - 1 (the last sampled token is never fed back).

Needs a reference checkout:   OMLM_REFERENCE_ROOT=<checkout> python tools/make_golden_generate_abspos.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_generate as G  # noqa: E402

ABS = dict(use_absolute_position_embeddings=True)
CASES = {
    # name: (stage, kwargs, conditioning shapes, prefix shape, max_time_steps, temperature, allow_eos)
    # coarse (q = 3) with a 2-step prefix: the first fed-back token is token 6 of the predicted sequence.
    # conditioning 5 and 12 tokens, predicted 6 + 24 - 1 = 29.  d = 64 keeps the fixture small; two layers
    "abspos_gen_coarse": ("coarse", dict(dim=64, depth=2, heads=2, clap_codebook_size=64, semantic_codebook_size=64,
                                         acoustic_codebook_size=64, num_clap_quantizers=4, num_coarse_quantizers=3,
                                         max_absolute_position_embeddings=29, **ABS),
                          [(2, 4), (2, 11)], (2, 2, 3), 10, 0.95, False),
    # fine (q = 5), eos allowed: conditioning 5 and 19 tokens, predicted 0 + 25 - 1 = 24; the last fed-back token is
    # quantizer 3 of the last time step
    "abspos_gen_fine_eos": ("fine", dict(dim=64, depth=1, heads=3, clap_codebook_size=64, acoustic_codebook_size=64,
                                         num_clap_quantizers=4, num_coarse_quantizers=3, num_fine_quantizers=5,
                                         max_absolute_position_embeddings=24, **ABS),
                            [(2, 4), (2, 6, 3)], None, 5, 1.0, True),
    # 20 sequences: the tensor-core decode path.  Conditioning 5 and 12 tokens, predicted 6 + 24 - 1 = 29
    "abspos_gen_coarse_b20": ("coarse", dict(dim=64, depth=1, heads=3, clap_codebook_size=64, semantic_codebook_size=64,
                                             acoustic_codebook_size=64, num_clap_quantizers=4, num_coarse_quantizers=3,
                                             max_absolute_position_embeddings=29, **ABS),
                              [(20, 4), (20, 11)], (20, 2, 3), 10, 0.95, False),
}

if __name__ == "__main__":
    G.CASES = CASES
    G.main()
