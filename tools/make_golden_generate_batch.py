"""Records tests/golden/gen_coarse_b20.pt: the REAL reference's generate with 20 sequences (more than the 16 the SIMT
decode kernels serve), so that test_generate_matches_reference_tokens_under_fixed_noise also covers the batched decode
path (csrc/decode_gemm.cu, attn_decode_mqa).  The recipe is oracle/make_golden_generate.py's -- same seeds, same
perturbed gammas / scales, same recorded Gumbel-noise stream -- run on this one case only, so that the existing gen_*.pt
fixtures are not rewritten.  The model is kept small (d = 64, one layer) to keep the fixture small.

Needs a reference checkout:   OMLM_REFERENCE_ROOT=<checkout> python tools/make_golden_generate_batch.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_generate as G  # noqa: E402

CASE = {
    # name: (stage, kwargs, conditioning shapes, prefix shape, max_time_steps, temperature, allow_eos)
    "gen_coarse_b20": ("coarse", dict(dim=64, depth=1, heads=3, clap_codebook_size=64, semantic_codebook_size=64,
                                      acoustic_codebook_size=64, num_clap_quantizers=4, num_coarse_quantizers=3),
                       [(20, 4), (20, 11)], (20, 2, 3), 10, 0.95, False),
}

if __name__ == "__main__":
    G.CASES = CASE
    G.main()
