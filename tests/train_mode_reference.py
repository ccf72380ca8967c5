"""The masks of a training-mode step and the fp32 oracle run under them, shared by tests/test_train_mode_cpu.py and
tests/test_train_mode_gpu.py.

A training step draws two masks from the device Philox stream (host replica: tests/test_philox_cpu.py):
  * the FFN dropout keep bits of layer l: ffn_norm_fwd under (seed, stream = l), row b * N + n of the engine's token
    order, one bit per inner channel, stored as uint8 [M, Fp / 8] (bit i of byte j is channel 8 j + i);
  * the forgetful causal mask: forgetful_mask under (seed, stream id), num_drop = min(int(N * mask_prob), N - 1) over
    the whole concatenated sequence, ANDed into the key mask after the conditioning pad / eos masking.
The reference (open_musiclm.py:374-376, transformer.py:148 / 159) holds the same masks as a [B, N] bool that
restatement.prepare_ids takes and per-layer [B, N, F] bools for the Dropout outputs.  The functions below convert
between the two layouts and run restatement.loss_and_logits under given masks."""
import dataclasses
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(__file__))
from test_philox_cpu import dropout_keep, forgetful_mask  # noqa: E402

from oracle import restatement as R  # noqa: E402

# gradient bounds (cos >=, rel-L2 <=) of test_parity_gpu.check_grads outside the rel-pos MLP (whose parameters have
# 0.995 / 1e-1, and net.3.bias an analytic zero)
GRAD_COS, GRAD_REL = 0.999, 2e-2
# the rel-L2 bound with OMLM_ACT16=bf16, bf16 forward operands (a diagnostics mode): the operand rounding alone moves
# the gradients of the d = 1024 conv stage (depth 2, h = 8, N = 501) by rel 2.47e-2 / cos 0.999697 in eval mode and
# 2.54e-2 / 0.999695 in training mode (fp16 operands: 9.1e-3 and 9.6e-3), measured on an H100 80GB HBM3 at 700 W
GRAD_REL_BF16 = 3.5e-2


def cfg_of(fx, ff_dropout, mask_prob=0.15) -> R.Cfg:
    """restatement config of an eval fixture (tests/golden/tiny_*.pt) with the given dropout probability."""
    kw = fx["kwargs"]
    common = dict(dim=kw["dim"], depth=kw["depth"], heads=kw["heads"], ff_dropout=ff_dropout, mask_prob=mask_prob,
                  grad_shrink_alpha=kw["grad_shrink_alpha"], ce_weights=list(fx["ce_weights"]),
                  use_conv_ff=kw.get("use_conv_ff", True), rel_pos_bias_type=kw.get("relative_position_bias_type", "continuous"),
                  abs_pos=kw.get("use_absolute_position_embeddings", False))
    cb = kw.get("clap_codebook_size", 1024)
    if fx["stage"] == "semantic":
        return R.semantic_cfg(codebook=cb, n_clap_q=kw["num_clap_quantizers"], **common)
    if fx["stage"] == "coarse":
        return R.coarse_cfg(codebook=cb, n_clap_q=kw["num_clap_quantizers"], n_coarse_q=kw["num_coarse_quantizers"], **common)
    return R.fine_cfg(codebook=cb, n_clap_q=kw["num_clap_quantizers"], n_coarse_q=kw["num_coarse_quantizers"],
                      n_fine_q=kw["num_fine_quantizers"], **common)


def padded_width(cfg: R.Cfg) -> int:
    """Fp: the inner FFN width rounded up to the engine's 128-channel groups."""
    return -(-cfg.ff_inner // 128) * 128


def num_drop(N, mask_prob):
    """utils.py:53."""
    return min(int(N * mask_prob), N - 1)


# ------------------------------------------------------------------------------------------------ layouts
def pack_keep(keep: np.ndarray) -> np.ndarray:
    """bool [M, Fp] -> the engine's uint8 [M, Fp / 8] keep bits (bit i of byte j is channel 8 j + i)."""
    return np.packbits(np.asarray(keep, dtype=bool), axis=1, bitorder="little")


def unpack_keep(bits) -> np.ndarray:
    """The engine's uint8 [M, Fp / 8] keep bits (numpy or a tensor on any device) -> bool [M, Fp]."""
    if isinstance(bits, torch.Tensor):
        bits = bits.cpu().numpy()
    return np.unpackbits(np.asarray(bits, dtype=np.uint8), axis=1, bitorder="little").astype(bool)


def keep_bnf(keep: np.ndarray, B, N, F) -> torch.Tensor:
    """bool [B N, Fp] in the engine's row order -> the reference's [B, N, F] Dropout keep mask."""
    return torch.from_numpy(np.ascontiguousarray(keep[:, :F])).reshape(B, N, F)


def keep_rows(keep_ref: torch.Tensor, Fp) -> np.ndarray:
    """The reference's [B, N, F] keep mask -> bool [B N, Fp] (padding channels dropped, as nothing reads them)."""
    B, N, F = keep_ref.shape
    out = np.zeros((B * N, Fp), dtype=bool)
    out[:, :F] = keep_ref.reshape(B * N, F).numpy()
    return out


# ------------------------------------------------------------------------------------------------ replica masks
def replica_keep_rows(seed, layer, B, N, Fp, p) -> np.ndarray:
    """bool [B N, Fp]: the keep bits ffn_norm_fwd writes for `layer` under `seed`."""
    return dropout_keep(seed, layer, np.arange(B * N), Fp, p)


def replica_keeps(seed, cfg: R.Cfg, B, N, p=None, layers=None):
    """Per layer, the reference's [B, N, F] keep mask of the engine's step under `seed` (layers: the stream of each
    layer, default l)."""
    p = cfg.ff_dropout if p is None else p
    Fp = padded_width(cfg)
    layers = list(range(cfg.depth)) if layers is None else layers
    return [keep_bnf(replica_keep_rows(seed, s, B, N, Fp, p), B, N, cfg.ff_inner) for s in layers]


def replica_forget(seed, stream_id, B, N, mask_prob) -> np.ndarray:
    """bool [B, N]: the forgetful causal mask the trainer draws under (seed, stream id), as prepare_ids takes it."""
    return forgetful_mask(seed, stream_id, B, N, num_drop(N, mask_prob)).astype(bool)


def seq_len(cfg: R.Cfg, tokens) -> int:
    """N of a training step (eos appended to every sequence, the last token of the last one dropped, start tokens)."""
    return sum(np.asarray(t).reshape(t.shape[0], -1).shape[1] + 1 for t in tokens) + len(tokens) - 1


# ------------------------------------------------------------------------------------------------ oracle under masks
def trainable_state(sd):
    return {k: v.detach().clone().requires_grad_(v.is_floating_point() and not k.endswith("beta")) for k, v in sd.items()}


def oracle_step(cfg: R.Cfg, sd, tokens, forget=None, keeps=None, scale=True):
    """restatement.loss_and_logits under the given masks (forget: [B, N] bool or None; keeps: per-layer [B, N, F] bool
    or None), then autograd.  scale=False leaves out dropout's 1 / (1 - p).  Returns (loss, logits, key mask, grads)."""
    if not scale:
        cfg = dataclasses.replace(cfg, ff_dropout=0.0)
    st = trainable_state(sd)
    loss, logits, _, _, mask = R.loss_and_logits(cfg, st, [np.asarray(t) for t in tokens], forget_mask=forget, drop_keeps=keeps)
    loss.backward()
    grads = {k: (v.grad.detach() if v.grad is not None else None) for k, v in st.items() if v.requires_grad}
    return float(loss.detach()), [lg.detach() for lg in logits], mask, grads


def grad_errors(got, gold):
    """(name, cos, rel) of every parameter gradient with a nonzero reference, rel-pos bias parameters aside."""
    out = []
    for k, g in gold.items():
        if g is None or "rel_pos_bias" in k or float(g.norm()) < 1e-6:
            continue
        a, b = got[k].detach().double().cpu().reshape(-1), g.double().cpu().reshape(-1)
        c = float((a @ b) / (a.norm() * b.norm()).clamp_min(1e-30))
        r = float((a - b).norm() / b.norm().clamp_min(1e-30))
        out.append((k, c, r))
    return out
