"""The per-sequence check of test_bench_step_gpu.py catches what a whole-tensor rel-L2 misses: an error confined to the
last sequence of bench.py's batch.  On tensors of the oracle's logits shapes at cfg2 (B = 16, 811 coarse rows) and cfg3
(B = 8, 1270 fine rows), the last 64 rows of sequence B - 1 are moved 8 % of the way toward the row one position
earlier (a kernel that leaks a neighbouring position into one tile of one sequence).  Logits of neighbouring positions
are about as far apart as independent rows (rel ~ 1.4 on the oracle's cfg2 logits), so random rows stand in for them."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import test_bench_step_gpu as T  # noqa: E402

import bench  # noqa: E402


def _leak(ref, rows=64, w=0.08):
    got = ref.clone()
    got[-1, -rows:] = (1 - w) * ref[-1, -rows:] + w * ref[-1, -rows - 1:-1]
    return got


@pytest.mark.parametrize("key,n_rows", [("cfg2", 811), ("cfg3", 1270)])
def test_per_sequence_check_catches_an_error_in_the_last_sequence(key, n_rows):
    B = bench.WORKLOADS[key]["batch"]
    ref = torch.randn(B, n_rows, 1025, generator=torch.Generator().manual_seed(B))
    got = _leak(ref)
    assert T.whole_rel(got, ref) < T.SEQ_BOUND                   # the whole-tensor bound passes it
    r = T.per_sequence_rel(got, ref)
    assert r[:-1] == [0.0] * (B - 1) and r[-1] > 2 * T.SEQ_BOUND
    fails = T.sequence_fails(got, ref, key)
    assert len(fails) == 1 and f"sequence {B - 1}:" in fails[0]
    assert not T.sequence_fails(ref, ref, key)


def test_per_sequence_ce_is_the_wrapper_loss_of_one_sequence():
    """per_sequence_ce of a one-sequence batch is restatement.wrapper_loss on it; unweighted sequences do not count."""
    from oracle import restatement as R
    g = torch.Generator().manual_seed(5)
    logits = [torch.randn(3, 7, 11, generator=g), torch.randn(3, 9, 11, generator=g)]
    labels = [torch.randint(0, 11, (3, 7), generator=g).numpy(), torch.randint(0, 11, (3, 9), generator=g).numpy()]
    cfg = R.coarse_cfg(depth=1, ce_weights=[0.0, 1.0])
    got = T.per_sequence_ce(logits, labels, [0.0, 1.0])
    for b in range(3):
        want = float(R.wrapper_loss(cfg, [lg[b:b + 1] for lg in logits], [lb[b:b + 1] for lb in labels]))
        assert got[b] == pytest.approx(want, rel=1e-6)
