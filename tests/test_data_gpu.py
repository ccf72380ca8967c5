"""Device side of the token pipeline and the checkpoint files: batches gathered in HBM (omlm_gather_windows) equal the
host crops; a trainer
saved in the reference's three-file format (trainer.py:359-391) loads into torch's own AdamW / LinearLR and back."""
import os
import random
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(__file__))


def test_device_batches_equal_host_crops(tmp_path):
    from open_musiclm_b200 import data as D
    from test_data_cpu import host_store, synth_items
    items = synth_items(6, seed=2)
    D.write_sqlite(str(tmp_path), items)
    for stage in ("semantic", "coarse", "fine"):
        dev = D.TokenStore.from_sqlite(str(tmp_path), stage)
        host = host_store(stage, items)
        ids = [3, 0, 5, 5, 1, 2, 4, 0]
        a = dev.sample_batch(len(ids), rng=random.Random(7), items=ids)
        b = host.sample_batch(len(ids), rng=random.Random(7), items=ids)
        for x, y in zip(a, b):
            assert x.dtype == torch.int64 and x.is_cuda and tuple(x.shape) == tuple(y.shape)
            assert torch.equal(x.cpu(), y)
        assert dev.bytes_resident() > 0


def test_training_from_the_token_store_and_checkpoint_files(tmp_path):
    """A few optimiser steps on batches drawn from the HBM-resident store; save in the reference's file format; the
    optimizer file loads into a plain torch.optim.AdamW built the reference's way; a fresh trainer resumes from the files."""
    import open_musiclm_b200 as O
    from open_musiclm_b200 import data as D
    from test_data_cpu import synth_items
    items = synth_items(4, seed=9)
    store = D.TokenStore.from_items("coarse", [{c: it[c] for c in D.STAGE_COLUMNS["coarse"]} for it in items])
    kw = dict(dim=128, depth=2, heads=2, num_coarse_quantizers=3, attn_dropout=0.0, ff_dropout=0.1)
    torch.manual_seed(0)
    m = O.create_coarse_transformer(**kw).cuda()
    tr = O.HotPathTrainer(m, cross_entropy_loss_weights=[0.0, 0.0, 1.0], lr=1e-3, lr_warmup=5, wd=0.01, use_cuda_graph=False)
    rng = random.Random(0)
    batch = store.sample_batch(2, rng=rng)
    assert [tuple(t.shape) for t in batch] == [(2, 12), (2, 199, 1), (2, 300, 3)]
    losses = [float(tr.train_step([store.sample_batch(2, rng=rng)])) for _ in range(3)]
    assert all(np.isfinite(l) for l in losses)
    paths = D.checkpoint_paths(str(tmp_path), "coarse", tr.steps)
    tr.save(*paths)
    assert D.latest_checkpoints(str(tmp_path))[1] == 3
    # the optimizer file is a torch AdamW state_dict with the reference's two parameter groups
    sd = torch.load(paths[1])
    assert len(sd["param_groups"]) == 2 and sd["param_groups"][1]["weight_decay"] == 0 and sd["param_groups"][0]["weight_decay"] == 0.01
    params = list(m.parameters())
    ref_opt = torch.optim.AdamW([{"params": [p for p in params if p.ndim >= 2]}, {"params": [p for p in params if p.ndim < 2], "weight_decay": 0}],
                                lr=1e-3, weight_decay=0.01, betas=(0.9, 0.99), eps=1e-8)
    ref_opt.load_state_dict(sd)
    st = ref_opt.state[params[0]]
    assert float(st["step"]) == 3 and st["exp_avg"].shape == params[0].shape and float(st["exp_avg"].abs().sum()) > 0
    sched = torch.optim.lr_scheduler.LinearLR(ref_opt, start_factor=1e-7, total_iters=5)
    sched.load_state_dict(torch.load(paths[2]))
    assert sched.last_epoch == 3
    # resume: a fresh model + trainer loaded from the files takes the same next step
    nxt = store.sample_batch(2, rng=random.Random(99))
    l_a = float(tr.train_step([nxt]))
    torch.manual_seed(1)
    m2 = O.create_coarse_transformer(**kw).cuda()
    tr2 = O.HotPathTrainer(m2, cross_entropy_loss_weights=[0.0, 0.0, 1.0], lr=1e-3, lr_warmup=5, wd=0.01, use_cuda_graph=False)
    assert tr2.load(*paths) == 3
    tr2.eng.seed.copy_(tr.eng.seed - 1); tr2._mask_draws = tr._mask_draws - 1      # same dropout / forgetful-mask draw as tr's step
    l_b = float(tr2.train_step([nxt]))
    assert abs(l_a - l_b) <= 1e-4 * abs(l_a), (l_a, l_b)
    for (k, a), (_, b) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert float((a - b).norm()) <= 1e-4 * float(a.norm()) + 1e-7, k
