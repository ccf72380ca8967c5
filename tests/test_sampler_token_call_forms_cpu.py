"""Host side of the sampler and token-path inventory (test_sampler_token_call_forms_gpu.py): plan_reference equals
oracle.restatement on the training form, its inference forms behave as include/omlm_b200.h states (pads only where the
offset sum is pad_id, out-of-table ids give -1 and their sequence's bit), the recorder's symbol dispatch follows
lib.sample, and every explicit case's key is in the covered set."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(__file__))
import test_sampler_token_call_forms_gpu as T  # noqa: E402


def test_plan_reference_equals_the_restatement_on_the_training_form():
    from oracle import restatement as R
    cfg = R.coarse_cfg(codebook=1024, n_clap_q=12, n_coarse_q=3)
    rng = np.random.default_rng(3)
    toks = [rng.integers(0, 1024, s) for s in [(3, 12), (3, 40), (3, 17, 3)]]
    toks[0][0, 0] = -1; toks[1][2, 3] = -1; toks[1][1, 7] = 1024; toks[2][0, 0, 0] = -1; toks[2][1, 2, 1] = -1
    ids_np, mask_np, labels_np = R.prepare_ids(cfg, toks, True)
    rows = R.embedding_rows(cfg, ids_np)
    bases = [0, 1025 * 12, 1025 * 12 + 1025]
    total = bases[2] + 1025 * 3
    ids_out, src, key, labels, err = T.plan_reference([t.reshape(3, -1) for t in toks], [1024] * 3, [12, 1, 3], bases,
                                                      [total, total + 1, total + 2], True, True, True, -1, None, None)
    exp = []
    for s, (r, pad) in enumerate(rows):
        exp += [np.full((3, 1), total + s), np.where(pad, -1, r + bases[s])]
    assert np.array_equal(ids_out, np.concatenate(ids_np, 1)) and np.array_equal(key, mask_np)
    assert np.array_equal(labels, np.concatenate(labels_np, 1)) and np.array_equal(src, np.concatenate(exp, 1)) and err == 0


def test_plan_reference_inference_form():
    """q = 3, codebook 10, base 100: a pad at quantizer 0 is a -1 row, at quantizer 1 it is row base + 9; an id past
    the table is -1 and sets bit 1; an empty last sequence has only its start row."""
    cond = np.array([[3, 4]])
    pred = np.array([[-1, -1, 5, 99, 0, 0]])
    _, src, key, _, err = T.plan_reference([cond, pred], [20, 10], [1, 3], [0, 100], [200, 201], False, False, False, -1, None, None)
    assert src.tolist() == [[200, 3, 4, 201, -1, 109, 125, -1, 110, 120]] and key.all() and err == 2
    _, src, _, _, err = T.plan_reference([cond, pred[:, :0]], [20, 10], [1, 3], [0, 100], [200, 201], False, False, False, -1, None, None)
    assert src.tolist() == [[200, 3, 4, 201]] and err == 0


def test_sample_symbol_follows_lib_sample():
    assert T.sample_symbol(None, (True, True, False), False) == ("omlm_sample_rows", False)
    assert T.sample_symbol(None, (True, True, True), False) == ("omlm_sample_rows", True)
    assert T.sample_symbol(0.9, (False, False, False), True) == ("omlm_sample_logprob", True)
    assert T.sample_symbol(1.0, (False, False, False), True) == ("omlm_sample_logprob", False)
    assert T.sample_symbol(0.9, (False, False, False), False) == ("omlm_sample_nucleus", True)
    assert T.sample_symbol(1.0, (False, False, False), False) == (None, False)


def test_plan_key_separates_a_last_sequence_that_ends_inside_a_time_step():
    """bench.py's cfg3 flattens the fine ids to 1269 = 253 x 5 + 4: a key of its own, apart from 1270 ids at q = 5 and
    from the coarse stage's whole steps; the explicit training plans cover it with and without forgetting and err_flag."""
    form = lambda n, q, forget, err: ([12, 762, n], [12, 3, q], True, True, True, False, forget, True, err)
    assert T.plan_key(*form(1269, 5, True, True)) != T.plan_key(*form(1270, 5, True, True))
    assert T.plan_key(*form(1269, 5, True, True))[-1] and not T.plan_key(*form(1270, 5, True, True))[-1]
    assert not T.plan_key([12, 197, 810], [12, 1, 3], True, True, True, False, True, True, True)[-1]
    assert not T.plan_key([12, 241], [12, 1], True, True, True, False, True, True, True)[-1]
    cov = T.covered_keys()
    for forget in (False, True):
        for err in (False, True):
            assert T.plan_key(*form(1269, 5, forget, err)) in cov
            assert T.plan_key([12, 241], [12, 1], True, True, True, False, forget, True, err) in cov


def test_explicit_cases_are_covered_and_distinct():
    cov = T.covered_keys()
    assert all(T.sampler_key(*c) in cov for c in T.EXPLICIT_SAMPLER) and all(T.plan_key(*c) in cov for c in T.EXPLICIT_PLAN)
    assert len({repr(c) for c in T.EXPLICIT_SAMPLER}) == len(T.EXPLICIT_SAMPLER)
    # C = 8200 passes the 48 KB default for both kernels; C = 1025 does not
    assert T.sampler_key("omlm_sample_rows", False, False, False, (True, True, False), "engine_seed", 8200, 8320)[-2]
    assert not T.sampler_key("omlm_sample_rows", True, False, False, (True, True, True), "engine_seed", 1025, 1152)[-2]
