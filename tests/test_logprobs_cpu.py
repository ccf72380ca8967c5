"""Token log-probabilities in generation without a GPU: the float64 statements (tests/logprob_reference.py) against
torch's log_softmax and a sort-based candidate set, the prefix label layout the per-row kernel reads, and the argument
checks of generate, the stages and GenerationSession, which raise before any device work."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))

from logprob_reference import candidate_set, model_logprob, sample_logprob  # noqa: E402
from norm_loss_reference import ce_ref  # noqa: E402
from test_sampling_nucleus_cpu import edge_logits  # noqa: E402


@pytest.mark.parametrize("C", [2, 65, 1025])
def test_model_logprob_is_the_negated_row_loss(C):
    g = torch.Generator().manual_seed(C)
    x = torch.randn(24, C, generator=g) * 4
    tok = torch.randint(0, C, (24,), generator=g)
    val, bound = model_logprob(x, tok)
    ref = ce_ref(x, tok, C, C, grad_scale=0.0)
    assert torch.allclose(val, -ref["loss"], rtol=0, atol=1e-12)
    assert torch.allclose(val, torch.log_softmax(x.double(), 1).gather(1, tok[:, None])[:, 0], rtol=0, atol=1e-12)
    assert bool((bound > 0).all()) and bool((bound < 1e-4 * (1 + val.abs())).all())


@pytest.mark.parametrize("top_p", [None, 0.5, 0.9])
@pytest.mark.parametrize("C", [3, 64, 1025])
def test_sample_logprob_is_a_distribution_over_the_candidate_set(C, top_p):
    """exp(sample_logprob) over every class of S sums to 1, S is inside K, and with k = C, no top_p and T = 1 it is
    log_softmax of the eos-masked row."""
    g = torch.Generator().manual_seed(C + 7)
    x = edge_logits(12, C, g)
    k, T = max(1, C // 3), 0.7
    S = candidate_set(x, k, T, False, top_p)
    for b in range(x.shape[0]):
        cls = S[b].nonzero()[:, 0]
        if len(cls) == 0 or not math.isfinite(float(x[b, cls].max())):
            continue
        vals = torch.stack([sample_logprob(x[b:b + 1], c.view(1), k, T, False, top_p)[0][0] for c in cls])
        finite = torch.isfinite(vals)
        assert abs(float(torch.exp(vals[finite]).sum()) - 1.0) < 1e-9
    y = torch.randn(6, C, generator=g)
    tok = torch.randint(0, C - 1, (6,), generator=g)
    ref = torch.log_softmax(torch.cat([y[:, :-1].double(), torch.full((6, 1), -math.inf, dtype=torch.float64)], 1), 1)
    got = sample_logprob(y, tok, C, 1.0, False, None)[0]
    assert torch.allclose(got, ref.gather(1, tok[:, None])[:, 0], rtol=0, atol=1e-12)


def test_prefix_labels_layout():
    """Group qi's row t reads label t q + qi through (offset qi, stride q, n + q per sequence); the row predicting the
    next token, and any token outside [0, C), reads -100."""
    from open_musiclm_b200.decode import prefix_labels
    q, C = 3, 10
    prompt = torch.tensor([[1, 2, 3, 4, 5, 6], [7, 8, -1, 9, 12, 0]])
    lab = prefix_labels(prompt, q, C)
    B, n = prompt.shape
    assert lab.shape == (B, n + q) and lab.dtype == torch.int32
    flat = lab.reshape(-1)
    for qi in range(q):
        cnt = (n + 1 - qi + q - 1) // q
        for b in range(B):
            for t in range(cnt):
                p = t * q + qi
                want = int(prompt[b, p]) if p < n and 0 <= int(prompt[b, p]) < C else -100
                assert int(flat[qi + b * (n + q) + t * q]) == want


class _NoEngine:
    @property
    def engine(self):
        raise AssertionError("device work before the argument check")


@pytest.mark.parametrize("bad", [1, 0, "yes", None, torch.tensor(True)])
def test_return_logprobs_must_be_a_bool(bad):
    import open_musiclm_b200 as O
    w = O.TokenConditionedTransformerWrapper.__new__(O.TokenConditionedTransformerWrapper)
    torch.nn.Module.__init__(w)
    with pytest.raises(ValueError, match="return_logprobs"):
        w.generate(conditioning_token_ids=[torch.zeros(1, 3, dtype=torch.int64)], return_logprobs=bad)
    with pytest.raises(ValueError, match="return_logprobs"):
        O.GenerationSession(w, slots=1, max_positions=8, return_logprobs=bad)


def test_stages_pass_return_logprobs_through():
    """Each stage hands return_logprobs to the wrapper's generate and returns what it returns."""
    from open_musiclm_b200 import stages

    class _W:
        token_sequences = [type("I", (), dict(codebook_size=8, num_quantizers=1))()]

        def generate(self, **kw):
            self.kw = kw
            return ("tokens", "logprobs", "sample_logprobs")

    for cls, kw in ((stages.SemanticStage, dict(clap_token_ids=torch.zeros(1, 2, dtype=torch.int64))),
                    (stages.CoarseStage, dict(clap_token_ids=torch.zeros(1, 2, dtype=torch.int64),
                                              semantic_token_ids=torch.zeros(1, 2, dtype=torch.int64))),
                    (stages.FineStage, dict(clap_token_ids=torch.zeros(1, 2, dtype=torch.int64),
                                            coarse_token_ids=torch.zeros(1, 2, 3, dtype=torch.int64)))):
        st = cls.__new__(cls)
        torch.nn.Module.__init__(st)
        st.transformer_wrapper = _W()
        st.clap = None
        out = st.generate(return_logprobs=True, **kw)
        assert out == ("tokens", "logprobs", "sample_logprobs")
        assert st.transformer_wrapper.kw["return_logprobs"] is True


def test_reconstruct_wave_with_logprobs_raises():
    from open_musiclm_b200 import stages
    for cls in (stages.CoarseStage, stages.FineStage):
        st = cls.__new__(cls)
        torch.nn.Module.__init__(st)
        with pytest.raises(ValueError, match="reconstruct_wave"):
            st.generate(semantic_token_ids=None, coarse_token_ids=None, reconstruct_wave=True, return_logprobs=True) \
                if cls is stages.CoarseStage else st.generate(coarse_token_ids=None, reconstruct_wave=True, return_logprobs=True)


@pytest.mark.parametrize("include_eos", [False, True])
def test_assemble_output_prefix_sampled_and_masked_positions(include_eos):
    """Two rows of different prefix lengths (ragged) and sample counts, an eos in row 0's samples: prefix columns take
    the prefix values (sample log p 0), sampled columns the decode's in order, columns past a row's end and every -1
    (after the eos, or the eos itself without include_eos) are 0; a non-ragged row is the plain concatenation."""
    from open_musiclm_b200.decode import assemble_output
    eos = 9
    n_real = torch.tensor([[2], [4]])
    n_end = n_real + torch.tensor([[4], [2]])
    tokens = torch.tensor([[1, 2, 5, eos, 6, 7], [3, 4, 5, 6, 8, 1]])
    prefix, new = tokens[:, :4], torch.tensor([[5, eos, 6, 7], [8, 1, 0, 0]])  # row 0: 2 prefix tokens; row 1: 4
    eos_mask = (tokens == eos).float()
    if include_eos:
        eos_mask = torch.nn.functional.pad(eos_mask, (1, -1))
    sampled = tokens.masked_fill(eos_mask.cumsum(-1) > 0, -1)
    pre = -torch.arange(1, 5, dtype=torch.float32).repeat(2, 1)                  # [2, 4]: -1 -2 -3 -4
    lp_new = -torch.arange(10, 14, dtype=torch.float32).repeat(2, 1)             # -10 -11 -12 -13
    slp_new = lp_new / 10
    out, lp, slp = (t[..., 0] for t in assemble_output(prefix, new, n_real, n_end, 6, eos, include_eos, 1, (pre, lp_new, slp_new)))
    assert torch.equal(out, sampled)
    want0 = [-1, -2, -10, -11 if include_eos else 0, 0, 0]
    assert lp[0].tolist() == want0
    assert torch.allclose(slp[0], torch.tensor([0, 0, -1.0, -1.1 if include_eos else 0, 0, 0]))
    assert lp[1].tolist() == [-1, -2, -3, -4, -10, -11] and torch.allclose(slp[1], torch.tensor([0, 0, 0, 0, -1.0, -1.1]))
    out, lp, slp = (t[..., 0] for t in assemble_output(prefix, new, n_real, n_real + torch.tensor([[4], [1]]), 6, eos, include_eos, 1,
                                                       (pre, lp_new, slp_new)))
    assert out[1, 5] == -1 and lp[1, 5] == 0 and slp[1, 5] == 0 and lp[1, 4] == -10    # padding of a shorter row
    out, lp, slp = (t[..., 0] for t in assemble_output(prefix, new[:, :0], 4, 4, 4, eos, include_eos, 1, (pre, None, None)))
    assert lp[1].tolist() == [-1, -2, -3, -4] and bool((slp == 0).all())


def test_session_pass_through_with_stubs():
    """GenerationSession(return_logprobs=True): a request that samples nothing is scored by generate's teacher-forced
    idiom with the session's eos settings, and finished() returns its triple of [n, q] rows."""
    import open_musiclm_b200 as O

    class _Info:
        codebook_size, num_quantizers, unique_consecutive = 8, 2, False

    class _M:
        heads, use_absolute_position_embeddings, device = 2, False, "cpu"

    class _W:
        token_sequences = [_Info(), _Info()]
        eos_ids = [8, 8]
        transformer = _M()

        def generate(self, **kw):
            self.kw = kw
            n = kw["pred_token_ids"].shape[1]
            return (kw["pred_token_ids"], -torch.ones(1, n, 2), torch.zeros(1, n, 2))

    w = _W()
    sess = O.GenerationSession(w, slots=2, max_positions=32, return_logprobs=True, include_eos_in_output=True)
    h = sess.add(conditioning_token_ids=[torch.zeros(1, 3, dtype=torch.int64)], pred_token_ids=torch.ones(1, 2, 2, dtype=torch.int64),
                 seed=1, max_time_steps=2)
    out = sess.finished()[h]
    assert w.kw["return_logprobs"] is True and w.kw["max_time_steps"] == 2 and w.kw["include_eos_in_output"] is True
    assert [tuple(t.shape) for t in out] == [(2, 2)] * 3 and bool((out[1] == -1).all())


@pytest.mark.parametrize("case", ["semantic", "coarse", "fine_eos"])
def test_restatement_reproduces_the_reference_fixture(case):
    """The oracle restatement, on the reference's weights and prompt, reproduces the fixture's raw rows, its
    log-softmax at the sampled tokens, its top-k sample log p and its prefix log-softmax (float32 CPU, 1e-4)."""
    from oracle import restatement as R
    gold = os.path.join(os.path.dirname(__file__), "golden")
    fx = torch.load(os.path.join(gold, f"logprobs_{case}.pt"), weights_only=False)
    sd = torch.load(os.path.join(gold, fx["weights"]), weights_only=False)["state_dict"]
    kw = fx["kwargs"]
    base = dict(dim=kw["dim"], depth=kw["depth"], heads=kw["heads"], codebook=kw.get("clap_codebook_size", 1024),
                n_clap_q=kw.get("num_clap_quantizers", 12))
    cfg = {"semantic": lambda: R.semantic_cfg(**base), "coarse": lambda: R.coarse_cfg(n_coarse_q=kw["num_coarse_quantizers"], **base),
           "fine": lambda: R.fine_cfg(n_coarse_q=kw["num_coarse_quantizers"], n_fine_q=kw["num_fine_quantizers"], **base)}[fx["stage"]]()
    B = fx["cond"][0].shape[0]
    cond = [torch.cat([t.reshape(B, -1), torch.full((B, 1), s.codebook_size)], 1).numpy() for t, s in zip(fx["cond"], cfg.seqs)]
    pre = fx["prefix"].reshape(B, -1) if fx["prefix"] is not None else torch.empty(B, 0, dtype=torch.long)
    flat = torch.cat([pre, fx["sampled"].t()], 1)
    n_pre, q = pre.shape[1], cfg.seqs[-1].num_quantizers
    with torch.no_grad():
        for s in range(fx["rows"].shape[0]):
            row = R.forward_logits(cfg, sd, cond + [flat[:, :n_pre + s].numpy()], None, only_final=True)[-1]
            assert torch.allclose(row[:, -1].double(), fx["rows"][s].double(), atol=1e-4, rtol=0)
            tok = fx["sampled"][s][:, None]
            assert torch.allclose(torch.log_softmax(row[:, -1].double(), -1).gather(1, tok)[:, 0], fx["logprobs"][s], atol=1e-4)
            masked = row[:, -1].clone()
            if not fx["allow_eos_in_output"] or (n_pre + s) % q != q - 1:
                masked[:, -1] = -math.inf
            filt = R.top_k_filter(masked, fx["filter_thres"]).double() / fx["temperature"]
            assert torch.allclose(torch.log_softmax(filt, -1).gather(1, tok)[:, 0], fx["sample_logprobs"][s], atol=1e-4)
            if s == 0 and n_pre:
                got = torch.log_softmax(row[:, :n_pre].double(), -1).gather(2, pre[:, :, None])[..., 0]
                assert torch.allclose(got, fx["prefix_logprobs"], atol=1e-4)
    out = fx["out"].reshape(B, -1)
    live = out[:, n_pre:] >= 0
    assert torch.equal(out[:, n_pre:][live], fx["sampled"].t()[live])
