"""The engine's phases for the call-form inventories (test_gemm_reference_gpu.py, test_norm_loss_reference_gpu.py,
test_attention_ffn_call_forms_gpu.py): one driver that runs training steps, eval_loss, generate and generation
sessions inside a recorder, so that every inventory sees the same calls.

A recorder is any object with a `phase` attribute; run() sets it before each phase, and the recorder files every call
it sees under the current phase.  Recorders read no device memory: generate and sessions capture CUDA graphs.

Models (MODELS): "d72" (d = 72, h = 3, codebooks whose C = 101 / 65 are not multiples of 64), "cfg2_depth1" (the
cfg2 layer dims at depth 1, h = 8) and "cfg2_h16" (d = 1024, h = 16, whose chunk unit U = 128 / gcd(h, 128) is 8; the
session phases only)."""
import math

import torch

# model kwargs, conditioning shapes (clap, semantic), predicted shape (time steps, quantizers), token range
MODELS = {
    "d72": (dict(dim=72, depth=1, heads=3, clap_codebook_size=100, semantic_codebook_size=100, acoustic_codebook_size=64,
                 num_clap_quantizers=4, num_coarse_quantizers=3), [(4,), (11,)], (10, 3), 64),
    "cfg2_depth1": (dict(dim=1024, depth=1, heads=8, num_coarse_quantizers=3), [(12,), (197,)], (270, 3), 1024),
    "cfg2_h16": (dict(dim=1024, depth=1, heads=16, num_coarse_quantizers=3), [(12,), (197,)], (270, 3), 1024),
}
SESSIONS_ONLY = {"cfg2_h16"}

# (phase, deterministic, frozen): "norms" freezes the LayerNorm gammas and the q/k scales, "relpos" the relative-position
# MLP (the attention backward then forms no bias gradient)
TRAIN_PHASES = [("default step", False, None), ("deterministic step", True, None), ("frozen norms step", False, "norms"),
                ("frozen norms deterministic step", True, "norms"), ("frozen relpos step", False, "relpos"),
                ("frozen relpos deterministic step", True, "relpos")]
GENERATE_PHASES = ["generate B=3", "generate B=20"]
SESSION_PHASES = ["session join", "session chunked", "session logprobs"]


def phases(model):
    if model in SESSIONS_ONLY:
        return list(SESSION_PHASES)
    return [p for p, _, _ in TRAIN_PHASES] + ["eval_loss"] + GENERATE_PHASES + SESSION_PHASES


def unit(heads):
    """Rows per chunk unit of a session's chunked prefill: 128 / gcd(heads, 128)."""
    return 128 // math.gcd(heads, 128)


def _freeze(m, frozen):
    for n, p in m.named_parameters():
        if frozen == "norms" and (n.endswith("gamma") or n.endswith("q_scale") or n.endswith("k_scale")):
            p.requires_grad_(False)
        if frozen == "relpos" and n.startswith("transformer.rel_pos_bias."):
            p.requires_grad_(False)


def _session_requests(g, cond_n, vocab, q, long_cond, n_req, prefixes):
    """Requests of mixed prompt lengths: semantic conditioning of long_cond tokens and less; prefixes of 0 ... 20 time steps."""
    reqs = []
    for i in range(n_req):
        n_sem = max(2, long_cond - 37 * i)
        cond = [torch.randint(0, min(vocab, 64), (1, cond_n[0][0]), generator=g).cuda(),
                torch.randint(0, min(vocab, 64), (1, n_sem), generator=g).cuda()]
        steps = (0, 20, 7, 13, 1)[i % 5] if prefixes else 0
        pred = torch.randint(0, min(vocab, 64), (1, steps, q), generator=g).cuda() if steps else None
        reqs.append(dict(conditioning_token_ids=cond, pred_token_ids=pred, seed=1000 + i, max_time_steps=steps + 3))
    return reqs


def _run_session(w, rec, phase, reqs, **kw):
    import open_musiclm_b200 as O
    rec.phase = phase
    sess = O.GenerationSession(w, slots=4, max_positions=512, max_queue=len(reqs), **kw)
    for r in reqs:
        sess.add(**r)
    while not sess.idle:
        sess.step()
    torch.cuda.synchronize()
    return sess.finished()


def run(rec, model, act16, monkeypatch):
    """Runs every phase of phases(model) with OMLM_ACT16 = act16, setting rec.phase before each."""
    import open_musiclm_b200 as O
    monkeypatch.setenv("OMLM_ACT16", act16)
    torch.manual_seed(0)
    kw, cond_n, pred_shape, vocab = MODELS[model]
    g = torch.Generator().manual_seed(1)

    def batch():
        toks = [torch.randint(0, min(vocab, 64), (4,) + s, generator=g) for s in cond_n + [pred_shape]]
        toks[0][1, -2:] = -1                     # pad tokens: their embedding rows are zero
        toks[1][2, -3:] = -1
        return [t.cuda() for t in toks]

    main = None
    if model not in SESSIONS_ONLY:
        # training: FFN dropout, pad tokens in the conditioning and the trainer's forgetful mask (mask_prob 0.15)
        for phase, det, frozen in TRAIN_PHASES:
            rec.phase = phase
            m = O.create_coarse_transformer(attn_dropout=0.0, ff_dropout=0.1, **kw).cuda()
            _freeze(m, frozen)
            tr = O.HotPathTrainer(m, cross_entropy_loss_weights=[0.0, 1.0, 1.0], lr=3e-4, wd=1e-2, use_cuda_graph=False)
            prev = torch.are_deterministic_algorithms_enabled()
            torch.use_deterministic_algorithms(det)
            try:
                tr.train_step([batch()])
                torch.cuda.synchronize()
            finally:
                torch.use_deterministic_algorithms(prev)
            if main is None:
                main = (m, tr)
        m, tr = main
        rec.phase = "eval_loss"
        tr.eval_loss(batch())
        torch.cuda.synchronize()
    else:
        m = O.create_coarse_transformer(attn_dropout=0.0, ff_dropout=0.1, **kw).cuda()
    m.eval()
    w = O.TokenConditionedTransformerWrapper(transformer=m, unique_consecutive=False)
    q = pred_shape[1]
    if model not in SESSIONS_ONLY:
        for B in (3, 20):          # B = 3: the SIMT decode; B = 20: the tensor-core decode; prefixes of their own lengths
            rec.phase = f"generate B={B}"
            cond = [torch.randint(0, min(vocab, 64), (B,) + s, generator=g).cuda() for s in cond_n]
            pred = torch.randint(0, min(vocab, 64), (B, 4, q), generator=g).cuda()
            w.generate(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=[1 + b % 4 for b in range(B)], max_time_steps=7)
            torch.cuda.synchronize()
    U = unit(kw["heads"])
    long_cond = max(cond_n[1][0], 2 * U + 37)      # prompts of several units, so that the chunked sessions split them
    _run_session(w, rec, "session join", _session_requests(g, cond_n, vocab, q, long_cond, 5, prefixes=True))
    _run_session(w, rec, "session chunked", _session_requests(g, cond_n, vocab, q, long_cond, 5, prefixes=False), prefill_rows=U)
    # chunk boundaries fall on multiples of U: at U = 128, conditioning of 2U - 30 tokens and less puts some of them
    # inside the prefixes
    lp_cond = 2 * U - 30 if U >= 64 else long_cond
    _run_session(w, rec, "session logprobs", _session_requests(g, cond_n, vocab, q, lp_cond, 5, prefixes=True), prefill_rows=2 * U,
                 return_logprobs=True)
