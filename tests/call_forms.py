"""The engine's phases for the call-form inventories (test_gemm_reference_gpu.py, test_norm_loss_reference_gpu.py,
test_attention_ffn_call_forms_gpu.py, test_sampler_token_call_forms_gpu.py) and the entry-point ledger
(test_entry_points_gpu.py): one driver that runs training steps, eval_loss, generate, scoring, generation sessions and
song sessions inside a recorder, so that every inventory sees the same calls.

A recorder is any object with a `phase` attribute; run() sets it before each phase, and the recorder files every call
it sees under the current phase.  Recorders read no device memory: generate and sessions capture CUDA graphs.

Models (MODELS): "d72" (d = 72, h = 3, codebooks whose C = 101 / 65 are not multiples of 64), "cfg2_depth1" (the
cfg2 layer dims at depth 1, h = 8), "d72_abspos" (d72 with absolute position embeddings: their rows in the
embedding gathers and the decode step), "cfg2_h16" (d = 1024, h = 16, whose chunk unit U = 128 / gcd(h, 128) is 8; the
session and score phases only) and "musiclm_prime" (the three stages of tests/golden/musiclm_prime.pt; song sessions
and song scoring only).

The bench models (BENCH_MODELS) are the workloads bench.py times, taken from bench.py itself (WORKLOADS, COMMON, TRAIN,
synth_batch), so that they follow it: "bench_cfg2" (the headline: coarse, B = 16, N = 1024), "bench_cfg3" (fine, B = 8,
N = 2048, the fine ids flattened to 1269 = 253 x 5 + 4: the remainder heads), "bench_cfg4" (h = 16, B = 16) and
"semantic" (the musiclm_small semantic stage, d = 1024, h = 8, N = 256, ce weights [0, 1], B = 16).  Each is built at
depth 1: the per-layer forms repeat unchanged across layers, so bench.py's depth 6 and cfg4's depth 24 add no form.  They
run bench.py's step (its batch, shapes, ce weights [0, 0, 1], FFN dropout 0.1 and the forgetful mask, eager: the
captured graph replays the same launches), its deterministic variant and eval_loss.  "semantic" also runs "bench
generation": MusicLM.generate_tokens with depth-1 musiclm_small semantic, coarse and fine stages at bench.py's batch 1
and 10 seconds, as bench.measure_generation does."""
import gc
import math

import torch

import bench

# model kwargs, conditioning shapes (clap, semantic), predicted shape (time steps, quantizers), token range
MODELS = {
    "d72": (dict(dim=72, depth=1, heads=3, clap_codebook_size=100, semantic_codebook_size=100, acoustic_codebook_size=64,
                 num_clap_quantizers=4, num_coarse_quantizers=3), [(4,), (11,)], (10, 3), 64),
    "cfg2_depth1": (dict(dim=1024, depth=1, heads=8, num_coarse_quantizers=3), [(12,), (197,)], (270, 3), 1024),
    "cfg2_h16": (dict(dim=1024, depth=1, heads=16, num_coarse_quantizers=3), [(12,), (197,)], (270, 3), 1024),
    "d72_abspos": (dict(dim=72, depth=1, heads=3, clap_codebook_size=100, semantic_codebook_size=100, acoustic_codebook_size=64,
                        num_clap_quantizers=4, num_coarse_quantizers=3, use_absolute_position_embeddings=True,
                        max_absolute_position_embeddings=320), [(4,), (11,)], (10, 3), 64),
}
SESSIONS_ONLY = {"cfg2_h16"}
SONGS_ONLY = {"musiclm_prime"}


def _bench_model(key):
    wl = bench.WORKLOADS[key]
    return dict(stage=wl["stage"], kw=dict(bench.COMMON, **dict(wl["model"], depth=1)), shapes=wl["shapes"], batch=wl["batch"],
                ce=list(bench.TRAIN["ce_weights"]))


# stage, model kwargs, token shapes per sequence, batch and ce weights of each bench model
BENCH_MODELS = {
    "bench_cfg2": _bench_model("cfg2"),
    "bench_cfg3": _bench_model("cfg3"),
    "bench_cfg4": _bench_model("cfg4"),
    # bench.py has no semantic training workload: the musiclm_small semantic stage of its generation (bench.measure_generation:
    # COMMON, h = 8) at the shapes of its cfg1 forward (bench.cpu_cfg1_forward: clap 12 + semantic 241, N = 256) and the
    # per-GPU training batch of its headline workload
    "semantic": dict(stage="semantic", kw=dict(bench.COMMON, depth=1, heads=8), shapes=[(12,), (241,)],
                     batch=bench.WORKLOADS["cfg2"]["batch"], ce=[0.0, 1.0]),
}
MODEL_KEYS = list(MODELS) + sorted(SONGS_ONLY) + list(BENCH_MODELS)

# (phase, deterministic, frozen): "norms" freezes the LayerNorm gammas and the q/k scales, "relpos" the relative-position
# MLP (the attention backward then forms no bias gradient)
TRAIN_PHASES = [("default step", False, None), ("deterministic step", True, None), ("frozen norms step", False, "norms"),
                ("frozen norms deterministic step", True, "norms"), ("frozen relpos step", False, "relpos"),
                ("frozen relpos deterministic step", True, "relpos")]
GENERATE_PHASES = ["generate B=3", "generate B=20", "generate sampling"]
SCORE_PHASES = ["score"]
SESSION_PHASES = ["session join", "session chunked", "session logprobs", "session sampling"]
SONG_PHASES = ["song session", "score songs"]
SCORE_MODELS = {"d72", "d72_abspos", "cfg2_h16"}
BENCH_PHASES = ["bench step", "bench deterministic step", "eval_loss"]
GENERATION_MODELS = {"semantic"}        # the bench models that also run "bench generation"


def train_spec(model):
    """Batch, token shapes per sequence and ce weights of a model's training phases."""
    if model in BENCH_MODELS:
        return {k: BENCH_MODELS[model][k] for k in ("batch", "shapes", "ce")}
    _, cond_n, pred_shape, _ = MODELS[model]
    return dict(batch=4, shapes=cond_n + [pred_shape], ce=[0.0, 1.0, 1.0])


def phases(model):
    if model in BENCH_MODELS:
        return BENCH_PHASES + (["bench generation"] if model in GENERATION_MODELS else [])
    if model in SONGS_ONLY:
        return list(SONG_PHASES)
    score = SCORE_PHASES if model in SCORE_MODELS else []
    if model in SESSIONS_ONLY:
        return score + SESSION_PHASES
    return [p for p, _, _ in TRAIN_PHASES] + ["eval_loss"] + GENERATE_PHASES + score + SESSION_PHASES


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


def _sampling_requests(g, cond_n, vocab, q, n_req):
    """Requests with their own filter_thres, temperature and top_p (None, 1.0 and nuclei), some with prefixes."""
    reqs = _session_requests(g, cond_n, vocab, q, cond_n[1][0], n_req, prefixes=True)
    for i, r in enumerate(reqs):
        r.update(filter_thres=(0.9, 0.5, 0.99, 0.0)[i % 4], temperature=(1.0, 0.7, 1.3)[i % 3], top_p=(None, 1.0, 0.9, 0.5, 0.75)[i % 5])
    return reqs


def _score(w, rec, g, cond_n, vocab, q):
    """TokenConditionedTransformerWrapper.score twice: with max_rows small enough that first-fit decreasing makes several
    forwards (the longest prompt, past max_rows, alone), and with the default max_rows (24 prompts in one forward).
    The two calls have semantic conditioning of different lengths; prefixes from 0 to 40 time steps."""
    rec.phase = "score"
    T = 40
    for B, n_sem, max_rows in ((7, cond_n[1][0], None), (24, max(2, cond_n[1][0] - 37), 16384)):
        cond = [torch.randint(0, min(vocab, 64), (B,) + cond_n[0], generator=g).cuda(),
                torch.randint(0, min(vocab, 64), (B, n_sem), generator=g).cuda()]
        pred = torch.randint(0, min(vocab, 64), (B, T, q), generator=g).cuda()
        lens = [(T, 0, 1, 13, 5, 22, 29)[b % 7] for b in range(B)]
        rows = sum(c[0] + 2 for c in cond_n[:1]) + n_sem + 2 + 1
        kw = dict(max_rows=rows + 17 * q + 1) if max_rows is None else dict(max_rows=max_rows)
        w.score(conditioning_token_ids=cond, pred_token_ids=pred, pred_lengths=lens, **kw)
    torch.cuda.synchronize()


def _songs(rec):
    """A MusicLMSession over a stream of songs (primes, per-stage top_p, coarse_only), then MusicLM.score_tokens on
    the songs it finished with all three stages, with a small max_rows and with the default."""
    import random
    import open_musiclm_b200 as O
    import test_musiclm_session_gpu as TM
    mlm = TM.h100_musiclm(TM.load()[1])
    rng, g = random.Random(3), torch.Generator().manual_seed(3)
    songs = TM.song_args(rng, g, 8, 4, 64, 3, 5, [2, 3, 4.5], [(9, 7), (3, 2)])
    for i, s in enumerate(songs):
        s["coarse_only"] = i % 4 == 1
    rec.phase = "song session"
    sess = O.MusicLMSession(mlm, slots=6, max_songs=4, max_queue=len(songs), **TM.FIX_WIN)
    res = TM.run_stream(sess, songs, rng)
    torch.cuda.synchronize()
    full = [r for r in res.values() if not r["args"]["coarse_only"]]
    rec.phase = "score songs"
    pk = ("prime_semantic_token_ids", "prime_coarse_token_ids", "prime_fine_token_ids")
    args = dict(clap_token_ids=[r["args"]["clap_token_ids"] for r in full], semantic_token_ids=[r["out"][1] for r in full],
                coarse_token_ids=[r["out"][2] for r in full], fine_token_ids=[r["out"][3] for r in full],
                output_seconds=[r["args"]["output_seconds"] for r in full], **{k: [r["args"].get(k) for r in full] for k in pk})
    for max_rows in (64, 16384):
        mlm.score_tokens(max_rows=max_rows, **args, **TM.FIX_WIN)
    torch.cuda.synchronize()


def _bench(rec, model):
    """bench.measure's step at depth 1: eager, then deterministic, then eval_loss, each on a batch of synth_batch."""
    import open_musiclm_b200 as O
    spec, ts = BENCH_MODELS[model], train_spec(model)
    make = {"coarse": O.create_coarse_transformer, "fine": O.create_fine_transformer, "semantic": O.create_semantic_transformer}
    m = make[spec["stage"]](**spec["kw"]).cuda()
    tr = O.HotPathTrainer(m, cross_entropy_loss_weights=ts["ce"], lr=bench.TRAIN["lr"], lr_warmup=bench.TRAIN["lr_warmup"],
                          wd=bench.TRAIN["wd"], max_grad_norm=bench.TRAIN["max_grad_norm"], grad_accum_every=1, use_cuda_graph=False)
    gen = torch.Generator().manual_seed(1234)
    batch = lambda: [t.cuda() for t in bench.synth_batch(ts["batch"], gen, ts["shapes"])]
    for phase, det in (("bench step", False), ("bench deterministic step", True)):
        rec.phase = phase
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(det)
        try:
            tr.train_step([batch()])
            torch.cuda.synchronize()
        finally:
            torch.use_deterministic_algorithms(prev)
    rec.phase = "eval_loss"
    tr.eval_loss(batch())
    torch.cuda.synchronize()
    del m, tr
    gc.collect()                # the d = 1024 workspaces at bench.py's batch: free them before the next phase or test
    if model in GENERATION_MODELS:
        rec.phase = "bench generation"
        _bench_generation()
        gc.collect()


def _bench_generation(seconds=10, batch=1):
    """bench.measure_generation's MusicLM.generate_tokens, with the three musiclm_small stages at depth 1 (its stage
    construction restated, since bench.py builds them inside the timed function)."""
    import open_musiclm_b200 as O
    mk = dict(bench.COMMON, depth=1, heads=8)
    sem = O.create_semantic_transformer(**mk).cuda().eval()
    coa = O.create_coarse_transformer(**mk, num_coarse_quantizers=3).cuda().eval()
    fin = O.create_fine_transformer(**mk, num_coarse_quantizers=3, num_fine_quantizers=5).cuda().eval()
    mlm = O.MusicLM(semantic_transformer=sem, coarse_transformer=coa, fine_transformer=fin)
    g = torch.Generator().manual_seed(1234)
    clap = torch.randint(0, 1024, (batch, 12), generator=g).cuda()
    mlm.generate_tokens(clap_token_ids=clap, output_seconds=seconds, return_all=True)
    torch.cuda.synchronize()


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
    if model in SONGS_ONLY:
        return _songs(rec)
    if model in BENCH_MODELS:
        return _bench(rec, model)
    kw, cond_n, pred_shape, vocab = MODELS[model]
    ts = train_spec(model)
    g = torch.Generator().manual_seed(1)

    def batch():
        toks = [torch.randint(0, min(vocab, 64), (ts["batch"],) + s, generator=g) for s in ts["shapes"]]
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
            tr = O.HotPathTrainer(m, cross_entropy_loss_weights=ts["ce"], lr=3e-4, wd=1e-2, use_cuda_graph=False)
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
        # the sampler's noise sources and modes: supplied uniforms, a scalar top_p, the shared Philox stream, per-row seeds
        # with log-probabilities
        rec.phase = "generate sampling"
        B, steps = 3, 4
        C1 = w.token_sequences[-1].codebook_size + 1
        cond = [torch.randint(0, min(vocab, 64), (B,) + s, generator=g).cuda() for s in cond_n]
        uni = torch.rand(steps * q, B, C1, generator=g).clamp_(1e-6, 1 - 1e-6)
        for extra in (dict(uniform_noise=uni), dict(top_p=0.8), dict(), dict(seeds=[5, 6, 7], return_logprobs=True, top_p=0.9)):
            w.generate(conditioning_token_ids=cond, max_time_steps=steps, **extra)
        torch.cuda.synchronize()
    U = unit(kw["heads"])
    if model in SCORE_MODELS:
        _score(w, rec, g, cond_n, vocab, q)
    long_cond = max(cond_n[1][0], 2 * U + 37)      # prompts of several units, so that the chunked sessions split them
    _run_session(w, rec, "session join", _session_requests(g, cond_n, vocab, q, long_cond, 5, prefixes=True))
    _run_session(w, rec, "session chunked", _session_requests(g, cond_n, vocab, q, long_cond, 5, prefixes=False), prefill_rows=U)
    # chunk boundaries fall on multiples of U: at U = 128, conditioning of 2U - 30 tokens and less puts some of them
    # inside the prefixes
    lp_cond = 2 * U - 30 if U >= 64 else long_cond
    _run_session(w, rec, "session logprobs", _session_requests(g, cond_n, vocab, q, lp_cond, 5, prefixes=True), prefill_rows=2 * U,
                 return_logprobs=True)
    reqs = _sampling_requests(g, cond_n, vocab, q, 10)
    _run_session(w, rec, "session sampling", reqs[:5])
    _run_session(w, rec, "session sampling", reqs[5:], return_logprobs=True)
