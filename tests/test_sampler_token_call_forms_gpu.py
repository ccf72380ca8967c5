"""The engine's sampler and token-path calls, recorded over every phase of tests/call_forms.py and replayed against
exact references.

The recorder wraps lib.sample (filed under the C symbol it dispatches to: omlm_sample, _seeded, _nucleus, _rows or
_logprob), lib.sample_rows_indexed (omlm_sample_rows_indexed(_logprob)), lib.token_plan, lib.forgetful_mask,
lib.embed_gather_pos_rows and lib.decode_advance_pos, and keeps each call's host-visible form: which arguments are
None, the scalars, C, the logits pitch, the sequence lengths and mode flags.  Nothing reads device memory: generate
and the sessions capture CUDA graphs, and song sessions run their stages on their own streams.  (lib.embed_gather's
forms, the decode step's included, are replayed by test_norm_loss_reference_gpu.py.)

Replays use fresh seeded inputs, outputs poisoned with a sentinel and rows past the outputs guarded:
- samplers: rows with their own k, temperature and top_p on the edge logits of test_generate_per_row_gpu.py, at
  sample indices 0 and 2, each token against the float64 Gumbel top-k / nucleus statement (check_nucleus, with its
  near-tie exclusion) under the host replica of the form's noise source (supplied uniforms, the Philox stream of the
  shared seed, or per-row seeds); log-probability forms also against the float64 statements of logprob_reference.py
  under their bounds; indexed forms with rows at, past and before their last sample index;
- token_plan: at the recorded batch, bit-exact against oracle.restatement for the training form and against plan_reference (below) for the
  inference forms, with pads at quantizer positions other than 0, an empty sequence and ids outside a table (a -1
  row and the sequence's err_flag bit);
- forgetful_mask against the replica ranking; embed_gather_pos_rows and decode_advance_pos against torch indexing,
  with positions outside [0, pos_rows) and negative source rows.

Coverage keys come from host-visible arguments only; a key that no explicit case (the family files' or EXPLICIT_*
below) covers fails the test and is named."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import call_forms  # noqa: E402
from logprob_reference import model_logprob, sample_logprob  # noqa: E402
from test_generate_per_row_gpu import SENTINEL, _kernel_case, _row_uniforms, _rows  # noqa: E402
from test_logprobs_gpu import _close  # noqa: E402
from test_philox_cpu import forgetful_mask as forgetful_replica  # noqa: E402
from test_sampling_gpu import seed_tensor  # noqa: E402
from test_sampling_nucleus_gpu import check_nucleus  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SMEM_DEFAULT = 48 * 1024            # dynamic shared memory a launch gets without the opt-in
NAMES = ("sample", "sample_rows_indexed", "token_plan", "forgetful_mask", "embed_gather_pos_rows", "decode_advance_pos")


def _lib():
    from open_musiclm_b200 import lib
    return lib


# ------------------------------------------------------------------------------------------------ coverage keys
def sample_symbol(top_p, rows, logprob):
    """The C symbol lib.sample dispatches to, and whether that launch runs the nucleus kernel.
    rows: (top_k_rows, temperature_rows, top_p_rows) present."""
    if logprob:
        return "omlm_sample_logprob", rows[2] or (top_p is not None and top_p < 1.0)
    if any(rows):
        return "omlm_sample_rows", rows[2]
    if top_p is not None and top_p != 1.0:
        return "omlm_sample_nucleus", True
    return None, False          # omlm_sample / omlm_sample_seeded: named by the noise source


def sampler_key(symbol, nucleus, row_step, logprob, rows, noise, C, ld):
    """symbol, the kernel's three template flags, the per-row arrays present, the noise source, C below one thread
    stride (256), past the 48 KB shared-memory default for those flags, and a logits pitch wider than C."""
    smem = (3 if nucleus else 2) * C * 4
    return ("sampler", symbol, bool(nucleus), bool(row_step), bool(logprob), tuple(bool(r) for r in rows), noise, C < 256,
            smem > SMEM_DEFAULT, ld > C)


def plan_key(lens, nqs, append_eos, drop_last, mask_cond, mask_in, forget, labels, err):
    """... and whether the last sequence ends inside a time step (ids not a multiple of its quantizer count: the fine
    stage's flattened 1269 = 253 x 5 + 4, whose heads see one row fewer for the last quantizer)."""
    return ("token_plan", len(lens), bool(append_eos), bool(drop_last), bool(mask_cond), bool(mask_in), bool(forget), bool(labels),
            bool(err), nqs[-1] > 1, max(lens) + 1 > 256, min(lens) == 0, lens[-1] % nqs[-1] != 0)


# explicit cases of the family files (their parametrizations, restated here; each runs with a contiguous C-wide pitch)
def family_sampler_keys():
    keys = set()
    for C in (65, 1025, 16384):
        for mode in ("uniform", "engine_seed", "per_sequence"):
            for nucleus in (False, True):       # test_generate_per_row_gpu: test_sample_rows_equals_the_references_row_by_row
                keys.add(sampler_key("omlm_sample_rows", nucleus, False, False, (True, True, nucleus), mode, C, C))
        for nucleus in (False, True):           # test_generate_session_gpu: test_indexed_sampler_against_the_references
            keys.add(sampler_key("omlm_sample_rows_indexed", nucleus, True, False, (True, True, nucleus), "per_sequence", C, C))
        # test_logprobs_gpu: test_sampler_logprobs_per_row_arguments
        keys.add(sampler_key("omlm_sample_logprob", True, False, True, (True, True, True), "per_sequence", C, C))
    for C in (2, 65, 1025, 16384):              # test_logprobs_gpu: test_sampler_logprobs_against_float64
        for noise in ("uniform", "engine_seed", "per_sequence"):
            for nucleus in (False, True):
                keys.add(sampler_key("omlm_sample_logprob", nucleus, False, True, (False, False, False), noise, C, C))
    return keys


# (symbol, nucleus, row_step, logprob, rows, noise, C, ld): the forms the engine issues that the family files do not run
EXPLICIT_SAMPLER = [
    # generate's and the stages' decode step: logits rows padded to the GEMM's width
    ("omlm_sample_rows", False, False, False, (True, True, False), "uniform", 65, 128),
    ("omlm_sample_rows", False, False, False, (True, True, False), "engine_seed", 65, 128),
    ("omlm_sample_rows", False, False, False, (True, True, False), "per_sequence", 65, 128),
    ("omlm_sample_rows", True, False, False, (True, True, True), "engine_seed", 65, 128),
    ("omlm_sample_rows", True, False, False, (True, True, True), "per_sequence", 65, 128),
    ("omlm_sample_rows", False, False, False, (True, True, False), "engine_seed", 1025, 1152),
    ("omlm_sample_rows", True, False, False, (True, True, True), "engine_seed", 1025, 1152),
    ("omlm_sample_rows", False, False, False, (True, True, False), "uniform", 1025, 1152),
    ("omlm_sample_rows", False, False, False, (True, True, False), "per_sequence", 1025, 1152),
    ("omlm_sample_rows", True, False, False, (True, True, True), "per_sequence", 1025, 1152),
    ("omlm_sample_logprob", False, False, True, (True, True, False), "per_sequence", 65, 128),
    ("omlm_sample_logprob", True, False, True, (True, True, True), "per_sequence", 65, 128),
    ("omlm_sample_logprob", False, False, True, (True, True, False), "per_sequence", 1025, 1152),
    ("omlm_sample_logprob", True, False, True, (True, True, True), "per_sequence", 1025, 1152),
    # sessions: the indexed sampler on padded rows, with and without log-probabilities
    ("omlm_sample_rows_indexed", False, True, False, (True, True, False), "per_sequence", 65, 128),
    ("omlm_sample_rows_indexed", True, True, False, (True, True, True), "per_sequence", 65, 128),
    ("omlm_sample_rows_indexed", False, True, False, (True, True, False), "per_sequence", 1025, 1152),
    ("omlm_sample_rows_indexed", True, True, False, (True, True, True), "per_sequence", 1025, 1152),
    ("omlm_sample_rows_indexed_logprob", False, True, True, (True, True, False), "per_sequence", 65, 128),
    ("omlm_sample_rows_indexed_logprob", True, True, True, (True, True, True), "per_sequence", 65, 128),
    ("omlm_sample_rows_indexed_logprob", False, True, True, (True, True, False), "per_sequence", 1025, 1152),
    ("omlm_sample_rows_indexed_logprob", True, True, True, (True, True, True), "per_sequence", 1025, 1152),
    # past the 48 KB opt-in with a padded pitch: C = 8200 (nucleus 96 KB, top-k 64 KB)
    ("omlm_sample_rows", True, False, False, (True, True, True), "per_sequence", 8200, 8320),
    ("omlm_sample_rows_indexed_logprob", False, True, True, (True, True, False), "per_sequence", 8200, 8320),
]

# (lens, nqs, append_eos, drop_last, mask_cond, mask_in, forget, labels, err): each sequence's ids per row (time steps
# times quantizers), the last one predicted
EXPLICIT_PLAN = [
    ([12, 40, 51], [12, 1, 3], True, True, True, False, False, True, False),        # training (test_kernels_gpu's form)
    ([12, 40, 51], [12, 1, 3], True, True, True, True, True, True, False),           # training with a mask and forgetting
    ([12, 40, 51], [12, 1, 3], True, True, True, False, False, True, True),          # the trainer's: err_flag, forgetting or not
    ([12, 40, 51], [12, 1, 3], True, True, True, False, True, True, True),
    ([12, 300, 0], [12, 1, 3], True, True, True, False, True, True, True),
    ([12, 197, 810], [12, 1, 3], True, True, True, False, False, True, True),        # at the cfg2 shapes: past 256 ids a row
    ([12, 197, 810], [12, 1, 3], True, True, True, False, True, True, True),
    ([12, 241], [12, 1], True, True, True, False, False, True, False),               # semantic training (bench.py's semantic
    ([12, 241], [12, 1], True, True, True, False, False, True, True),                # stage): eval_loss and the step, with
    ([12, 241], [12, 1], True, True, True, False, True, True, False),                # and without forgetting and err_flag
    ([12, 241], [12, 1], True, True, True, False, True, True, True),
    ([12, 762, 1269], [12, 3, 5], True, True, True, False, False, True, False),      # fine training at bench.py's cfg3: the
    ([12, 762, 1269], [12, 3, 5], True, True, True, False, False, True, True),       # last sequence ends 4 ids into a step
    ([12, 762, 1269], [12, 3, 5], True, True, True, False, True, True, False),
    ([12, 762, 1269], [12, 3, 5], True, True, True, False, True, True, True),
    ([12, 30, 40], [12, 3, 5], True, True, True, False, True, True, True),           # fine training on whole steps
    ([4, 11, 30], [4, 1, 3], False, False, False, False, False, False, True),       # inference: generate, score, sessions
    ([4, 11, 0], [4, 1, 3], False, False, False, False, False, False, True),        # a request with no prefix
    ([4, 11, 0], [4, 1, 3], True, False, True, False, False, False, True),
    ([4, 11, 30], [4, 1, 3], True, False, True, False, False, False, True),         # decode.py's prompt plan
    ([12, 197, 60], [12, 1, 3], True, False, True, False, False, False, True),
    ([12, 197, 0], [12, 1, 3], True, False, True, False, False, False, True),
    ([12, 197, 60], [12, 1, 3], False, False, False, False, False, False, True),
    ([12, 197, 0], [12, 1, 3], False, False, False, False, False, False, True),
    ([12, 300, 0], [12, 1, 3], False, False, False, False, False, False, True),
    ([12, 300, 600], [12, 1, 3], False, False, False, False, False, False, True),
    ([12, 300, 600], [12, 1, 3], True, False, True, False, False, False, True),
    ([12, 300, 0], [12, 1, 3], True, False, True, False, False, False, True),
    ([4, 300], [4, 1], True, False, True, False, False, False, True),                 # the semantic stage
    ([4, 0], [4, 1], True, False, True, False, False, False, True),
    ([4, 300], [4, 1], False, False, False, False, False, False, True),
    ([4, 0], [4, 1], False, False, False, False, False, False, True),
    ([4, 11], [4, 1], True, False, True, False, False, False, True),
    ([4, 11], [4, 1], False, False, False, False, False, False, True),
    ([4, 30, 40], [4, 3, 5], True, False, True, False, False, False, True),           # the fine stage
    ([4, 30, 0], [4, 3, 5], True, False, True, False, False, False, True),
    ([4, 30, 40], [4, 3, 5], False, False, False, False, False, False, True),
    ([4, 30, 0], [4, 3, 5], False, False, False, False, False, False, True),
    ([4, 300, 400], [4, 3, 5], False, False, False, False, False, False, True),
    ([4, 300, 400], [4, 3, 5], True, False, True, False, False, False, True),
]


def covered_keys():
    keys = family_sampler_keys()
    keys |= {sampler_key(*c) for c in EXPLICIT_SAMPLER}
    keys |= {plan_key(*c) for c in EXPLICIT_PLAN}
    keys |= {("forgetful_mask",), ("embed_gather_pos_rows",), ("decode_advance_pos",)}     # exact at every form
    return keys


# ------------------------------------------------------------------------------------------------ the recorder
class _Recorder:
    """Wraps lib's sampler and token-path wrappers (the engine looks them up as module attributes at call time)."""

    def __init__(self, lib):
        self.lib, self.forms, self.phase, self.seen = lib, set(), None, set()
        self.orig = {n: getattr(lib, n) for n in NAMES}

    def _add(self, name, form):
        self.forms.add((name, form))
        self.seen.add((self.phase, form[0] if name in ("sample", "sample_rows_indexed") else name))

    def __enter__(self):
        o = self.orig

        def sample(logits, C, top_k, temperature, allow_eos, uniform, seed, tokens, next_row, row_offset, counters, pos, B, seeds=None,
                   top_p=None, top_k_rows=None, temperature_rows=None, top_p_rows=None, logprobs=None, sample_logprobs=None):
            rows = (top_k_rows is not None, temperature_rows is not None, top_p_rows is not None)
            sym, nucleus = sample_symbol(top_p, rows, logprobs is not None)
            noise = "uniform" if uniform is not None else "per_sequence" if seeds is not None else "engine_seed"
            if sym is None:
                sym = "omlm_sample" if seeds is None else "omlm_sample_seeded"
            self._add("sample", (sym, nucleus, False, logprobs is not None, rows, noise, C, logits.stride(0), B, top_k, float(temperature),
                                 None if top_p is None else float(top_p)))
            return o["sample"](logits, C, top_k, temperature, allow_eos, uniform, seed, tokens, next_row, row_offset, counters, pos, B,
                               seeds=seeds, top_p=top_p, top_k_rows=top_k_rows, temperature_rows=temperature_rows, top_p_rows=top_p_rows,
                               logprobs=logprobs, sample_logprobs=sample_logprobs)

        def sample_rows_indexed(logits, C, allow_eos, seeds, tokens, next_row, row_offset, step_rows, n_rows, top_k_rows, temperature_rows,
                                top_p_rows=None, logprobs=None, sample_logprobs=None):
            lp = logprobs is not None
            sym = "omlm_sample_rows_indexed_logprob" if lp else "omlm_sample_rows_indexed"
            self._add("sample", (sym, top_p_rows is not None, True, lp, (True, True, top_p_rows is not None), "per_sequence", C,
                                 logits.stride(0), logits.shape[0], 1, 1.0, None))
            return o["sample_rows_indexed"](logits, C, allow_eos, seeds, tokens, next_row, row_offset, step_rows, n_rows, top_k_rows,
                                            temperature_rows, top_p_rows, logprobs=logprobs, sample_logprobs=sample_logprobs)

        def token_plan(ids_list, codebooks, nqs, emb_row_base, start_row, *, append_eos, drop_last, mask_cond, pad_id=-1, mask_in=None,
                       forget_keep=None, want_labels=True, err_flag=None):
            lens = tuple(t.reshape(t.shape[0], -1).shape[1] for t in ids_list)
            self._add("token_plan", (lens, tuple(int(c) for c in codebooks), tuple(int(q) for q in nqs), ids_list[0].shape[0],
                                     bool(append_eos), bool(drop_last), bool(mask_cond), int(pad_id), mask_in is not None,
                                     forget_keep is not None, bool(want_labels), err_flag is not None))
            return o["token_plan"](ids_list, codebooks, nqs, emb_row_base, start_row, append_eos=append_eos, drop_last=drop_last,
                                   mask_cond=mask_cond, pad_id=pad_id, mask_in=mask_in, forget_keep=forget_keep, want_labels=want_labels,
                                   err_flag=err_flag)

        def forgetful_mask(B, N, num_drop, seed_tensor, stream_id, device):
            self._add("forgetful_mask", (B, N, num_drop))
            return o["forgetful_mask"](B, N, num_drop, seed_tensor, stream_id, device)

        def embed_gather_pos_rows(table, src_row, pos, pos_offset, pos_row_base, pos_rows, x):
            self._add("embed_gather_pos_rows", (x.shape[0], x.shape[1], table.shape[0], pos_row_base, pos_rows))
            return o["embed_gather_pos_rows"](table, src_row, pos, pos_offset, pos_row_base, pos_rows, x)

        def decode_advance_pos(pos, pos_last):
            self._add("decode_advance_pos", (pos.numel(),))
            return o["decode_advance_pos"](pos, pos_last)

        for n in NAMES:
            setattr(self.lib, n, locals()[n])
        return self

    def __exit__(self, *exc):
        for n, f in self.orig.items():
            setattr(self.lib, n, f)


def _record(act16, model, monkeypatch):
    with _Recorder(_lib()) as rec:
        call_forms.run(rec, model, act16, monkeypatch)
    if model in call_forms.SONGS_ONLY:
        expected = {("song session", n) for n in ("omlm_sample_rows_indexed", "token_plan", "decode_advance_pos")} | \
            {("score songs", "token_plan")}
    elif model in call_forms.BENCH_MODELS:
        expected = {(p, "token_plan") for p in call_forms.BENCH_PHASES} | {("bench step", "forgetful_mask"),
                                                                           ("bench deterministic step", "forgetful_mask")}
        if model in call_forms.GENERATION_MODELS:
            expected |= {("bench generation", "omlm_sample_rows"), ("bench generation", "token_plan")}
    else:
        expected = {(p, n) for p in call_forms.SESSION_PHASES for n in ("token_plan", "decode_advance_pos")} | \
            {("session logprobs", "omlm_sample_rows_indexed_logprob"), ("session join", "omlm_sample_rows_indexed"),
             ("session sampling", "omlm_sample_rows_indexed"), ("session sampling", "omlm_sample_rows_indexed_logprob")}
    if model in call_forms.SCORE_MODELS:
        expected.add(("score", "token_plan"))
    if model in call_forms.MODELS and model not in call_forms.SESSIONS_ONLY:
        expected |= {("default step", "token_plan"), ("default step", "forgetful_mask"), ("generate B=3", "omlm_sample_rows"),
                     ("generate sampling", "omlm_sample_rows"), ("generate sampling", "omlm_sample_logprob")}
    if model in call_forms.MODELS and call_forms.MODELS[model][0].get("use_absolute_position_embeddings"):
        expected |= {(p, "embed_gather_pos_rows") for p in ("generate B=3", "generate B=20", "session join")}
    assert expected <= rec.seen, f"entry points the engine did not call through lib: {sorted(expected - rec.seen)}"
    return rec.forms


# ------------------------------------------------------------------------------------------------ sampler replays
def replay_sampler(symbol, nucleus, row_step, logprob, rows, noise, C, ld, step_late=0):
    """One launch of the form at sample indices 0 and 2 (indexed: per-row indices, some rows at or past their last)
    against float64 -> failures.  step_late: the host replica's stream taken that many steps late (a planted fault)."""
    lib = _lib()
    from open_musiclm_b200.decode import seeds_tensor
    B = 24
    x, ks, temps, tops, seed, seeds, uni = _kernel_case(C, noise, B)
    if not nucleus:
        tops = [None] * B
    ra = _rows(ks, temps, tops, nucleus)
    kw = {n: ra[n] if present else None for n, present in zip(("top_k_rows", "temperature_rows", "top_p_rows"), rows)}
    k0, T0 = (ks[0], temps[0])
    if not rows[0]:
        ks = [k0] * B
    if not rows[1]:
        temps = [T0] * B
    scalar_p = tops[1] if nucleus and not rows[2] else None
    if nucleus and not rows[2]:
        tops = [scalar_p] * B
    xp = torch.full((B + 1, ld), float("nan"))
    xp[:B, :C] = x
    xd = xp.to(DEV)[:B]
    seed_t = torch.tensor([seed - 2 ** 64 if seed >= 2 ** 63 else seed], device=DEV)
    seeds_t = seeds_tensor(seeds, B, DEV)
    W = 6
    fails = []
    tag = f"sampler form {(symbol, nucleus, row_step, logprob, rows, noise, C, ld)}"
    for step, allow in ((0, False), (2, True)):
        # the log-probability samplers' one allocation: tokens [B, W], then logprobs and sample_logprobs (float32 [B, W]
        # each), then guard words; without them, tokens has a guard row B
        store = torch.zeros(2 * B * W + W, device=DEV, dtype=torch.int64)
        tokens = store[:B * W].view(B, W) if logprob else torch.empty(B + 1, W, device=DEV, dtype=torch.int64)
        after = store[B * W:].view(torch.float32)
        after.fill_(float("nan"))
        after[2 * B * W:] = 7.0
        lp, slp = (after[:B * W].view(B, W), after[B * W:2 * B * W].view(B, W)) if logprob else (None, None)
        tokens.fill_(SENTINEL)
        next_row = torch.full((B + 1,), SENTINEL, device=DEV, dtype=torch.int32)
        if row_step:
            t0 = [(step + b) % W for b in range(B)]
            n = [t + 1 + b % 3 for b, t in enumerate(t0)]
            t0[3], n[3] = 4, 4                           # has all its samples
            t0[4], n[4] = 5, 2                           # past them
            t0[5] = -1                                   # a free slot's index
            t_dev = torch.tensor(t0, device=DEV, dtype=torch.int32)
            lib.sample_rows_indexed(xd, C, allow, seeds_t, tokens[:B], next_row, 5, t_dev, torch.tensor(n, device=DEV, dtype=torch.int32),
                                    kw["top_k_rows"], kw["temperature_rows"], kw["top_p_rows"],
                                    logprobs=lp[:B] if logprob else None, sample_logprobs=slp[:B] if logprob else None)
            idx = [t if 0 <= t < min(nn, W) else None for t, nn in zip(t0, n)]
        else:
            counters = torch.tensor([step, 0], device=DEV, dtype=torch.int32)
            lib.sample(xd, C, k0, T0, allow, uni if noise == "uniform" else None, seed_t if noise == "engine_seed" else None, tokens[:B],
                       next_row, 5, counters, None, B, seeds=seeds_t if noise == "per_sequence" else None, top_p=scalar_p,
                       logprobs=lp[:B] if logprob else None, sample_logprobs=slp[:B] if logprob else None, **kw)
            idx = [step] * B
        torch.cuda.synchronize()
        tok, nr = tokens.cpu(), next_row.cpu()
        guard = bool((after[2 * B * W:] == 7.0).all()) if logprob else bool((tok[B] == SENTINEL).all())
        if not (guard and int(nr[B]) == SENTINEL):
            fails.append(f"{tag}: a word past the outputs was written")
        if row_step:
            want_t = [t + (i is not None) for t, i in zip(t0, idx)]
            if t_dev.cpu().tolist() != want_t:
                fails.append(f"{tag}: step_rows {t_dev.cpu().tolist()}, want {want_t} (t + 1 where a row samples)")
        written = torch.zeros(B, W, dtype=torch.bool)
        for b, t in enumerate(idx):
            if t is not None:
                written[b, t] = True
        if not bool((tok[:B][~written] == SENTINEL).all()):
            fails.append(f"{tag}: tokens written outside each row's sample index")
        if logprob and not all(bool(torch.isnan(a.cpu()[~written]).all()) for a in (lp, slp)):
            fails.append(f"{tag}: log-probabilities written outside each row's sample index")
        for b in range(B):
            t = idx[b]
            if t is None:
                if int(nr[b]) != SENTINEL:
                    fails.append(f"{tag}: row {b} wrote next_row without sampling")
                continue
            if int(nr[b]) != int(tok[b, t]) + 5 and int(tok[b, t]) < C:
                fails.append(f"{tag}: row {b}: next_row {int(nr[b])} for token {int(tok[b, t])}")
            if row_step or noise == "per_sequence":
                from test_generate_seeded_cpu import seeded_uniforms
                u = torch.from_numpy(seeded_uniforms(seeds[b], t + step_late, C))[None]
            else:
                u = _row_uniforms(noise, uni, seed, seeds, t + step_late, B, C)[b:b + 1]
            top = None if tops[b] in (None, 1.0) else tops[b]
            T = float(np.float32(temps[b]))
            try:
                check_nucleus(tok[b:b + 1, t], x[b:b + 1], u, ks[b], T, allow, top, (tag, b, t))
            except AssertionError as e:
                fails.append(f"{tag}: row {b} step {t}: {str(e).splitlines()[0][:200]}")
                continue
            if logprob and 0 <= int(tok[b, t]) < C:
                xt, tt = x[b:b + 1].to(DEV), tok[b:b + 1, t].to(DEV)
                try:
                    v, bnd = model_logprob(xt, tt)
                    _close(lp[b:b + 1, t], v, bnd)
                    v, bnd = sample_logprob(xt, tt, ks[b], T, allow, top)
                    _close(slp[b:b + 1, t], v, bnd)
                except AssertionError as e:
                    fails.append(f"{tag}: row {b} step {t}: log-probabilities {str(e)[:200]}")
    return fails


# ------------------------------------------------------------------------------------------------ token plan replays
def plan_reference(ids, codebooks, nqs, emb_row_base, start_row, append_eos, drop_last, mask_cond, pad_id, mask_in, forget):
    """numpy statement of omlm_token_plan (include/omlm_b200.h): (ids_out, src_row, key_mask, labels, err bits).
    Per sequence s: a start-token row, then its tokens (eos = codebook appended in wrapper mode; the last sequence
    loses its last token with drop_last); conditioning pads and eos masked out and zeroed with mask_cond; the key
    mask that one, or mask_in instead when given, AND forget_keep when given; the row is
    emb_row_base + id + codebook * (t mod q) for q > 1, -1 where that sum equals pad_id, and -1 with err bit s where
    it lies outside [0, (codebook + 1) q)."""
    B, S = ids[0].shape[0], len(ids)
    ids_out, src, keym, labels, err = [], [], [], [], 0
    for s, x in enumerate(ids):
        last = s == S - 1
        cb, q = codebooks[s], nqs[s]
        full = np.concatenate([x, np.full((B, 1), cb)], 1) if append_eos else x.copy()
        labels.append(full.astype(np.int32))
        tok = full[:, :-1] if (last and drop_last) else full.copy()
        m = np.ones(tok.shape, bool)
        if mask_cond and not last:
            m = (tok != pad_id) & (tok != cb)
            tok = np.where(m, tok, 0)
        ids_out.append(tok)
        c = tok + (cb * (np.arange(tok.shape[1]) % q))[None] if q > 1 else tok
        pad = c == pad_id
        oob = ~pad & ((c < 0) | (c >= (cb + 1) * q))
        if oob.any():
            err |= 1 << s
        src.append(np.full((B, 1), start_row[s]))
        src.append(np.where(pad | oob, -1, emb_row_base[s] + c))
        keym.append(np.ones((B, 1), bool))
        keym.append(np.ones(tok.shape, bool) if not (mask_cond and not last) else m)
    key = np.concatenate(keym, 1)
    if mask_in is not None:
        key = mask_in.astype(bool)
    if forget is not None:
        key = key & forget.astype(bool)
    return np.concatenate(ids_out, 1), np.concatenate(src, 1).astype(np.int32), key, np.concatenate(labels, 1), err


def replay_plan(lens, nqs, append_eos, drop_last, mask_cond, mask_in, forget, labels, err, B=5, seed=None, start_shift=0):
    """One token_plan launch at the form with fresh ids (pads at quantizer positions 0 and others, eos ids in the
    conditioning, and with err ids outside their tables in two sequences, the last non-empty one and one the seed picks)
    against plan_reference and the bits planted -> failures.
    start_shift: the reference's start rows shifted by one (a planted fault)."""
    lib = _lib()
    seed = sum(lens) + 7 * len(lens) if seed is None else seed
    g = torch.Generator().manual_seed(seed)
    S = len(lens)
    cbs = [100 + 7 * s for s in range(S)]
    bases = [sum((cbs[i] + 1) * nqs[i] for i in range(s)) for s in range(S)]
    total = bases[-1] + (cbs[-1] + 1) * nqs[-1]
    starts = [total + s for s in range(S)]
    ids = []
    for s, n in enumerate(lens):
        x = torch.randint(0, cbs[s], (B, n), generator=g)
        if x.shape[1]:
            flat = x.view(-1)
            pick = torch.randint(0, flat.numel(), (max(1, flat.numel() // 9),), generator=g)
            flat[pick] = -1                                      # pads, at every quantizer position
            if s < S - 1:
                flat[pick[: len(pick) // 2] // 2] = cbs[s]       # eos ids in the conditioning
        ids.append(x)
    bad = set()
    if err:     # ids past their tables: in the last non-empty sequence (at quantizer q - 1) and one other the seed picks
        live = [s for s in range(S) if ids[s].shape[1]]
        bad = {live[-1]} | ({live[seed % (len(live) - 1)]} if len(live) > 1 else set())
        for s in bad:
            q, n = nqs[s], ids[s].shape[1]
            t = (n // 2) // q * q + q - 1 if n >= q else n - 1
            ids[s][(B - 1 + s) % B, t] = 10 * (cbs[s] + 1) * q + 3
    n_tok = [l + (1 if append_eos else 0) - (1 if (drop_last and s == S - 1) else 0) for s, l in enumerate(x.shape[1] for x in ids)]
    N = sum(n + 1 for n in n_tok)
    mi = (torch.rand(B, N, generator=g) > 0.2).to(torch.uint8) if mask_in else None
    fk = (torch.rand(B, N, generator=g) > 0.3).to(torch.uint8) if forget else None
    ef = torch.tensor([1 << 20, 0], device=DEV, dtype=torch.int32) if err else None        # a bit latched earlier stays
    ids_out, src_row, key_mask, lab, nt = lib.token_plan([x.to(DEV) for x in ids], cbs, nqs, bases, starts, append_eos=append_eos,
                                                         drop_last=drop_last, mask_cond=mask_cond, mask_in=None if mi is None else mi.to(DEV),
                                                         forget_keep=None if fk is None else fk.to(DEV), want_labels=labels,
                                                         err_flag=None if ef is None else ef[:1])
    torch.cuda.synchronize()
    ref = plan_reference([x.numpy() for x in ids], cbs, nqs, bases, [r + start_shift for r in starts], append_eos, drop_last, mask_cond, -1,
                         None if mi is None else mi.numpy(), None if fk is None else fk.numpy())
    tag = f"token_plan form {(lens, nqs, append_eos, drop_last, mask_cond, mask_in, forget, labels, err)} shift={start_shift}"
    fails = []
    if list(nt) != n_tok:
        fails.append(f"{tag}: n_tok {nt}")
    for name, got, want in (("ids_out", ids_out, ref[0]), ("src_row", src_row, ref[1]), ("key_mask", key_mask, ref[2])):
        got = got.cpu().numpy()
        if name == "key_mask":
            got = got.astype(bool)
        if got.shape != want.shape or not np.array_equal(got, want):
            at = np.argwhere(got != want)[:4].tolist() if got.shape == want.shape else (got.shape, want.shape)
            fails.append(f"{tag}: {name} differs at {at}")
    if labels and not np.array_equal(lab.cpu().numpy(), ref[3]):
        fails.append(f"{tag}: labels differ")
    if err:
        e, want = ef.cpu().tolist(), sum(1 << s for s in bad)
        if ref[4] != want or e != [want | 1 << 20, 0]:
            fails.append(f"{tag}: err_flag {e}, want bits {want} (reference {ref[4]}) on top of bit 20, the word after it 0")
    return fails


def replay_training_plan():
    """The training form bit-exact against oracle.restatement.prepare_ids / embedding_rows."""
    from oracle import restatement as R
    lib = _lib()
    cfg = R.coarse_cfg(codebook=1024, n_clap_q=12, n_coarse_q=3)
    g = torch.Generator().manual_seed(8)
    toks = [torch.randint(0, 1024, s, generator=g) for s in [(3, 12), (3, 300), (3, 90, 3)]]
    toks[0][0, 0] = -1; toks[1][1, 257] = -1; toks[1][2, 3] = 1024; toks[2][0, 0, 0] = -1; toks[2][1, 2, 1] = -1; toks[2][2, 88, 2] = -1
    ids_np, mask_np, labels_np = R.prepare_ids(cfg, [t.numpy() for t in toks], True)
    rows = R.embedding_rows(cfg, ids_np)
    bases = [0, 1025 * 12, 1025 * 12 + 1025]
    total = bases[2] + 1025 * 3
    ids_out, src_row, key_mask, labels, _ = lib.token_plan([t.to(DEV) for t in toks], [1024] * 3, [12, 1, 3], bases,
                                                           [total, total + 1, total + 2], append_eos=True, drop_last=True, mask_cond=True)
    exp = []
    for s, (r, pad) in enumerate(rows):
        exp.append(np.full((3, 1), total + s))
        exp.append(np.where(pad, -1, r + bases[s]))
    assert np.array_equal(ids_out.cpu().numpy(), np.concatenate(ids_np, 1))
    assert np.array_equal(key_mask.cpu().numpy().astype(bool), mask_np)
    assert np.array_equal(labels.cpu().numpy(), np.concatenate(labels_np, 1).astype(np.int32))
    assert np.array_equal(src_row.cpu().numpy(), np.concatenate(exp, 1).astype(np.int32))


# ------------------------------------------------------------------------------------------------ the other four
def replay_forgetful(B, N, num_drop):
    lib = _lib()
    for seed, sid in ((12345, 7), (0x0123456789ABCDEF, (5 << 32) + 3)):
        keep = lib.forgetful_mask(B, N, num_drop, seed_tensor(seed), sid, DEV).cpu().numpy()
        if not np.array_equal(keep, forgetful_replica(seed, sid, B, N, num_drop)):
            return [f"forgetful_mask {(B, N, num_drop)} seed {seed}: differs from the replica"]
    return []


def replay_gather_pos_rows(M, D, rows, base, lim, g):
    lib = _lib()
    table = torch.randn(rows, D, generator=g).to(DEV)
    src = torch.randint(-3, base, (M,), generator=g, dtype=torch.int32)
    pos = torch.randint(-5, lim + 5, (M,), generator=g, dtype=torch.int32)
    off = torch.randint(-8, 8, (M,), generator=g, dtype=torch.int32)
    pos[0], off[0], pos[-1], off[-1] = lim, 0, 0, -1                    # just past each end
    xb = torch.full((M + 1, D), float("nan"), device=DEV)
    xb[M:] = 7.0
    lib.embed_gather_pos_rows(table, src.to(DEV), pos.to(DEV), off.to(DEV), base, lim, xb[:M])
    torch.cuda.synchronize()
    tab = table.cpu()
    want = tab[src.long().clamp_min(0)] * (src >= 0)[:, None]
    p = (pos + off).long()
    inside = (p >= 0) & (p < lim)
    want = want + tab[(base + p.clamp(0, lim - 1))] * inside[:, None]
    out = xb.cpu()
    fails = [] if torch.equal(out[:M], want) else [f"embed_gather_pos_rows {(M, D, rows, base, lim)}: differs from torch indexing"]
    if not bool((out[M:] == 7.0).all()):
        fails.append(f"embed_gather_pos_rows {(M, D, rows, base, lim)}: the row past M was written")
    return fails


def replay_advance(B, g):
    lib = _lib()
    last = torch.randint(-2, 50, (B + 1,), generator=g, dtype=torch.int32)
    pos = last + torch.randint(-3, 3, (B + 1,), generator=g, dtype=torch.int32)
    pd, ld = pos.to(DEV), last.to(DEV)
    lib.decode_advance_pos(pd[:B], ld[:B])
    want = pos.clone()
    want[:B] += (pos[:B] < last[:B]).int()
    return [] if torch.equal(pd.cpu(), want) and torch.equal(ld.cpu(), last) else [f"decode_advance_pos B={B}: differs"]


# ------------------------------------------------------------------------------------------------ the tests
@pytest.mark.parametrize("model", call_forms.MODEL_KEYS)
@pytest.mark.parametrize("act16", ["fp16", "bf16"])
def test_engine_call_forms_replayed_and_covered(act16, model, monkeypatch):
    forms = sorted(_record(act16, model, monkeypatch), key=repr)
    g = torch.Generator().manual_seed(41)
    fails, keys = [], set()
    samp = {}
    for name, f in forms:
        if name == "sample":
            sym, nucleus, row_step, lp, rows, noise, C, ld = f[:8]
            samp.setdefault(sampler_key(sym, nucleus, row_step, lp, rows, noise, C, ld), f[:8])
        elif name == "token_plan":
            lens, cbs, nqs, B, ae, dl, mc, pad, mi, fk, lab, err = f
            assert pad == -1, f
            k = plan_key(lens, nqs, ae, dl, mc, mi, fk, lab, err)
            if k not in keys:
                fails += replay_plan(list(lens), list(nqs), ae, dl, mc, mi, fk, lab, err, B=B, seed=len(keys))
            keys.add(k)
        elif name == "forgetful_mask":
            fails += replay_forgetful(*f)
            keys.add(("forgetful_mask",))
        elif name == "embed_gather_pos_rows":
            M, D, rows_t, base, lim = f
            fails += replay_gather_pos_rows(M, D, rows_t, base, lim, g)
            keys.add(("embed_gather_pos_rows",))
        elif name == "decode_advance_pos":
            fails += replay_advance(f[0], g)
            keys.add(("decode_advance_pos",))
    for k, f in samp.items():
        fails += replay_sampler(*f)
        keys.add(k)
    print(f"act16={act16} {model}: {len(keys)} keys issued by the engine")
    for k in sorted(keys, key=repr):
        print("   ", k)
    assert not fails, "\n".join(fails[:40])
    missing = sorted((k for k in keys if k not in covered_keys()), key=repr)
    assert not missing, f"engine call forms without an explicit case: {missing}"


@pytest.mark.parametrize("case", EXPLICIT_SAMPLER, ids=lambda c: f"{c[0][5:]}-{'p' if c[1] else 'k'}-{c[5]}-C{c[6]}-ld{c[7]}")
def test_explicit_sampler_forms(case):
    fails = replay_sampler(*case)
    assert not fails, "\n".join(fails[:20])


@pytest.mark.parametrize("case", EXPLICIT_PLAN, ids=lambda c: f"{'-'.join(map(str, c[0]))}-q{c[1][-1]}-{''.join(str(int(v)) for v in c[2:])}")
def test_explicit_token_plan_forms(case):
    fails = replay_plan(*case)
    assert not fails, "\n".join(fails)


def test_training_token_plan_equals_the_restatement():
    replay_training_plan()


def test_other_token_path_forms_exact():
    g = torch.Generator().manual_seed(2)
    fails = replay_forgetful(4, 2, 1) + replay_forgetful(3, 777, 116) + replay_forgetful(2, 1500, 1499)
    fails += replay_gather_pos_rows(37, 72, 300, 200, 90, g) + replay_gather_pos_rows(256, 1024, 1200, 1100, 100, g)
    fails += replay_advance(1, g) + replay_advance(256, g)
    assert not fails, "\n".join(fails)


# ------------------------------------------------------------------------------------------------ discrimination
def test_sampler_replay_rejects_a_philox_counter_one_step_late():
    """The replay passes with the stream at each row's own sample index and fails when the replica is one step late."""
    case = ("omlm_sample_rows", True, False, False, (True, True, True), "engine_seed", 1025, 1152)
    assert not replay_sampler(*case)
    assert replay_sampler(*case, step_late=1)
    case = ("omlm_sample_rows_indexed", False, True, False, (True, True, False), "per_sequence", 65, 128)
    assert not replay_sampler(*case)
    assert replay_sampler(*case, step_late=1)


def test_token_plan_replay_rejects_a_start_row_shifted_by_one():
    case = ([12, 197, 60], [12, 1, 3], True, False, True, False, False, False, True)
    assert not replay_plan(*case)
    assert replay_plan(*case, start_shift=1)
