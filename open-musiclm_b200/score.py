"""Teacher-forced log-likelihoods of given token sequences: `TokenConditionedTransformerWrapper.score` for rows of one
stage and `MusicLM.score_tokens` for whole songs through MusicLM's sliding windows.

A scored row is one prompt (conditioning sequences with their eos, then the predicted sequence's tokens) and the range
of its predicted tokens whose log p is wanted.  The rows are packed back to back without padding into forwards of at
most max_rows rows (pack_groups), each one Engine.forward_packed over a session.PackedPrefill plan with its prefix
rows scored: the varlen attention and FFN-up kernels give every row what the fixed-length kernels give its prompt
alone, and the logit heads and omlm_token_logprob are those of generate's prefill, so every value is bit for bit what
generate(pred_token_ids=<the prompt's tokens>, max_time_steps=<their steps>, return_logprobs=True) reports for that
row alone (DESIGN section 4, "Scoring").

Rows are given as index arrays into flat token sources (ScoreRow), so that thousands of windows cut from a few streams
cost a handful of gathers instead of one slice per window.  song_rows turns the window plans of stages.plan_song into
such rows; it is host code only.
"""
import numbers
from typing import List, NamedTuple

import numpy as np
import torch

from . import lib
from .decode import bias_table, check_pred_lengths
from .session import PackedPrefill

MAX_ROWS = 16384          # default rows per packed forward


class ScoreRow(NamedTuple):
    """One prompt to score.  cond: per conditioning sequence, int64 indices into its flat source (the eos is added);
    pred: int64 indices into the flat source of predicted tokens, the prompt's predicted tokens in order; its tokens
    first ... len(pred) - 1 are scored, their log p going to the flat output at `out` (len(pred) - first indices)."""
    cond: list
    pred: np.ndarray
    first: int
    out: np.ndarray


def check_max_rows(max_rows, where: str) -> int:
    if isinstance(max_rows, bool) or not isinstance(max_rows, numbers.Integral) or max_rows < 1:
        raise ValueError(f"{where}: max_rows must be an int >= 1, not {max_rows!r}")
    return int(max_rows)


def check_ids(t: torch.Tensor, codebook: int, what: str, where: str, mask=None):
    """ValueError unless every id of t (where mask is true) lies in [0, codebook)."""
    bad = (t < 0) | (t >= codebook)
    if mask is not None:
        bad &= mask
    if bool(bad.any()):
        raise ValueError(f"{where}: {what} holds ids outside the codebook [0, {codebook})")


def prompt_rows(row: ScoreRow) -> int:
    """The packed rows of a row's prompt: each sequence after its start token, conditioning sequences with their eos."""
    return sum(len(c) + 2 for c in row.cond) + len(row.pred) + 1


def pack_groups(lengths, max_rows: int) -> List[List[int]]:
    """Prompts of the given lengths (rows) -> groups of their indices, each one packed forward of at most max_rows rows,
    a prompt longer than max_rows alone in its own: first-fit decreasing (longest first, each into the first group
    with room), indices ascending within a group.  The grouping changes no value."""
    order = sorted(range(len(lengths)), key=lambda i: (-lengths[i], i))
    groups, room = [], []
    shortest = min(lengths, default=0)
    open_ = []                                       # groups that still have room for the shortest prompt
    for i in order:
        n = lengths[i]
        for g in open_:
            if n <= room[g]:
                groups[g].append(i)
                room[g] -= n
                break
        else:
            groups.append([i])
            room.append(max_rows - n)
            open_.append(len(groups) - 1)
        open_ = [g for g in open_ if room[g] >= shortest]
    return [sorted(g) for g in groups]


def score_rows(wrapper, cond_src, pred_src, rows: List[ScoreRow], out: torch.Tensor, max_rows: int = MAX_ROWS):
    """Scores `rows` of the wrapper's stage into the flat float32 `out`: cond_src (one flat int64 device tensor per
    conditioning sequence) and pred_src (flat int64) hold the tokens the rows index, every id checked.  One token plan
    per distinct conditioning shape, then one packed forward per group of pack_groups."""
    eng = wrapper.transformer.engine
    dev, q, C = eng.dev, eng.seqs[-1].num_quantizers, eng.seqs[-1].codebook_size + 1
    live = [i for i, r in enumerate(rows) if len(r.out)]
    if not live:
        return
    pad = pred_src.numel()                          # pred_ext[pad] = 0 (padding), pred_ext[pad + 1] = -100 (no label)
    pred_ext = torch.cat([pred_src, pred_src.new_tensor([0, -100])])
    cond_ext = [torch.cat([c, c.new_tensor([e])]) for c, e in zip(cond_src, wrapper.eos_ids)]    # its last id: the eos
    # token plans: the rows of one conditioning shape in one lib.token_plan call, padded to their longest prediction;
    # row i's prompt is then src[at[i] : at[i] + P_i]
    buckets = {}
    for i in live:
        buckets.setdefault(tuple(len(c) for c in rows[i].cond), []).append(i)
    src, at, base = [], {}, 0
    for shape, idx in buckets.items():
        T = max(len(rows[i].pred) for i in idx)
        host = [np.stack([np.append(rows[i].cond[s], len(cond_src[s])) for i in idx]) for s in range(len(shape))]
        host.append(np.stack([np.pad(rows[i].pred, (0, T - len(rows[i].pred)), constant_values=pad) for i in idx]))
        up = torch.from_numpy(np.concatenate([h.reshape(-1) for h in host]).astype(np.int64)).to(dev, non_blocking=True)
        ids, o = [], 0
        for s, h in enumerate(host):
            ext = cond_ext[s] if s < len(shape) else pred_ext
            ids.append(ext[up[o:o + h.size]].view(h.shape))
            o += h.size
        _, src_row, _, _, _ = lib.token_plan(ids, [s.codebook_size for s in eng.seqs], [s.num_quantizers for s in eng.seqs],
                                             eng.emb_row_base, eng.start_row, append_eos=False, drop_last=False, mask_cond=False,
                                             want_labels=False, err_flag=eng.err_flag)
        N = src_row.shape[1]
        for b, i in enumerate(idx):
            at[i] = base + b * N
        src.append(src_row.view(-1))
        base += src_row.numel()
    src = torch.cat(src) if len(src) > 1 else src[0]
    n_tok = {i: [len(c) + 1 for c in rows[i].cond] + [len(rows[i].pred)] for i in live}
    P = [prompt_rows(rows[i]) for i in live]
    groups = [[live[j] for j in g] for g in pack_groups(P, max_rows)]
    size = dict(zip(live, P))
    ws = eng.packed_workspace(max(sum(size[i] for i in g) for g in groups),
                              max(len(g) + sum(len(rows[i].pred) for i in g) for g in groups))
    table = bias_table(eng, max(P))["table"]
    for g in groups:
        k = len(g)
        plan = PackedPrefill([n_tok[i] for i in g], np.arange(k), max(P), q, eng.h, eng.abs_row_base if eng.abs_pos else None,
                             logprob=True)
        dv = plan.to_device(dev)
        tok_src = np.concatenate([rows[i].pred for i in g])
        tok_dst = np.concatenate([np.concatenate([np.full(rows[i].first, -1), rows[i].out]) for i in g])
        lab = plan.label_idx                        # head row -> its token among the group's predicted tokens (-1: next token)
        label_src = np.where(lab < 0, pad + 1, tok_src[np.maximum(lab, 0)])
        dst = tok_dst[lab[k:]]
        sel = k + np.flatnonzero(dst >= 0)
        dst = dst[dst >= 0]
        host = [np.concatenate([at[i] + np.arange(size[i]) for i in g]), label_src, sel, dst]
        up = torch.from_numpy(np.concatenate(host).astype(np.int64)).to(dev, non_blocking=True)
        cut = np.cumsum([0] + [len(h) for h in host])
        src_idx, label_idx, sel_d, dst_d = (up[a:b] for a, b in zip(cut[:-1], cut[1:]))
        dv.src_row = src[src_idx]
        eng.forward_packed(ws, dv, table)
        lp = torch.empty(plan.head_rows, device=dev, dtype=torch.float32)
        lib.token_logprob(ws["logits"][:plan.head_rows], pred_ext[label_idx].to(torch.int32), C, lp)
        out.index_copy_(0, dst_d, lp[sel_d])


def score_batch(wrapper, conditioning_token_ids, pred_token_ids, pred_lengths, max_rows):
    """TokenConditionedTransformerWrapper.score: checks, then one ScoreRow per row with real tokens."""
    where = "open_musiclm_b200 score"
    max_rows = check_max_rows(max_rows, where)
    infos = wrapper.token_sequences
    q, cb = infos[-1].num_quantizers, infos[-1].codebook_size
    if not isinstance(conditioning_token_ids, (list, tuple)) or len(conditioning_token_ids) != len(infos) - 1:
        raise ValueError(f"{where}: conditioning_token_ids must be a list of {len(infos) - 1} tensors")
    x = pred_token_ids
    if not isinstance(x, torch.Tensor) or not ((x.dim() == 3 and x.shape[2] == q) or (x.dim() == 2 and q == 1)):
        got = list(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__
        raise ValueError(f"{where}: pred_token_ids must be [b, t, {q}] (whole time steps), not {got}")
    B, T = x.shape[0], x.shape[1]
    for s, t in enumerate(conditioning_token_ids):
        if not isinstance(t, torch.Tensor) or t.dim() < 1 or t.shape[0] != B:
            raise ValueError(f"{where}: conditioning sequence {s} must be a tensor of {B} rows, [{B}, ...]")
        check_ids(t, infos[s].codebook_size, f"conditioning sequence {s}", where)
    lengths = check_pred_lengths(pred_lengths, x, B, caller="score")
    lengths = [T] * B if lengths is None else lengths
    real = torch.arange(T, device=x.device)[None] < torch.tensor(lengths, device=x.device)[:, None]
    check_ids(x.reshape(B, T, q), cb, "pred_token_ids", where, real[..., None])
    m = wrapper.transformer
    n_cond = [t[0].numel() for t in conditioning_token_ids]
    if m.use_absolute_position_embeddings and any(lengths):             # the reference's nn.Embedding lookup (generate)
        lim = int(m.max_absolute_position_embeddings)
        for s, n in enumerate(n_cond):
            if n + 1 > lim:
                raise IndexError(f"{where}: conditioning sequence {s} has {n + 1} tokens but max_absolute_position_embeddings is {lim}")
        for b, n in enumerate(lengths):
            if n * q > lim:
                raise IndexError(f"{where}: the predicted sequence of row {b} has {n * q} tokens but max_absolute_position_embeddings is {lim}")
    dev = m.device
    cond = [t.to(dev, torch.int64).reshape(-1) for t in conditioning_token_ids]
    pred = x.to(dev, torch.int64).reshape(-1)
    out = torch.zeros(B * T * q, device=dev, dtype=torch.float32)
    rows = []
    for b, n in enumerate(lengths):
        idx = b * T * q + np.arange(n * q)
        rows.append(ScoreRow([b * c + np.arange(c) for c in n_cond], idx, 0, idx))
    score_rows(wrapper, cond, pred, rows, out, max_rows)
    return out.view(B, T, q)


# ---------------------------------------------------------------------------------------- songs through the windows
class _Layout(NamedTuple):
    """Where one song's generated stream (as MusicLM.generate_tokens builds it internally, the window jobs' frame)
    sits in what generate_tokens returns: that output is `pre` prime steps, then the stream from step `lo` on.  The
    stream's first `plen0` steps are the prime steps `tail` ... of the prime (the first window's prefix, copied in)."""
    pre: int
    lo: int
    plen0: int
    tail: int
    q: int


def song_layouts(plan, prime_lengths, qs):
    """{stream: _Layout} of a song's plan (stages.plan_song) and prime lengths (None: no prime); qs: quantizers per
    stream.  ValueError when generate_tokens' crop of a stream reaches past the prime steps at its start: the output
    then lacks generated tokens the windows read or wrote, so a prime this short is inconsistent with the plan.  (Every
    window reads its streams at or after their crop, or inside the prime steps before it.)"""
    from .stages import STREAMS
    tp = prime_lengths or (0, 0, 0)
    lo = dict(semantic=plan.sem_lo, coarse=0 if plan.coarse_only else plan.coarse_lo, fine=plan.fine_lo)
    out = {}
    for st, name in enumerate(STREAMS[:2 if plan.coarse_only else 3]):
        first = next((j for j in plan.jobs if j.stage == st), None)
        ref = first.prefix if first is not None else None
        tail, plen0 = (ref[1], ref[2] - ref[1]) if ref is not None and ref[0].startswith("prime_") else (0, 0)
        pre = 0 if name == "semantic" or plan.coarse_only or prime_lengths is None else tp[st]
        if lo[name] > plen0:
            raise ValueError(f"open_musiclm_b200 MusicLM.score_tokens: a prime of {tp[st]} {name} steps is shorter than the "
                             f"{lo[name]} steps generate_tokens crops from that stream, so its output lacks generated tokens")
        out[name] = _Layout(pre, lo[name], plen0, tail, qs[st])
    return out


def output_length(plan, layout: _Layout, name: str) -> int:
    """Time steps of generate_tokens' output stream `name` for this plan."""
    return layout.pre + plan.length[name] - layout.lo


def song_rows(plans, layouts, seg, primes, out_off, clap):
    """The ScoreRows of every window job of the songs, per stage (semantic, coarse, fine): plans and layouts (song_layouts)
    per song; seg[name][i] (time steps): where song i's segment of stream `name` starts in that stream's flat source,
    the segment being the song's prime (primes[name][i] steps, 0 without one) followed by its output; out_off[name][i]:
    where song i's output starts in the flat scores of `name`; clap[i]: the token indices of song i's clap ids.

    Window j of stage st appends its generate output's steps drop ... steps - 1 to its stream at dest.  Its prompt is
    its conditioning (clap ids, then its cond slice), its prefix (plen steps), then the stream's steps
    dest + max(plen - drop, 0) ... dest + steps - drop - 1, which its generate call returned after the prefix.  Those
    are scored; the prefix and the prime steps a first window copies into its stream are not."""
    from .stages import STREAMS
    rows = [[], [], []]
    for i, (plan, lay) in enumerate(zip(plans, layouts)):
        def steps(name, a, b):
            """Source steps of stream (or prime) `name`'s steps a ... b - 1."""
            p = np.arange(a, b)
            if name.startswith("prime_"):
                return seg[name[6:]][i] + p
            L = lay[name]
            return seg[name][i] + np.where(p < L.lo, L.tail + p, primes[name][i] + L.pre + p - L.lo)

        def tokens(name, s):
            q = lay[name.replace("prime_", "")].q
            return (s[:, None] * q + np.arange(q)).reshape(-1)

        for job in plan.jobs:
            name = STREAMS[job.stage]
            plen = 0 if job.prefix is None else job.prefix[2] - job.prefix[1]
            a, b = job.dest + max(plen - job.drop, 0), job.dest + job.steps - job.drop
            if b <= a:
                continue
            L = lay[name]
            cond = [clap[i]] + ([] if job.cond is None else [tokens(job.cond[0], steps(*job.cond))])
            pre = np.zeros(0, dtype=np.int64) if job.prefix is None else tokens(job.prefix[0], steps(*job.prefix))
            pred = np.concatenate([pre, tokens(name, steps(name, a, b))])
            out = tokens(name, out_off[name][i] + L.pre + np.arange(a, b) - L.lo)
            rows[job.stage].append(ScoreRow(cond, pred, len(pre), out))
    return rows


def _songs(t, n: int, what: str, where: str):
    """A batch argument -> one entry per song: a list or tuple of n entries as it is, a tensor [n, ...] row by row."""
    if isinstance(t, (list, tuple)):
        if len(t) != n:
            raise ValueError(f"{where}: {what} has {len(t)} entries for {n} songs")
        return list(t)
    if not isinstance(t, torch.Tensor) or t.dim() < 1 or t.shape[0] != n:
        got = list(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
        raise ValueError(f"{where}: {what} must be a tensor [{n}, ...] or a list of {n} tensors [1, ...], not {got}")
    return [t[i:i + 1] for i in range(n)]


def _steps(t, q: int, what: str, where: str) -> torch.Tensor:
    """One song's stream [1, T, q] ([1, T] when q = 1) -> [1, T, q], or ValueError."""
    if isinstance(t, torch.Tensor) and t.dim() == 2 and q == 1:
        t = t.unsqueeze(-1)
    if not isinstance(t, torch.Tensor) or t.dim() != 3 or t.shape[0] != 1 or t.shape[2] != q:
        got = list(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
        raise ValueError(f"{where}: each song's {what} must be [1, T, {q}], not {got}")
    return t


def score_songs(mlm, *, clap_token_ids, semantic_token_ids, coarse_token_ids, fine_token_ids, output_seconds, windowing: dict,
                primes, coarse_only, max_rows):
    """MusicLM.score_tokens (its docstring states the contract): checks, the songs' plans and layouts, the flat
    token sources of each stream (per song its prime, then its output), song_rows, and one score_rows per stage."""
    from .stages import STREAMS, _check_prime, plan_song
    where = "open_musiclm_b200 MusicLM.score_tokens"
    max_rows = check_max_rows(max_rows, where)
    if not isinstance(coarse_only, bool):
        raise ValueError(f"{where}: coarse_only must be a bool, not {coarse_only!r}")
    if coarse_only != (fine_token_ids is None):
        raise ValueError(f"{where}: fine_token_ids is {'not taken with' if coarse_only else 'needed without'} coarse_only")
    stages = (mlm.semantic, mlm.coarse, mlm.fine)
    infos = [s.transformer_wrapper.token_sequences for s in stages]
    qs = tuple(inf[-1].num_quantizers for inf in infos)
    names = STREAMS[:2 if coarse_only else 3]
    listed = isinstance(semantic_token_ids, (list, tuple))
    n = len(semantic_token_ids) if listed else semantic_token_ids.shape[0] if isinstance(semantic_token_ids, torch.Tensor) else None
    if not n:
        raise ValueError(f"{where}: semantic_token_ids must be a tensor [b, T] or a non-empty list of tensors [1, T]")
    given = {name: [_steps(t, qs[st], f"{name} tokens", where)
                    for t in _songs((semantic_token_ids, coarse_token_ids, fine_token_ids)[st], n, f"{name}_token_ids", where)]
             for st, name in enumerate(names)}
    clap = [t.reshape(1, -1) if isinstance(t, torch.Tensor) else t for t in _songs(clap_token_ids, n, "clap_token_ids", where)]
    if not all(isinstance(t, torch.Tensor) for t in clap):
        raise ValueError(f"{where}: clap_token_ids must hold tensors")
    # primes: all three or none, per song
    if all(p is None for p in primes):
        song_primes = [None] * n
    elif any(p is None for p in primes):
        raise ValueError(f"{where}: pass all three prime token streams or none")
    else:
        per = []
        for st, (p, what) in enumerate(zip(primes, ("prime_semantic_token_ids", "prime_coarse_token_ids", "prime_fine_token_ids"))):
            if isinstance(p, (list, tuple)):
                per.append([None if t is None else _check_prime(t, 1, qs[st], what, "MusicLM.score_tokens") for t in _songs(p, n, what, where)])
            else:
                p = _check_prime(p, n, qs[st], what, "MusicLM.score_tokens")
                per.append([p[0:1] if p.shape[0] == 1 else p[i:i + 1] for i in range(n)])
        song_primes = []
        for i in range(n):
            ps = [per[st][i] for st in range(3)]
            if any((t is None) != (ps[0] is None) for t in ps):
                raise ValueError(f"{where}: song {i} has some prime token streams but not all three")
            song_primes.append(None if ps[0] is None else ps)
    secs = list(output_seconds) if isinstance(output_seconds, (list, tuple)) else [output_seconds] * n
    if len(secs) != n:
        raise ValueError(f"{where}: output_seconds has {len(secs)} values for {n} songs")
    for s in secs:
        if isinstance(s, bool) or not isinstance(s, numbers.Real) or not 0 < float(s) < float("inf"):
            raise ValueError(f"{where}: output_seconds must be positive numbers, not {s!r}")
    plans, layouts = [], []
    for i in range(n):
        tp = None if song_primes[i] is None else tuple(t.shape[1] for t in song_primes[i])
        plan = plan_song(output_seconds=secs[i], prime_lengths=tp, coarse_only=coarse_only, **windowing)
        lay = song_layouts(plan, tp, qs)
        for name in names:
            want, got = output_length(plan, lay[name], name), given[name][i].shape[1]
            if got != want:
                raise ValueError(f"{where}: song {i}'s {name} stream has {got} steps; its plan gives {want}")
        plans.append(plan)
        layouts.append(lay)
    # flat sources: per stream, every song's prime steps (if any), then its output
    seg, pre_steps, out_off, src = {}, {}, {}, {}
    for st, name in enumerate(names):
        parts, seg[name], pre_steps[name], out_off[name] = [], [], [], []
        at = out = 0
        for i in range(n):
            p = [] if song_primes[i] is None else [song_primes[i][st]]
            seg[name].append(at)
            pre_steps[name].append(sum(t.shape[1] for t in p))
            out_off[name].append(out)
            parts += p + [given[name][i]]
            at += pre_steps[name][-1] + given[name][i].shape[1]
            out += given[name][i].shape[1]
        dev = stages[st].device
        src[name] = torch.cat([t.to(dev, torch.int64).reshape(-1) for t in parts])
    clap_at = np.cumsum([0] + [t.shape[1] for t in clap])
    clap_src = torch.cat([t.to(stages[0].device, torch.int64).reshape(-1) for t in clap])
    check_ids(clap_src, infos[0][0].codebook_size, "clap_token_ids", where)
    for st, name in enumerate(names):
        check_ids(src[name], infos[st][-1].codebook_size, f"the {name} tokens (or their prime)", where)
    rows = song_rows(plans, layouts, seg, pre_steps, out_off, [clap_at[i] + np.arange(t.shape[1]) for i, t in enumerate(clap)])
    result = []
    for st, name in enumerate(names):
        T = [t.shape[1] for t in given[name]]
        dev = stages[st].device
        out = torch.zeros(sum(T) * qs[st], device=dev, dtype=torch.float32)
        cond = [clap_src.to(dev)] + ([] if st == 0 else [src[STREAMS[st - 1]].to(dev)])
        score_rows(stages[st].transformer_wrapper, cond, src[name], rows[st], out, max_rows)
        arg = (semantic_token_ids, coarse_token_ids, fine_token_ids)[st]
        if listed:
            lp = [out[o * qs[st]:(o + t) * qs[st]].view(1, t, qs[st]) for o, t in zip(out_off[name], T)]
            result.append([v.view(a.shape) for v, a in zip(lp, arg)])
        else:
            result.append(out.view(arg.shape))
    return tuple(result) + ((None,) if coarse_only else ())
