"""Continuous batching on the KV-cache decode path: a generation session whose rows join and leave while the others
keep decoding.

A `GenerationSession` holds one decode state of `slots` rows over one `TokenConditionedTransformerWrapper`.  `add`
queues a request (conditioning, optional prefix, seed, sampling arguments); at the next time-step boundary it takes a
free slot: the prompts of every row that joins at that boundary are prefilled together, packed back to back in one
forward (Engine.forward_packed: the regular layers with the varlen attention and FFN-up kernels), and installed into
their slots, and from then on it decodes with the others, one quantizer slot per step.  A row that has all its
tokens leaves at the end of that time step and its slot is refilled at the next boundary.  The tokens of a request,
and the logits they were sampled from, are bit for bit those of `generate` with that row alone and its seed, whatever
the slot, the join step and the other rows (DESIGN section 4, "Generation sessions").

Every prefix is whole time steps, so all rows sit at the same quantizer slot at every step and share the logit head
and the per-slot CUDA graphs; the arrays those graphs read (positions, sample indices, seeds, offsets, sampling
arguments) change at a join, the graphs do not.  `SlotSchedule` is the host bookkeeping, without device work.
"""
import math
import numbers
import types
from collections import deque

import numpy as np
import torch

from . import lib
from .decode import (MAX_BATCH, DecodeSession, GraphCache, assemble_output, check_abs_positions, check_sampling_rows, plan_rows,
                     row_arrays, seeds_tensor)


PACK_ROWS = 16384     # rows of a session's packed-prefill workspace: max(max_positions, this), at most slots * max_positions


def split_joiners(prompt_lens, capacity: int):
    """The joiners of one boundary (prompt lengths in admission order, each <= capacity) -> lists of their indices,
    consecutive in admission order, each list's prompts together at most capacity rows: one packed prefill each."""
    groups, total = [], capacity
    for i, n in enumerate(prompt_lens):
        if total + n > capacity:
            groups.append([])
            total = 0
        groups[-1].append(i)
        total += n
    return groups


def lpt_work(seq_lens, h: int, p0=None):
    """The attention work list of a packed forward: every (sequence, 128-row block of its len * h folded query rows)
    once, as int32 [n, 2], heaviest first (the block's key tiles, min(len - 1, last row's position) // 128 + 1; ties by
    sequence, then later blocks first), as omlm_attn_fwd_tc orders its fixed-length grid.  p0: each sequence is a chunk
    whose first row is position p0[b] of its prompt (p0[b] * h a multiple of 128); blocks are counted from the chunk's
    first row and its key tiles from position 0, min(p0 + len - 1, last row's position) // 128 + 1."""
    b = np.concatenate([np.full((n * h + 127) // 128, i) for i, n in enumerate(seq_lens)]).astype(np.int64)
    rb = np.concatenate([np.arange((n * h + 127) // 128) for n in seq_lens]).astype(np.int64)
    lens = np.asarray(seq_lens, dtype=np.int64)[b]
    p = np.zeros_like(lens) if p0 is None else np.asarray(p0, dtype=np.int64)[b]
    tiles = np.minimum(p + lens - 1, (p * h + rb * 128 + 127) // h) // 128 + 1
    order = np.lexsort((-rb, b, -tiles))
    return np.stack([b[order], rb[order]], 1).astype(np.int32)


def check_seed(seed, where: str) -> int:
    """A request's seed: one int or a one-element int64 tensor -> the int; anything else raises ValueError."""
    if isinstance(seed, torch.Tensor):
        if seed.dtype != torch.int64 or seed.numel() != 1:
            raise ValueError(f"{where}: seed must be one int or a one-element int64 tensor, not a {seed.dtype} tensor of "
                             f"{seed.numel()} elements")
        seed = int(seed.reshape(-1)[0])
    if isinstance(seed, bool) or not isinstance(seed, numbers.Integral):
        raise ValueError(f"{where}: seed must be one int, not {seed!r}")
    return seed


class PackedPrefill:
    """Host plan of one packed prefill: the prompts of k joiners back to back, without padding.  n_tok: per joiner the
    token counts of its sequences (conditioning sequences with their eos, then its prefix of whole time steps), as
    lib.token_plan returns them; its prompt is sum(n + 1) rows (each sequence after its start token).  slots: the
    joiners' slots in a decode state of n_max positions per slot; q: quantizers of the last sequence; h: heads;
    abs_row_base (absolute position embeddings): the first row of each sequence's position table.  logprob: also
    plan the rows that score the prefix tokens.  chunks: per joiner (p0, length), the positions p0 ... p0 + length - 1
    of its prompt that this prefill runs (p0 a multiple of 128 / gcd(h, 128)); None: each whole prompt, (0, P).  A
    chunk that ends its prompt is final: only final chunks have a next-token logits row and install conv history.

    Arrays (numpy): start, P, p0, end (each chunk's first packed row, length, first and one-past-last position), final
    [k] (bool), row_pos [M] (position within its prompt), src_row2 [M] (position-table rows, -1 for start tokens; None
    without absolute positions), work (lpt_work), last_row [k_final] (each final chunk's last row, whose head-0 logits
    predict the first sampled token: every prefix is whole time steps, so the next token is at quantizer 0),
    prefix_rows[qi] (the rows whose head-qi logits score the prefix tokens at quantizer qi, joiner by joiner),
    dest_row [M] (row -> final-norm output row, -1 when no head reads it: last rows first, then prefix_rows[0], [1],
    ...), groups [(qi, base, cnt)] (head qi on output rows base .. base + cnt - 1), prefix_off [k] and label_idx
    [head_rows] (each output row's prefix token in the joiners' concatenated prefixes, -1 for the last rows),
    prefix_span [k] (the range j_lo, j_hi of each joiner's prefix tokens scored here), kv_dst [M] (flat cache row
    slot * n_max + row_pos), kv_start [k] (slot * n_max), hist_idx [M] (the slot at the first row of a chunk with p0 > 0,
    whose conv history is rows 2 slot, 2 slot + 1 of the session's history buffer; -1 elsewhere), hist_src, hist_dst
    (non-final chunks: rows end - 2, end - 1 -> history rows slot * 2 + j), and for final chunks conv_src and conv_dst
    (prompt rows P - 2, P - 1 -> flat conv-history rows slot * 2 + j), conv_hsrc and conv_hdst (those of the two rows
    that precede the chunk: from the history buffer) and conv_zero (flat conv rows before a prompt's first row)."""

    def __init__(self, n_tok, slots, n_max: int, q: int, h: int, abs_row_base=None, logprob: bool = False, chunks=None):
        k = len(n_tok)
        self.k = k
        full = np.array([sum(n + 1 for n in t) for t in n_tok], dtype=np.int64)
        if chunks is None:
            chunks = [(0, int(n)) for n in full]
        self.p0 = np.array([c[0] for c in chunks], dtype=np.int64)
        self.P = np.array([c[1] for c in chunks], dtype=np.int64)
        self.end = self.p0 + self.P
        assert (self.P >= 1).all() and (self.end <= full).all()
        self.final = self.end == full
        self.start = np.concatenate([[0], np.cumsum(self.P)[:-1]]).astype(np.int64)
        self.M = int(self.P.sum())
        self.max_len = int(self.P.max())
        self.max_end = int(self.end.max())
        self.row_pos = np.concatenate([np.arange(a, e) for a, e in zip(self.p0, self.end)]).astype(np.int32)
        self.src_row2 = None
        if abs_row_base is not None:
            r2 = []
            for t, a, e in zip(n_tok, self.p0, self.end):
                whole = np.concatenate([np.concatenate([[-1], abs_row_base[s] + np.arange(n)]) for s, n in enumerate(t)])
                r2.append(whole[a:e])
            self.src_row2 = np.concatenate(r2).astype(np.int32)
        self.work = lpt_work(self.P.tolist(), h, self.p0)
        fin = np.flatnonzero(self.final)
        self.k_final = len(fin)
        self.last_row = (self.start + self.P - 1)[fin]
        n_pre = [t[-1] if logprob else 0 for t in n_tok]
        pred0 = [sum(n + 1 for n in t[:-1]) for t in n_tok]         # each predicted sequence's start token (position)
        # prefix token j is scored by the row at position pred0 + j: the tokens j_lo ... j_hi - 1 fall in this chunk
        self.prefix_span = [(int(min(max(a - p, 0), n)), int(max(min(e - p, n), 0))) for a, e, p, n in zip(self.p0, self.end, pred0, n_pre)]
        self.prefix_off = np.concatenate([[0], np.cumsum(n_pre)[:-1]]).astype(np.int64)
        span = lambda i, qi: np.arange(self.prefix_span[i][0] + (qi - self.prefix_span[i][0]) % q, self.prefix_span[i][1], q)
        self.prefix_rows = [np.concatenate([np.zeros(0)] + [self.start[i] + pred0[i] + span(i, qi) - self.p0[i] for i in range(k)]).astype(np.int64)
                            for qi in range(q)]
        prefix_tok = [np.concatenate([np.zeros(0)] + [self.prefix_off[i] + span(i, qi) for i in range(k)]).astype(np.int64) for qi in range(q)]
        out_rows = [self.last_row] + self.prefix_rows
        self.head_rows = sum(len(r) for r in out_rows)
        self.dest_row = np.full(self.M, -1, dtype=np.int32)
        self.dest_row[np.concatenate(out_rows)] = np.arange(self.head_rows)
        self.groups, base = [], 0
        for qi in range(q):
            cnt = len(self.prefix_rows[qi]) + (self.k_final if qi == 0 else 0)
            if cnt:
                self.groups.append((qi, base, cnt))
            base += cnt
        self.label_idx = np.concatenate([np.full(self.k_final, -1, dtype=np.int64)] + prefix_tok)
        slot = np.asarray(slots, dtype=np.int64)
        self.slots = slot
        self.kv_dst = np.repeat(slot * n_max, self.P) + self.row_pos
        self.kv_start = slot * n_max
        self.hist_idx = np.full(self.M, -1, dtype=np.int32)
        cont = self.p0 > 0
        self.hist_idx[self.start[cont]] = slot[cont]
        part = np.flatnonzero(~self.final)
        assert (self.P[part] >= 2).all()                                             # non-final chunks are whole units
        self.hist_dst = (slot[part, None] * 2 + np.arange(2)[None]).reshape(-1)
        self.hist_src = (self.start[part, None] + self.P[part, None] + np.arange(-2, 0)[None]).reshape(-1)
        hist = self.end[fin, None] + np.arange(-2, 0)[None]                           # prompt rows P - 2, P - 1
        rel = hist - self.p0[fin, None]                                               # < 0: before the chunk
        self.conv_dst = (slot[fin, None] * 2 + np.arange(2)[None]).reshape(-1)
        self.conv_src = (self.start[fin, None] + np.maximum(rel, 0)).reshape(-1)
        self.conv_zero = self.conv_dst[(hist < 0).reshape(-1)]
        before = ((hist >= 0) & (rel < 0)).reshape(-1)
        self.conv_hdst = self.conv_dst[before]
        self.conv_hsrc = (slot[fin, None] * 2 + rel + 2).reshape(-1)[before]          # history row of position p0 - 2 + j
        self.fin_slots = slot[fin]

    def to_device(self, dev):
        """The device arrays, sent in one non-blocking copy (staged from pageable memory, as decode.row_arrays does, so
        that it never waits for the device): a namespace of the arrays above that the forward and the install read."""
        arrays = dict(row_pos=self.row_pos, work=self.work, seq_start=self.start.astype(np.int32), seq_len=self.P.astype(np.int32),
                      q_off=self.p0.astype(np.int32), kv_start=self.kv_start.astype(np.int32), hist_idx=self.hist_idx,
                      dest_row=self.dest_row, kv_dst=self.kv_dst, label_idx=self.label_idx)
        optional = ("src_row2", "conv_dst", "conv_src", "conv_zero", "conv_hdst", "conv_hsrc", "hist_dst", "hist_src", "fin_slots")
        for name in optional:                   # None when absent or empty
            a = getattr(self, name)
            if a is not None and len(a):
                arrays[name] = a
        parts, where, off = [], {}, 0
        for name, a in arrays.items():
            raw = np.ascontiguousarray(a).reshape(-1).view(np.uint8)
            where[name] = (off, a.dtype, a.shape)
            parts += [raw, np.zeros(-len(raw) % 8, dtype=np.uint8)]
            off += len(raw) + (-len(raw) % 8)
        buf = torch.from_numpy(np.concatenate(parts)).to(dev, non_blocking=True)
        dv = dict(M=self.M, max_len=self.max_len, max_end=self.max_end, k_final=self.k_final, groups=self.groups,
                  **{name: None for name in optional})
        for name, (o, dt, shape) in where.items():
            tdt = torch.int32 if dt == np.int32 else torch.int64
            dv[name] = buf[o:o + int(np.prod(shape)) * dt.itemsize].view(tdt).view(shape)
        return types.SimpleNamespace(**dv)


class _PackedCapture:
    """Receives a packed prefill's per-layer K/V rows and pre-conv FFN rows (Engine.forward_packed) into the joiners'
    slots of a DecodeSession: every chunk row's K/V at its position; for a final chunk, prompt rows P - 2, P - 1 as conv
    history (zero before a prompt's first row, from the history buffer `hist` when they precede the chunk); for any
    other chunk, its last two rows into `hist` (the decode step shifts every slot's conv history at every step, so a
    prefilling slot's history lives outside it).  One gather or scatter per layer and kind, as _PromptCapture does per
    row."""

    def __init__(self, dec, dv, hist=None):
        self.dec, self.dv, self.hist = dec, dv, hist

    def after_kv(self, l, kvn):
        self.dec.cache[l].view(-1, 128).index_copy_(0, self.dv.kv_dst, kvn)

    def after_u(self, l, u):
        dv = self.dv
        conv = self.dec.conv[l].view(-1, u.shape[-1])
        if dv.conv_dst is not None:
            conv.index_copy_(0, dv.conv_dst, u.index_select(0, dv.conv_src))
        if dv.conv_hdst is not None:
            conv.index_copy_(0, dv.conv_hdst, self.hist[l].index_select(0, dv.conv_hsrc))
        if dv.conv_zero is not None:
            conv.index_fill_(0, dv.conv_zero, 0)
        if dv.hist_dst is not None:
            self.hist[l].index_copy_(0, dv.hist_dst, u.index_select(0, dv.hist_src))


class _Row:
    """One request: prompt length P (= the position its first decode step processes), n tokens to sample, its
    predicted sequence's start position pred_start, and its progress: filled (prompt rows prefilled so far, counting
    the chunk planned at this boundary), chunk ((p0, length) of that chunk) and t (tokens sampled so far)."""

    def __init__(self, handle, P, n, pred_start, payload=None):
        self.handle, self.P, self.n, self.pred_start, self.payload = handle, P, n, pred_start, payload
        self.t = 0
        self.filled = 0
        self.chunk = None
        self.slot = None
        self.join_step = None
        self.snapshot = None           # a suspended running row's decode state (GenerationSession._snapshot)

    @property
    def prefilled(self) -> bool:
        return self.filled == self.P

    def device_state(self):
        """The values the device arrays hold for this row after its t samples: sample index, position, last position,
        predicted-sequence offset.  It is installed at position P - 1 so that the advance after its first sample
        moves it to P, as the running rows' advance moves them."""
        pos_last = self.P + max(self.n, 1) - 2
        return dict(t=self.t, pos=min(self.P - 1 + self.t, pos_last), pos_last=pos_last, pos_offset=-(self.pred_start + 1))


class SlotSchedule:
    """Slot allocation of a session: requests wait in a FIFO queue (at most `max_queue` beyond the free slots), take
    the lowest free slot at a time-step boundary, sample q tokens per time step and leave when they have n.

    prefill_rows: at most that many prompt rows are prefilled per boundary (None: no bound).  A prompt that does not
    fit is prefilled in chunks over consecutive boundaries, each but the last a multiple of `unit` rows; its request
    holds its slot meanwhile and samples from the boundary of its last chunk on.

    Between boundaries a row can be cancelled (it leaves wherever it is and its slot is free at once), suspended (a
    queued row leaves the queue; a prefilled row leaves its slot, keeping its progress; a row part-way through its
    prompt cannot be) and resumed.  A suspended row holds no slot and no queue place.  Resumed rows wait in `resumed`,
    ahead of the queue, in the order they were resumed; a prefilled one takes a slot without prefill or budget."""

    def __init__(self, slots: int, q: int, max_queue: int = 0, prefill_rows=None, unit: int = 1):
        self.slots, self.q, self.max_queue = slots, q, max_queue
        self.prefill_rows, self.unit = prefill_rows, unit
        self.free = list(range(slots))
        self.rows = {}                 # slot -> _Row (prefilling rows included)
        self.queue = deque()
        self.resumed = deque()         # resumed rows, ahead of the queue
        self.suspended = {}            # handle -> suspended _Row
        self.live = {}                 # handle -> _Row of every queued, resumed, slotted or suspended row
        self.prefilling = []           # rows part-way through their prompt, in admission order
        self.restored = []             # the prefilled rows the last admit put back into slots
        self.steps = 0                 # time steps run

    def check_room(self):
        """Raises ValueError when every slot is taken or promised to a waiting row and the queue is full."""
        waiting = len(self.queue) + len(self.resumed)
        if len(self.rows) + waiting >= self.slots + self.max_queue:
            raise ValueError(f"open_musiclm_b200 GenerationSession.add: all {self.slots} slots are taken and the queue holds "
                             f"{waiting} of max_queue = {self.max_queue} requests")

    def submit(self, row: _Row):
        self.check_room()
        self.queue.append(row)
        self.live[row.handle] = row

    def status(self, row: _Row) -> str:
        if row.handle in self.suspended:
            return "suspended"
        if row.slot is None:
            return "queued"
        return "running" if row.prefilled else "prefilling"

    def _leave(self, row: _Row):
        """Takes a row out of the queue, the resumed rows or its slot (freed at once)."""
        if row.slot is not None:
            del self.rows[row.slot]
            self.free.append(row.slot)
            row.slot = None
            if row in self.prefilling:
                self.prefilling.remove(row)
        elif row in self.resumed:
            self.resumed.remove(row)
        else:
            self.queue.remove(row)

    def cancel(self, row: _Row):
        if self.suspended.pop(row.handle, None) is None:
            self._leave(row)
        del self.live[row.handle]

    def suspend(self, row: _Row):
        assert row.handle not in self.suspended and (row.slot is None or row.prefilled)
        self._leave(row)
        self.suspended[row.handle] = row

    def resume(self, row: _Row):
        del self.suspended[row.handle]
        self.resumed.append(row)

    def admit(self):
        """The boundary: the budget of prompt rows goes in FIFO order, first to the rows part-way through their
        prompt, then to resumed rows and then queued rows, which take free slots (lowest first) while there are any.  A
        row gets a chunk only if it can take min(unit, its remaining rows): its whole remainder if that fits, else the
        largest multiple of unit that does; the first row that cannot ends the boundary's admissions, so no row
        overtakes an earlier one.  A resumed row that was prefilled when it was suspended needs no chunk: it takes a slot
        whatever is left of the budget and goes to `restored`.  Returns the rows with a chunk at this boundary
        (row.chunk = (p0, length)); without a budget, the rows that joined, each with its whole prompt."""
        left = float("inf") if self.prefill_rows is None else self.prefill_rows
        out = []
        self.restored = []

        def take(row):
            nonlocal left
            rem = row.P - row.filled
            n = rem if rem <= left else int(left) // self.unit * self.unit
            if n == 0:
                return False
            row.chunk = (row.filled, n)
            row.filled += n
            left -= n
            out.append(row)
            return True

        blocked = not all(take(row) for row in self.prefilling)
        while self.free and (self.resumed or self.queue):
            line = self.resumed if self.resumed else self.queue
            row = line[0]
            if row.prefilled:
                self.restored.append(row)
            elif blocked or not take(row):
                break
            line.popleft()
            row.slot = min(self.free)
            self.free.remove(row.slot)
            row.join_step = self.steps
            self.rows[row.slot] = row
        self.prefilling = [r for r in self.prefilling if not r.prefilled] + [r for r in out if r.chunk[0] == 0 and not r.prefilled]
        return out

    def advance(self):
        """One time step: every active row samples q tokens.  Returns the rows that now have all theirs (their slots
        are free again)."""
        self.steps += 1
        done = []
        for slot, row in sorted(self.rows.items()):
            if not row.prefilled:
                continue
            row.t += self.q
            if row.t >= row.n:
                done.append(row)
        for row in done:
            del self.rows[row.slot]
            del self.live[row.handle]
            self.free.append(row.slot)
        return done


class _SlotDecode(DecodeSession):
    """DecodeSession over `slots` rows with, on top of its per-row state, one sample index and token count per row,
    device arrays that installs rewrite."""

    def __init__(self, eng, slots: int, max_positions: int, logprob: bool):
        rows = row_arrays(eng.dev, slots, pos=0, pos_last=0, pos_offset=0, top_k=0, temperature=1.0, top_p=1.0)
        super().__init__(eng, slots, max_positions, max_positions, rows, seeded=True, logprob=logprob)
        self.t = torch.zeros(slots, device=eng.dev, dtype=torch.int32)
        self.n_rows = torch.zeros(slots, device=eng.dev, dtype=torch.int32)

    def sample_rows(self, qi: int, allow_eos: bool, nucleus: bool):
        """Every row with tokens left samples the token of quantizer slot qi at its own sample index; then every
        position advances (up to its row's last)."""
        lib.sample_rows_indexed(self.logits, self.eng.C[-1], allow_eos, self.seeds, self.tokens, self.next_row, self.row_offset(qi),
                                self.t, self.n_rows, self.top_k, self.temperature, self.top_p if nucleus else None,
                                logprobs=self.lp, sample_logprobs=self.slp)
        lib.decode_advance_pos(self.pos, self.pos_last)


class GenerationSession:
    """Continuous batching over one TokenConditionedTransformerWrapper: up to `slots` (1 ... 256) seeded rows decode
    together; rows join at time-step boundaries and leave when they have their tokens.

        sess = GenerationSession(wrapper, slots=64, max_positions=1400)
        h = sess.add(conditioning_token_ids=[clap_1xn, sem_1xm], pred_token_ids=None, seed=1234, max_time_steps=300,
                     temperature=0.95, filter_thres=0.9, top_p=None)
        while not sess.idle:
            sess.step()
            for h, tokens in sess.finished().items(): ...          # tokens: [n, q] int64, as generate(...)[0]

    allow_eos_in_output, include_eos_in_output and append_eos_to_conditioning_tokens hold for every row, as in
    `generate`.  max_positions bounds every row's prompt (its conditioning sequences with their start tokens and eos,
    and its prefix) plus the tokens it samples; the caches hold max_positions positions per slot.  max_queue: how many
    requests may wait beyond the free slots (0: `add` raises once every slot is taken or promised).
    use_cuda_graph: replay each step from one CUDA graph per (quantizer slot, kind, nucleus or not), captured on first
    use and never again.  trace_logits (tests): run eagerly and keep the [n, codebook+1] logits each row's tokens were
    sampled from, returned by `traced_logits(handle)` once the row has finished.
    return_logprobs: `finished()` maps each handle to (tokens, logprobs, sample_logprobs), each [n, q], with the
    definitions of `generate(..., return_logprobs=True)`; the prefix values come from the row's rows of the packed prefill.
    prefill_rows: None (every request's whole prompt is prefilled at the boundary where it joins), or the most prompt
    rows prefilled at one boundary, across all requests, an int >= U = 128 / gcd(heads, 128).  A longer prompt is then
    prefilled in chunks over consecutive boundaries (each but the last a multiple of U rows) while the other rows keep
    decoding in between, so a mass join stalls the running rows for a bounded time.  The budget goes first to requests
    part-way through their prompt, then to queued ones, in arrival order; a request takes its slot with its first
    chunk and samples from the boundary of its last.  Time steps in which a request only prefills count for `step`.

    Between steps, `status(h)` reports where a request is, `cancel(h)` drops it and frees its slot at once, and
    `suspend(h)` / `resume(h)` take a running row out of its slot and later put it back into any free slot, restored
    from a device snapshot of its decode state.  None of them changes another row's values, and a resumed row's values
    are those of the row never suspended.  They add no CUDA graph and no host synchronisation.

    The transformer's weights are packed when the session is created; train it between sessions, not during one.
    Every row gets exactly what `generate` gives that row alone with seeds=[seed] and the same arguments; free and
    finished slots keep computing values nobody reads."""

    def __init__(self, wrapper, slots: int, max_positions: int, allow_eos_in_output=False, include_eos_in_output=False,
                 append_eos_to_conditioning_tokens=True, max_queue: int = 0, use_cuda_graph=True, trace_logits=False,
                 return_logprobs=False, prefill_rows=None):
        if not isinstance(return_logprobs, bool):
            raise ValueError(f"open_musiclm_b200 GenerationSession: return_logprobs must be a bool, not {return_logprobs!r}")
        for name, v in (("slots", slots), ("max_positions", max_positions), ("max_queue", max_queue)):
            if isinstance(v, bool) or not isinstance(v, numbers.Integral):
                raise ValueError(f"open_musiclm_b200 GenerationSession: {name} must be an int, not {v!r}")
        if not 1 <= slots <= MAX_BATCH:
            raise ValueError(f"open_musiclm_b200 GenerationSession: slots = {slots} lies outside [1, {MAX_BATCH}]")
        if max_positions < 1 or max_queue < 0:
            raise ValueError(f"open_musiclm_b200 GenerationSession: max_positions = {max_positions} must be >= 1 and "
                             f"max_queue = {max_queue} >= 0")
        m = wrapper.transformer
        if m.heads > 16:
            raise ValueError(f"open_musiclm_b200 GenerationSession: seeded generation supports at most 16 heads ({m.heads} given)")
        unit = 128 // math.gcd(m.heads, 128)
        if prefill_rows is not None and (isinstance(prefill_rows, bool) or not isinstance(prefill_rows, numbers.Integral)
                                         or prefill_rows < unit):
            raise ValueError(f"open_musiclm_b200 GenerationSession: prefill_rows must be None or an int >= {unit} "
                             f"(128 / gcd(heads, 128)), not {prefill_rows!r}")
        self.prefill_rows = None if prefill_rows is None else int(prefill_rows)
        self.w, self.m = wrapper, m
        info = wrapper.token_sequences[-1]
        self.q, self.C, self.eos = info.num_quantizers, info.codebook_size + 1, wrapper.eos_ids[-1]
        self.slots, self.max_positions = int(slots), int(max_positions)
        self.allow_eos, self.include_eos, self.append_eos = bool(allow_eos_in_output), bool(include_eos_in_output), \
            bool(append_eos_to_conditioning_tokens)
        self.use_graph, self.trace = bool(use_cuda_graph) and not trace_logits, bool(trace_logits)
        self.logprob = return_logprobs
        self.sched = SlotSchedule(self.slots, self.q, int(max_queue), self.prefill_rows, unit)
        self._next_handle = 0
        self._cancelled = set()
        self._done = {}
        self._traced = {}
        self._trace = []               # trace mode: the [slots, C] logits of every sample point since _trace_base
        self._trace_base = 0
        self._graphs = GraphCache(self.use_graph)
        self.eng = self.dec = None     # the engine and the slots' device state, made by the first step that runs a row
        self._pack_ws = None           # the packed prefill's workspace, made at the first join
        self._hist = None              # with prefill_rows: per layer the conv history of prefilling slots, [2 slots, 2 Fp]

    def _device_state(self):
        if self.dec is None:
            self.eng = self.m.engine
            self.dec = _SlotDecode(self.eng, self.slots, self.max_positions, self.logprob)
        return self.dec

    # ------------------------------------------------------------------------------------------------ requests
    def _prompt_lengths(self, cond_lens, n_pre):
        """Host-side token plan of one row: (P, pred_start) = its prompt length and its predicted sequence's start
        position, as Engine.plan computes them from lib.token_plan's counts."""
        n_tok = list(cond_lens) + [n_pre]
        return sum(n + 1 for n in n_tok), sum(n + 1 for n in n_tok[:-1])

    def add(self, *, conditioning_token_ids, pred_token_ids=None, seed, max_time_steps=512, temperature=1.0, filter_thres=0.9,
            top_p=None):
        """Queues one request and returns its handle (an int).  It joins at the next time-step boundary with a free
        slot.  The arguments are those of `generate` for one row, with one seed; every check runs before any device
        work and raises ValueError (IndexError for the absolute-position limit, as `generate` raises).  A request that
        samples nothing finishes at once."""
        S = len(self.w.token_sequences)
        where = "open_musiclm_b200 GenerationSession.add"
        seed = check_seed(seed, where)
        if not isinstance(conditioning_token_ids, (list, tuple)) or len(conditioning_token_ids) != S - 1:
            raise ValueError(f"{where}: conditioning_token_ids must be a list of {S - 1} tensors")
        for t in conditioning_token_ids:
            if not isinstance(t, torch.Tensor) or t.dim() < 1 or t.shape[0] != 1:
                raise ValueError(f"{where}: each conditioning sequence must be a tensor of one row, [1, ...]")
        q = self.q
        if pred_token_ids is not None:
            shape = tuple(pred_token_ids.shape)
            if not ((len(shape) == 3 and shape[0] == 1 and shape[2] == q) or (q == 1 and len(shape) == 2 and shape[0] == 1)):
                raise ValueError(f"{where}: pred_token_ids must be [1, time steps, {q}] (whole time steps), not {list(shape)}")
        one = lambda v: v if isinstance(v, (list, tuple)) or (isinstance(v, torch.Tensor) and v.dim() == 1) else \
            [v.item() if isinstance(v, torch.Tensor) else v]
        temperature, top_k, top_p, max_time_steps = check_sampling_rows(1, self.C, one(temperature), one(filter_thres), one(top_p),
                                                                        one(max_time_steps))
        (n_pre,), (n,) = plan_rows(pred_token_ids, 1, q, None, max_time_steps)
        cond_lens = [t.numel() + (1 if self.append_eos else 0) for t in conditioning_token_ids]
        P, pred_start = self._prompt_lengths(cond_lens, n_pre)
        if self.m.use_absolute_position_embeddings:
            check_abs_positions(where, int(self.m.max_absolute_position_embeddings), cond_lens, [n_pre], [n])
        if P + n > self.max_positions:
            raise ValueError(f"{where}: the prompt's {P} positions plus {n} sampled tokens exceed max_positions = {self.max_positions}")
        if n > 0:
            self.sched.check_room()
        handle = self._next_handle
        self._next_handle += 1
        dev = self.m.device
        cond = [t.to(dev, torch.int64).reshape(1, -1) for t in conditioning_token_ids]
        prefix = pred_token_ids.to(dev, torch.int64).reshape(1, -1) if pred_token_ids is not None else \
            torch.empty(1, 0, device=dev, dtype=torch.int64)
        if n == 0:
            if self.logprob:             # nothing to sample: generate's teacher-forced scoring of the prefix
                self._done[handle] = tuple(t[0] for t in self.w.generate(
                    conditioning_token_ids=cond, pred_token_ids=pred_token_ids, max_time_steps=max_time_steps, return_logprobs=True,
                    include_eos_in_output=self.include_eos, append_eos_to_conditioning_tokens=self.append_eos))
            else:
                self._done[handle] = self._output(prefix[0], prefix.new_empty(0))
            if self.trace:
                self._traced[handle] = torch.empty(0, self.C, device=dev)
            return handle
        if self.append_eos:                                                                        # open_musiclm.py:288-290
            cond = [torch.cat([t, torch.full((1, 1), e, device=dev, dtype=torch.int64)], 1) for t, e in zip(cond, self.w.eos_ids)]
        self.sched.submit(_Row(handle, P, n, pred_start, payload=dict(
            ids=cond + [prefix], n_tok=cond_lens + [n_pre], prefix=prefix, seed=seed, top_k=top_k, temperature=float(temperature),
            top_p=top_p)))
        return handle

    @property
    def idle(self) -> bool:
        """No row is decoding, prefilling or queued (suspended rows wait for `resume` and keep no session busy)."""
        return not self.sched.rows and not self.sched.queue and not self.sched.resumed

    # ------------------------------------------------------------------------------------------------ cancel, suspend
    def _state(self, handle, where: str) -> str:
        if not isinstance(handle, bool) and isinstance(handle, numbers.Integral):
            row = self.sched.live.get(handle)
            if row is not None:
                return self.sched.status(row)
            if 0 <= handle < self._next_handle and handle not in self._cancelled:
                return "finished"
            if handle in self._cancelled:
                raise ValueError(f"open_musiclm_b200 GenerationSession.{where}: request {handle} was cancelled")
        raise ValueError(f"open_musiclm_b200 GenerationSession.{where}: {handle!r} is not a handle of this session")

    def status(self, handle) -> str:
        """"queued", "prefilling" (part-way through a chunked prefill), "running", "suspended" or "finished" (its result
        waits in `finished()` or was returned).  Host state only.  ValueError for a handle `add` never returned or a
        cancelled one."""
        return self._state(handle, "status")

    def cancel(self, handle) -> bool:
        """Removes a queued, prefilling, running or suspended request: its slot is free for the next boundary, it never
        appears in `finished()`, and no other row changes.  Returns False, leaving the result where it is, for a
        finished request.  Called between steps, like `add`; no device work.  ValueError for a handle `add` never
        returned or a cancelled one."""
        if self._state(handle, "cancel") == "finished":
            return False
        row = self.sched.live[handle]
        self.sched.cancel(row)
        row.snapshot = row.payload = None
        self._cancelled.add(handle)
        return True

    def suspend(self, handle):
        """A running row gives up its slot: its decode state is copied into a snapshot the session keeps on the row's
        device (torch copies on the current stream), and `resume` later continues it bit for bit in whatever slot it
        gets.  A queued request leaves the queue, keeping its arguments.  A suspended request holds no slot and no
        queue place.  Called between steps.  ValueError, before any device work, under trace_logits and for a request
        that is not queued or running: part-way through a chunked prefill (`status` says when it has finished),
        suspended, finished, cancelled or unknown."""
        state = self._state(handle, "suspend")
        if self.trace:
            raise ValueError("open_musiclm_b200 GenerationSession.suspend: not available with trace_logits=True")
        if state not in ("queued", "running"):
            raise ValueError(f"open_musiclm_b200 GenerationSession.suspend: request {handle} is {state}; only queued and running "
                             f"requests can be suspended")
        row = self.sched.live[handle]
        if state == "running":
            self._snapshot(row)
        self.sched.suspend(row)

    def resume(self, handle):
        """Puts a suspended request at the head of the queue, behind the requests resumed before it and ahead of every
        request `add` queued: it takes the lowest free slot at the next boundary with one.  A row that was running is
        restored from its snapshot there and runs no prefill (it uses none of prefill_rows); a request suspended while
        queued is prefilled as usual.  Never raises for lack of room.  ValueError for a request that is not suspended."""
        state = self._state(handle, "resume")
        if state != "suspended":
            raise ValueError(f"open_musiclm_b200 GenerationSession.resume: request {handle} is {state}, not suspended")
        self.sched.resume(self.sched.live[handle])

    _ROW_STATE = ("next_row", "pos", "pos_last", "pos_offset", "t", "n_rows", "top_k", "temperature", "top_p", "seeds")

    def _snapshot(self, row):
        """Copies out what the next time step reads of the row's slot: the K/V of its live positions (those before
        its current position P - 1 + t, which the next step writes), its conv history, its per-row arrays and its
        samples so far."""
        dec, s, t = self.dec, row.slot, row.t
        pos = row.P - 1 + t
        snap = dict(cache=[c[s, :pos].clone() for c in dec.cache], conv=[c[s].clone() for c in dec.conv],
                    rows={name: getattr(dec, name)[s:s + 1].clone() for name in self._ROW_STATE},
                    out=[o[s, :t].clone() for o in ((dec.tokens, dec.lp, dec.slp) if self.logprob else (dec.tokens,))])
        row.snapshot = snap

    def _restore(self, rows):
        """Writes the snapshots of `rows` (restored by the schedule at this boundary) into their new slots, before the
        boundary step reads them."""
        dec = self.dec
        for row in rows:
            s, snap = row.slot, row.snapshot
            pos = snap["cache"][0].shape[0]
            for c, v in zip(dec.cache, snap["cache"]):
                c[s, :pos].copy_(v)
            for c, v in zip(dec.conv, snap["conv"]):
                c[s].copy_(v)
            for name, v in snap["rows"].items():
                getattr(dec, name)[s:s + 1].copy_(v)
            for o, v in zip((dec.tokens, dec.lp, dec.slp), snap["out"]):
                o[s, :v.shape[0]].copy_(v)
            row.snapshot = None

    @property
    def graph_count(self) -> int:
        return len(self._graphs.graphs)

    def finished(self):
        """{handle: [n, q] int64 tokens} of the rows that finished since the last call (device tensors): exactly
        generate(...)[0] for that row alone.  With return_logprobs: {handle: (tokens, logprobs, sample_logprobs)}."""
        done, self._done = self._done, {}
        return done

    def traced_logits(self, handle):
        """trace_logits mode: the [n, codebook+1] logits a finished row's tokens were sampled from."""
        return self._traced.pop(handle)

    # ------------------------------------------------------------------------------------------------ decoding
    def _output(self, prefix, new, lp=None):
        """generate's output for one row from its prefix [n_pre] and samples [n]: [n_pre + n, q] tokens; with lp =
        (prefix logprobs or None, new logprobs, new sample logprobs): (tokens, logprobs, sample_logprobs)."""
        out = assemble_output(prefix[None], new[None], prefix.shape[0], prefix.shape[0] + new.shape[0], prefix.shape[0] + new.shape[0],
                              self.eos, self.include_eos, self.q, None if lp is None else tuple(None if t is None else t[None] for t in lp))
        return out[0] if lp is None else tuple(t[0] for t in out)

    def _install(self, rows):
        """Prefills the chunks the schedule gave `rows` at this boundary, packed back to back (_prefill_packed; in
        consecutive groups when they exceed the packed workspace), writes their K/V rows into the slots and, for each
        row whose prompt is now complete, its conv history and last logits, then sets the slots' arrays.  Runs after the
        boundary step (which writes every slot's cache and conv history at the slot's old position) and before the
        boundary sample.  A row still prefilling is parked: it samples nothing (n = 0), and its position stays at its
        first unfilled one, whose K/V the next chunk overwrites before anything reads it (pos_offset = -pos keeps the
        absolute-position row of every step in range)."""
        eng, dec, dev = self.eng, self.dec, self.eng.dev
        if self._pack_ws is None:
            self._pack_rows = min(max(self.max_positions, PACK_ROWS), self.slots * self.max_positions)
            if self.prefill_rows is not None:
                self._pack_rows = min(self._pack_rows, self.prefill_rows)
                self._hist = [torch.empty(2 * self.slots, 2 * eng.Fp, device=dev, dtype=eng.a16) for _ in range(eng.L)]
            self._pack_ws = eng.packed_workspace(self._pack_rows, self._pack_rows if self.logprob else self.slots)
        for group in split_joiners([r.chunk[1] for r in rows], self._pack_rows):
            self._prefill_packed([rows[i] for i in group])
        states = [r.device_state() if r.prefilled else dict(pos=r.filled, pos_last=r.filled, pos_offset=-r.filled) for r in rows]
        vals = row_arrays(dev, len(rows), slot=[r.slot for r in rows], pos=[s["pos"] for s in states],
                          pos_last=[s["pos_last"] for s in states], pos_offset=[s["pos_offset"] for s in states], t=0,
                          n=[r.n if r.prefilled else 0 for r in rows], top_k=[r.payload["top_k"] for r in rows],
                          temperature=[r.payload["temperature"] for r in rows], top_p=[r.payload["top_p"] for r in rows])
        idx = vals["slot"].long()
        for name, dst in (("pos", dec.pos), ("pos_last", dec.pos_last), ("pos_offset", dec.pos_offset), ("t", dec.t), ("n", dec.n_rows),
                          ("top_k", dec.top_k), ("temperature", dec.temperature)):
            dst[idx] = vals[name]
        if vals["top_p"] is not None:
            dec.top_p[idx] = vals["top_p"]
        else:                                   # not dec.top_p[idx] = 1.0: a Python scalar goes up in a blocking copy
            dec.top_p.index_fill_(0, idx, 1.0)
        dec.seeds[idx] = seeds_tensor([r.payload["seed"] for r in rows], len(rows), dev)

    def _prefill_packed(self, rows):
        """One packed forward over the rows' chunks (Engine.forward_packed, its attention reading each slot's K/V
        cache), installed by _PackedCapture; the last rows' head-0 logits of the final chunks go to the slots' logits
        rows, and with return_logprobs each row's prefix log-probabilities are scored from the same heads and rows as
        prefix_logprobs scores them in `generate`'s prefill, chunk by chunk."""
        eng, dec, ws = self.eng, self.dec, self._pack_ws
        plan = PackedPrefill([r.payload["n_tok"] for r in rows], [r.slot for r in rows], dec.n_max, self.q, eng.h,
                             eng.abs_row_base if eng.abs_pos else None, self.logprob, [r.chunk for r in rows])
        dv = plan.to_device(eng.dev)
        src = []
        for r in rows:                        # the token plan of each prompt, as decode.prefill makes it
            if "src_row" not in r.payload:
                _, src_row, _, _, _ = lib.token_plan(r.payload["ids"], [s.codebook_size for s in eng.seqs],
                                                     [s.num_quantizers for s in eng.seqs], eng.emb_row_base, eng.start_row,
                                                     append_eos=False, drop_last=False, mask_cond=False, want_labels=False,
                                                     err_flag=eng.err_flag)
                r.payload["src_row"] = src_row.view(-1)
            p0, n = r.chunk
            src.append(r.payload["src_row"][p0:p0 + n])
        dv.src_row = torch.cat(src) if len(src) > 1 else src[0]
        eng.forward_packed(ws, dv, dec.table, capture=_PackedCapture(dec, dv, self._hist), kv=dec.cache, hist=self._hist)
        k, Cp = plan.k_final, eng.Cp[-1]
        if k:
            dec.logits[:, :Cp].index_copy_(0, dv.fin_slots, ws["logits"][:k])
        if self.logprob:
            pre = [r.payload["prefix"][0] for r in rows]
            lp = torch.zeros(sum(p.shape[0] for p in pre), device=eng.dev, dtype=torch.float32)
            if plan.head_rows > k:
                ids = torch.cat(pre)
                tok = torch.where((ids >= 0) & (ids < self.C), ids, -100)[dv.label_idx[k:]]
                labels = torch.cat([tok.new_full((k,), -100), tok]).to(torch.int32)
                out = torch.empty(plan.head_rows, device=eng.dev, dtype=torch.float32)
                lib.token_logprob(ws["logits"][:plan.head_rows], labels, self.C, out)
                lp.index_copy_(0, dv.label_idx[k:], out[k:])
            for r, o, p, (j0, j1) in zip(rows, plan.prefix_off.tolist(), pre, plan.prefix_span):
                n = p.shape[0]
                if n and (j0, j1) == (0, n):
                    r.payload["prefix_lp"] = lp[o:o + n]
                elif n:                               # the prefix spans chunks: gather it in a buffer of its own
                    if r.payload.get("prefix_lp") is None:
                        r.payload["prefix_lp"] = torch.zeros(n, device=eng.dev, dtype=torch.float32)
                    if j1 > j0:
                        r.payload["prefix_lp"][j0:j1].copy_(lp[o + j0:o + j1])
                else:
                    r.payload["prefix_lp"] = None

    def _sample_point(self):
        if self.trace:
            self._trace.append(self.dec.logits[:, :self.C].clone())

    @torch.no_grad()
    def step(self, n_time_steps: int = 1):
        """Runs n_time_steps time steps (q tokens per active row each).  Each starts at a boundary, where resumed and
        queued rows take free slots (resumed rows that were running are restored from their snapshots there):
        the running rows' step to quantizer slot 0, the prefill of this boundary's chunks and the
        install of the prompts they complete, then the sample of slot 0 for every row; slots 1 ... q-1 follow as step
        and sample.  Rows with all their tokens leave
        at the end of the time step; `finished` returns them.  A time step with no row to run does nothing."""
        if isinstance(n_time_steps, bool) or not isinstance(n_time_steps, numbers.Integral) or n_time_steps < 0:
            raise ValueError(f"open_musiclm_b200 GenerationSession.step: n_time_steps must be an int >= 0, not {n_time_steps!r}")
        q, sched = self.q, self.sched
        allow = lambda qi: bool(self.allow_eos and qi == q - 1)                                   # open_musiclm.py:311-313
        for _ in range(n_time_steps):
            running = bool(sched.rows)
            chunked = sched.admit()
            if not sched.rows:
                break
            dec = self._device_state()
            if sched.restored:            # back in their slots before the boundary step, which runs them as it runs the others
                self._restore(sched.restored)
                running = True
            if self.trace and not running:
                self._trace, self._trace_base = [], self._trace_base + len(self._trace)
            for row in chunked:
                if row.prefilled:
                    row.trace_start = self._trace_base + len(self._trace)
            nucleus = any(r.payload["top_p"] is not None for r in sched.rows.values())
            for qi in range(q):
                if qi == 0 and chunked:
                    if running:
                        self._graphs.run(("step", 0), lambda: dec.step(0))
                    self._install(chunked)
                    self._sample_point()
                    self._graphs.run(("sample", 0, nucleus), lambda: dec.sample_rows(0, allow(0), nucleus))
                elif self.trace:
                    dec.step(qi)
                    self._sample_point()
                    dec.sample_rows(qi, allow(qi), nucleus)
                else:
                    self._graphs.run(("full", qi, nucleus), lambda qi=qi: (dec.step(qi), dec.sample_rows(qi, allow(qi), nucleus)))
            for row in sched.advance():
                a = row.payload
                lp = (a["prefix_lp"], dec.lp[row.slot, :row.n].clone(), dec.slp[row.slot, :row.n].clone()) if self.logprob else None
                self._done[row.handle] = self._output(a["prefix"][0], dec.tokens[row.slot, :row.n].clone(), lp)
                if self.trace:
                    lo = row.trace_start - self._trace_base
                    self._traced[row.handle] = torch.stack([lg[row.slot] for lg in self._trace[lo:lo + row.n]])
