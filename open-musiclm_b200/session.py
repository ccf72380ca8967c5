"""Continuous batching on the KV-cache decode path: a generation session whose rows join and leave while the others
keep decoding.

A `GenerationSession` holds one decode state of `slots` rows over one `TokenConditionedTransformerWrapper`.  `add`
queues a request (conditioning, optional prefix, seed, sampling arguments); at the next time-step boundary it takes a
free slot: its prompt is prefilled alone (the regular wgmma forward, as `generate` runs it for one row) and installed
into that slot, and from then on it decodes with the others, one quantizer slot per step.  A row that has all its
tokens leaves at the end of that time step and its slot is refilled at the next boundary.  The tokens of a request,
and the logits they were sampled from, are bit for bit those of `generate` with that row alone and its seed, whatever
the slot, the join step and the other rows (DESIGN section 4, "Generation sessions").

Every prefix is whole time steps, so all rows sit at the same quantizer slot at every step and share the logit head
and the per-slot CUDA graphs; the arrays those graphs read (positions, sample indices, seeds, offsets, sampling
arguments) change at a join, the graphs do not.  `SlotSchedule` is the host bookkeeping, without device work.
"""
import numbers
from collections import deque

import torch

from . import lib
from .decode import (MAX_BATCH, DecodeSession, GraphCache, assemble_output, check_abs_positions, check_sampling_rows, plan_rows,
                     prefill, prefix_logprobs, row_arrays, seeds_tensor)


class _Row:
    """One request: prompt length P (= the position its first decode step processes), n tokens to sample, its
    predicted sequence's start position pred_start, and its progress t (tokens sampled so far)."""

    def __init__(self, handle, P, n, pred_start, payload=None):
        self.handle, self.P, self.n, self.pred_start, self.payload = handle, P, n, pred_start, payload
        self.t = 0
        self.slot = None
        self.join_step = None

    def device_state(self):
        """The values the device arrays hold for this row after its t samples: sample index, position, last position,
        predicted-sequence offset.  It is installed at position P - 1 so that the advance after its first sample
        moves it to P, as the running rows' advance moves them."""
        pos_last = self.P + max(self.n, 1) - 2
        return dict(t=self.t, pos=min(self.P - 1 + self.t, pos_last), pos_last=pos_last, pos_offset=-(self.pred_start + 1))


class SlotSchedule:
    """Slot allocation of a session: requests wait in a FIFO queue (at most `max_queue` beyond the free slots), take
    the lowest free slot at a time-step boundary, sample q tokens per time step and leave when they have n."""

    def __init__(self, slots: int, q: int, max_queue: int = 0):
        self.slots, self.q, self.max_queue = slots, q, max_queue
        self.free = list(range(slots))
        self.rows = {}                 # slot -> _Row
        self.queue = deque()
        self.steps = 0                 # time steps run

    def check_room(self):
        """Raises ValueError when every slot is taken or promised to a queued row and the queue is full."""
        if len(self.rows) + len(self.queue) >= self.slots + self.max_queue:
            raise ValueError(f"open_musiclm_b200 GenerationSession.add: all {self.slots} slots are taken and the queue holds "
                             f"{len(self.queue)} of max_queue = {self.max_queue} requests")

    def submit(self, row: _Row):
        self.check_room()
        self.queue.append(row)

    def admit(self):
        """The boundary: queued rows take free slots (lowest first), in order.  Returns the rows that joined."""
        joined = []
        while self.queue and self.free:
            row = self.queue.popleft()
            row.slot = min(self.free)
            self.free.remove(row.slot)
            row.join_step = self.steps
            self.rows[row.slot] = row
            joined.append(row)
        return joined

    def advance(self):
        """One time step: every active row samples q tokens.  Returns the rows that now have all theirs (their slots
        are free again)."""
        self.steps += 1
        done = []
        for slot, row in sorted(self.rows.items()):
            row.t += self.q
            if row.t >= row.n:
                done.append(row)
        for row in done:
            del self.rows[row.slot]
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
    definitions of `generate(..., return_logprobs=True)`; the prefix values come from the row's own prefill.

    The transformer's weights are packed when the session is created; train it between sessions, not during one.
    Every row gets exactly what `generate` gives that row alone with seeds=[seed] and the same arguments; free and
    finished slots keep computing values nobody reads."""

    def __init__(self, wrapper, slots: int, max_positions: int, allow_eos_in_output=False, include_eos_in_output=False,
                 append_eos_to_conditioning_tokens=True, max_queue: int = 0, use_cuda_graph=True, trace_logits=False,
                 return_logprobs=False):
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
        self.w, self.m = wrapper, m
        info = wrapper.token_sequences[-1]
        self.q, self.C, self.eos = info.num_quantizers, info.codebook_size + 1, wrapper.eos_ids[-1]
        self.slots, self.max_positions = int(slots), int(max_positions)
        self.allow_eos, self.include_eos, self.append_eos = bool(allow_eos_in_output), bool(include_eos_in_output), \
            bool(append_eos_to_conditioning_tokens)
        self.use_graph, self.trace = bool(use_cuda_graph) and not trace_logits, bool(trace_logits)
        self.logprob = return_logprobs
        self.sched = SlotSchedule(self.slots, self.q, int(max_queue))
        self._next_handle = 0
        self._done = {}
        self._traced = {}
        self._trace = []               # trace mode: the [slots, C] logits of every sample point since _trace_base
        self._trace_base = 0
        self._graphs = GraphCache(self.use_graph)
        self.eng = self.dec = None     # the engine and the slots' device state, made by the first step that runs a row

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
        if isinstance(seed, torch.Tensor):
            if seed.dtype != torch.int64 or seed.numel() != 1:
                raise ValueError(f"{where}: seed must be one int or a one-element int64 tensor, not a {seed.dtype} tensor of "
                                 f"{seed.numel()} elements")
            seed = int(seed.reshape(-1)[0])
        if isinstance(seed, bool) or not isinstance(seed, numbers.Integral):
            raise ValueError(f"{where}: seed must be one int, not {seed!r}")
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
        self.sched.submit(_Row(handle, P, n, pred_start, payload=dict(
            cond=cond, prefix=prefix, seed=seed, top_k=top_k, temperature=float(temperature), top_p=top_p)))
        return handle

    @property
    def idle(self) -> bool:
        """No row is decoding or queued."""
        return not self.sched.rows and not self.sched.queue

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
        """Prefills each joining row alone and writes its prompt's K/V rows, conv history and last logits into its
        slot, then sets the slot's arrays.  Runs after the boundary step (which writes every slot's cache and conv
        history at the slot's old position) and before the boundary sample."""
        eng, dec, dev = self.eng, self.dec, self.eng.dev
        for row in rows:
            a = row.payload
            pl, ws = prefill(self.w, a["cond"], a["prefix"], self.append_eos, dec, slice(row.slot, row.slot + 1),
                             torch.full((1,), row.P, device=dev))
            assert pl.N == row.P and pl.pos0[-1] == row.pred_start, (pl.N, row.P)
            if self.logprob:
                a["prefix_lp"] = prefix_logprobs(eng, pl, ws, a["prefix"], self.q, self.C)[0] if a["prefix"].shape[1] else None
        idx = torch.tensor([r.slot for r in rows], device=dev)
        states = [r.device_state() for r in rows]
        vals = row_arrays(dev, len(rows), pos=[s["pos"] for s in states], pos_last=[s["pos_last"] for s in states],
                          pos_offset=[s["pos_offset"] for s in states], t=0, n=[r.n for r in rows],
                          top_k=[r.payload["top_k"] for r in rows], temperature=[r.payload["temperature"] for r in rows],
                          top_p=[r.payload["top_p"] for r in rows])
        for name, dst in (("pos", dec.pos), ("pos_last", dec.pos_last), ("pos_offset", dec.pos_offset), ("t", dec.t), ("n", dec.n_rows),
                          ("top_k", dec.top_k), ("temperature", dec.temperature)):
            dst[idx] = vals[name]
        dec.top_p[idx] = vals["top_p"] if vals["top_p"] is not None else 1.0
        dec.seeds[idx] = seeds_tensor([r.payload["seed"] for r in rows], len(rows), dev)

    def _sample_point(self):
        if self.trace:
            self._trace.append(self.dec.logits[:, :self.C].clone())

    @torch.no_grad()
    def step(self, n_time_steps: int = 1):
        """Runs n_time_steps time steps (q tokens per active row each).  Each starts at a boundary, where queued rows
        take free slots: the running rows' step to quantizer slot 0, the joiners' prefill and install, then the
        sample of slot 0 for every row; slots 1 ... q-1 follow as step and sample.  Rows with all their tokens leave
        at the end of the time step; `finished` returns them.  A time step with no row to run does nothing."""
        if isinstance(n_time_steps, bool) or not isinstance(n_time_steps, numbers.Integral) or n_time_steps < 0:
            raise ValueError(f"open_musiclm_b200 GenerationSession.step: n_time_steps must be an int >= 0, not {n_time_steps!r}")
        q, sched = self.q, self.sched
        allow = lambda qi: bool(self.allow_eos and qi == q - 1)                                   # open_musiclm.py:311-313
        for _ in range(n_time_steps):
            running = bool(sched.rows)
            joined = sched.admit()
            if not sched.rows:
                break
            dec = self._device_state()
            if self.trace and not running:
                self._trace, self._trace_base = [], self._trace_base + len(self._trace)
            for row in joined:
                row.trace_start = self._trace_base + len(self._trace)
            nucleus = any(r.payload["top_p"] is not None for r in sched.rows.values())
            for qi in range(q):
                if qi == 0 and joined:
                    if running:
                        self._graphs.run(("step", 0), lambda: dec.step(0))
                    self._install(joined)
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
