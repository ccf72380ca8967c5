"""Continuous batching of whole songs: MusicLM's semantic, coarse and fine windows as requests on three generation
sessions, with the acoustic tokens streamed out as they become final.

A song is the window jobs of `plan_song` (stages.py), the plan `MusicLM.generate_tokens` runs.  Each job is a
seeded request on its stage's `GenerationSession`, added as soon as the stream tokens it reads exist: coarse windows
start while semantic windows remain, fine windows while coarse windows remain, and the independent fine windows of a
song run side by side.  A seeded session row is bit for bit `generate` with that row alone and its seed, and every
job's seed is window_seed(song seed, stage, window), so each song is bit for bit `generate_tokens(seeds=[seed])` for
that song alone, whatever else runs beside it (DESIGN section 4, "Song sessions").

Each stage runs on a CUDA stream of its own, so the three stages' decode steps overlap on the GPU.  Within one time
step they share no data: a window reads another stage's stream only after that window has finished, and events order
those reads (DESIGN section 4, "Song sessions on three streams").
"""
import numbers
import sys
from collections import deque

import torch

from .decode import MAX_BATCH
from .session import GenerationSession, check_seed
from .stages import COARSE, FINE, SEMANTIC, STREAMS, _check_prime, _stage_top_p, plan_song, song_output

_WHERE = "open_musiclm_b200 MusicLM"


def _positions(cond_tokens, steps: int, q: int) -> int:
    """Decode positions of one request: each conditioning sequence with its eos and start token, the predicted
    sequence's start token and its steps * q tokens (GenerationSession's prompt plus sampled tokens)."""
    return sum(n + 2 for n in cond_tokens) + 1 + steps * q


class _Song:
    """One song in flight: its plan, its streams (the generated ones preallocated at their final lengths, the primes),
    how much of each generated stream is written from its start (`done`) and which written pieces lie beyond that,
    the next job of each stage to submit, the jobs not yet finished, and the output rows handed out so far."""

    def __init__(self, handle, plan, clap, primes, given):
        self.handle, self.plan, self.clap, self.primes, self.given = handle, plan, clap, primes, given
        self.streams = dict(primes)
        self.done = {name: 0 for name in STREAMS}
        self.pieces = {name: {} for name in STREAMS}
        self.by_stage = [[j for j in plan.jobs if j.stage == s] for s in (SEMANTIC, COARSE, FINE)]
        self.next = [0, 0, 0]
        self.left = len(plan.jobs)
        self.sent = 0                  # output rows known to be final
        self.handed = 0                # output rows handed out by ready()
        self.live = set()              # (stage, request handle) of its submitted jobs that have not finished
        self.held = None               # suspended: the (stage, request handle) pairs suspend() suspended

    def write(self, job, tokens):
        """A finished job's tokens [steps, q] -> its stream."""
        name, n = STREAMS[job.stage], job.steps - job.drop
        if n > 0:
            self.streams[name][0, job.dest:job.dest + n] = tokens[job.drop:]
            self.pieces[name][job.dest] = job.dest + n
            while self.done[name] in self.pieces[name]:
                self.done[name] = self.pieces[name].pop(self.done[name])
        self.left -= 1

    def runnable(self):
        """The jobs whose input streams now exist and that were not submitted yet, stage by stage in plan order."""
        out = []
        for s, jobs in enumerate(self.by_stage):
            while self.next[s] < len(jobs) and all(self.done[k] >= v for k, v in jobs[self.next[s]].needs.items()):
                out.append(jobs[self.next[s]])
                self.next[s] += 1
        return out

    def part(self, ref):
        return None if ref is None else self.streams[ref[0]][:, ref[1]:ref[2]]

    def final_rows(self) -> int:
        """How many rows of the output tensor are final: coarse_only, the written coarse stream; else the acoustic
        rows whose prime or generated coarse and fine tokens all exist."""
        p = self.plan
        if p.coarse_only:
            return self.done["coarse"]
        tc = self.primes["prime_coarse"].shape[1] if p.primed else 0
        tf = self.primes["prime_fine"].shape[1] if p.primed else 0
        return min(tc + max(self.done["coarse"] - p.coarse_lo, 0), tf + max(self.done["fine"] - p.fine_lo, 0))

    def rows(self, a: int, b: int):
        """Rows a ... b - 1 of the output tensor, [1, b - a, q]."""
        p = self.plan
        if p.coarse_only:
            return self.streams["coarse"][:, a:b]

        def part(prime, name, lo):     # rows a ... b - 1 of cat([prime, stream[:, lo:]], 1)
            t = prime.shape[1] if prime is not None else 0
            pieces = []
            if a < t:
                pieces.append(prime[:, a:min(b, t)])
            if b > t:
                pieces.append(self.streams[name][:, lo + max(a - t, 0):lo + b - t])
            return torch.cat(pieces, 1) if len(pieces) > 1 else pieces[0]
        return torch.cat([part(self.primes.get("prime_coarse"), "coarse", p.coarse_lo),
                          part(self.primes.get("prime_fine"), "fine", p.fine_lo)], -1)


class MusicLMSession:
    """Continuous batching of seeded songs through MusicLM's three stages, one `GenerationSession` per stage.

        sess = MusicLMSession(musiclm, slots=(16, 32, 64), semantic_window_seconds=10, max_songs=64, max_queue=0)
        h = sess.add(clap_token_ids=clap_1xn, seed=1234, output_seconds=12, top_p=None)
        while not sess.idle:
            sess.step()
            for h, rows in sess.ready().items(): ...     # [1, t, q] output rows that became final, in order
            for h, out in sess.finished().items(): ...   # generate_tokens(..., seeds=[seed], return_all=True) alone

    slots: rows of each stage's session, one int or (semantic, coarse, fine).  The windowing arguments are those of
    `generate_tokens`, fixed for the session; with them and the clap length (clap_length; default one time step of
    the semantic stage's clap quantizers) they bound every window's context, and so each stage's max_positions.
    max_songs: songs in flight at once; max_queue: songs that may wait beyond them (`add` raises past that).

    A window job is added to its stage's session as soon as the streams it reads exist; each stage's session serves
    its requests first come, first served.  `step` runs one time step of every stage session with work, writes the
    windows that finished into their songs' streams and adds the jobs they unblock.  `ready` hands out, per song, the
    rows of its output tensor (the acoustic tokens [1, T, coarse + fine quantizers], or the coarse stream with
    coarse_only) that became final since the last call; the prime's rows are final at once.  Concatenated, a song's
    rows are its `finished` output's first tensor.  Songs are seeded; there is no noise stream.

    Between steps, `status(h)` reports where a song is, `cancel(h)` drops it and frees its stage slots and its place
    under max_songs, and `suspend(h)` / `resume(h)` stop a song's windows and later continue them bit for bit.

    Streams: every stage's device work (its session's adds, steps, prefills and graph replays, and the writes of its
    windows into the songs' streams) runs on `streams[stage]`, a CUDA stream the session owns on that stage's device.
    Events order the rest, and `step` never waits for the device once the stage sessions have captured their graphs:
    a stage stream waits on the caller's current stream before it reads what the caller passed to `add`, and on a
    stage's `written` event (recorded after that stage's writes) before a window reads that stage's stream; `ready` and
    `finished` make the caller's current stream wait on every stage's event, so what they return is usable on it as
    is.  Tensors used on a stream other than the one they were allocated on are recorded on it (record_stream)."""

    def __init__(self, musiclm, slots=64, *, semantic_window_seconds=10, coarse_window_seconds=4, fine_window_seconds=2,
                 semantic_steps_per_second=50, acoustic_steps_per_second=75, semantic_sliding_window_step_percent=0.5,
                 coarse_sliding_window_step_percent=0.5, fine_sliding_window_step_percent=1, max_songs=64, max_queue=0,
                 clap_length=None):
        where = f"{_WHERE}Session"
        slots = tuple(slots) if isinstance(slots, (list, tuple)) else (slots,) * 3
        stages = (musiclm.semantic, musiclm.coarse, musiclm.fine)
        if clap_length is None:
            clap_length = stages[0].transformer_wrapper.token_sequences[0].num_quantizers
        for name, v in (("max_songs", max_songs), ("max_queue", max_queue), ("clap_length", clap_length)) + \
                tuple((f"slots[{i}]", s) for i, s in enumerate(slots)):
            if isinstance(v, bool) or not isinstance(v, numbers.Integral):
                raise ValueError(f"{where}: {name} must be an int, not {v!r}")
        if len(slots) != 3:
            raise ValueError(f"{where}: slots must be one int or three (semantic, coarse, fine), got {len(slots)}")
        if not all(1 <= n <= MAX_BATCH for n in slots):
            raise ValueError(f"{where}: slots = {slots} lie outside [1, {MAX_BATCH}]")
        if max_songs < 1 or max_queue < 0 or clap_length < 1:
            raise ValueError(f"{where}: max_songs = {max_songs} must be >= 1, max_queue = {max_queue} >= 0 and "
                             f"clap_length = {clap_length} >= 1")
        self.window_args = dict(semantic_window_seconds=semantic_window_seconds, coarse_window_seconds=coarse_window_seconds,
                                fine_window_seconds=fine_window_seconds, semantic_steps_per_second=semantic_steps_per_second,
                                acoustic_steps_per_second=acoustic_steps_per_second,
                                semantic_sliding_window_step_percent=semantic_sliding_window_step_percent,
                                coarse_sliding_window_step_percent=coarse_sliding_window_step_percent,
                                fine_sliding_window_step_percent=fine_sliding_window_step_percent)
        self.mlm, self.clap_length = musiclm, int(clap_length)
        self.max_songs, self.max_queue = int(max_songs), int(max_queue)
        self.qc = musiclm.coarse.num_coarse_quantizers
        self.qf = musiclm.fine.transformer_wrapper.token_sequences[-1].num_quantizers
        self.devices = [st.device for st in stages]
        # a window's context: clap ids, its conditioning window, and at most one window of predicted steps
        sps, aps = semantic_steps_per_second, acoustic_steps_per_second
        fwin = int(fine_window_seconds * aps)
        self.max_positions = (_positions([self.clap_length], int(semantic_window_seconds * sps), 1),
                              _positions([self.clap_length, int(coarse_window_seconds * sps - 1)], int(coarse_window_seconds * aps), self.qc),
                              _positions([self.clap_length, fwin * self.qc], fwin, self.qf))
        self.sessions = [GenerationSession(st.transformer_wrapper, slots=int(n), max_positions=p, max_queue=sys.maxsize)
                         for st, n, p in zip(stages, slots, self.max_positions)]
        # one stream per stage (None on a CPU device); each starts after the caller's work so far, such as weight updates
        self.streams = [torch.cuda.Stream(d) if torch.device(d).type == "cuda" else None for d in self.devices]
        self.written = [torch.cuda.Event() if s is not None else None for s in self.streams]
        for s in self.streams:
            if s is not None:
                s.wait_stream(torch.cuda.current_stream(s.device))
        self._next_handle = 0
        self._songs = {}               # handle -> _Song in flight, in admission order
        self._queue = deque()          # (handle, plan, claps, primes, given) waiting for room
        self._jobs = [{}, {}, {}]      # per stage: request handle -> (song, job)
        self._ready = {}               # handle -> _Song with final rows not handed out yet
        self._done = {}                # handle -> finished _Song
        self._held = {}                # handle -> queue entry of a song suspended while queued
        self._cancelled = set()

    # ------------------------------------------------------------------------------------------------ streams
    def _caller_event(self):
        """An event on the caller's current stream, after the work it enqueued so far (None without a GPU stage)."""
        if not any(self.streams):
            return None
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        return ev

    def _wait_writes(self):
        """The caller's current stream waits on every stage's writes so far; returns it (None without a GPU stage)."""
        if not any(self.streams):
            return None
        cur = torch.cuda.current_stream()
        for ev in self.written:
            if ev is not None:
                cur.wait_event(ev)
        return cur

    @staticmethod
    def _record_on(cur, songs):
        """`ready` and `finished` read the songs' streams on the caller's stream: as slices they hand out and as inputs
        of the concatenations they make there.  Every stream buffer of those songs (generated ones, allocated on a
        stage stream, and the primes) is recorded on it, so that no stage stream reuses a buffer before the caller's
        reads are done, whether or not the caller keeps a view of it."""
        if cur is not None:
            for song in songs:
                for t in song.streams.values():
                    t.record_stream(cur)

    # ------------------------------------------------------------------------------------------------ songs
    def add(self, *, clap_token_ids, seed, output_seconds=8, top_p=None, prime_semantic_token_ids=None,
            prime_coarse_token_ids=None, prime_fine_token_ids=None, coarse_only=False):
        """Queues one song and returns its handle (an int): `generate_tokens`' arguments for one prompt, with one seed.
        It starts at once while fewer than max_songs are in flight, else waits (up to max_queue songs).  Every check
        runs before any device work and raises ValueError."""
        where = f"{_WHERE}Session.add"
        seed = check_seed(seed, where)
        top_p = _stage_top_p(top_p, "MusicLMSession.add")
        if isinstance(output_seconds, bool) or not isinstance(output_seconds, numbers.Real) or not output_seconds > 0:
            raise ValueError(f"{where}: output_seconds must be a number > 0, not {output_seconds!r}")
        if not isinstance(clap_token_ids, torch.Tensor) or tuple(clap_token_ids.shape) != (1, self.clap_length):
            got = tuple(clap_token_ids.shape) if isinstance(clap_token_ids, torch.Tensor) else type(clap_token_ids).__name__
            raise ValueError(f"{where}: clap_token_ids must be [1, {self.clap_length}] (the session's clap length), got {got}")
        primes = (prime_semantic_token_ids, prime_coarse_token_ids, prime_fine_token_ids)
        primed = prime_semantic_token_ids is not None
        if any((p is not None) != primed for p in primes):
            raise ValueError(f"{where}: pass all three prime token streams or none")
        if primed:
            primes = [_check_prime(t, 1, q, what, "MusicLMSession.add") for t, q, what in
                      zip(primes, (1, self.qc, self.qf), ("prime_semantic_token_ids", "prime_coarse_token_ids", "prime_fine_token_ids"))]
        plan = plan_song(output_seconds=output_seconds, **self.window_args, prime_lengths=[t.shape[1] for t in primes] if primed else None,
                         coarse_only=bool(coarse_only), top_p=top_p, seed=seed)
        q_cond = (1, 1, self.qc)
        q_out = (1, self.qc, self.qf)
        for job in plan.jobs:
            cond = [self.clap_length] + ([(job.cond[2] - job.cond[1]) * q_cond[job.stage]] if job.cond else [])
            n = _positions(cond, job.steps, q_out[job.stage])
            if n > self.max_positions[job.stage]:
                raise ValueError(f"{where}: {STREAMS[job.stage]} window {job.window} needs {n} positions, more than the "
                                 f"{self.max_positions[job.stage]} its window bounds (a prefix longer than one window)")
        if len(self._songs) >= self.max_songs and len(self._queue) >= self.max_queue:
            raise ValueError(f"{where}: {len(self._songs)} songs are in flight (max_songs = {self.max_songs}) and the queue "
                             f"holds {len(self._queue)} of max_queue = {self.max_queue}")
        handle = self._next_handle
        self._next_handle += 1
        # on the caller's stream: the clap ids on every stage's device and the primes on theirs, then an event that
        # the stage streams wait on before they read them
        claps = [clap_token_ids.to(d, torch.int64) for d in self.devices]
        primes = dict(zip(("prime_semantic", "prime_coarse", "prime_fine"),
                          (t.to(d, torch.int64) for t, d in zip(primes, self.devices)))) if primed else {}
        self._queue.append((handle, plan, claps, primes, self._caller_event()))
        self._admit()
        return handle

    def _admit(self):
        while self._queue and len(self._songs) < self.max_songs:
            handle, plan, claps, primes, given = self._queue.popleft()
            song = _Song(handle, plan, claps, primes, given)
            q = (1, self.qc, self.qf)
            for s, name in enumerate(STREAMS):
                if plan.length[name]:
                    # allocated on the stage stream that writes it; recorded on every other stream that reads it
                    with torch.cuda.stream(self.streams[s]):
                        song.streams[name] = torch.empty(1, plan.length[name], q[s], device=self.devices[s], dtype=torch.int64)
            self._songs[handle] = song
            self._emit(song)
            self._submit(song)

    def _submit(self, song):
        if song.held is not None:      # a suspended song submits nothing until it is resumed
            return
        for job in song.runnable():
            s = job.stage
            with torch.cuda.stream(self.streams[s]):
                self._wait_inputs(song, job)
                cond = song.part(job.cond)
                h = self.sessions[s].add(conditioning_token_ids=[song.clap[s]] + ([cond] if cond is not None else []),
                                         pred_token_ids=song.part(job.prefix), seed=job.seed, max_time_steps=job.max_time_steps,
                                         temperature=job.temperature, top_p=job.top_p)
            self._jobs[s][h] = (song, job)
            song.live.add((s, h))

    def _wait_inputs(self, song, job):
        """Orders a job's reads on its stage stream: after the caller's `add` (clap ids, primes) and after the writes of
        the stage whose stream it reads; those tensors are recorded on the stage stream, whose reads may outlast the
        caller's and the producer's references."""
        st = self.streams[job.stage]
        if st is None:
            return
        if song.given is not None:
            st.wait_event(song.given)
        song.clap[job.stage].record_stream(st)
        for ref in (job.cond, job.prefix):
            if ref is None:
                continue
            src = STREAMS.index(ref[0]) if ref[0] in STREAMS else None
            if src != job.stage:
                if src is not None:
                    st.wait_event(self.written[src])
                song.streams[ref[0]].record_stream(st)

    def _emit(self, song):
        """Marks the song's output rows that became final since the last call for `ready` (host bookkeeping: `ready`
        slices them on the caller's stream)."""
        n = song.final_rows()
        if n > song.sent:
            self._ready[song.handle] = song
            song.sent = n

    @property
    def idle(self) -> bool:
        """No song in flight or queued, but suspended ones (they wait for `resume` and keep no session busy)."""
        return not self._queue and all(song.held is not None for song in self._songs.values())

    # ------------------------------------------------------------------------------------------------ cancel, suspend
    def _state(self, handle, where: str) -> str:
        if not isinstance(handle, bool) and isinstance(handle, numbers.Integral):
            song = self._songs.get(handle)
            if song is not None:
                if song.held is not None:
                    return "suspended"
                running = any(self.sessions[s].status(h) in ("running", "prefilling") for s, h in song.live)
                return "running" if running else "waiting"
            if handle in self._held:
                return "suspended"
            if any(entry[0] == handle for entry in self._queue):
                return "queued"
            if handle in self._cancelled:
                raise ValueError(f"{_WHERE}Session.{where}: song {handle} was cancelled")
            if 0 <= handle < self._next_handle:
                return "finished"
        raise ValueError(f"{_WHERE}Session.{where}: {handle!r} is not a song handle of this session")

    def status(self, handle) -> str:
        """"queued" (waiting for room under max_songs), "running" (a window of it decodes), "waiting" (admitted, no
        window decoding at the moment), "suspended" or "finished" (its output waits in `finished()` or was returned).
        Host state only.  ValueError for a handle `add` never returned or a cancelled one."""
        return self._state(handle, "status")

    def cancel(self, handle) -> bool:
        """Drops a queued, admitted or suspended song: its windows leave the three stage sessions (their slots are
        free at the next step), its jobs are never submitted, its place under max_songs goes to the next queued song
        at once, and it never appears in `ready()` or `finished()` again (rows `ready()` returned stay returned).  No
        other song changes.  Returns False for a finished song, whose output stays where it is.  Called between steps;
        ValueError for a handle `add` never returned or a cancelled one."""
        state = self._state(handle, "cancel")
        if state == "finished":
            return False
        if handle in self._held:
            del self._held[handle]
        elif state == "queued":
            self._queue.remove(next(e for e in self._queue if e[0] == handle))
        else:
            song = self._songs.pop(handle)
            for s, h in sorted(song.live):
                self.sessions[s].cancel(h)
                del self._jobs[s][h]
            self._ready.pop(handle, None)
        self._cancelled.add(handle)
        self._admit()
        return True

    def suspend(self, handle):
        """An admitted song stops: its windows' rows give up their stage slots (running ones keep a device snapshot
        of their decode state, GenerationSession.suspend; the snapshots are taken on the stage streams after the
        caller's current stream) and none of its jobs is submitted until `resume`.  It keeps its place under
        max_songs (cancel it to free that).  A queued song leaves the queue.  Called between steps; ValueError for a
        song that is suspended, finished, cancelled or unknown."""
        state = self._state(handle, "suspend")
        if state not in ("queued", "running", "waiting"):
            raise ValueError(f"{_WHERE}Session.suspend: song {handle} is {state}; only queued and admitted songs can be suspended")
        if state == "queued":
            entry = next(e for e in self._queue if e[0] == handle)
            self._queue.remove(entry)
            self._held[handle] = entry
            return
        song = self._songs[handle]
        ev = self._caller_event()
        song.held = []
        for s, h in sorted(song.live):
            if self.sessions[s].status(h) not in ("queued", "running"):
                continue
            with torch.cuda.stream(self.streams[s]):
                if ev is not None and self.streams[s] is not None:
                    self.streams[s].wait_event(ev)
                self.sessions[s].suspend(h)
            song.held.append((s, h))

    def resume(self, handle):
        """A suspended song continues: its windows' rows go back to the head of their stage sessions' queues, in the
        order they were submitted, and its jobs are submitted again as their inputs exist.  Its output and its
        `ready()` rows are bit for bit those of the song never suspended.  A song suspended while queued goes back to
        the head of the queue.  ValueError for a song that is not suspended."""
        state = self._state(handle, "resume")
        if state != "suspended":
            raise ValueError(f"{_WHERE}Session.resume: song {handle} is {state}, not suspended")
        if handle in self._held:
            self._queue.appendleft(self._held.pop(handle))
            self._admit()
            return
        song = self._songs[handle]
        for s, h in song.held:
            self.sessions[s].resume(h)
        song.held = None
        self._submit(song)

    def step(self):
        """One time step of every stage session with work; then the windows that finished go into their songs'
        streams, the jobs they unblock are added, and finished songs make room for queued ones."""
        for stage, sess in enumerate(self.sessions):
            if not sess.idle:
                with torch.cuda.stream(self.streams[stage]):
                    sess.step()
        touched = {}
        for stage, sess in enumerate(self.sessions):
            done = sess.finished()
            if not done:
                continue
            with torch.cuda.stream(self.streams[stage]):
                for h, tokens in done.items():
                    if h not in self._jobs[stage]:      # a window of a cancelled song that finished at its add
                        continue
                    song, job = self._jobs[stage].pop(h)
                    song.live.discard((stage, h))
                    song.write(job, tokens)
                    touched[song.handle] = song
                if self.written[stage] is not None:
                    self.written[stage].record(self.streams[stage])
        for song in sorted(touched.values(), key=lambda s: s.handle):
            self._emit(song)
            if song.left:
                self._submit(song)
                continue
            del self._songs[song.handle]
            self._done[song.handle] = song
        self._admit()

    def ready(self):
        """{handle: [1, t, q] rows} of each song's output tensor that became final since the last call, in order."""
        if not self._ready:
            return {}
        cur = self._wait_writes()
        out = {h: song.rows(song.handed, song.sent) for h, song in self._ready.items()}
        for song in self._ready.values():
            song.handed = song.sent
        self._record_on(cur, self._ready.values())
        self._ready = {}
        return out

    def finished(self):
        """{handle: output} of the songs that finished since the last call: exactly
        generate_tokens(..., seeds=[seed], return_all=True) for that song alone."""
        if not self._done:
            return {}
        cur = self._wait_writes()
        out = {h: song_output(song.plan, song.streams, True) for h, song in self._done.items()}
        self._record_on(cur, self._done.values())
        self._done = {}
        return out
