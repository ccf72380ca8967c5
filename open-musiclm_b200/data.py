"""Token data pipeline for the H100 training path: the reference's pre-tokenised dataset, resident in HBM.

The reference trains each stage from `preprocessed.db` (sqlite; one row per audio file with the clap / semantic / coarse /
fine token arrays, written by open_musiclm/preprocess.py:200,279 with numpy-serialised blobs) through
`PreprocessedDataset` (open_musiclm/data.py:304-438): per item one sqlite query, two `random.randint` draws and a few
Python slices, collated by a single-process DataLoader.  At >1 M tokens/s per GPU that path is the bottleneck, and the
whole token corpus is small next to 180 GB of HBM (a 30 s clip is ~12 k int16 tokens), so here

  * `TokenStore.from_sqlite` reads the same database ONCE into flat int16 arrays + per-item offsets and uploads them;
  * `TokenStore.sample_batch` draws the crops on the host with the reference's arithmetic (whole-second outer window of
    `semantic_window_seconds`, inner window for the coarse / fine stages; data.py:356-366, 388-434) and assembles the
    batch with one `omlm_gather_windows` launch per sequence, entirely on the device: the tensors it returns are what
    `HotPathTrainer.train_step` takes.

`write_sqlite` produces a database in the reference's format (tests, synthetic corpora).
"""
import io
import os
import random
import sqlite3
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import lib

STAGE_COLUMNS = {"semantic": ("clap", "semantic"), "coarse": ("clap", "semantic", "coarse"), "fine": ("clap", "coarse", "fine")}


def _blob(arr: np.ndarray) -> bytes:
    out = io.BytesIO()
    np.save(out, arr)           # the reference's sqlite adapter (data.py:33-41)
    return out.getvalue()


def _unblob(b: bytes) -> np.ndarray:
    return np.load(io.BytesIO(b))


def write_sqlite(folder: str, items: Sequence[dict]) -> str:
    """items: dicts with 'clap' [L - W + 1, q_clap], 'semantic' [1, Ts], 'coarse' [1, Ta, qc], 'fine' [1, Ta, qf] (uint16),
    optional 'path'.  Schema and serialisation of preprocess.py:200,279."""
    os.makedirs(folder, exist_ok=True)
    path = os.path.join(folder, "preprocessed.db")
    conn = sqlite3.connect(path)
    cur = conn.cursor()
    cur.execute("CREATE TABLE IF NOT EXISTS tokens(idx integer primary key, path text, clap array, semantic array, coarse array, fine array)")
    for i, it in enumerate(items):
        cur.execute("INSERT INTO tokens VALUES (?, ?, ?, ?, ?, ?)",
                    (i, it.get("path", f"item{i}"), *[sqlite3.Binary(_blob(np.asarray(it[k]))) for k in ("clap", "semantic", "coarse", "fine")]))
    conn.commit()
    conn.close()
    return path


class TokenStore:
    """One training stage's view of the token corpus, resident on `device`."""

    def __init__(self, stage: str, arrays: dict, lengths: np.ndarray, *, semantic_window_seconds=10, coarse_window_seconds=4,
                 fine_window_seconds=2, semantic_steps_per_second=50, acoustic_steps_per_second=75, device="cuda"):
        assert stage in STAGE_COLUMNS
        self.stage, self.device = stage, torch.device(device)
        self.sw, self.cw, self.fw = semantic_window_seconds, coarse_window_seconds, fine_window_seconds
        self.sps, self.aps = semantic_steps_per_second, acoustic_steps_per_second
        self.audio_len = lengths                                    # whole seconds per item
        self.flat, self.offset, self.width = {}, {}, {}
        for name, (flat, off) in arrays.items():
            self.width[name] = flat.shape[1]
            self.offset[name] = off                                 # first row of item i in the flat array (numpy int64)
            self.flat[name] = torch.from_numpy(flat.astype(np.int16, copy=False)).to(self.device)
        self.n_items = len(lengths)

    # ---------------------------------------------------------------------------------------------- loading
    @classmethod
    def from_sqlite(cls, folder: str, stage: str, **kw) -> "TokenStore":
        conn = sqlite3.connect(os.path.join(folder, "preprocessed.db"))
        cols = STAGE_COLUMNS[stage]
        rows = conn.execute(f"SELECT {', '.join(cols)} FROM tokens ORDER BY idx").fetchall()
        conn.close()
        return cls.from_items(stage, [dict(zip(cols, (_unblob(b) for b in r))) for r in rows], **kw)

    @classmethod
    def from_items(cls, stage: str, items: Sequence[dict], **kw) -> "TokenStore":
        sw = kw.get("semantic_window_seconds", 10)
        sps, aps = kw.get("semantic_steps_per_second", 50), kw.get("acoustic_steps_per_second", 75)
        cols = STAGE_COLUMNS[stage]
        per = {c: [] for c in cols}
        lengths = []
        for it in items:
            # get_and_assert_audio_length_from_tokens, data.py:334-346: every token stream implies the same audio length
            ls = []
            for c in cols:
                a = np.asarray(it[c])
                if c == "clap":
                    ls.append(a.shape[0] + sw - 1)
                    per[c].append(a.reshape(a.shape[0], -1))
                elif c == "semantic":
                    ls.append((a.shape[1] + 1) // sps)
                    per[c].append(a.reshape(a.shape[1], -1))
                else:
                    ls.append(a.shape[1] // aps)
                    per[c].append(a.reshape(a.shape[1], -1))
            assert len(set(int(l) for l in ls)) == 1, "audio lengths are not equal"
            lengths.append(int(ls[0]))
        arrays = {}
        for c in cols:
            off = np.zeros(len(items) + 1, np.int64)
            off[1:] = np.cumsum([a.shape[0] for a in per[c]])
            arrays[c] = (np.concatenate(per[c], 0).astype(np.uint16).view(np.int16), off[:-1])
        return cls(stage, arrays, np.asarray(lengths, np.int64), **kw)

    # ---------------------------------------------------------------------------------------------- crops
    def crop_plan(self, item: int, rng) -> dict:
        """Row ranges (start, length) of one random crop of `item`, with the reference's draws: an outer window of
        semantic_window_seconds at a whole-second offset, and for coarse / fine an inner window inside it
        (compute_crop_indices, data.py:356-366; crop_* 348-354; get_clap_tokens 346)."""
        L = int(self.audio_len[item])
        o0 = rng.randint(0, L - self.sw)
        plan = {"clap": (o0, 1)}
        if self.stage == "semantic":
            plan["semantic"] = (o0 * self.sps, (o0 + self.sw) * self.sps - 1 - o0 * self.sps)
            return plan
        inner = self.cw if self.stage == "coarse" else self.fw
        i0 = rng.randint(o0, o0 + self.sw - inner)
        i1 = i0 + inner
        if self.stage == "coarse":
            plan["semantic"] = (i0 * self.sps, i1 * self.sps - 1 - i0 * self.sps)
            plan["coarse"] = (i0 * self.aps, (i1 - i0) * self.aps)
        else:
            plan["coarse"] = (i0 * self.aps, (i1 - i0) * self.aps)
            plan["fine"] = (i0 * self.aps, (i1 - i0) * self.aps)
        return plan

    def sample_batch(self, batch_size: int, rng: Optional[random.Random] = None, items: Optional[Sequence[int]] = None) -> List[torch.Tensor]:
        """One training batch, on the device, in the stage's order: (clap [B, q], semantic [B, Ts, 1], coarse [B, Ta, qc])
        for the coarse stage etc. — the tuple the reference's dataloader yields (data.py:388-434, concatenate_fn)."""
        rng = rng or random
        items = list(items) if items is not None else [rng.randrange(self.n_items) for _ in range(batch_size)]
        plans = [self.crop_plan(i, rng) for i in items]
        out = []
        for name in STAGE_COLUMNS[self.stage]:
            length = plans[0][name][1]
            assert all(p[name][1] == length for p in plans)
            start = torch.tensor([int(self.offset[name][i]) + p[name][0] for i, p in zip(items, plans)], dtype=torch.int64).to(self.device, non_blocking=True)
            dst = torch.empty(len(items), length, self.width[name], dtype=torch.int64, device=self.device)
            lib.gather_windows(self.flat[name], start, dst)
            out.append(dst[:, 0] if name == "clap" else dst)
        return out

    def bytes_resident(self) -> int:
        return sum(t.numel() * 2 for t in self.flat.values())


# ---------------------------------------------------------------------------------------------------- checkpoints
def checkpoint_paths(results_folder: str, stage: str, steps: int) -> Tuple[str, str, str]:
    """File names of SingleStageTrainer's periodic save (trainer.py:540-542)."""
    return tuple(os.path.join(results_folder, f"{stage}.{kind}.{steps}.pt") for kind in ("transformer", "optimizer", "scheduler"))


def latest_checkpoints(results_folder: str, max_step: Optional[int] = None):
    """scripts/train_utils.py:19-46: newest aligned (transformer, optimizer[, scheduler]) triple of a results folder."""
    best = {"transformer": (-1, None), "optimizer": (-1, None), "scheduler": (-1, None)}
    limit = float("inf") if max_step is None else max_step
    for f in os.listdir(results_folder):
        if not f.endswith(".pt"):
            continue
        for kind in best:
            if kind in f:
                step = int(f.split(".")[2])
                if best[kind][0] < step <= limit:
                    best[kind] = (step, os.path.join(results_folder, f))
                break
    assert best["transformer"][0] == best["optimizer"][0], "transformer and optimizer checkpoints are not aligned"
    if best["scheduler"][1] is not None:
        assert best["transformer"][0] == best["scheduler"][0], "transformer and scheduler checkpoints are not aligned"
    return (best["transformer"][1], best["optimizer"][1], best["scheduler"][1]), best["transformer"][0]
