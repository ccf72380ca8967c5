"""Stage wrappers and the three-stage windowed generation on top of the H100 TokenConditionedTransformer.

Mirrors the orchestration layer of the reference (open_musiclm/open_musiclm.py:514-1035): `SemanticStage`,
`CoarseStage`, `FineStage` (each a TokenConditionedTransformerWrapper plus the optional tokenizer objects) and
`MusicLM.forward`, which chains them through sliding windows: semantic tokens are grown window by window conditioned on
the tail of what exists, every coarse window is conditioned on a slice of the semantic stream plus the tail of the coarse
stream, every fine window on a slice of the coarse stream.  All arithmetic here is integer bookkeeping on token tensors;
the compute is `TokenConditionedTransformerWrapper.generate` (KV-cache decode, decode.py).

The tokenizers (CLAP-RVQ, MERT/HuBERT k-means, Encodec) are outside the hot path (SURVEY section 2): the stages accept
them as opaque callables exactly like the reference and never need them when token ids are passed in.
"""
from typing import List, Optional

import torch
from torch import nn

from .decode import TokenConditionedTransformerWrapper
from .model import TokenConditionedTransformer


class NoiseStream:
    """A pre-drawn stream of uniform(0,1) tensors [n, b, C], handed out in order to successive generate() calls
    (parity runs: the stream torch's default generator would have produced for the reference)."""

    def __init__(self, uniforms: torch.Tensor):
        self.u, self.at = uniforms, 0

    def take(self, n: int) -> torch.Tensor:
        assert self.at + n <= self.u.shape[0], "noise stream exhausted"
        out = self.u[self.at:self.at + n]
        self.at += n
        return out


_MASK64 = (1 << 64) - 1
SEMANTIC, COARSE, FINE = 0, 1, 2       # stage numbers of window_seed


def splitmix64(x: int) -> int:
    """The splitmix64 output function (Steele, Lea and Flood, "Fast splittable pseudorandom number generators", 2014)
    of the 64-bit value x: x + 0x9E3779B97F4A7C15, then two xor-shift-multiply rounds and a final xor-shift."""
    z = (x + 0x9E3779B97F4A7C15) & _MASK64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _MASK64
    return z ^ (z >> 31)


def window_seed(seed: int, stage: int, window: int) -> int:
    """The seed MusicLM.generate_tokens hands one sequence's generate call for window `window` (0, 1, ... in the order
    of generation) of stage `stage` (SEMANTIC, COARSE, FINE), given that sequence's seed:
        splitmix64(seed ^ splitmix64(stage << 32 | window))   (all values unsigned 64-bit)."""
    return splitmix64((int(seed) & _MASK64) ^ splitmix64((stage << 32) | window))


def _n_new(pred_token_ids, max_time_steps: int, q: int) -> int:
    init = 0 if pred_token_ids is None else pred_token_ids.shape[1]
    return max(0, (max_time_steps - init) * q)


class _Stage(nn.Module):
    """Common part of the three stages: the wrapper, the device, the conditioning order."""

    def __init__(self, transformer: TokenConditionedTransformer, pad_id, unique_consecutive, cross_entropy_loss_weights, mask_prob,
                 wrapper=None):
        super().__init__()
        self.transformer_wrapper = wrapper if wrapper is not None else TokenConditionedTransformerWrapper(
            transformer=transformer, pad_id=pad_id, unique_consecutive=unique_consecutive,
            cross_entropy_loss_weights=cross_entropy_loss_weights, mask_prob=mask_prob)

    @property
    def device(self):
        return self.transformer_wrapper.device

    def _generate(self, conditioning: List[torch.Tensor], pred, noise: Optional[NoiseStream], **kw):
        q = self.transformer_wrapper.token_sequences[-1].num_quantizers
        if noise is not None:
            kw["uniform_noise"] = noise.take(_n_new(pred, kw["max_time_steps"], q))
        return self.transformer_wrapper.generate(conditioning_token_ids=conditioning, pred_token_ids=pred, **kw)


def _clap_ids(clap_token_ids, clap, conditioning_audio, conditioning_text):
    """get_or_compute_clap_token_ids, open_musiclm.py:476-485."""
    if clap_token_ids is None:
        assert (conditioning_audio is not None) ^ (conditioning_text is not None), "either condition on text or audio"
        assert clap is not None, "a CLAP quantizer is needed to turn text / audio into clap token ids"
        clap_token_ids = clap(text_input=conditioning_text) if conditioning_text is not None else clap(audio_input=conditioning_audio)
    return clap_token_ids


class SemanticStage(_Stage):
    """open_musiclm.py:514-603: clap tokens -> semantic tokens."""

    def __init__(self, *, semantic_transformer: TokenConditionedTransformer, wav2vec=None, clap=None, pad_id=-1,
                 unique_consecutive=False, cross_entropy_loss_weights: Optional[List[float]] = None, mask_prob=0.15, wrapper=None):
        super().__init__(semantic_transformer, pad_id, unique_consecutive, cross_entropy_loss_weights, mask_prob, wrapper)
        self.wav2vec, self.clap = wav2vec, clap

    @torch.no_grad()
    def generate(self, *, conditioning_text=None, conditioning_audio=None, input_audio=None, clap_token_ids=None,
                 semantic_token_ids=None, filter_thres=0.9, temperature=1., max_time_steps=30 * 25, include_eos_in_output=False,
                 append_eos_to_conditioning_tokens=True, noise: Optional[NoiseStream] = None, **kwargs):
        clap_token_ids = _clap_ids(clap_token_ids, self.clap, conditioning_audio, conditioning_text)
        if semantic_token_ids is None and input_audio is not None:
            assert self.wav2vec is not None
            semantic_token_ids = self.wav2vec(input_audio, flatten=False)
        return self._generate([clap_token_ids], semantic_token_ids, noise, max_time_steps=max_time_steps, filter_thres=filter_thres,
                              temperature=temperature, include_eos_in_output=include_eos_in_output,
                              append_eos_to_conditioning_tokens=append_eos_to_conditioning_tokens, **kwargs)

    def forward(self, *, raw_wave_for_clap=None, raw_wave_for_semantic=None, clap_token_ids=None, semantic_token_ids=None,
                return_loss=False, **kwargs):
        clap_token_ids = _clap_ids(clap_token_ids, self.clap, raw_wave_for_clap, None)
        if semantic_token_ids is None:
            assert raw_wave_for_semantic is not None and self.wav2vec is not None
            semantic_token_ids = self.wav2vec(raw_wave_for_semantic, flatten=False)
        return self.transformer_wrapper.forward(all_token_ids=[clap_token_ids, semantic_token_ids], return_loss=return_loss, **kwargs)


class CoarseStage(_Stage):
    """open_musiclm.py:606-716: clap + semantic tokens -> coarse acoustic tokens."""

    def __init__(self, *, coarse_transformer: TokenConditionedTransformer, wav2vec=None, clap=None, neural_codec=None, pad_id=-1,
                 unique_consecutive=False, cross_entropy_loss_weights: Optional[List[float]] = None, mask_prob=0.15, wrapper=None):
        super().__init__(coarse_transformer, pad_id, unique_consecutive, cross_entropy_loss_weights, mask_prob, wrapper)
        self.wav2vec, self.clap, self.neural_codec = wav2vec, clap, neural_codec
        self.num_coarse_quantizers = self.transformer_wrapper.token_sequences[-1].num_quantizers

    @torch.no_grad()
    def generate(self, *, semantic_token_ids, coarse_token_ids=None, conditioning_text=None, conditioning_audio=None,
                 clap_token_ids=None, filter_thres=0.9, temperature=1., max_time_steps=10 * 600, include_eos_in_output=False,
                 append_eos_to_conditioning_tokens=True, reconstruct_wave=False, noise: Optional[NoiseStream] = None, **kwargs):
        clap_token_ids = _clap_ids(clap_token_ids, self.clap, conditioning_audio, conditioning_text)
        out = self._generate([clap_token_ids, semantic_token_ids], coarse_token_ids, noise, max_time_steps=max_time_steps,
                             filter_thres=filter_thres, temperature=temperature, include_eos_in_output=include_eos_in_output,
                             append_eos_to_conditioning_tokens=append_eos_to_conditioning_tokens, **kwargs)
        if reconstruct_wave:
            assert self.neural_codec is not None
            return self.neural_codec.decode_from_codebook_indices(out)[:, 0]
        return out

    def forward(self, *, clap_token_ids, semantic_token_ids, coarse_token_ids, return_loss=False, **kwargs):
        return self.transformer_wrapper.forward(all_token_ids=[clap_token_ids, semantic_token_ids, coarse_token_ids],
                                                return_loss=return_loss, **kwargs)


class FineStage(_Stage):
    """open_musiclm.py:719-814: clap + coarse tokens -> fine acoustic tokens."""

    def __init__(self, *, fine_transformer: TokenConditionedTransformer, clap=None, neural_codec=None, pad_id=-1,
                 unique_consecutive=False, cross_entropy_loss_weights: Optional[List[float]] = None, mask_prob=0.15, wrapper=None):
        super().__init__(fine_transformer, pad_id, unique_consecutive, cross_entropy_loss_weights, mask_prob, wrapper)
        self.clap, self.neural_codec = clap, neural_codec
        self.num_coarse_quantizers = self.transformer_wrapper.token_sequences[1].num_quantizers

    @torch.no_grad()
    def generate(self, *, coarse_token_ids, fine_token_ids=None, conditioning_text=None, conditioning_audio=None,
                 clap_token_ids=None, filter_thres=0.9, temperature=1., max_time_steps=3 * 600, include_eos_in_output=False,
                 append_eos_to_conditioning_tokens=True, reconstruct_wave=False, noise: Optional[NoiseStream] = None, **kwargs):
        clap_token_ids = _clap_ids(clap_token_ids, self.clap, conditioning_audio, conditioning_text)
        out = self._generate([clap_token_ids, coarse_token_ids], fine_token_ids, noise, max_time_steps=max_time_steps,
                             filter_thres=filter_thres, temperature=temperature, include_eos_in_output=include_eos_in_output,
                             append_eos_to_conditioning_tokens=append_eos_to_conditioning_tokens, **kwargs)
        if reconstruct_wave:
            assert self.neural_codec is not None
            return self.neural_codec.decode_from_codebook_indices(torch.cat([coarse_token_ids, out], -1))[:, 0]
        return out

    def forward(self, *, clap_token_ids, coarse_token_ids, fine_token_ids, return_loss=False, **kwargs):
        return self.transformer_wrapper.forward(all_token_ids=[clap_token_ids, coarse_token_ids, fine_token_ids],
                                                return_loss=return_loss, **kwargs)


def _windows(tokens: torch.Tensor, size: int, step: int):
    """[b, T, q] -> list of [b, size, q] windows at stride `step` (torch.unfold semantics: only complete windows)."""
    T = tokens.shape[1]
    return [tokens[:, s:s + size] for s in range(0, T - size + 1, step)]


class MusicLM(nn.Module):
    """open_musiclm.py:817-1035: text (clap tokens) -> semantic -> coarse -> fine token streams through sliding windows."""

    def __init__(self, *, semantic_transformer=None, coarse_transformer=None, fine_transformer=None, wav2vec=None, clap=None,
                 neural_codec=None, stages=None):
        super().__init__()
        if stages is not None:          # pre-built stages (tests plug oracle-backed wrappers in here)
            self.semantic, self.coarse, self.fine = stages
        else:
            st, ct, ft = semantic_transformer.token_sequences, coarse_transformer.token_sequences, fine_transformer.token_sequences
            assert st[1].codebook_size == ct[1].codebook_size
            assert ct[2].codebook_size == ft[2].codebook_size and ct[2].num_quantizers == ft[1].num_quantizers
            self.semantic = SemanticStage(semantic_transformer=semantic_transformer, wav2vec=wav2vec, clap=clap)
            self.coarse = CoarseStage(coarse_transformer=coarse_transformer, wav2vec=wav2vec, clap=clap, neural_codec=neural_codec)
            self.fine = FineStage(fine_transformer=fine_transformer, clap=clap, neural_codec=neural_codec)
        self.wav2vec, self.clap, self.neural_codec = wav2vec, clap, neural_codec

    @torch.no_grad()
    def generate_tokens(self, *, clap_token_ids, output_seconds=8, semantic_window_seconds=10, coarse_window_seconds=4,
                        fine_window_seconds=2, semantic_steps_per_second=50, acoustic_steps_per_second=75,
                        semantic_sliding_window_step_percent=0.5, coarse_sliding_window_step_percent=0.5,
                        fine_sliding_window_step_percent=1, noise: Optional[NoiseStream] = None, return_all=False, seeds=None):
        """The token-level body of MusicLM.forward (open_musiclm.py:925-1031, no audio prompt): returns the acoustic tokens
        [b, T, coarse + fine quantizers] the reference would hand to the codec (return_all: also the three streams).
        seeds (optional): one unsigned 64-bit seed per prompt (list of ints or int64 tensor).  Every generate call then gets
        the per-sequence seeds window_seed(seeds[b], stage, window index), so the whole song of prompt b is a function
        of (prompt b, seeds[b]), whatever else is in the batch.  Excludes noise."""
        if seeds is not None and noise is not None:
            raise ValueError("open_musiclm_b200 MusicLM.generate_tokens: seeds and noise exclude each other")
        if seeds is not None:
            seeds = seeds.reshape(-1).tolist() if isinstance(seeds, torch.Tensor) else [int(s) for s in seeds]
            if len(seeds) != clap_token_ids.shape[0]:
                raise ValueError(f"open_musiclm_b200 MusicLM.generate_tokens: {len(seeds)} seeds for {clap_token_ids.shape[0]} prompts")
        counter = {}

        def seeded(stage):             # the per-sequence seeds of this stage's next window (none when unseeded)
            if seeds is None:
                return {}
            w = counter.get(stage, 0)
            counter[stage] = w + 1
            return dict(seeds=[window_seed(s, stage, w) for s in seeds])

        sps, aps = semantic_steps_per_second, acoustic_steps_per_second
        common = dict(clap_token_ids=clap_token_ids, include_eos_in_output=False, append_eos_to_conditioning_tokens=True, noise=noise)
        # ---- semantic stream: first window from scratch, then windows conditioned on the tail of the stream (:930-949)
        sem = self.semantic.generate(semantic_token_ids=None, max_time_steps=int(min(output_seconds, semantic_window_seconds) * sps),
                                     **common, **seeded(SEMANTIC))
        keep = int(semantic_window_seconds * sps * (1 - semantic_sliding_window_step_percent))
        while sem.shape[1] < int(output_seconds * sps):
            nxt = self.semantic.generate(semantic_token_ids=sem[:, -keep:], max_time_steps=int(semantic_window_seconds * sps), **common,
                                         **seeded(SEMANTIC))
            sem = torch.cat([sem, nxt[:, keep:]], 1)
        # ---- coarse stream: one window of semantic tokens per generate, conditioned on the coarse tail (:956-985)
        win = int(coarse_window_seconds * sps - 1)
        coarse, keep = None, int(coarse_window_seconds * aps * (1 - coarse_sliding_window_step_percent))
        for sem_win in _windows(sem, win, int(win * coarse_sliding_window_step_percent)):
            pred = self.coarse.generate(semantic_token_ids=sem_win, coarse_token_ids=None if coarse is None else coarse[:, -keep:],
                                        max_time_steps=int(coarse_window_seconds * aps), temperature=0.95, **common, **seeded(COARSE))
            coarse = pred if coarse is None else torch.cat([coarse, pred[:, keep:]], 1)
        # ---- fine stream: one window of coarse tokens per generate (:995-1024)
        fwin = int(fine_window_seconds * aps)
        fine, keep = None, int(fwin * (1 - fine_sliding_window_step_percent))
        for coarse_win in _windows(coarse, fwin, int(fwin * fine_sliding_window_step_percent)):
            cond = fine[:, -keep:] if (fine is not None and keep > 0) else None
            pred = self.fine.generate(coarse_token_ids=coarse_win, fine_token_ids=cond, max_time_steps=fwin, temperature=0.4, **common,
                                      **seeded(FINE))
            fine = pred if fine is None else torch.cat([fine, pred[:, keep:]], 1)
        acoustic = torch.cat([coarse, fine], -1)                                                       # :1032
        return (acoustic, sem, coarse, fine) if return_all else acoustic

    @torch.no_grad()
    def forward(self, *, text: Optional[List[str]] = None, prime_wave=None, prime_wave_sample_hz=None, clap_token_ids=None, **kwargs):
        """open_musiclm.py:860-1035 without the audio-prompt branch: text -> waveform (needs the CLAP quantizer and the codec)."""
        if prime_wave is not None:
            raise NotImplementedError("open_musiclm_b200 MusicLM.forward: audio continuation (prime_wave) needs the wav2vec / codec "
                                      "tokenizers, which are outside the H100 hot path")
        clap_token_ids = _clap_ids(clap_token_ids, self.clap, None, text)
        acoustic = self.generate_tokens(clap_token_ids=clap_token_ids, **kwargs)
        assert self.neural_codec is not None, "a neural codec is needed to turn acoustic tokens into a waveform"
        return self.neural_codec.decode_from_codebook_indices(acoustic)[:, 0]
