"""Stage wrappers and the three-stage windowed generation on top of the H100 TokenConditionedTransformer.

Mirrors the orchestration layer of the reference (open_musiclm/open_musiclm.py:514-1035): `SemanticStage`,
`CoarseStage`, `FineStage` (each a TokenConditionedTransformerWrapper plus the optional tokenizer objects) and
`MusicLM.forward`, which chains them through sliding windows: semantic tokens are grown window by window conditioned on
the tail of what exists, every coarse window is conditioned on a slice of the semantic stream plus the tail of the coarse
stream, every fine window on a slice of the coarse stream.  All arithmetic here is integer bookkeeping on token tensors;
the compute is `TokenConditionedTransformerWrapper.generate` (KV-cache decode, decode.py).

The tokenizers (CLAP-RVQ, MERT/HuBERT k-means, Encodec) are outside the hot path (SURVEY section 2): the stages accept
them as opaque callables exactly like the reference and never need them when token ids are passed in.  Audio
continuation (MusicLM.forward(prime_wave=...)) and best-of-N sampling (MusicLM.generate_top_match) call the caller's
wav2vec, codec and CLAP objects for the prime tokens and the similarity scores; the generation itself is the same
prefill + KV-cache decode, driven with the prime's tokens as the predicted sequence's prefix.
"""
from typing import List, Optional

import torch
import torch.nn.functional as F
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


# ---------------------------------------------------------------------------------------- audio helpers (utils.py:147-166)
def _resample(wave: torch.Tensor, orig_hz, new_hz) -> torch.Tensor:
    from torchaudio.functional import resample
    return resample(wave, orig_hz, new_hz)


def int16_to_float32(x: torch.Tensor) -> torch.Tensor:
    return (x / 32767.0).type(torch.float32)


def float32_to_int16(x: torch.Tensor) -> torch.Tensor:
    return (torch.clamp(x, min=-1., max=1.) * 32767.).type(torch.int16)


def zero_mean_unit_var_norm(x: torch.Tensor) -> torch.Tensor:
    return (x - x.mean(dim=-1, keepdim=True)) / torch.sqrt(x.var(dim=-1, keepdim=True) + 1e-7)


def prepare_audio(data: torch.Tensor, sample_hz, target_sample_hz, normalize=True, target_length_seconds=None) -> torch.Tensor:
    """A [channels, n] wave -> the [1, m] mono wave a tokenizer at target_sample_hz takes: the channel mean (more than
    one channel), optionally zero mean / unit variance, cropped to target_length_seconds, resampled, then rounded
    through int16 as a file would store it."""
    if data.shape[0] > 1:
        data = data.mean(dim=0, keepdim=True)
    if normalize:
        data = zero_mean_unit_var_norm(data)
    if target_length_seconds is not None and data.shape[1] > target_length_seconds * sample_hz:
        data = data[:, :int(target_length_seconds * sample_hz)]
    return int16_to_float32(float32_to_int16(_resample(data, sample_hz, target_sample_hz)))


def _prime(t: torch.Tensor, b: int, q: int, device, what: str) -> torch.Tensor:
    """Prime tokens [1 or b, T, q] ([1 or b, T] for the semantic stream) -> [b, T, q] int64 on `device`."""
    if t.dim() == 2 and q == 1:
        t = t.unsqueeze(-1)
    if t.dim() != 3 or t.shape[-1] != q or t.shape[0] not in (1, b):
        raise ValueError(f"open_musiclm_b200 MusicLM.generate_tokens: {what} must be [1 or {b}, T, {q}], got {tuple(t.shape)}")
    return t.to(device, torch.int64).expand(b, -1, -1).contiguous()


class MusicLM(nn.Module):
    """open_musiclm.py:817-1071: text (clap tokens), optionally continuing a prime wave -> semantic -> coarse -> fine token
    streams through sliding windows; best-of-N sampling scored by CLAP (generate_top_match)."""

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
                        fine_sliding_window_step_percent=1, noise: Optional[NoiseStream] = None, return_all=False, seeds=None,
                        prime_semantic_token_ids=None, prime_coarse_token_ids=None, prime_fine_token_ids=None, coarse_only=False):
        """The token-level body of MusicLM.forward (open_musiclm.py:913-1032): returns the acoustic tokens
        [b, T, coarse + fine quantizers] the reference would hand to the codec (return_all: also the three streams).
        seeds (optional): one unsigned 64-bit seed per prompt (list of ints or int64 tensor).  Every generate call then gets
        the per-sequence seeds window_seed(seeds[b], stage, window index), so the whole song of prompt b is a function
        of (prompt b, prime, seeds[b]), whatever else is in the batch.  Excludes noise.
        prime_{semantic,coarse,fine}_token_ids (audio continuation, all three or none): the tokens of a prime wave,
        [1 or b, Ts, 1], [1 or b, Ta, coarse quantizers], [1 or b, Ta, fine quantizers].  The first window of every
        stage is conditioned on the prime's tail, the streams are cropped so that the stages line up, and the full
        prime acoustic streams come first in the output.  A prime with batch 1 is used for all b prompts, one with
        batch b row by row (the reference tokenizes a single prime wave and so continues a single prompt).  With a fine
        condition length > 0 (fine_sliding_window_step_percent < 1) the reference's streams cannot be joined; here the
        coarse stream drops the prime tokens the first fine window was conditioned on, so both start after the prime.
        coarse_only: stop after the coarse stage and return its stream [b, T, coarse quantizers] as it stands before
        the crop that lines it up with the fine windows (forward's return_coarse_generated_wave)."""
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
        primes = (prime_semantic_token_ids, prime_coarse_token_ids, prime_fine_token_ids)
        primed = prime_semantic_token_ids is not None
        if any((p is not None) != primed for p in primes):
            raise ValueError("open_musiclm_b200 MusicLM.generate_tokens: pass all three prime token streams or none")
        # ---- audio continuation: condition lengths, the prime's tails and the crops that line the stages up (:913-926)
        sem_prime = coarse_prime = fine_prime = None
        sem_adj = coarse_adj = fine_adj = 0
        if primed:
            B = clap_token_ids.shape[0]
            qc = self.coarse.num_coarse_quantizers
            qf = self.fine.transformer_wrapper.token_sequences[-1].num_quantizers
            prime_sem = _prime(prime_semantic_token_ids, B, 1, self.semantic.device, "prime_semantic_token_ids")
            prime_coarse = _prime(prime_coarse_token_ids, B, qc, self.coarse.device, "prime_coarse_token_ids")
            prime_fine = _prime(prime_fine_token_ids, B, qf, self.fine.device, "prime_fine_token_ids")
            cond_sem = int(sps * semantic_window_seconds * (1 - semantic_sliding_window_step_percent))
            cond_coarse = int(aps * coarse_window_seconds * (1 - coarse_sliding_window_step_percent))
            cond_fine = int(aps * fine_window_seconds * (1 - fine_sliding_window_step_percent))
            sem_prime = prime_sem[:, -cond_sem:] if prime_sem.shape[1] >= cond_sem else prime_sem
            coarse_prime = prime_coarse[:, -cond_coarse:]
            fine_prime = prime_fine[:, -cond_fine:] if cond_fine > 0 else None
            sem_adj = cond_sem - int(sps * coarse_window_seconds * (1 - coarse_sliding_window_step_percent))
            coarse_adj = cond_coarse - int(aps * fine_window_seconds * (1 - fine_sliding_window_step_percent))
            fine_adj = cond_fine
        common = dict(clap_token_ids=clap_token_ids, include_eos_in_output=False, append_eos_to_conditioning_tokens=True, noise=noise)
        # ---- semantic stream: first window from the prime's tail (or scratch), then windows conditioned on the tail of
        # the stream (:930-949); cropped to line up with the coarse windows (:952)
        sem = self.semantic.generate(semantic_token_ids=sem_prime, max_time_steps=int(min(output_seconds, semantic_window_seconds) * sps),
                                     **common, **seeded(SEMANTIC))
        keep = int(semantic_window_seconds * sps * (1 - semantic_sliding_window_step_percent))
        while sem.shape[1] < int(output_seconds * sps):
            nxt = self.semantic.generate(semantic_token_ids=sem[:, -keep:], max_time_steps=int(semantic_window_seconds * sps), **common,
                                         **seeded(SEMANTIC))
            sem = torch.cat([sem, nxt[:, keep:]], 1)
        sem = sem[:, sem_adj:]
        # ---- coarse stream: one window of semantic tokens per generate, conditioned on the coarse tail, the first one
        # on the prime's (:956-985)
        win = int(coarse_window_seconds * sps - 1)
        coarse, keep = None, int(coarse_window_seconds * aps * (1 - coarse_sliding_window_step_percent))
        for sem_win in _windows(sem, win, int(win * coarse_sliding_window_step_percent)):
            pred = self.coarse.generate(semantic_token_ids=sem_win, coarse_token_ids=coarse_prime if coarse is None else coarse[:, -keep:],
                                        max_time_steps=int(coarse_window_seconds * aps), temperature=0.95, **common, **seeded(COARSE))
            coarse = pred if coarse is None else torch.cat([coarse, pred[:, keep:]], 1)
        if coarse_only:                                                                                 # :986-989
            return coarse
        coarse = coarse[:, coarse_adj:]                                                                 # :992
        # ---- fine stream: one window of coarse tokens per generate, the first one conditioned on the prime's tail (:995-1024)
        fwin = int(fine_window_seconds * aps)
        fine, keep = None, int(fwin * (1 - fine_sliding_window_step_percent))
        for coarse_win in _windows(coarse, fwin, int(fwin * fine_sliding_window_step_percent)):
            cond = fine_prime if fine is None else (fine[:, -keep:] if keep > 0 else None)
            pred = self.fine.generate(coarse_token_ids=coarse_win, fine_token_ids=cond, max_time_steps=fwin, temperature=0.4, **common,
                                      **seeded(FINE))
            fine = pred if fine is None else torch.cat([fine, pred[:, keep:]], 1)
        fine = fine[:, fine_adj:]                                                                       # :1026
        # the coarse stream still starts with the fine_adj prime tokens the first fine window was conditioned on; the
        # reference keeps them, so with a fine condition length > 0 its coarse and fine streams differ in length and
        # cannot be joined.  Dropping them lines both up on the first token after the prime (no-op when fine_adj = 0).
        coarse = coarse[:, fine_adj:]
        if primed:                                                                                      # :1028-1030
            fine, coarse = torch.cat([prime_fine, fine], 1), torch.cat([prime_coarse, coarse], 1)
        acoustic = torch.cat([coarse, fine], -1)                                                       # :1032
        return (acoustic, sem, coarse, fine) if return_all else acoustic

    def prime_token_ids(self, prime_wave: torch.Tensor, prime_wave_sample_hz, semantic_window_seconds=10):
        """A [channels, n] prime wave -> the prime_{semantic,coarse,fine}_token_ids of generate_tokens (batch 1), through
        the caller's wav2vec (semantic ids at wav2vec.target_sample_hz, normalised wave) and codec (acoustic ids at
        neural_codec.sample_rate, wave as it is), each fed the first semantic_window_seconds (open_musiclm.py:897-912)."""
        if self.wav2vec is None or self.neural_codec is None:
            raise ValueError("open_musiclm_b200 MusicLM: audio continuation (prime_wave) needs the wav2vec and neural_codec "
                             "tokenizers; pass them to MusicLM(wav2vec=..., neural_codec=...)")
        if prime_wave_sample_hz is None:
            raise ValueError("open_musiclm_b200 MusicLM: prime_wave needs prime_wave_sample_hz")
        wave_sem = prepare_audio(prime_wave, prime_wave_sample_hz, self.wav2vec.target_sample_hz, normalize=True,
                                 target_length_seconds=semantic_window_seconds)
        wave_codec = prepare_audio(prime_wave, prime_wave_sample_hz, self.neural_codec.sample_rate, normalize=False,
                                   target_length_seconds=semantic_window_seconds)
        sem = self.wav2vec(wave_sem, flatten=False)                                                     # :489-495
        if isinstance(self.neural_codec, nn.Module):
            self.neural_codec.eval()
        indices = self.neural_codec(wave_codec, return_encoded=True)[1]                                 # :499-510
        qc = self.coarse.num_coarse_quantizers
        return dict(prime_semantic_token_ids=sem.reshape(sem.shape[0], -1, 1), prime_coarse_token_ids=indices[..., :qc],
                    prime_fine_token_ids=indices[..., qc:])

    @torch.no_grad()
    def forward(self, *, text: Optional[List[str]] = None, prime_wave=None, prime_wave_sample_hz=None, clap_token_ids=None,
                semantic_window_seconds=10, return_coarse_generated_wave=False, **kwargs):
        """open_musiclm.py:860-1035: text (or clap token ids) -> waveform [b, n] through the codec.  prime_wave ([channels, n]
        at prime_wave_sample_hz): continue that audio (prime_token_ids, then generate_tokens); it needs the wav2vec and
        the codec.  return_coarse_generated_wave: decode the coarse stream alone, before its crop (generate_tokens'
        coarse_only).  Every other keyword goes to generate_tokens."""
        clap_token_ids = _clap_ids(clap_token_ids, self.clap, None, text)
        if prime_wave is not None:
            kwargs.update(self.prime_token_ids(prime_wave, prime_wave_sample_hz, semantic_window_seconds))
        tokens = self.generate_tokens(clap_token_ids=clap_token_ids, semantic_window_seconds=semantic_window_seconds,
                                      coarse_only=return_coarse_generated_wave, **kwargs)
        assert self.neural_codec is not None, "a neural codec is needed to turn acoustic tokens into a waveform"
        return self.neural_codec.decode_from_codebook_indices(tokens)[:, 0]

    @torch.no_grad()
    def generate_top_match(self, *, text: List[str], num_samples=4, num_top_matches=1, **kwargs):
        """open_musiclm.py:1039-1071: for every prompt, num_samples songs in one batch (forward(**kwargs)), scored by the
        cosine similarity of the caller's CLAP embeddings of the prompt and of each song (resampled from
        neural_codec.sample_rate to clap.sample_rate and rounded through int16).  Returns, per prompt, the
        num_top_matches best waves [num_top_matches, n] and their similarities (on the CPU), best first.  seeds, if
        given, holds one seed per sample and is used for every prompt."""
        if self.clap is None or self.neural_codec is None:
            raise ValueError("open_musiclm_b200 MusicLM.generate_top_match needs the clap and neural_codec models")
        all_samples, all_similarities = [], []
        for prompt in text:
            samples = self.forward(text=[prompt] * num_samples, **kwargs)
            text_latents = self.clap(text_input=[prompt], return_embedding=True).repeat(num_samples, 1)
            clap_input = int16_to_float32(float32_to_int16(_resample(samples, self.neural_codec.sample_rate, self.clap.sample_rate)))
            audio_latents = self.clap(audio_input=clap_input, return_embedding=True)
            sim = F.cosine_similarity(text_latents.to(audio_latents.device), audio_latents, dim=-1)
            top = sim.topk(num_top_matches, dim=0, sorted=True).indices
            all_similarities.append(sim[top].detach().cpu())
            all_samples.append(samples[top])
        return all_samples, all_similarities
