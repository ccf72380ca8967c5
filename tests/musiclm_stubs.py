"""Stand-ins for the models MusicLM calls around generation (a wav2vec semantic tokenizer, a neural codec, a CLAP
quantizer), shared by oracle/make_golden_musiclm_prime.py and the tests.  They ignore the audio they tokenize and
return fixed ids, so that a fixture recorded with them pins the token bookkeeping of audio continuation and of
best-of-N sampling; every wave handed to them is kept in `.seen` so a test can check what the caller prepared."""
import zlib

import torch
import torch.nn.functional as F
from torch import nn


class Wav2Vec:
    """Semantic tokenizer: returns `ids` ([b, Ts], as the k-means tokenizer does with flatten=False)."""

    def __init__(self, ids: torch.Tensor, target_sample_hz: int, codebook_size: int = 64):
        self.ids, self.target_sample_hz, self.codebook_size, self.seen = ids, target_sample_hz, codebook_size, []

    def __call__(self, wave, flatten=True):
        assert not flatten
        self.seen.append(wave.detach().cpu().clone())
        return self.ids.clone().to(wave.device)


class Codec(nn.Module):
    """Neural codec: encoding returns (None, `ids` [b, Ta, q], None); decoding returns the ids themselves as a
    [b, 1, T * q] float "wave"."""

    def __init__(self, ids: torch.Tensor, sample_rate: int):
        super().__init__()
        self.ids, self.sample_rate, self.seen = ids, sample_rate, []

    def forward(self, wave, return_encoded=True):
        assert return_encoded
        self.seen.append(wave.detach().cpu().clone())
        return None, self.ids.clone().to(wave.device), None

    def decode_from_codebook_indices(self, ids):
        return ids.reshape(ids.shape[0], 1, -1).float()


def _prompt_generator(prompt: str) -> torch.Generator:
    return torch.Generator().manual_seed(zlib.crc32(prompt.encode()))


class Clap:
    """CLAP quantizer: the token ids and the embedding of a text are drawn from a generator seeded by the text; the
    embedding of audio [b, n] is `proj` applied to its average over `proj.shape[0]` equal time bins."""

    def __init__(self, codebook_size: int, num_quantizers: int, proj: torch.Tensor, sample_rate: int):
        self.codebook_size, self.num_quantizers, self.proj, self.sample_rate = codebook_size, num_quantizers, proj, sample_rate
        self.seen = []

    def text_ids(self, prompt: str) -> torch.Tensor:
        return torch.randint(0, self.codebook_size, (self.num_quantizers,), generator=_prompt_generator(prompt))

    def text_embedding(self, prompt: str) -> torch.Tensor:
        g = _prompt_generator(prompt)
        torch.randint(0, self.codebook_size, (self.num_quantizers,), generator=g)
        return torch.randn(self.proj.shape[1], generator=g)

    def __call__(self, text_input=None, audio_input=None, return_embedding=False):
        if text_input is not None:
            f = self.text_embedding if return_embedding else self.text_ids
            return torch.stack([f(t) for t in text_input])
        assert return_embedding, "the stub CLAP embeds audio, it does not tokenize it"
        self.seen.append(audio_input.detach().cpu().clone())
        pooled = F.adaptive_avg_pool1d(audio_input.float()[:, None], self.proj.shape[0])[:, 0]
        return pooled @ self.proj.to(pooled.device)
