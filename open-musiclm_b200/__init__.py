"""open-musiclm hot path, H100-native (sm_90a): package root.

Only what the TokenConditionedTransformer training path needs lives here:
  csrc/       hand-written CUDA kernels + the C ABI (libomlm_b200.so)
  lib.py      ctypes binding of that ABI (no fallback)
  engine.py   parameter arena, packed weights, kernel sequencing (forward / backward)
  model.py    drop-in `TokenConditionedTransformer`, `create_{semantic,coarse,fine}_transformer`
  trainer.py  H100-native SingleStageTrainer step loop (`HotPathTrainer`)
  decode.py   `TokenConditionedTransformerWrapper.generate`: KV-cache autoregressive decoding
  stages.py   `SemanticStage` / `CoarseStage` / `FineStage` and the windowed three-stage `MusicLM` generation
"""
__version__ = "0.1.0"

from .model import (TokenConditionedTransformer, TokenSequenceInfo, create_coarse_transformer,  # noqa: F401
                    create_fine_transformer, create_semantic_transformer)
from .trainer import HotPathTrainer  # noqa: F401
from .decode import TokenConditionedTransformerWrapper  # noqa: F401
from .stages import CoarseStage, FineStage, MusicLM, NoiseStream, SemanticStage, prepare_audio  # noqa: F401
