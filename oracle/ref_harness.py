"""ORACLE — test infrastructure only.

Imports the REAL reference (`$OMLM_REFERENCE_ROOT/open_musiclm`, a checkout of zhvng/open-musiclm) with the two stub modules SURVEY.md §8c
describes, so that its TokenConditionedTransformer / Wrapper / Stage classes run on CPU.  Only
usable where that checkout exists; the tests compare against golden data recorded from it (tests/golden/).
"""
import os
import sys
import types

REF_ROOT = os.environ.get("OMLM_REFERENCE_ROOT", "")


def available() -> bool:
    return bool(REF_ROOT) and os.path.isdir(os.path.join(REF_ROOT, "open_musiclm"))


def import_reference():
    """Returns the module `open_musiclm.open_musiclm` of the reference."""
    if not available():
        raise RuntimeError(f"reference tree not found at {REF_ROOT}")
    if "open_musiclm.open_musiclm" in sys.modules:
        return sys.modules["open_musiclm.open_musiclm"]
    os.environ.pop("USE_BEARTYPE", None)
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    # package shell without running open_musiclm/__init__.py (it imports config -> trainer -> accelerate)
    pkg = types.ModuleType("open_musiclm")
    pkg.__path__ = [os.path.join(REF_ROOT, "open_musiclm")]
    sys.modules["open_musiclm"] = pkg
    cq = types.ModuleType("open_musiclm.clap_quantized")
    cq.ClapQuantized = type("ClapQuantized", (), {})
    mt = types.ModuleType("open_musiclm.model_types")
    mt.NeuralCodec = type("NeuralCodec", (), {})
    mt.Wav2Vec = type("Wav2Vec", (), {})
    sys.modules["open_musiclm.clap_quantized"] = cq
    sys.modules["open_musiclm.model_types"] = mt
    import importlib
    return importlib.import_module("open_musiclm.open_musiclm")
