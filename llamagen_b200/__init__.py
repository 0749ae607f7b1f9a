"""llamagen_b200 — H100-native (sm_90a) drop-in for LlamaGen's sampling hot path.

Public surface mirrors the reference modules on the path (SURVEY §8b):
    GPT_models, generate          <- autoregressive/models/gpt.py, autoregressive/models/generate.py
    VQ_models                     <- tokenizer/tokenizer_image/vq_model.py
All compute runs in hand-written CUDA behind the C-ABI library (include/llamagen_b200.h); importing the
package on a CPU-only machine works (for the registries / ABI tests) but any compute call fails loudly.
"""
from .gpt import GPT_models, ModelArgs, Transformer            # noqa: F401
from .generate import generate, sample                         # noqa: F401
from .vq_model import VQ_models, VQModel                       # noqa: F401
from ._lib import LgError                                      # noqa: F401

__all__ = ["GPT_models", "VQ_models", "generate", "sample", "Transformer", "VQModel", "ModelArgs", "LgError"]
