"""kakveda_b200 -- H100-native engine for Kakveda's GFKB fingerprint-match path.

Scope: the one data-parallel hot path of prateekdevisingh/kakveda -- the scan of incoming trace
fingerprints against the Global Failure Knowledge Base (``SimilarityEngine.score``,
services/shared/similarity.py:14-20, as called by services/gfkb/app.py:86) -- as hand-written
sm_90a CUDA behind a C ABI (include/kakveda_b200.h).  See DESIGN.md.
"""
from .fingerprint import fingerprint_text, fingerprint_u64, normalize_prompt, signature_text
from .denseindex import DenseIndex
from .hashindex import HashIndex
from .jaccardindex import JaccardIndex
from .similarity import FeatureBatch, GfkbIndex, SimilarityEngine, Vocabulary
from .store import GfkbStore
from . import patterns

__all__ = [
    "SimilarityEngine", "GfkbIndex", "Vocabulary", "FeatureBatch", "HashIndex", "DenseIndex", "JaccardIndex",
    "GfkbStore", "patterns", "signature_text", "fingerprint_text", "fingerprint_u64", "normalize_prompt",
]
__version__ = "0.1.0"
