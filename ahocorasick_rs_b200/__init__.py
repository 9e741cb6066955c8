"""H100-native multi-pattern matcher with the ``ahocorasick_rs`` Python API.

Mirrors the reference's pysrc/ahocorasick_rs/__init__.py:1-23 (same exported
names, including the deprecated MATCHKIND_* constants); the scan runs in
hand-written sm_90a CUDA kernels behind the C ABI in include/acb200.h."""
from .matcher import AhoCorasick, BytesAhoCorasick, TokenAhoCorasick, TokenVocabulary, MatchKind, Implementation

# Backwards compatibility (reference: pysrc/ahocorasick_rs/__init__.py:10-12)
MATCHKIND_STANDARD = MatchKind.Standard
MATCHKIND_LEFTMOST_FIRST = MatchKind.LeftmostFirst
MATCHKIND_LEFTMOST_LONGEST = MatchKind.LeftmostLongest

__all__ = [
    "AhoCorasick",
    "BytesAhoCorasick",
    "TokenAhoCorasick",
    "TokenVocabulary",
    "MatchKind",
    "Implementation",
    "MATCHKIND_STANDARD",
    "MATCHKIND_LEFTMOST_FIRST",
    "MATCHKIND_LEFTMOST_LONGEST",
]
