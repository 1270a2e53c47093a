"""parseable_b200 — H100-native columnar query hot path for Parseable.

The product is ``libparseable_b200.so`` (hand-written sm_90a CUDA behind the C
ABI in include/parseable_b200.h).  This package only binds it (``_lib``),
mirrors the reference's query surface on top of it (``query``) and generates the
synthetic log tables the tests and the bench use (``synth``).
"""
__version__ = "0.1.0"
