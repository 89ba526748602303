"""multiply_b200 — H100-native (sm_90a) implementation of MultiPly's volume-rendering hot path."""
__version__ = "0.1.0"
