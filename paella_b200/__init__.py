"""paella_b200 — H100-native (sm_90a) implementation of Paella's sampling hot path.

Python mirror of the reference's class surface (``Paella``, ``sample``, ``VQModel`` ...) over the
C ABI in ``include/paella_b200.h`` (``libpaella_b200.so``, hand-written CUDA).  No CPU fallback.
"""
__version__ = "0.1.0"
