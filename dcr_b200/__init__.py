"""dcr_b200 -- H100-native (sm_90a) engine for DCR's embed -> match -> top-k (+FID) hot path.

Python host code mirrors the reference's call surface (diff_retrieval.py / embedding_search / metrics.fid) and
calls libdcr_b200.so (hand-written CUDA) through ctypes.  See DESIGN.md / INTEGRATION.md.
"""
__version__ = "0.1.0"
