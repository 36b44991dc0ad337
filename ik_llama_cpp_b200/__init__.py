"""ik_llama_cpp_b200 — Hopper (sm_90a) quantized mat-mul hot path behind the ggml-backend boundary of ik_llama.cpp.

Product = ik_llama_cpp_b200/libb200q.so (CUDA, C ABI in include/b200q.h).  This Python package is the host-side
mirror of the reference operator interface used by tests and bench.py.
"""
from ._lib import B200QError, LIB_PATH, header_symbols, lib  # noqa: F401
