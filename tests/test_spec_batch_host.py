"""Speculative decoding over several sequences, host side (no GPU): argument checks of cl_engine_set_speculate_batch and
cl_decode_verify_batch that need no engine, and the cl_spec_stats layout with multi_passes."""
import ctypes as C

import numpy as np

from crowdllama_b200 import engine as eng


def test_spec_stats_layout_with_multi_passes():
    st = eng.SpecStats
    assert C.sizeof(st) == 72                                   # unchanged: multi_passes took reserved[0]
    assert st.multi_passes.offset == 40 and st.reserved.offset == 48 and len(st().reserved) == 3
    assert st.tokens_emitted.offset == 32


def test_set_speculate_batch_and_verify_batch_refuse_a_null_engine():
    L = eng.lib()
    for n in (1, 4, 0, 33):
        assert L.cl_engine_set_speculate_batch(None, n) == eng.CL_ERR_INVALID_ARG
    seqs, x0, ks = np.zeros(2, np.int32), np.zeros(2, np.int32), np.zeros(2, np.int32)
    ids, n = np.zeros(2, np.int32), np.zeros(2, np.int32)
    p = eng._ptr
    assert L.cl_decode_verify_batch(None, p(seqs), 2, p(x0), None, p(ks), None, None, p(ids), p(n), None) == eng.CL_ERR_INVALID_ARG


def test_new_symbols_are_exported():
    for name in ("cl_engine_set_speculate_batch", "cl_decode_verify_batch"):
        assert name in eng.EXPORTS
        assert hasattr(eng.lib(), name)
