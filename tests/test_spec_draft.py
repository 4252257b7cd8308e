"""Speculative decoding, host side (no GPU): the prompt-lookup drafter cl_draft_ngram against a statement of its rule,
and the config field that switches speculation on."""
import ctypes as C
import random

import numpy as np
import pytest

from crowdllama_b200 import engine as eng


def draft_rule(hist, k):
    """The longest suffix of length 3, else 2, that also occurs earlier; the up to k ids after its most recent earlier
    occurrence, cut at the end of hist."""
    n = len(hist)
    for g in (3, 2):
        if n < g + 1:
            continue
        suffix = hist[n - g:]
        for i in range(n - g - 1, -1, -1):
            if hist[i:i + g] == suffix:
                return hist[i + g:i + g + k]
    return []


@pytest.mark.parametrize("k", range(1, 16))
def test_draft_matches_the_rule_on_random_and_repetitive_ids(k):
    rng = random.Random(k)
    for trial in range(200):
        n = rng.randrange(0, 80)
        vocab = rng.choice([2, 3, 5, 50, 128256])
        hist = [rng.randrange(vocab) for _ in range(n)]
        if trial % 3 == 0 and n > 8:            # a repeated run, then its start again
            a = rng.randrange(0, n // 2)
            hist = hist + hist[a:a + rng.randrange(2, 12)]
        got = eng.draft_ngram(hist, k).tolist()
        assert got == draft_rule(hist, k), (hist, k)


def test_draft_cases():
    # most recent earlier occurrence wins
    assert eng.draft_ngram([1, 2, 3, 10, 11, 1, 2, 3, 20, 21, 1, 2, 3], 2).tolist() == [20, 21]
    # a trigram match is preferred over a more recent bigram match
    assert eng.draft_ngram([7, 1, 2, 30, 9, 9, 1, 2, 40, 7, 1, 2], 1).tolist() == [30]
    # bigram fallback when the trigram never occurred before
    assert eng.draft_ngram([5, 1, 2, 40, 6, 1, 2], 3).tolist() == [40, 6, 1]
    # overlapping occurrence: a constant run drafts more of itself
    assert eng.draft_ngram([4, 4, 4, 4], 15).tolist() == [4]
    assert eng.draft_ngram([1, 2, 1, 2, 1], 5).tolist() == [2, 1]
    # the continuation stops at the end of the history
    assert eng.draft_ngram([1, 2, 3, 8, 1, 2, 3], 15).tolist() == [8, 1, 2, 3]
    # no match, too short
    assert eng.draft_ngram([1, 2, 3, 4, 5, 6], 4).size == 0
    assert eng.draft_ngram([1, 1], 4).size == 0
    assert eng.draft_ngram([], 4).size == 0


def test_draft_rejects_bad_k():
    for k in (0, 16):
        with pytest.raises(eng.EngineError) as ei:
            eng.draft_ngram([1, 2, 1, 2], k)
        assert ei.value.status == eng.CL_ERR_INVALID_ARG


def test_config_default_and_layout():
    cfg = eng.EngineConfig()
    eng.lib().cl_default_engine_config(C.byref(cfg))
    assert cfg.speculate == 0
    assert list(cfg.reserved) == [0] * 6
    # the field comes out of `reserved`: the struct keeps its size and every other offset (ABI version 2)
    assert C.sizeof(eng.EngineConfig) == EngineConfigV2.size()
    for name, _ in EngineConfigV2._fields_:
        if name != "reserved":
            assert getattr(eng.EngineConfig, name).offset == getattr(EngineConfigV2, name).offset, name
    assert eng.EngineConfig.speculate.offset == EngineConfigV2.reserved.offset
    assert eng.lib().cl_abi_version() == 2


class EngineConfigV2(C.Structure):
    """cl_engine_config as ABI version 2 first declared it, with reserved[7]."""
    _fields_ = [("abi_version", C.c_int32), ("device", C.c_int32), ("model_name", C.c_char_p), ("preset", C.c_char_p),
                ("model", eng.ModelConfig), ("weights_path", C.c_char_p), ("weights_seed", C.c_uint64),
                ("kv_pool_bytes", C.c_int64), ("page_size", C.c_int32), ("max_batch", C.c_int32),
                ("max_seqs", C.c_int32), ("use_cuda_graph", C.c_int32), ("decode_path", C.c_int32),
                ("start_scheduler", C.c_int32), ("prefix_cache", C.c_int32), ("reserved", C.c_int32 * 7)]

    @classmethod
    def size(cls):
        return C.sizeof(cls)


def test_spec_stats_struct_layout():
    assert C.sizeof(eng.SpecStats) == 4 + 4 + 8 * 4 + 8 * 4
    assert np.dtype(np.int64).itemsize == 8
