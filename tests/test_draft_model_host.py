"""Draft-model speculative decoding, host side: the new C-ABI symbols, the refusals that need no device, the Python and
worker plumbing, and the cl_spec_stats layout."""
import ctypes as C

import pytest

from crowdllama_b200 import engine as eng
from crowdllama_b200 import worker


@pytest.fixture(autouse=True)
def _no_env_override(monkeypatch):
    for k in ("CL_SPECULATE", "CL_DRAFT_MODEL", "CL_DRAFT_SEED", "CL_CONTEXT_LENGTH"):
        monkeypatch.delenv(k, raising=False)


def _target(preset="llama3-8b", speculate=3):
    cfg = eng.EngineConfig()
    eng.lib().cl_default_engine_config(C.byref(cfg))
    cfg.preset = preset.encode()
    cfg.speculate = speculate
    return cfg


def _create(cfg, draft):
    h = C.c_void_p()
    rc = eng.lib().cl_engine_create_with_draft(C.byref(cfg), C.byref(draft) if draft is not None else None, C.byref(h))
    return rc, eng.lib().cl_last_error().decode()


def test_symbols_are_exported():
    L = eng.lib()
    for s in ("cl_engine_create_with_draft", "cl_draft_model"):
        assert s in eng.EXPORTS and hasattr(L, s)


def test_create_with_draft_needs_a_device():
    if eng.device_count() > 0:
        pytest.skip("GPU present")
    keep = []
    rc, _ = _create(_target(), eng.draft_engine_config("llama3.2-1b", None, None, 1, keep))
    assert rc == eng.CL_ERR_NO_DEVICE


def test_refusals_before_the_device():
    keep = []
    rc, err = _create(_target(), eng.draft_engine_config("tiny-test", None, None, 1, keep))
    assert rc == eng.CL_ERR_INVALID_ARG and "vocabulary" in err
    rc, err = _create(_target(speculate=0), eng.draft_engine_config("llama3.2-1b", None, None, 1, keep))
    assert rc == eng.CL_ERR_INVALID_ARG and "speculate" in err
    rc, _ = _create(_target(), eng.draft_engine_config("no-such-model", None, None, 1, keep))
    assert rc == eng.CL_ERR_UNKNOWN_MODEL


def test_env_switch_reaches_plain_create(monkeypatch):
    h = C.c_void_p()
    monkeypatch.setenv("CL_DRAFT_MODEL", "tiny-test")
    assert eng.lib().cl_engine_create(C.byref(_target()), C.byref(h)) == eng.CL_ERR_INVALID_ARG
    assert "vocabulary" in eng.lib().cl_last_error().decode()
    monkeypatch.setenv("CL_DRAFT_MODEL", "llama3.2-1b")
    monkeypatch.setenv("CL_DRAFT_SEED", "x")   # not a number: strtoull takes 0; still a draft, refused for speculate 0
    assert eng.lib().cl_engine_create(C.byref(_target(speculate=0)), C.byref(h)) == eng.CL_ERR_INVALID_ARG
    assert "speculate" in eng.lib().cl_last_error().decode()


def test_draft_model_without_an_engine():
    assert eng.lib().cl_draft_model(None, None, 0, None, None, None, None, None, None, None) == eng.CL_ERR_INVALID_ARG


def test_python_draft_config():
    keep = []
    assert eng.draft_engine_config(None, None, None, 5, keep) is None
    d = eng.draft_engine_config("llama3.2-1b", None, None, 5, keep)
    assert d.preset == b"llama3.2-1b" and d.weights_seed == 5 and d.weights_path is None
    d = eng.draft_engine_config(None, dict(n_layers=1, d_model=256, n_heads=4, n_kv_heads=2, head_dim=64, d_ff=512,
                                           vocab_size=512, max_seq_len=512, rope_theta=1e4, rms_eps=1e-5), "/x", 9, keep)
    assert d.preset is None and d.model.n_layers == 1 and d.weights_path == b"/x" and d.weights_seed == 9


def test_worker_draft_arguments(tmp_path):
    assert worker.draft_kwargs(None, 3) == {}
    assert worker.draft_kwargs("llama3.2-1b", None) == dict(draft_preset="llama3.2-1b")
    assert worker.draft_kwargs("llama3.2-1b", 7) == dict(draft_preset="llama3.2-1b", draft_seed=7)
    assert worker.draft_kwargs(str(tmp_path), None) == dict(draft_weights_path=str(tmp_path))


def test_spec_stats_layout_is_unchanged():
    st = eng.SpecStats
    assert C.sizeof(st) == 72 and st.reserved.offset == 48   # draft_rows, draft_ns, draft_pages_used took reserved[0..2]
