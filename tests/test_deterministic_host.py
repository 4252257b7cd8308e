"""Deterministic mode, host side (no GPU): the config field's layout, the refusals cl_engine_create makes before it touches
a device, the env / Python / worker plumbing, and the split-K plan that does not depend on the card's SM count."""
import ctypes as C
import shutil
import subprocess
import sys
from pathlib import Path

import pytest

from crowdllama_b200 import engine as eng
from crowdllama_b200 import worker

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(autouse=True)
def _no_env(monkeypatch):
    for k in ("CL_DETERMINISTIC", "CL_SPECULATE", "CL_DRAFT_MODEL", "CL_CONTEXT_LENGTH"):
        monkeypatch.delenv(k, raising=False)


def _create(preset="llama3-8b", deterministic=1, page_size=32, max_batch=8):
    cfg = eng.EngineConfig()
    eng.lib().cl_default_engine_config(C.byref(cfg))
    cfg.preset = preset.encode()
    cfg.page_size = page_size
    cfg.max_batch = max_batch
    cfg.reserved[3] = deterministic
    h = C.c_void_p()
    rc = eng.lib().cl_engine_create(C.byref(cfg), C.byref(h))
    if rc == eng.CL_OK:
        eng.lib().cl_engine_destroy(h)
    return rc, eng.lib().cl_last_error().decode()


def test_config_layout(tmp_path):
    """deterministic sits where the ctypes struct's reserved[3] does, and the struct keeps its size"""
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "clengine.h"\n'
                   'int main(void) {\n'
                   '  printf("%zu %zu %d", sizeof(cl_engine_config), offsetof(cl_engine_config, deterministic), CL_ABI_VERSION); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True, capture_output=True)
    size, off, abi = map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split())
    assert C.sizeof(eng.EngineConfig) == size and abi == 2
    assert eng.EngineConfig.reserved.offset + 3 * 4 == off
    cfg = eng.EngineConfig()
    eng.lib().cl_default_engine_config(C.byref(cfg))
    assert cfg.reserved[3] == 0   # off by default


@pytest.mark.parametrize("preset,page,max_batch", [("tiny-test", 32, 8), ("llama3.2-1b", 32, 8), ("tinyllama-1.1b", 32, 8),
                                                   ("llama3-8b", 16, 8), ("llama3-8b", 64, 8), ("llama3-8b", 32, 129)])
def test_refusals(preset, page, max_batch):
    rc, err = _create(preset, 1, page, max_batch)
    assert rc == eng.CL_ERR_INVALID_ARG and "deterministic" in err


def test_accepted_shapes_reach_the_device():
    if eng.device_count() > 0:
        pytest.skip("GPU present")
    for preset in ("llama3-8b", "mistral-7b"):
        assert _create(preset)[0] == eng.CL_ERR_NO_DEVICE
    assert _create("llama3-8b", max_batch=128)[0] == eng.CL_ERR_NO_DEVICE


def test_env_overrides_the_field(monkeypatch):
    monkeypatch.setenv("CL_DETERMINISTIC", "1")
    assert _create("tiny-test", deterministic=0)[0] == eng.CL_ERR_INVALID_ARG
    monkeypatch.setenv("CL_DETERMINISTIC", "0")
    assert _create("tiny-test", deterministic=1)[0] != eng.CL_ERR_INVALID_ARG


def _captured_config(monkeypatch, **kw):
    """the cl_engine_config eng.Engine(**kw) hands to cl_engine_create"""
    seen = {}

    class Stop(Exception):
        pass

    def create(cfg, h):
        seen["cfg"] = C.cast(cfg, C.POINTER(eng.EngineConfig)).contents
        raise Stop()

    monkeypatch.setattr(eng.lib(), "cl_engine_create", create)
    with pytest.raises(Stop):
        eng.Engine(preset="llama3-8b", **kw)
    return seen["cfg"]


def test_python_engine_sets_the_field(monkeypatch):
    assert _captured_config(monkeypatch).reserved[3] == 0
    assert _captured_config(monkeypatch, deterministic=True).reserved[3] == 1


def test_worker_flag(monkeypatch):
    got = {}
    monkeypatch.setattr(worker, "serve", lambda *a, **kw: got.update(kw))
    monkeypatch.setattr(sys, "argv", ["worker.py", "--deterministic"])
    worker.main()
    assert got["deterministic"] is True
    monkeypatch.setattr(sys, "argv", ["worker.py"])
    worker.main()
    assert got["deterministic"] is False


def _plan(n, k, sms, det):
    ks = C.c_int32()
    assert eng.lib().cl_gemm_split_plan(n, k, sms, det, C.byref(ks)) == eng.CL_OK
    return ks.value


SHAPES = [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336), (3072, 2048), (2048, 2048), (16384, 2048), (2048, 8192)]


@pytest.mark.parametrize("n,k", SHAPES)
def test_split_plan_does_not_depend_on_the_sm_count(n, k):
    det = {sms: _plan(n, k, sms, 1) for sms in (78, 114, 132, 144)}
    assert len(set(det.values())) == 1
    assert det[132] == _plan(n, k, 132, 0)   # an H100 SXM runs its default plan
    nkb = (k + 63) // 64
    s = det[132]
    assert 1 <= s <= 16 and (nkb + s - 1) // s * (s - 1) < nkb   # every split owns a k-block (gemm_splits_supported)


def test_default_plan_follows_the_sm_count():
    assert any(_plan(n, k, 114, 0) != _plan(n, k, 132, 0) for n, k in SHAPES)


def test_split_plan_arguments():
    ks = C.c_int32()
    assert eng.lib().cl_gemm_split_plan(0, 4096, 132, 0, C.byref(ks)) == eng.CL_ERR_INVALID_ARG
    assert eng.lib().cl_gemm_split_plan(4096, 4096, 0, 0, C.byref(ks)) == eng.CL_ERR_INVALID_ARG
    assert eng.lib().cl_gemm_split_plan(4096, 4096, 0, 1, None) == eng.CL_ERR_INVALID_ARG
