"""Host-side rules of long context (no GPU): the served window of cl_engine_config.context_length as
cl_resolve_model_config (the function cl_engine_create calls) applies it, the ctypes layout of the new field, and the split
plan of the split-KV prefill attention (cl_attn_prefill_long_plan)."""
import ctypes as C
import json
import shutil
import subprocess
from pathlib import Path

import pytest

from crowdllama_b200 import engine as eng

ROOT = Path(__file__).resolve().parents[1]
MAX_CONTEXT = 131072


@pytest.fixture(autouse=True)
def _no_env(monkeypatch):
    for k in ("CL_CONTEXT_LENGTH", "CL_CONTEXT_SHIFT", "CL_NUM_KEEP"):
        monkeypatch.delenv(k, raising=False)


def resolve(preset=None, weights_path=None, model=None, context_length=0, page_size=32, context_shift=False, num_keep=0):
    """(status, max_seq_len) of cl_resolve_model_config"""
    L = eng.lib()
    cfg = eng.EngineConfig()
    L.cl_default_engine_config(C.byref(cfg))
    keep = []
    if preset:
        keep.append(preset.encode())
        cfg.preset = keep[-1]
    if weights_path:
        keep.append(str(weights_path).encode())
        cfg.weights_path = keep[-1]
    if model:
        cfg.model = eng.ModelConfig(**model)
    cfg.page_size = page_size
    cfg.reserved[0] = 1 if context_shift else 0
    cfg.reserved[1] = num_keep
    cfg.reserved[2] = context_length
    out = eng.ModelConfig()
    rc = L.cl_resolve_model_config(C.byref(cfg), C.byref(out))
    return rc, out.max_seq_len


def model_dir(tmp_path, max_pos=131072, window=None):
    d = tmp_path / f"m{max_pos}_{window}"
    d.mkdir(exist_ok=True)
    cfg = {"num_hidden_layers": 2, "hidden_size": 4096, "num_attention_heads": 32, "num_key_value_heads": 8,
           "intermediate_size": 14336, "vocab_size": 128256, "max_position_embeddings": max_pos, "rope_theta": 5e5,
           "rope_scaling": {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                            "original_max_position_embeddings": 8192}}
    if window:
        cfg["sliding_window"] = window
    (d / "config.json").write_text(json.dumps(cfg))
    return d


def test_model_dir_default_window_unchanged(tmp_path):
    assert resolve(weights_path=model_dir(tmp_path)) == (eng.CL_OK, 32768)
    assert resolve(weights_path=model_dir(tmp_path, max_pos=8192)) == (eng.CL_OK, 8192)
    assert resolve(weights_path=model_dir(tmp_path, max_pos=32768, window=4096)) == (eng.CL_OK, 4096)


@pytest.mark.parametrize("n", [65536, 131072])
def test_model_dir_long_windows_accepted(tmp_path, n):
    assert resolve(weights_path=model_dir(tmp_path), context_length=n) == (eng.CL_OK, n)


def test_model_dir_refusals(tmp_path):
    assert resolve(weights_path=model_dir(tmp_path, max_pos=65536), context_length=65537)[0] == eng.CL_ERR_INVALID_ARG
    assert "max_position_embeddings" in eng.lib().cl_last_error().decode()
    assert resolve(weights_path=model_dir(tmp_path, max_pos=131072, window=32768), context_length=32800)[0] == eng.CL_ERR_INVALID_ARG
    assert "sliding_window" in eng.lib().cl_last_error().decode()
    assert resolve(weights_path=model_dir(tmp_path, max_pos=131072, window=32768), context_length=32768) == (eng.CL_OK, 32768)
    # below the model's default is allowed too
    assert resolve(weights_path=model_dir(tmp_path), context_length=4096) == (eng.CL_OK, 4096)


@pytest.mark.parametrize("preset", ["llama3.1-8b", "llama3.2-1b", "tiny-test", "mistral-7b"])
def test_presets(preset):
    base = eng.ModelConfig()
    assert eng.lib().cl_model_preset(preset.encode(), C.byref(base)) == eng.CL_OK
    assert resolve(preset=preset) == (eng.CL_OK, base.max_seq_len)          # 0: the preset's window
    assert resolve(preset=preset, context_length=MAX_CONTEXT) == (eng.CL_OK, MAX_CONTEXT)
    assert resolve(preset=preset, context_length=96) == (eng.CL_OK, 96)


def test_explicit_model_config():
    m = eng.ModelConfig()
    eng.lib().cl_model_preset(b"tiny-test", C.byref(m))
    assert resolve(model=m.as_dict()) == (eng.CL_OK, m.max_seq_len)
    assert resolve(model=m.as_dict(), context_length=65536) == (eng.CL_OK, 65536)


@pytest.mark.parametrize("page", [16, 32, 64])
def test_range(page):
    assert resolve(preset="tiny-test", page_size=page, context_length=MAX_CONTEXT + 1)[0] == eng.CL_ERR_INVALID_ARG
    assert resolve(preset="tiny-test", page_size=page, context_length=2 * page - 1)[0] == eng.CL_ERR_INVALID_ARG
    assert resolve(preset="tiny-test", page_size=page, context_length=2 * page) == (eng.CL_OK, 2 * page)
    assert resolve(preset="tiny-test", page_size=page, context_length=-5)[0] == eng.CL_ERR_INVALID_ARG


def test_env_overrides(monkeypatch):
    monkeypatch.setenv("CL_CONTEXT_LENGTH", "65536")
    assert resolve(preset="llama3.1-8b") == (eng.CL_OK, 65536)
    assert resolve(preset="llama3.1-8b", context_length=MAX_CONTEXT) == (eng.CL_OK, 65536)
    monkeypatch.setenv("CL_CONTEXT_LENGTH", "0")
    assert resolve(preset="llama3.1-8b", context_length=MAX_CONTEXT) == (eng.CL_OK, 32768)


def test_num_keep_checked_against_the_final_window():
    # tiny-test's own window allows num_keep 1000 when it is long enough; a 1024-token context_length leaves < 2 pages
    m = eng.ModelConfig()
    eng.lib().cl_model_preset(b"tiny-test", C.byref(m))
    keep = 1000
    assert m.max_seq_len - keep >= 64 or m.max_seq_len < keep
    assert resolve(preset="tiny-test", context_length=4096, context_shift=True, num_keep=keep) == (eng.CL_OK, 4096)
    assert resolve(preset="tiny-test", context_length=1024, context_shift=True, num_keep=keep)[0] == eng.CL_ERR_INVALID_ARG
    assert resolve(preset="tiny-test", context_length=1064, context_shift=True, num_keep=keep) == (eng.CL_OK, 1064)
    assert resolve(preset="tiny-test", context_length=1024, context_shift=False, num_keep=keep) == (eng.CL_OK, 1024)


def test_engine_config_layout(tmp_path):
    """the ctypes struct is the C struct: same size, and context_length where C reads it"""
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "clengine.h"\n'
                   'int main(void) { printf("%zu %zu", sizeof(cl_engine_config), offsetof(cl_engine_config, context_length)); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True, capture_output=True)
    size, off = map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split())
    assert C.sizeof(eng.EngineConfig) == size
    assert eng.EngineConfig.reserved.offset + 2 * 4 == off
    assert resolve(preset="tiny-test", context_length=640) == (eng.CL_OK, 640)


def plan(pos0, t, n_heads=32, sms=132, nsplit=0):
    ns, part = C.c_int32(), C.c_int64()
    assert eng.lib().cl_attn_prefill_long_plan(pos0, t, n_heads, sms, nsplit, C.byref(ns), C.byref(part)) == eng.CL_OK
    return ns.value, part.value


def coverage(pos0, t, ns):
    """per (tile, split): the KV blocks [kb0, kb1) the kernel's items cover (attn_prefill_tc.cu get_item)"""
    out = {}
    for tile in range((t + 127) // 128):
        nblk = (pos0 + min(tile * 128 + 128, t) - 1) // 64 + 1
        out[tile] = (nblk, [(s * nblk // ns, (s + 1) * nblk // ns) for s in range(ns)])
    return out


@pytest.mark.parametrize("pos0", [0, 1000, 10240, 32768, 65535, 100000, MAX_CONTEXT - 4096])
@pytest.mark.parametrize("t", [1, 2, 16, 17, 64, 128, 129, 300, 1024, 2047, 4096])
@pytest.mark.parametrize("n_heads", [8, 32])
def test_split_plan(pos0, t, n_heads):
    sms = 132
    ns, part = plan(pos0, t, n_heads, sms)
    items = (t + 127) // 128 * n_heads
    assert ns >= 1
    if items >= sms:
        assert ns == 1                                          # the unsplit items fill the SMs
    nblk0 = (pos0 + min(128, t) - 1) // 64 + 1
    if ns > 1:
        assert nblk0 // ns >= 32                                # the minimum blocks per split
        assert items * ns * 128 * 130 <= part                   # the workspace bound
    for nblk, ranges in coverage(pos0, t, ns).values():         # every block exactly once, no empty split
        assert ranges[0][0] == 0 and ranges[-1][1] == nblk
        assert all(a < b for a, b in ranges)
        assert all(ranges[i][1] == ranges[i + 1][0] for i in range(ns - 1))


def test_split_plan_fills_the_sms_behind_a_long_cache():
    assert plan(100000, 16)[0] >= 4                             # one tile x 32 heads on 132 SMs
    assert plan(100000, 300)[0] == 1                            # 96 items: 2 splits would take as many waves
    assert plan(100000, 4096)[0] == 1
    assert plan(1000, 16)[0] == 1                               # too few blocks to split


@pytest.mark.parametrize("force", [1, 2, 7, 1000])
def test_forced_splits_are_clamped(force):
    for pos0, t in [(10241 - 17, 17), (0, 4096), (131072 - 300, 300), (0, 1)]:
        ns, _ = plan(pos0, t, nsplit=force)
        nblk0 = (pos0 + min(128, t) - 1) // 64 + 1
        assert ns == min(force, nblk0)
        for nblk, ranges in coverage(pos0, t, ns).values():
            assert all(a < b for a, b in ranges) and ranges[-1][1] == nblk
