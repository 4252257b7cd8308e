"""Context shift on the CPU oracle's side, and its float64 bound.

oracle_shift runs oc_seq_shift (tests/oracle_shift.c), which restates cl_seq_shift's contract on an oracle sequence: the
kept K rotated by -delta in fp32 with row delta of the oracle's own cos/sin table, every product and sum rounded, then
rounded to bf16; V moved; len dropped by delta.  That file compiles llama_oracle.c into its own shared object so that it
works on the oracle's private structs through their one definition; it is built here on first use, into a temporary
directory, with the oracle Makefile's flags."""
from __future__ import annotations

import ctypes as C
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

from oracle import oracle as oc

_SRC = Path(__file__).resolve().parent / "oracle_shift.c"
_CFLAGS = ["-O3", "-mavx2", "-mfma", "-fopenmp", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-fno-math-errno",
           "-ffp-contract=off", "-fvisibility=hidden"]
_lib = None


def _shift_lib():
    global _lib
    if _lib is None:
        out = Path(tempfile.mkdtemp(prefix="oracle_shift_")) / "liboracle_shift.so"
        cc = shutil.which("gcc") or "/usr/bin/gcc"
        subprocess.run([cc, *_CFLAGS, "-shared", "-o", str(out), str(_SRC), "-lm"], check=True, capture_output=True)
        L = C.CDLL(str(out))
        L.oc_seq_shift.restype, L.oc_seq_shift.argtypes = C.c_int, [C.c_void_p, C.c_int32, C.c_int32]
        L.oc_rope_row.restype, L.oc_rope_row.argtypes = C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]
        _lib = L
    return _lib


def oracle_rope_row(m: oc.Model, row: int) -> np.ndarray:
    """Row `row` of the oracle's fp32 table [head_dim / 2][2] (cos, sin): the engine builds the same table bit for bit."""
    out = np.empty((m.cfg["head_dim"] // 2, 2), np.float32)
    if _shift_lib().oc_rope_row(m._h, row, out.ctypes.data_as(C.c_void_p)):
        raise ValueError(f"oc_rope_row({row})")
    return out


def oracle_rope_table(m: oc.Model) -> np.ndarray:
    """The oracle's whole table [max_seq_len][head_dim / 2][2]."""
    return np.stack([oracle_rope_row(m, r) for r in range(m.cfg["max_seq_len"])])


def oracle_shift(seq: oc.Seq, n_keep: int, n_discard: int):
    """oc_seq_shift: tokens [n_keep, n_keep + n_discard) leave the oracle sequence, as cl_seq_shift does in the engine."""
    if _shift_lib().oc_seq_shift(seq._h, n_keep, n_discard):
        raise ValueError(f"oc_seq_shift({n_keep}, {n_discard}) on a sequence of {len(seq)} tokens")


def rotate_back(k: np.ndarray, cs: np.ndarray) -> np.ndarray:
    """bf16(R(-delta) k) in fp32: k [..., hd] (bf16 values as fp32), cs [hd/2][2] = row delta.  a c + b s, b c - a s."""
    half = k.shape[-1] // 2
    a, b = k[..., :half].astype(np.float32), k[..., half:].astype(np.float32)
    c, s = cs[:, 0].astype(np.float32), cs[:, 1].astype(np.float32)
    return oc.np_bf16_round(np.concatenate([a * c + b * s, b * c - a * s], axis=-1))


def rope_table(cfg: dict, rows: int) -> np.ndarray:
    """The engine's / oracle's table expression in numpy (double angle, fp32 cos / sin), "llama3" scaling included."""
    D = cfg["head_dim"]
    i = np.arange(D // 2, dtype=np.float64)
    inv = np.power(np.float64(np.float32(cfg["rope_theta"])), -2.0 * i / D)
    f = float(np.float32(cfg.get("rope_factor", 0.0)))
    if f > 1.0 and cfg.get("rope_original_max_pos", 0) > 0:
        lo, hi = float(np.float32(cfg["rope_low_freq_factor"])), float(np.float32(cfg["rope_high_freq_factor"]))
        old = float(cfg["rope_original_max_pos"])
        wl = 2 * np.pi / inv
        smooth = (old / wl - lo) / (hi - lo)
        inv = np.where(wl < old / hi, inv, np.where(wl > old / lo, inv / f, (1 - smooth) * inv / f + smooth * inv))
    ang = np.arange(rows, dtype=np.float64)[:, None] * inv[None, :]
    return np.stack([np.cos(ang).astype(np.float32), np.sin(ang).astype(np.float32)], axis=-1)


def shift_bound(k_old: np.ndarray, cs: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """The float64 rotation of k_old by -delta and the per-element bound on a shifted K: 1 bf16 ulp of the result plus
    2^-22 (|a c| + |b s|) for the fp32 products and sum."""
    half = k_old.shape[-1] // 2
    a, b = k_old[..., :half].astype(np.float64), k_old[..., half:].astype(np.float64)
    c, s = cs[:, 0].astype(np.float64), cs[:, 1].astype(np.float64)
    ref = np.concatenate([a * c + b * s, b * c - a * s], axis=-1)
    mag = np.concatenate([np.abs(a * c) + np.abs(b * s), np.abs(b * c) + np.abs(a * s)], axis=-1)
    ulp = np.exp2(np.floor(np.log2(np.maximum(np.abs(ref), 1e-38))) - 7)
    return ref, ulp + 2.0 ** -22 * mag


def shift_err(k_new: np.ndarray, k_old: np.ndarray, cs: np.ndarray) -> float:
    """max |k_new - rotation| / bound (<= 1 passes)."""
    ref, bound = shift_bound(k_old, cs)
    return float((np.abs(k_new.astype(np.float64) - ref) / bound).max()) if ref.size else 0.0
