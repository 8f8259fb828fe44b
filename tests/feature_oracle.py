"""ctypes loader of tests/feature_oracle.c: the CPU oracle (oracle/snn_oracle.c, unchanged) extended by the
MulticompartmentConnection features Probability, Mask and Intensity.  TEST INFRASTRUCTURE: the library exports the
oracle's own entry points, so ``FeatureOracleBackend`` is ``oracle.oracle.OracleBackend`` with this library in place of
libsnn_oracle.so.  Also the draw's vectorised twin, for the golden generator and the tests."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from bindsnet_b200 import _abi
from oracle import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "feature_oracle.c")
LIB = os.path.join(HERE, "libsnn_feature_oracle.so")
_DEPS = [SRC, os.path.join(ROOT, "oracle", "snn_oracle.c"), os.path.join(ROOT, "include", "snn_b200.h")]
_lib = None


def build(force: bool = False) -> str:
    """The oracle's compiler and flags (oracle/Makefile)."""
    stale = (not os.path.exists(LIB)) or any(os.path.getmtime(f) > os.path.getmtime(LIB) for f in _DEPS)
    if force or stale:
        cmd = ["/usr/bin/gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-Wall", "-Wextra",
               "-shared", "-o", LIB, SRC, "-lm"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("building the feature oracle failed:\n" + res.stderr[-4000:])
    return LIB


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        vp, i32 = C.c_void_p, C.c_int32
        L.snn_oracle_run_window.restype = C.c_int
        L.snn_oracle_run_window.argtypes = [C.POINTER(_abi.SnnNet), C.POINTER(_abi.SnnRunOpts), C.c_int, C.c_int]
        L.snn_oracle_delta_apply.restype = C.c_int
        L.snn_oracle_delta_apply.argtypes = [vp, vp, vp, i32, i32, i32, C.c_float, C.c_float, i32, i32, C.c_float]
        L.snn_oracle_conn_compute.restype = C.c_int
        L.snn_oracle_conn_compute.argtypes = [C.POINTER(_abi.SnnConn), i32, i32, i32, vp, vp]
        L.snn_oracle_conn_update.restype = C.c_int
        L.snn_oracle_conn_update.argtypes = [C.POINTER(_abi.SnnNet), i32, i32]
        L.snn_oracle_conn_normalize.restype = C.c_int
        L.snn_oracle_conn_normalize.argtypes = [C.POINTER(_abi.SnnConn), i32, i32]
        L.snn_oracle_abi_version.restype = C.c_int
        assert L.snn_oracle_abi_version() == _abi.SNN_ABI_VERSION
        _lib = L
    return _lib


class FeatureOracleBackend(oracle.OracleBackend):
    """``OracleBackend`` (host API on CPU tensors -> the oracle) running on the feature-capable oracle library."""

    def __enter__(self):
        self._prev_lib = oracle._lib
        oracle._lib = lib()
        return super().__enter__()

    def __exit__(self, *exc):
        super().__exit__(*exc)
        oracle._lib = self._prev_lib
        return False


def _fmix32(h: np.ndarray) -> np.ndarray:
    h = h ^ (h >> np.uint32(16))
    h = h * np.uint32(0x85EBCA6B)
    h = h ^ (h >> np.uint32(13))
    h = h * np.uint32(0xC2B2AE35)
    return h ^ (h >> np.uint32(16))


def draw_matrix(seed: int, t: int, conn: int, n_src: int, n_tgt: int) -> np.ndarray:
    """``snn_synapse_draw(seed, t, conn, i, j)`` for every synapse: [n_src, n_tgt] uint32 (the twin of
    ``_abi.synapse_draw``, vectorised)."""
    u = lambda x: np.uint32(x & 0xFFFFFFFF)
    with np.errstate(over="ignore"):
        h = _fmix32(np.array([u(seed) ^ np.uint32(0x53594E41)], dtype=np.uint32))
        h = _fmix32(h ^ u(0x9E3779B9 * (t + 1)))
        h = _fmix32(h ^ u(0x85EBCA6B * (conn + 1)))
        rows = _fmix32(h ^ (np.uint32(0xC2B2AE35) * (np.arange(n_src, dtype=np.uint32) + np.uint32(1))))
        cols = np.uint32(0x27D4EB2F) * (np.arange(n_tgt, dtype=np.uint32) + np.uint32(1))
        return _fmix32(rows[:, None] ^ cols[None, :])


def transmit_matrix(p: np.ndarray, seed: int, t: int, conn: int) -> np.ndarray:
    """``snn_synapse_transmits`` for every synapse of a [n_src, n_tgt] probability matrix: float32 0 / 1."""
    h = draw_matrix(seed, t, conn, *p.shape)
    u = (h >> np.uint32(8)).astype(np.float32) * np.float32(2.0**-24)
    return (u < p.astype(np.float32)).astype(np.float32)
