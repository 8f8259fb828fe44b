"""ctypes loader of tests/weight_norm_oracle.c: the feature oracle (tests/feature_oracle.c and oracle/snn_oracle.c,
both unchanged) extended by per-target norm tensors and per-step Weight normalisation.  TEST INFRASTRUCTURE: the library exports the
oracle's own entry points, so ``WeightNormOracleBackend`` is ``oracle.oracle.OracleBackend`` with this library in place of
libsnn_oracle.so."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from bindsnet_b200 import _abi
from oracle import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "weight_norm_oracle.c")
LIB = os.path.join(HERE, "libsnn_weight_norm_oracle.so")
_DEPS = [SRC, os.path.join(HERE, "feature_oracle.c"), os.path.join(ROOT, "oracle", "snn_oracle.c"),
         os.path.join(ROOT, "include", "snn_b200.h")]
_lib = None


def build(force: bool = False) -> str:
    """The oracle's compiler and flags (oracle/Makefile)."""
    stale = (not os.path.exists(LIB)) or any(os.path.getmtime(f) > os.path.getmtime(LIB) for f in _DEPS)
    if force or stale:
        cmd = ["/usr/bin/gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-Wall", "-Wextra",
               "-shared", "-o", LIB, SRC, "-lm"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("building the weight norm oracle failed:\n" + res.stderr[-4000:])
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


class WeightNormOracleBackend(oracle.OracleBackend):
    """``OracleBackend`` (host API on CPU tensors -> the oracle) running on this library."""

    def __enter__(self):
        self._prev_lib = oracle._lib
        oracle._lib = lib()
        return super().__enter__()

    def __exit__(self, *exc):
        super().__exit__(*exc)
        oracle._lib = self._prev_lib
        return False
