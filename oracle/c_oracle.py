"""ctypes wrapper of the C oracle oracle/cw_oracle.c (TEST INFRASTRUCTURE)."""
from __future__ import annotations

import ctypes
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cw_oracle.c")
SO = os.path.join(HERE, "libcw_oracle.so")


def build(force: bool = False) -> str:
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < os.path.getmtime(SRC):
        subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-pthread", "-o", SO, SRC])
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
        _lib.orc_load.restype = ctypes.c_void_p
        _lib.orc_load.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
        _lib.orc_total_signals.restype = ctypes.c_uint64
        _lib.orc_total_signals.argtypes = [ctypes.c_void_p]
        _lib.orc_n_inputs.restype = ctypes.c_uint32
        _lib.orc_n_inputs.argtypes = [ctypes.c_void_p]
        _lib.orc_run.restype = ctypes.c_int32
        _lib.orc_run.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        _lib.orc_r1cs_check.restype = ctypes.c_int64
        _lib.orc_r1cs_check.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        _lib.orc_apply.restype = ctypes.c_int
        _lib.orc_apply.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p,
                                   ctypes.c_void_p, ctypes.c_void_p]
        _lib.orc_free.argtypes = [ctypes.c_void_p]
        _lib.orc_run_many.restype = ctypes.c_long
        _lib.orc_run_many.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long, ctypes.c_int]
        _lib.orc_poly_eval.restype = ctypes.c_int
        _lib.orc_poly_eval.argtypes = [ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_int,
                                       ctypes.c_void_p]
    return _lib


class COracle:
    """the circuit description executed by the C restatement of the reference runtime"""

    def __init__(self, desc_bytes: bytes):
        self._blob = bytes(desc_bytes)
        self._h = lib().orc_load(self._blob, len(self._blob))
        if not self._h:
            raise ValueError("oracle: cannot parse circuit description")
        self.n_signals = lib().orc_total_signals(self._h)
        self.n_inputs = lib().orc_n_inputs(self._h)

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_free(self._h)
            self._h = None

    def run(self, inputs: np.ndarray, threads: int = 1):
        """inputs uint64 [batch][n_inputs][4] -> (witness [batch][n_signals][4], status [batch])"""
        inputs = np.ascontiguousarray(inputs, dtype=np.uint64).reshape(-1, self.n_inputs, 4)
        B = inputs.shape[0]
        wit = np.zeros((B, self.n_signals, 4), dtype=np.uint64)
        st = np.zeros(B, dtype=np.int32)

        def one(i):
            st[i] = lib().orc_run(self._h, inputs[i].ctypes.data, wit[i].ctypes.data)
        if threads > 1:
            with ThreadPoolExecutor(threads) as ex:
                list(ex.map(one, range(B)))
        else:
            for i in range(B):
                one(i)
        return wit, st

    def run_many(self, inputs: np.ndarray, threads: int) -> int:
        """throughput mode (witnesses are not kept): returns how many instances finished with status 0"""
        inputs = np.ascontiguousarray(inputs, dtype=np.uint64).reshape(-1, self.n_inputs, 4)
        return int(lib().orc_run_many(self._h, inputs.ctypes.data, inputs.shape[0], threads))

    def r1cs_check(self, witness: np.ndarray) -> np.ndarray:
        witness = np.ascontiguousarray(witness, dtype=np.uint64).reshape(-1, self.n_signals, 4)
        return np.array([lib().orc_r1cs_check(self._h, witness[i].ctypes.data) for i in range(witness.shape[0])],
                        dtype=np.int64)


def poly_eval(prime_id: int, coef: np.ndarray, x: int, threads: int = 0) -> int:
    """sum_i coef[i] x^i mod q for canonical coefficients uint64 [n][4] (Horner's rule on `threads` threads, 0: one per
    CPU)"""
    coef = np.ascontiguousarray(coef, dtype=np.uint64).reshape(-1, 4)
    xs = (ctypes.c_uint64 * 4)(*[(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)])
    r = (ctypes.c_uint64 * 4)()
    if not lib().orc_poly_eval(prime_id, coef.ctypes.data, coef.shape[0], xs, threads or os.cpu_count() or 1, r):
        raise ValueError("unknown prime id %d" % prime_id)
    return sum(int(r[i]) << (64 * i) for i in range(4))


def apply(prime_id: int, op: int, a: int, b: int = 0, c: int = 0) -> int:
    def enc(v):
        return (ctypes.c_uint64 * 4)(*[(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)])
    r = (ctypes.c_uint64 * 4)()
    ok = lib().orc_apply(prime_id, op, enc(a), enc(b), enc(c), r)
    if not ok:
        raise ZeroDivisionError
    return sum(int(r[i]) << (64 * i) for i in range(4))
