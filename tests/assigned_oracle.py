"""Checkers of halo2-base's own witness form (the N cells with n in place of every Rational(n, d), the (index, d) pairs of
the Rational cells, the looked-up cells as virtual-column indices), for the tests only:
  assigned_witness   the C restatement tests/cpp/assigned_witness_oracle.c (batch_invert_assigned, then assign_raw), built
                     on first use into a temporary directory and linked against the oracle's field arithmetic;
  apply_rational     the plain-integer formula that pins the C;
  evaluated_inputs   the form turned into the evaluated witness and looked-up values that oracle/prover_ref.py takes."""
from __future__ import annotations
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
import numpy as np
from oracle import oracle as orc, pyref

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "cpp", "assigned_witness_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        so_oracle = orc.build()
        tmp = tempfile.mkdtemp(prefix="h2b_assigned_oracle_")
        atexit.register(shutil.rmtree, tmp, True)  # the loaded library stays mapped; the directory goes with the process
        out = os.path.join(tmp, "libassigned_oracle.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        d = os.path.dirname(so_oracle)
        subprocess.check_call([cc, "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", _SRC, "-o", out,
                               f"-L{d}", "-loracle", f"-Wl,-rpath,{d}"])
        _lib = C.CDLL(out)
        _lib.aw_assigned_witness.restype = C.c_int
    return _lib


def assigned_witness(values, index, den, lookup_index, k, L):
    """-> (rc, evaluated cells N x 4, lookup columns L x 2^k x 4); rc 0, -1 layout overflow, -2 index >= N,
    -3 Rational indices not strictly increasing"""
    v = np.ascontiguousarray(values, dtype=np.uint64).reshape(-1, 4)
    ix = np.ascontiguousarray(index, dtype=np.uint64).reshape(-1)
    d = np.ascontiguousarray(den, dtype=np.uint64).reshape(-1, 4)
    lk = np.ascontiguousarray(lookup_index, dtype=np.uint64).reshape(-1)
    assert len(ix) == len(d)
    out = np.empty_like(v)
    cols = np.empty((L, 1 << k, 4), dtype=np.uint64)
    p = lambda a: C.c_void_p(a.ctypes.data) if a.size else None
    rc = lib().aw_assigned_witness(p(v), C.c_size_t(len(v)), p(ix), p(d), C.c_size_t(len(ix)), p(lk), C.c_size_t(len(lk)),
                                   C.c_uint(k), C.c_size_t(L), p(out), p(cols))
    return rc, out, cols


def apply_rational(values, rational):
    """plain integers: `values` holds n for every Rational(n, d) cell, `rational` the (index, d) pairs.  Returns what
    batch_invert_assigned yields: values[index] = n / d, and 0 where d = 0."""
    out = [v % pyref.R for v in values]
    for idx, d in rational:
        out[idx] = out[idx] * pow(d, -1, pyref.R) % pyref.R if d % pyref.R else 0
    return out


def evaluated_inputs(values, rational, lookup_index):
    """the form -> (evaluated virtual column, looked-up values in assign_raw order), plain integers"""
    v = apply_rational(values, rational)
    return v, [v[i] for i in lookup_index]
