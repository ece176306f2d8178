"""halo2's permutation keygen on halo2-base's copy calls, restated for the tests of halo2_lib_b200.keygen
(tests/test_gpu_keygen.py, tests/test_oracle_keygen.py).  Cells are ids c 2^k + r, c the permutation column in
[c, a0.., a{A-1}, l0.., l{L-1}] order (flex_gate/mod.rs:121-136, then the range config).

  Assembly         halo2's permutation::keygen::Assembly (mapping / aux / sizes) and its `copy`, literally: return when both
                   cells are in one cycle, else relabel the smaller cycle in aux and swap mapping[left] and mapping[right];
  assembly_c       the same restated in C (tests/cpp/keygen_oracle.c), for the full-size comparisons where Python is too slow;
  copy_sequence    the copy calls of BaseCircuitBuilder::synthesize in halo2-base's order (gates/circuit/mod.rs:179-199):
                   the break copies (single_phase.rs:243-250), LookupAnyManager::assign_raw's copies (lookups.rs:138-151),
                   the advice equalities sorted by (a, b), the constant equalities sorted by (constant, cell) with each
                   distinct constant at the next row of c (copy_constraints.rs:129-167);
  closed_form      sigma = t_1 o .. o t_F over the copies that join two classes when made (Kruskal's forest by call index),
                   evaluated by the walk that crosses, from x, the largest forest edge below the last one crossed;
  sigma_values     delta^c' omega^r' of every mapping entry, as Montgomery limbs."""
from __future__ import annotations
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
import numpy as np
from oracle import pyref
from util import mont
import builder_oracle as bo

R = pyref.R
_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


class Assembly:
    """halo2's permutation Assembly over flat cell ids"""

    def __init__(self, n_cells: int):
        self.mapping = list(range(n_cells))
        self.aux = list(range(n_cells))
        self.sizes = [1] * n_cells

    def copy(self, left: int, right: int):
        left_cycle, right_cycle = self.aux[left], self.aux[right]
        if left_cycle == right_cycle:
            return
        if self.sizes[left_cycle] < self.sizes[right_cycle]:
            left_cycle, right_cycle = right_cycle, left_cycle
        self.sizes[left_cycle] += self.sizes[right_cycle]
        i = right_cycle
        while True:
            self.aux[i] = left_cycle
            i = self.mapping[i]
            if i == right_cycle:
                break
        self.mapping[left], self.mapping[right] = self.mapping[right], self.mapping[left]


def assembly(n_cells: int, pairs) -> np.ndarray:
    a = Assembly(n_cells)
    for x, y in np.asarray(pairs, dtype=np.int64).reshape(-1, 2).tolist():
        a.copy(x, y)
    return np.array(a.mapping, dtype=np.uint32)


def _c_lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="h2b_keygen_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        out = os.path.join(tmp, "libkeygen_oracle.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.check_call([cc, "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", os.path.join(_HERE, "cpp", "keygen_oracle.c"), "-o", out])
        _lib = C.CDLL(out)
        _lib.ko_assembly.restype = C.c_int
    return _lib


def assembly_c(n_cells: int, pairs) -> np.ndarray:
    p = np.ascontiguousarray(pairs, dtype=np.uint32).reshape(-1, 2)
    out = np.empty(n_cells, dtype=np.uint32)
    rc = _c_lib().ko_assembly(C.c_uint32(n_cells), C.c_void_p(p.ctypes.data if p.size else None), C.c_size_t(len(p)),
                              C.c_void_p(out.ctypes.data))
    assert rc == 0, "a copy names a cell outside the columns"
    return out


def closed_form(n_cells: int, pairs) -> np.ndarray:
    """Kruskal by call index, then the walk with descending edge indices"""
    parent = list(range(n_cells))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    adj = {}
    for e, (x, y) in enumerate(np.asarray(pairs, dtype=np.int64).reshape(-1, 2).tolist()):
        rx, ry = find(x), find(y)
        if rx == ry:
            continue
        parent[rx] = ry
        adj.setdefault(x, []).append((e, y))
        adj.setdefault(y, []).append((e, x))
    sigma = np.arange(n_cells, dtype=np.uint32)
    for x, lst in adj.items():
        cur, bound = x, None
        while True:
            below = [(e, o) for e, o in adj[cur] if bound is None or e < bound]
            if not below:
                break
            bound, cur = max(below)
        sigma[x] = cur
    return sigma


def _raw_ids(bps, n: int, p) -> np.ndarray:
    """the cell ids of virtual indices p (a break cell belongs to the column it ends)"""
    p = np.asarray(p, dtype=np.int64).reshape(-1)
    starts = np.concatenate([[0], np.cumsum(np.asarray(bps, dtype=np.int64))])
    j = np.searchsorted(starts[1:], p, side="left")
    return (1 + j) * n + (p - starts[j])


def copy_sequence(k: int, A: int, L: int, max_rows: int, b: dict):
    """(pairs: the copy calls as (E, 2) cell ids in call order, c_rows: {canonical constant: row of c}, break points).
    b: a builder of builder_oracle.make_builder's form, constants canonical (< 2^64)."""
    n = 1 << k
    bps = bo.assign_with_constraints(b["contexts"], A, max_rows, record=False)[0]
    parts = [np.array([[(2 + j) * n, (1 + j) * n + bp] for j, bp in enumerate(bps)], dtype=np.int64).reshape(-1, 2)]
    if L:
        i = np.arange(len(b["lookups"]), dtype=np.int64)
        parts.append(np.stack([_raw_ids(bps, n, b["lookups"]), (1 + A + i % L) * n + i // L], axis=1))
    E = np.asarray(b["advice_equalities"], dtype=np.int64).reshape(-1, 2)
    E = E[np.lexsort((E[:, 1], E[:, 0]))]
    parts.append(np.stack([_raw_ids(bps, n, E[:, 0]), _raw_ids(bps, n, E[:, 1])], axis=1).reshape(-1, 2))
    consts = np.asarray(b["constants"], dtype=np.uint64)
    idx = np.asarray(b["constant_index"], dtype=np.int64)
    order = np.lexsort((idx, consts))
    distinct, row = np.unique(consts[order], return_inverse=True)
    parts.append(np.stack([row.astype(np.int64), _raw_ids(bps, n, idx[order])], axis=1).reshape(-1, 2))
    c_rows = {int(v): r for r, v in enumerate(distinct.tolist())}
    return np.concatenate(parts).astype(np.int64), c_rows, [int(x) for x in bps]


def sigma_values(mapping, n_cols: int, k: int) -> np.ndarray:
    """(n_cols, 2^k, 4) Montgomery limbs of delta^c' omega^r' for mapping[c 2^k + r] = c' 2^k + r'"""
    n = 1 << k
    w = pyref.omega_for(k)
    wp = [1] * n
    for r in range(1, n):
        wp[r] = wp[r - 1] * w % R
    dp = [pow(pyref.DELTA, c, R) for c in range(n_cols)]
    m = np.asarray(mapping, dtype=np.int64)
    vals = [dp[int(x) >> k] * wp[int(x) & (n - 1)] % R for x in m.tolist()]
    return mont(vals, R).reshape(n_cols, n, 4)
