"""halo2-base's keygen pass and halo2's MockProver restated literally on Python integers, for a builder in its keygen form
(witness_gen_only = false): the yardstick of halo2_lib_b200.MockProver (tests/test_gpu_mock_prover.py).  It shares no method
with the device: the walk goes cell by cell, the constants are sorted as tuples, every gate and lookup is evaluated row by row.

  assign_with_constraints   halo2-base/src/gates/flex_gate/threads/single_phase.rs:193-263, with its panics;
  assign_lookups_in_phase   halo2-base/src/gates/circuit/builder.rs:327-376, with its asserts;
  assign_constants          CopyConstraintManager::assign_raw (virtual_region/copy_constraints.rs:129-173) on one constants
                            column: sort by (constant, cell), each distinct constant at the next fixed row;
  verify                    MockProver's gate, lookup and equality semantics over the resulting columns.

Cells are virtual-column indices (the contexts' ctx.advice concatenated); values are canonical integers.  `make_builder`
builds synthetic keygen-form builders: chains of vertical gates overlapping at distance 3 as mul_add chains do, bit cells
tied to constants, looked-up limbs, and one advice equality per chain."""
from __future__ import annotations
import bisect
import numpy as np
from oracle import pyref

R = pyref.R
BLINDING_FACTORS = 6
ROTATIONS = 4


class Panic(Exception):
    """a panic of halo2-base's keygen pass (or an error of halo2's MockProver::run), with its message"""


def not_enough_columns(max_rows):
    return Panic("NOT ENOUGH ADVICE COLUMNS. Perhaps blinding factors were not taken into account. The max non-poisoned rows is %d" % max_rows)


def assign_with_constraints(contexts, num_cols: int, max_rows: int, record: bool = True):
    """contexts: one selector list per context.  Returns (break_points, raw, q): raw[p] = the (column, row) assigned_advices
    records for virtual cell p, q[j] = the rows where q_enable of column j is enabled (both only with `record`)."""
    break_points, raw, q = [], [], [set() for _ in range(num_cols)]
    gate_index = row_offset = base = 0
    for sel in contexts:
        if len(sel) == 0:
            continue
        if gate_index >= num_cols:
            raise not_enough_columns(max_rows)
        for i, qi in enumerate(sel):
            if record:
                raw.append((gate_index, row_offset))
            if (qi and row_offset + ROTATIONS > max_rows) or row_offset >= max_rows - 1:
                break_points.append(row_offset)
                row_offset = 0
                gate_index += 1
                if ROTATIONS > 1 and i + 2 >= ROTATIONS:
                    for delta in range(1, ROTATIONS - 1):
                        if sel[i - delta]:
                            raise Panic("We do not support overlaps with delta = %d" % delta)
                if gate_index >= num_cols:
                    raise not_enough_columns(max_rows)
            if qi and record:
                q[gate_index].add(row_offset)
            row_offset += 1
        base += len(sel)
    return break_points, raw, q


def spans(break_points, N: int):
    """(start, cells) of every column the walk fills: column j holds virtual cells start_j .. start_j + cells_j - 1"""
    out, s = [], 0
    for b in break_points:
        out.append((s, b + 1))
        s += b
    if N:
        out.append((s, N - s))
    return out


def raw_cell(break_points, p: int):
    """the cell assigned_advices records for p: a break cell belongs to the column it ends"""
    starts = np.cumsum([0] + list(break_points))
    j = bisect.bisect_left(starts[1:].tolist(), p)
    return (j, p - int(starts[j]))


def assign_lookups_in_phase(lookup_index, raw_of, N: int, A: int, L: int, selector_lookup: bool, max_rows: int):
    """("q_lookup", rows) with the selector lookup, ("lookup", index columns) with L lookup-advice columns (column t row r =
    the cell index[r L + t]), None without lookups"""
    if len(lookup_index) == 0:
        return None
    if selector_lookup and L == 0:
        assert A == 1
        rows = set()
        for idx in lookup_index:
            if idx >= N:
                raise Panic("virtual cell not assigned")
            col, row = raw_of(int(idx))
            if row >= max_rows:
                raise Panic("range lookup assigned to an unusable row")
            assert col == 0, "lookup column does not match"
            rows.add(row)
        return ("q_lookup", rows)
    if L == 0:
        raise Panic("range lookups require lookup advice columns")
    if -(-len(lookup_index) // L) > max_rows:
        raise Panic("range lookups would be assigned to unusable rows")
    if any(int(i) >= N for i in lookup_index):
        raise Panic("virtual cell not assigned")
    return ("lookup", [list(lookup_index[t::L]) for t in range(L)])


def assign_constants(constant_equalities, u: int, k: int):
    """{constant: row of the constants column}: the equalities sorted by (constant, cell), each new constant at the next row"""
    rows = {}
    for c, _ in sorted((int(c) % R, int(i)) for c, i in constant_equalities):
        if c not in rows:
            if len(rows) >= u:
                raise Panic("NotEnoughRowsAvailable { current_k: %d }" % k)
            rows[c] = len(rows)
    return rows


def _report(items, max_report):
    items = sorted(set(items))
    return (len(items), items[:max_report])


def run(k: int, A: int, L: int, selector_lookup: bool, lookup_bits: int, max_rows: int, b: dict, values, max_report: int = 16,
        gate_rows=None, record: bool = True) -> dict:
    """MockProver::run + verify: the keygen pass's layout, then every check.  values[p]: the canonical value of cell p (the
    witness after batch_invert_assigned).  gate_rows: {column: rows} restricts the gate checks (default: every row < u)."""
    n = 1 << k
    u = n - (BLINDING_FACTORS + 1)
    values = [int(x) for x in values]
    N = len(values)
    sel = selector_lookup and L == 0
    n_lookups = L if L else (1 if sel else 0)
    bps, raw, q = assign_with_constraints(b["contexts"], A, max_rows, record)
    raw_of = (lambda p: raw[p]) if record else (lambda p: raw_cell(bps, p))
    lk = assign_lookups_in_phase(b["lookups"], raw_of, N, A, L, selector_lookup, max_rows)
    assign_constants(zip(b["constants"], b["constant_index"]), u, k)
    for x, y in b["advice_equalities"]:
        if x >= N or y >= N:
            raise Panic("virtual cell not assigned")
    if any(int(i) >= N for i in b["constant_index"]):
        raise Panic("virtual cell not assigned")
    sp = spans(bps, N)
    if not record:
        sel_bytes = np.concatenate([np.asarray(s, dtype=bool) for s in b["contexts"]]) if N else np.zeros(0, dtype=bool)
        q = [set() for _ in range(A)]
        for j, (s, cnt) in enumerate(sp):
            end = cnt - 1 if j + 1 < len(sp) else cnt
            q[j] = set((np.flatnonzero(sel_bytes[s:s + end])).tolist())

    def adv(j, r):
        if r >= u or j >= len(sp) or r >= sp[j][1]:
            return 0
        return values[sp[j][0] + r] % R
    gates = []
    for j in range(A):
        bad = []
        rows = range(u) if gate_rows is None else sorted(gate_rows.get(j, ()))
        for r in rows:
            if r in q[j] and (adv(j, r) + adv(j, (r + 1) % n) * adv(j, (r + 2) % n) - adv(j, (r + 3) % n)) % R:
                bad.append(r)
        gates.append(_report(bad, max_report))
    table = set(range(1 << lookup_bits))
    lookups = []
    for t in range(n_lookups):
        bad = []
        if lk is None:
            pass
        elif sel:
            bad = [r for r in lk[1] if r < u and adv(0, r) not in table]
        else:
            col = lk[1][t]
            bad = [r for r in range(min(len(col), u)) if values[int(col[r])] % R not in table]
        lookups.append(_report(bad, max_report))
    E = b["advice_equalities"]
    eq = _report([i for i, (x, y) in enumerate(E) if values[int(x)] % R != values[int(y)] % R], max_report)
    co = _report([i for i, (c, x) in enumerate(zip(b["constants"], b["constant_index"])) if values[int(x)] % R != int(c) % R], max_report)
    return {"gates": gates, "lookups": lookups, "equalities": eq, "constants": co,
            "equality_cells": [(raw_of(int(E[i][0])), raw_of(int(E[i][1]))) for i in eq[1]],
            "constant_cells": [raw_of(int(b["constant_index"][i])) for i in co[1]],
            "break_points": [int(x) for x in bps], "satisfied": not any(c for c, _ in gates + lookups + [eq, co]), "q": q,
            "q_lookup": lk[1] if lk is not None and lk[0] == "q_lookup" else None}


# ------------------------------------------------------------------------------------------------ synthetic builders
def make_builder(rng: np.random.Generator, k: int, A: int, L: int, selector_lookup: bool, lookup_bits: int, max_rows: int,
                 fill: float = 1.0, contexts: int = 1) -> dict:
    """A satisfied keygen-form builder filling about `fill` of the A gate columns.  Chains of 1..8 vertical gates
    x_{t+1} = x_t + b_t c_t laid out [x0, b0, c0, x1, b1, c1, .., x_len, y] with q_enable at every x_t (t < len): consecutive
    gates overlap at distance 3.  b_t is looked up (all of them with the selector lookup, as many as L lookup columns hold
    otherwise), every bit c_t is tied to its constant, every 7th chain's x0 to its own constant, and y copies x_len (one
    advice equality per chain).  Values are canonical and small (uint64).  Returns the builder dict and, under "meta", where
    the cells are (for planting violations)."""
    target = int(fill * (A * (max_rows - 3) - 2))  # every column takes at least max_rows - 3 new cells before it breaks
    lens = []
    total = 0
    while True:
        ln = int(rng.integers(1, 9))
        if total + 3 * ln + 2 > target:
            break
        lens.append(ln)
        total += 3 * ln + 2
    if not lens:
        raise ValueError("make_builder: no room for a chain")
    lens = np.array(lens, dtype=np.int64)
    nch, G = len(lens), int(lens.sum())
    off = np.concatenate([[0], np.cumsum(3 * lens + 2)[:-1]]).astype(np.int64)
    cid = np.repeat(np.arange(nch), lens)
    pos = np.arange(G) - np.repeat(np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
    x_idx = off[cid] + 3 * pos
    b = rng.integers(0, 1 << lookup_bits, size=G, dtype=np.int64).astype(np.uint64)
    c = rng.integers(0, 2, size=G, dtype=np.int64).astype(np.uint64)
    x0 = rng.integers(0, 1 << 32, size=nch, dtype=np.int64).astype(np.uint64)
    inc = b * c
    cs = np.cumsum(inc)
    before = np.concatenate([[0], cs])[np.concatenate([[0], np.cumsum(lens)[:-1]])]  # cs before each chain's first gate
    x_after = x0[cid] + cs - before[cid].astype(np.uint64)                               # x_{t+1}
    x_before = x_after - inc
    N = total
    values = np.zeros(N, dtype=np.uint64)
    values[x_idx], values[x_idx + 1], values[x_idx + 2], values[x_idx + 3] = x_before, b, c, x_after
    y_idx = off + 3 * lens + 1
    values[y_idx] = values[y_idx - 1]
    selectors = np.zeros(N, dtype=np.uint8)
    selectors[x_idx] = 1
    if L == 0 and selector_lookup:
        lookups = x_idx + 1
    elif L:
        lookups = (x_idx + 1)[: min(G, L * (max_rows - 1))]
    else:
        lookups = np.zeros(0, dtype=np.int64)
    tied = off[::7]
    const_index = np.concatenate([x_idx + 2, tied])
    consts = values[const_index]
    cuts = np.sort(rng.choice(np.arange(1, N), size=contexts - 1, replace=False)) if contexts > 1 else np.zeros(0, dtype=np.int64)
    bounds = np.concatenate([[0], cuts, [N]]).astype(np.int64)
    ctx_sel = [selectors[bounds[i]:bounds[i + 1]] for i in range(len(bounds) - 1)]
    return {"values": values, "selectors": selectors, "contexts": ctx_sel,
            "advice_equalities": np.stack([y_idx - 1, y_idx], axis=1).astype(np.uint64),
            "constants": consts.astype(np.uint64), "constant_index": const_index.astype(np.uint64), "lookups": lookups.astype(np.uint64),
            "meta": {"x": x_idx, "b": x_idx + 1, "c": c, "y": y_idx, "chain_start": off, "tied": tied, "lens": lens}}


def plant(rng: np.random.Generator, b: dict, lookup_bits: int, many: int = 0) -> np.ndarray:
    """values with one violation of each kind (gate, lookup, advice equality, constant equality) and `many` more broken advice
    equalities; returns the new values (the builder is not changed)"""
    v = b["values"].copy()
    m = b["meta"]
    free = np.setdiff1d(m["chain_start"], m["tied"])
    v[free[len(free) // 2]] += 1                                    # a chain's x0: its first gate
    looked = set(int(i) for i in b["lookups"])
    zero_c = [int(i) for i, c in zip(m["b"], m["c"]) if c == 0 and int(i) in looked]
    if zero_c:
        v[zero_c[len(zero_c) // 3]] = (1 << lookup_bits) + 5       # a limb outside the table, in a gate with c = 0
    ys = m["y"]
    for y in rng.choice(ys, size=min(len(ys), 1 + many), replace=False):
        v[y] += 1                                                    # y != x_len
    v[m["tied"][-1]] += 2                                            # a tied x0: its constant and its first gate
    return v
