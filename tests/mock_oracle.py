"""MockProver::verify restated literally on Python integers, for the constraint system the resident prover proves (A gate
columns with the vertical gate, the selector lookup or L lookup-advice columns, equality on [c, a0.., l0..]).  It is the
yardstick of ProverSession.check (tests/test_gpu_check.py) and shares no method with the device: every gate is evaluated
row by row, the table is a Python set, and sigma is decoded through a dict {delta^c omega^r: (c, r)} built from the
definition (no v^n trick, no hash table of omega powers, no sort).

Values are canonical integers.  The values checked are those a proof commits before blinding: the assigned columns with
rows >= u read as 0 (u = n - (BLINDING_FACTORS + 1)); the fixed columns as they are.  Reports have the device's form:
(failure count, the first max_report failing rows in ascending order)."""
from oracle import pyref

R = pyref.R
BLINDING_FACTORS = 6


def assign(k: int, A: int, L: int, virtual, break_points, lookup_cells):
    """the A + L advice columns the assignment lays out (halo2-base's column walk and assign_raw)"""
    n = 1 << k
    cols = pyref.assign_witnesses([list(virtual)], [int(b) for b in break_points], A, n)
    if L:
        cols += pyref.assign_lookups(list(lookup_cells), L, n)
    return [list(c) for c in cols]


def sigma_dict(k: int, n_cols: int, cells=None) -> dict:
    """{delta^c omega^r: (c, r)} for every cell (c, r) of the permutation, or only for `cells`"""
    n, w = 1 << k, pyref.omega_for(k)
    if cells is None:
        cells = [(c, r) for c in range(n_cols) for r in range(n)]
    return {pow(pyref.DELTA, c, R) * pow(w, r, R) % R: (c, r) for c, r in cells}


def decode_sigma(k: int, sigma, cells=None, targets=None):
    """(targets of the cells, malformed cells): sigma_c(r) looked up in sigma_dict; `cells` restricts which entries are decoded,
    `targets` which cells the dict holds (both default to every cell)"""
    n, npc = 1 << k, len(sigma)
    d = sigma_dict(k, npc, targets)
    cells = [(c, r) for c in range(npc) for r in range(n)] if cells is None else cells
    out, bad = {}, []
    for c, r in cells:
        t = d.get(sigma[c][r] % R)
        if t is None:
            bad.append((c, r))
        else:
            out[(c, r)] = t
    return out, bad


def _report(rows, max_report):
    rows = sorted(set(rows))
    return (len(rows), rows[:max_report])


def verify(k: int, A: int, L: int, sel: bool, fixed: dict, sigma, cols, max_report: int = 16, only=None) -> dict:
    """the three checks over every row, or (`only`) over the rows the caller names: a dict with keys "gates" {j: rows},
    "lookups" {t: rows}, "copies" {c: rows} (missing keys: nothing checked there) and "targets" (the cells sigma_dict holds).
    A malformed sigma entry raises ValueError naming it."""
    n = 1 << k
    u = n - (BLINDING_FACTORS + 1)
    npc = 1 + A + L
    sel = sel and L == 0
    n_lookups = L if L else (1 if sel else 0)
    val = lambda col, r: col[r] % R if r < u else 0  # an advice cell as committed before blinding
    pick = lambda key, i, default: default if only is None else sorted(only.get(key, {}).get(i, ()))
    gates = []
    for j in range(A):
        q, a = fixed["q%d" % j], cols[j]
        bad = []
        for r in pick("gates", j, range(u)):
            g = q[r] * (val(a, r) + val(a, (r + 1) % n) * val(a, (r + 2) % n) - val(a, (r + 3) % n)) % R
            if g:
                bad.append(r)
        gates.append(_report(bad, max_report))
    table = {fixed["table"][r] % R for r in range(u)} if n_lookups else set()
    lookups = []
    for t in range(n_lookups):
        bad = []
        for r in pick("lookups", t, range(u)):
            x = fixed["q_lookup"][r] * val(cols[0], r) % R if L == 0 else val(cols[A + t], r)
            if x not in table:
                bad.append(r)
        lookups.append(_report(bad, max_report))
    value = lambda c, r: fixed["c"][r] % R if c == 0 else val(cols[c - 1], r)
    cells = None if only is None else [(c, r) for c in range(npc) for r in pick("copies", c, ())]
    targets, malformed = decode_sigma(k, sigma, cells, None if only is None else only["targets"])
    if malformed:
        raise ValueError("sigma entry at (column, row) %s is not delta^c omega^r" % (malformed[0],))
    copies = []
    for c in range(npc):
        rows = range(n) if only is None else pick("copies", c, ())
        copies.append(_report([r for r in rows if value(c, r) != value(*targets[(c, r)])], max_report))
    reps = gates + lookups + copies
    return {"satisfied": not any(cnt for cnt, _ in reps), "gates": gates, "lookups": lookups, "copies": copies}


def malformed_sigma(k: int, sigma, max_report: int = 16):
    """per permutation column: the report of the sigma entries that name no cell"""
    _, bad = decode_sigma(k, sigma)
    return [_report([r for c2, r in bad if c2 == c], max_report) for c in range(len(sigma))]
