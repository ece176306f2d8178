// h2b200_mock.hpp — MockProver::run + verify for a halo2-base builder in its keygen form (witness_gen_only = false), on the
// device, with no SRS, no sigma and no proving key: what `BaseTester::run_builder` asks of halo2's MockProver
// (halo2-base/src/utils/testing.rs:164-188).  DESIGN.md §4.7.
//
// The builder is passed as halo2-base holds it, every ContextCell mapped by the caller to its index in the virtual column
// (the contexts' ctx.advice concatenated in thread order; index = the context's start + the offset):
//   cells / rational pairs   the witness in either form ProverSession takes (see AssignedWitness);
//   selectors                ctx.selector, one byte per virtual cell;
//   advice_equalities        the copy manager's (ContextCell, ContextCell) pairs as index pairs;
//   constant_equalities      its (F, ContextCell) pairs: Montgomery constants + indices;
//   lookup_index             L > 0: the looked-up cells in assign_raw order; L = 0 with the selector lookup: the cells whose
//                            raw row gets q_lookup;
//   instance_index           per instance column m < n_instance_columns, its assigned_instances as n_instance[m] indices;
//   instance_values          per instance column (MockProver only), the n_instance[m] public values (Montgomery).
// MockProver builds what the keygen pass would assign (assign_with_constraints: break points, advice and q_j columns;
// assign_lookups_in_phase: q_lookup or the lookup-advice columns) and checks, on the device:
//   gates[j]    rows r < u with q_j(r) (a_j(r) + a_j(r+1) a_j(r+2) - a_j(r+3)) != 0, u = 2^k - 7 (rows >= u read as 0);
//   lookups[t]  rows r < u whose input (q_lookup * a0, or l_t) is not among the table's values 0 .. 2^lookup_bits - 1;
//   equalities  advice equalities i with value(a_i) != value(b_i);
//   constants   constant equalities i with value(cell_i) != c_i;
//   instances[m] rows r of instance column m with value(instance_index_m[r]) != instance_values_m[r].
// One deliberate difference from halo2's MockProver: a copy failure is counted per violated equality, not per cell against its
// sigma image; both are zero exactly when every equality holds.  The lookup-advice copies of assign_raw hold by construction (the
// columns are filled from the indices).  The number F of constants columns (num_fixed) changes no value check, only where the
// constants fit: D distinct constants need D <= F u (DESIGN.md §4.11), and MockReport::distinct_constants returns D, the number
// calculate_params sizes num_fixed from.
#pragma once
#include <algorithm>
#include <string>

#include "h2b200_prover.hpp"

namespace h2b {

struct BuilderView {
    const Fr* cells = nullptr;
    size_t n_cells = 0;
    const uint64_t* rational_index = nullptr;
    const Fr* rational_den = nullptr;
    size_t n_rational = 0;
    const uint8_t* selectors = nullptr;  // n_cells bytes
    const uint64_t* advice_equalities = nullptr;  // 2 x n_advice_equalities: (a, b) pairs
    size_t n_advice_equalities = 0;
    const Fr* constants = nullptr;  // n_constant_equalities Montgomery constants, with constant_index[i] the cell tied to constants[i]
    const uint64_t* constant_index = nullptr;
    size_t n_constant_equalities = 0;
    const uint64_t* lookup_index = nullptr;
    size_t n_lookup = 0;
    const uint64_t* const* instance_index = nullptr;
    const Fr* const* instance_values = nullptr;
    const size_t* n_instance = nullptr;
    size_t n_instance_columns = 0;
};

// a cell of the assignment: gate-advice column and row
struct RawCell {
    uint64_t column = 0, row = 0;
    bool operator==(const RawCell& o) const { return column == o.column && row == o.row; }
};

struct MockReport {
    bool satisfied = true;
    std::vector<uint64_t> break_points;
    std::vector<ReportItem> gates, lookups;
    ReportItem equalities, constants;
    std::vector<std::pair<RawCell, RawCell>> equality_cells;  // both raw cells of every reported advice equality
    std::vector<RawCell> constant_cells;                      // the raw advice cell of every reported constant equality
    std::vector<ReportItem> instances;                        // per instance column: the failing rows
    std::vector<std::vector<RawCell>> instance_cells;         // per instance column: the raw advice cell of every reported row
    uint64_t distinct_constants = 0;                          // D: the distinct constants among the constant equalities
};

// ------------------------------------------------------------------------------------------------ what MockProver and keygen share
// the shape of a builder, checked; messages start with `who`.  max_rows = 2^k - unusable_rows, as calculate_params gets it; it
// must leave the blinding rows alone (<= 2^k - 7)
inline CircuitShape builder_shape(const std::string& who, uint32_t k, size_t A, size_t L, bool selector_lookup, uint32_t lookup_bits, size_t max_rows,
                                  size_t I = 0, size_t F = 1) {
    if (k < 3 || k > 28) throw Error(H2B_ERR_ARG, who + ": k out of range (3..28)");
    if (F >= (size_t(1) << 32)) throw Error(H2B_ERR_ARG, who + ": too many constants columns");
    CircuitShape s(k, A, L, selector_lookup, I, F);
    if (A < 1) throw Error(H2B_ERR_ARG, who + ": no gate columns");
    if (s.selector_lookup && A != 1) throw Error(H2B_ERR_ARG, who + ": the selector lookup needs exactly one gate column");
    if (max_rows < 1 || max_rows > s.u) throw Error(H2B_ERR_ARG, who + ": max_rows must be in 1..2^k - 7");
    if (s.n_lookups && (lookup_bits > 28 || (size_t(1) << lookup_bits) > s.u))
        throw Error(H2B_ERR_ARG, who + ": the lookup table does not fit the usable rows");
    return s;
}

// the range table 0 .. 2^bits - 1 (Montgomery), zero-padded to n rows
inline std::vector<Fr> lookup_table(size_t n, uint32_t bits) {
    std::vector<Fr> t(n, Fr{});
    Fr x{}, one = HostFr::one();
    for (size_t i = 0; i < (size_t(1) << bits); i++, x = HostFr::add(x, one)) t[i] = x;
    return t;
}

// assign_with_constraints' break points by its closed form (O(1) selector probes per column).  In column j the walk breaks
// at the first row r >= r_min (0 in column 0, 1 after a break: row 0 holds the copied break cell) where
// (selector && r + 4 > max_rows) || r >= max_rows - 1, i.e. at r in {max_rows - 3, max_rows - 2} with the selector set or
// else at max_rows - 1, if that cell exists.  Panics of the walk -> H2B_ERR_ARG with halo2-base's text.  The overlap
// assertion reads the two cells before the break in the virtual column (halo2-base reads them within the break's context).
inline std::vector<uint64_t> break_points_of(const uint8_t* sel, size_t N, size_t A, size_t max_rows) {
    std::vector<uint64_t> bps;
    const std::string no_cols = "NOT ENOUGH ADVICE COLUMNS. Perhaps blinding factors were not taken into account. The max non-poisoned rows is " +
                                std::to_string(max_rows);
    if (N == 0) return bps;
    if (A == 0) throw Error(H2B_ERR_ARG, no_cols);
    size_t s = 0, r_min = 0;
    for (;;) {
        size_t r = std::max(r_min, max_rows >= 3 ? max_rows - 3 : size_t(0));
        while (r < max_rows - 1 && !(s + r < N && sel[s + r])) r++;
        const size_t p = s + r;
        if (p >= N) return bps;
        for (size_t delta = 1; delta <= 2; delta++)
            if (p >= 2 && sel[p - delta]) throw Error(H2B_ERR_ARG, "We do not support overlaps with delta = " + std::to_string(delta));
        bps.push_back(r);
        if (bps.size() >= A) throw Error(H2B_ERR_ARG, no_cols);
        s = p;
        r_min = 1;
    }
}

// the host side of a builder's keygen pass: every count > 0 needs its array (with `values`, the cells and the Rational pairs
// too), the break points, and the two range-lookup panics of assign_lookups_in_phase
inline std::vector<uint64_t> builder_break_points(const CircuitShape& s, const std::string& who, size_t max_rows, const BuilderView& b, bool values) {
    if ((b.n_cells && !(b.selectors && (b.cells || !values))) || (values && b.n_rational && !(b.rational_index && b.rational_den)) ||
        (b.n_advice_equalities && !b.advice_equalities) || (b.n_constant_equalities && !(b.constants && b.constant_index)) || (b.n_lookup && !b.lookup_index))
        throw Error(H2B_ERR_ARG, who + ": a count > 0 needs its array");
    check_instances(who, s, b.instance_index, b.n_instance, b.n_instance_columns, values);  // keygen: the copies find rows >= u
    if (values) check_instances(who, s, b.instance_values, b.n_instance, b.n_instance_columns);
    std::vector<uint64_t> bps = break_points_of(b.selectors, b.n_cells, s.A, max_rows);
    if (b.n_lookup) {
        if (s.L && (b.n_lookup + s.L - 1) / s.L > max_rows) throw Error(H2B_ERR_ARG, "range lookups would be assigned to unusable rows");
        if (!s.L && !s.selector_lookup) throw Error(H2B_ERR_ARG, "range lookups require lookup advice columns");
    }
    return bps;
}

// halo2-base's panics for what the device found, in the order of the keygen pass: the lookups, then assign_raw (constants
// placed first, then the equalities resolved).  assign_raw places distinct constant d at row d div F of constants column
// d mod F, so the first one that does not fit is d = F u, whose row reaches u: D > F u distinct constants is halo2's
// NotEnoughRowsAvailable.  calculate_params sizes F by 2^k, not u, so F u < D <= F 2^k fails in halo2-base too.  With F = 0
// the first constant indexes an empty column list (`config[0]`).
inline void builder_panics(const CircuitShape& s, bool lookup_unassigned, bool unusable_row, uint64_t distinct_constants, bool equality_unassigned) {
    if (lookup_unassigned) throw Error(H2B_ERR_ARG, "virtual cell not assigned");
    if (unusable_row) throw Error(H2B_ERR_ARG, "range lookup assigned to an unusable row");
    if (distinct_constants && s.F == 0) throw Error(H2B_ERR_ARG, "index out of bounds: the len is 0 but the index is 0");
    if (distinct_constants > s.F * s.u)
        throw Error(H2B_ERR_ARG, "NotEnoughRowsAvailable { current_k: " + std::to_string(s.k) + " }: " + std::to_string(distinct_constants) +
                                     " distinct constants for the " + std::to_string(s.F * s.u) + " usable cells of " + std::to_string(s.F) +
                                     " constants column" + (s.F > 1 ? "s" : ""));
    if (equality_unassigned) throw Error(H2B_ERR_ARG, "virtual cell not assigned");
}

class MockProver : public CircuitShape {
public:
    // max_rows as for builder_shape; F constants columns
    MockProver(const Context& ctx, uint32_t k, size_t A, size_t L, bool selector_lookup, uint32_t lookup_bits, size_t max_rows, size_t I = 0,
               size_t F = 1)
        : CircuitShape(builder_shape("MockProver", k, A, L, selector_lookup, lookup_bits, max_rows, I, F)), ctx(ctx), lookup_bits(lookup_bits),
          max_rows(max_rows) {
        adv = std::make_unique<Poly>(ctx, n * (A + L));
        q = std::make_unique<Poly>(ctx, n * A);
        if (n_lookups) {
            table = std::make_unique<Poly>(ctx, n);
            table->upload(lookup_table(n, lookup_bits).data(), n);
        }
        if (this->selector_lookup) {
            q_lookup = std::make_unique<Poly>(ctx, n);
            input = std::make_unique<Poly>(ctx, n);
        }
        gate = add_vertical_gate(ev, 0);  // bound to q{j}, a{j} per gate column
    }

    // the cell assigned_advices records for virtual index p: a break cell belongs to the column it ends
    static RawCell raw_cell(const std::vector<uint64_t>& bps, uint64_t p) {
        uint64_t s = 0;
        for (size_t j = 0; j < bps.size(); j++) {
            if (p <= s + bps[j]) return {j, p - s};
            s += bps[j];
        }
        return {bps.size(), p - s};
    }

    MockReport run(const BuilderView& b, size_t max_report = 16) {
        const size_t N = b.n_cells, M = b.n_advice_equalities, Mc = b.n_constant_equalities;
        h2b_ctx* c = ctx.raw();
        if (max_report < 1 || max_report > H2B_CHECK_MAX_REPORT) throw Error(H2B_ERR_ARG, "MockProver: max_report out of range");
        MockReport out;
        out.break_points = builder_break_points(*this, "MockProver", max_rows, b, true);
        // element 0 of the report block: the verdict words (rational, lookup index, q_lookup, advice eq, constant eq, distinct);
        // then the reports (gates, lookups, equalities, constants, instances); then one status word per instance column
        const size_t W = max_report + 1, n_items = A + n_lookups + 2 + I, rep_elems = 1 + (n_items * W + 3) / 4, elems = rep_elems + (I + 7) / 8;
        Poly* rep = grown(ctx, rep_, elems);
        const Fr zero{};
        rep->upload(&zero, 1);
        uint32_t* verdict = static_cast<uint32_t*>(rep->at(0));
        auto at = [&](size_t i) { return static_cast<char*>(rep->at(1)) + 8 * W * i; };
        WitnessView w;
        w.cells = b.cells;
        w.n_cells = N;
        w.break_points = out.break_points.data();
        w.n_break_points = out.break_points.size();
        w.rational_index = b.rational_index;
        w.rational_den = b.rational_den;
        w.n_rational = b.n_rational;
        if (L) {
            w.lookup_index = b.lookup_index;
            w.n_lookup = b.n_lookup;
        }
        assign_witness(ctx, *this, w, true, verdict, adv->at(), wit_);
        const void* cells = wit_.cells->at();
        const uint64_t* bp = out.break_points.empty() ? nullptr : out.break_points.data();
        upload_bytes(ctx, sel_, b.selectors, N);
        ctx.check(h2b_mock_selectors_dev(c, sel_->at(), N, bp, out.break_points.size(), k, A, q->at()));
        if (selector_lookup) {
            upload_bytes(ctx, wit_.lookups, b.lookup_index, 8 * b.n_lookup);
            ctx.check(h2b_mock_lookup_selector_dev(c, wit_.lookups->at(), b.n_lookup, N, max_rows, k, q_lookup->at(), verdict + 2));
            ctx.check(h2b_fr_mul_elementwise_dev(c, q_lookup->at(), adv->at(), n, input->at()));
        }
        upload_bytes(ctx, eq_, b.advice_equalities, 16 * M);
        ctx.check(h2b_check_equalities_dev(c, cells, N, eq_->at(), M, max_report, at(A + n_lookups), verdict + 3));
        upload_bytes(ctx, const_, b.constants, 32 * Mc);
        upload_bytes(ctx, const_idx_, b.constant_index, 8 * Mc);
        ctx.check(h2b_check_constants_dev(c, cells, N, const_->at(), const_idx_->at(), Mc, max_report, at(A + n_lookups + 1), verdict + 4));
        ctx.check(h2b_count_distinct_dev(c, const_->at(), Mc, verdict + 5));
        // the instance copies of assign_instances, as the constant check: cell instance_index_m[r] against public value r
        inst_.resize(2 * I);
        for (size_t m = 0; m < I; m++) {
            upload_bytes(ctx, inst_[2 * m], b.instance_values[m], 32 * b.n_instance[m]);
            upload_bytes(ctx, inst_[2 * m + 1], b.instance_index[m], 8 * b.n_instance[m]);
            ctx.check(h2b_check_constants_dev(c, cells, N, inst_[2 * m]->at(), inst_[2 * m + 1]->at(), b.n_instance[m], max_report,
                                              at(A + n_lookups + 2 + m), static_cast<uint32_t*>(rep->at(rep_elems)) + m));
        }
        for (size_t j = 0; j < A; j++) {
            const BoundGraph g(ev, gate, {q->at(j * n)}, {adv->at(j * n)});
            ctx.check(h2b_check_graph_dev(c, g.get(), k, u, max_report, at(j)));
        }
        for (size_t t = 0; t < n_lookups; t++)
            ctx.check(h2b_check_lookup_dev(c, L ? adv->at((A + t) * n) : input->at(), table->at(), k, u, max_report, at(A + t)));
        const std::vector<Fr> raw = rep->download(0, elems);
        const uint32_t* v = reinterpret_cast<const uint32_t*>(raw[0].data());
        if (v[0] & 1) throw Error(H2B_ERR_ARG, "MockProver: a Rational index is >= the witness length");
        if (v[0] & 2) throw Error(H2B_ERR_ARG, "MockProver: the Rational indices do not strictly increase");
        builder_panics(*this, (v[1] | v[2]) & 1, v[2] & 2, v[5], (v[3] | v[4]) & 1);
        const uint32_t* inst_status = reinterpret_cast<const uint32_t*>(raw[rep_elems].data());
        for (size_t m = 0; m < I; m++)
            if (inst_status[m] & 1) throw Error(H2B_ERR_ARG, "instance not assigned");
        out.distinct_constants = v[5];
        const std::vector<ReportItem> items = decode_reports(raw[1].data(), n_items, max_report, out.satisfied);
        out.gates.assign(items.begin(), items.begin() + A);
        out.lookups.assign(items.begin() + A, items.begin() + A + n_lookups);
        out.equalities = items[A + n_lookups];
        out.constants = items[A + n_lookups + 1];
        for (uint64_t i : out.equalities.second)
            out.equality_cells.push_back({raw_cell(out.break_points, b.advice_equalities[2 * i]), raw_cell(out.break_points, b.advice_equalities[2 * i + 1])});
        for (uint64_t i : out.constants.second) out.constant_cells.push_back(raw_cell(out.break_points, b.constant_index[i]));
        out.instances.assign(items.begin() + A + n_lookups + 2, items.end());
        for (size_t m = 0; m < I; m++) {
            out.instance_cells.emplace_back();
            for (uint64_t r : out.instances[m].second) out.instance_cells[m].push_back(raw_cell(out.break_points, b.instance_index[m][r]));
        }
        return out;
    }

    // a column of the last run, for tests: a{j}, l{t}, q{j}, q_lookup, table (2^k Lagrange values each)
    NamedColumn column(const std::string& name) const {
        auto idx = [&](const char* p, size_t count) -> size_t {
            const size_t len = std::strlen(p);
            if (name.compare(0, len, p) != 0 || name.size() == len || name.find_first_not_of("0123456789", len) != std::string::npos) return SIZE_MAX;
            const size_t i = std::stoul(name.substr(len));
            return i < count ? i : SIZE_MAX;
        };
        if (name == "q_lookup" && q_lookup) return {{q_lookup.get(), 0}, n};
        if (name == "table" && table) return {{table.get(), 0}, n};
        if (idx("a", A) != SIZE_MAX) return {{adv.get(), idx("a", A) * n}, n};
        if (idx("l", L) != SIZE_MAX) return {{adv.get(), (A + idx("l", L)) * n}, n};
        if (idx("q", A) != SIZE_MAX) return {{q.get(), idx("q", A) * n}, n};
        throw Error(H2B_ERR_ARG, "MockProver: no column " + name);
    }

    const Context& ctx;
    uint32_t lookup_bits;
    size_t max_rows;

private:
    GraphEvaluator ev;
    ValueSource gate{};
    PolyPtr adv, q, q_lookup, input, table;
    WitnessBuffers wit_;
    PolyPtr sel_, eq_, const_, const_idx_, rep_;
    std::vector<PolyPtr> inst_;  // per instance column: its public values, its indices
};

}  // namespace h2b
