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
//                            raw row gets q_lookup.
// MockProver builds what the keygen pass would assign (assign_with_constraints: break points, advice and q_j columns;
// assign_lookups_in_phase: q_lookup or the lookup-advice columns) and checks, on the device:
//   gates[j]    rows r < u with q_j(r) (a_j(r) + a_j(r+1) a_j(r+2) - a_j(r+3)) != 0, u = 2^k - 7 (rows >= u read as 0);
//   lookups[t]  rows r < u whose input (q_lookup * a0, or l_t) is not among the table's values 0 .. 2^lookup_bits - 1;
//   equalities  advice equalities i with value(a_i) != value(b_i);
//   constants   constant equalities i with value(cell_i) != c_i.
// One deliberate difference from halo2's MockProver: a copy failure is counted per violated equality, not per cell against its
// sigma image; both are zero exactly when every equality holds.  Instance columns and several constants columns are not
// covered; the lookup-advice copies of assign_raw hold by construction (the columns are filled from the indices).
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
};

// a cell of the assignment: gate-advice column and row
struct RawCell {
    uint64_t column = 0, row = 0;
    bool operator==(const RawCell& o) const { return column == o.column && row == o.row; }
};

// each report: (failure count, the first min(count, max_report) failing rows or equality indices, ascending)
struct MockReport {
    bool satisfied = true;
    std::vector<uint64_t> break_points;
    std::vector<std::pair<uint64_t, std::vector<uint64_t>>> gates, lookups;
    std::pair<uint64_t, std::vector<uint64_t>> equalities, constants;
    std::vector<std::pair<RawCell, RawCell>> equality_cells;  // both raw cells of every reported advice equality
    std::vector<RawCell> constant_cells;                      // the raw advice cell of every reported constant equality
};

class MockProver {
public:
    static constexpr size_t BLINDING_FACTORS = 6;

    // max_rows = 2^k - unusable_rows, as calculate_params gets it; it must leave the blinding rows alone (<= 2^k - 7)
    MockProver(const Context& ctx, uint32_t k, size_t A, size_t L, bool selector_lookup, uint32_t lookup_bits, size_t max_rows)
        : ctx(ctx), k(k), A(A), L(L), selector_lookup(selector_lookup && L == 0), lookup_bits(lookup_bits), max_rows(max_rows) {
        if (k < 3 || k > 28) throw Error(H2B_ERR_ARG, "MockProver: k out of range (3..28)");
        n = size_t(1) << k;
        u = n - (BLINDING_FACTORS + 1);
        if (A < 1) throw Error(H2B_ERR_ARG, "MockProver: no gate columns");
        if (this->selector_lookup && A != 1) throw Error(H2B_ERR_ARG, "MockProver: the selector lookup needs exactly one gate column");
        if (max_rows < 1 || max_rows > u) throw Error(H2B_ERR_ARG, "MockProver: max_rows must be in 1..2^k - 7");
        n_lookups = L ? L : (this->selector_lookup ? 1 : 0);
        adv = std::make_unique<Poly>(ctx, n * (A + L));
        q = std::make_unique<Poly>(ctx, n * A);
        if (n_lookups) {
            if (lookup_bits > 28 || (size_t(1) << lookup_bits) > u) throw Error(H2B_ERR_ARG, "MockProver: the lookup table does not fit the usable rows");
            std::vector<Fr> t(n, Fr{});
            Fr x{}, one = HostFr::one();
            for (size_t i = 0; i < (size_t(1) << lookup_bits); i++, x = HostFr::add(x, one)) t[i] = x;
            table = std::make_unique<Poly>(ctx, n);
            table->upload(t.data(), n);
        }
        if (this->selector_lookup) {
            q_lookup = std::make_unique<Poly>(ctx, n);
            input = std::make_unique<Poly>(ctx, n);
        }
        // the vertical gate on fixed slot 0 / advice slot 0, bound to q{j}, a{j} per gate column
        const uint32_t r0 = ev.add_rotation(0), r1 = ev.add_rotation(1), r2 = ev.add_rotation(2), r3 = ev.add_rotation(3);
        auto a = [&](uint32_t rot) { return ev.add_calculation(Calculation::Store(ValueSource::Advice(0, rot))); };
        const ValueSource qs = ev.add_calculation(Calculation::Store(ValueSource::Fixed(0, r0)));
        const ValueSource a0 = a(r0), a1 = a(r1), a2 = a(r2), a3 = a(r3);
        const ValueSource sum = ev.add_calculation(Calculation::Add(a0, ev.add_calculation(Calculation::Mul(a1, a2))));
        gate = ev.add_calculation(Calculation::Mul(qs, ev.add_calculation(Calculation::Sub(sum, a3))));
        program = ev.program();
    }

    // assign_with_constraints' break points by its closed form (O(1) selector probes per column).  In column j the walk breaks
    // at the first row r >= r_min (0 in column 0, 1 after a break: row 0 holds the copied break cell) where
    // (selector && r + 4 > max_rows) || r >= max_rows - 1, i.e. at r in {max_rows - 3, max_rows - 2} with the selector set or
    // else at max_rows - 1, if that cell exists.  Panics of the walk -> H2B_ERR_ARG with halo2-base's text.  The overlap
    // assertion reads the two cells before the break in the virtual column (halo2-base reads them within the break's context).
    static std::vector<uint64_t> break_points_of(const uint8_t* sel, size_t N, size_t A, size_t max_rows) {
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
        const size_t N = b.n_cells, M = b.n_advice_equalities, Mc = b.n_constant_equalities, R = b.n_rational;
        h2b_ctx* c = ctx.raw();
        if (max_report < 1 || max_report > H2B_CHECK_MAX_REPORT) throw Error(H2B_ERR_ARG, "MockProver: max_report out of range");
        if ((N && !(b.cells && b.selectors)) || (R && !(b.rational_index && b.rational_den)) || (M && !b.advice_equalities) ||
            (Mc && !(b.constants && b.constant_index)) || (b.n_lookup && !b.lookup_index))
            throw Error(H2B_ERR_ARG, "MockProver: a count > 0 needs its array");
        MockReport out;
        out.break_points = break_points_of(b.selectors, N, A, max_rows);
        if (b.n_lookup) {
            if (L && (b.n_lookup + L - 1) / L > max_rows) throw Error(H2B_ERR_ARG, "range lookups would be assigned to unusable rows");
            if (!L && !selector_lookup) throw Error(H2B_ERR_ARG, "range lookups require lookup advice columns");
        }
        // element 0 of the report block: the verdict words (rational, lookup index, q_lookup, advice eq, constant eq, distinct)
        const size_t W = max_report + 1, n_items = A + n_lookups + 2, elems = 1 + (n_items * W + 3) / 4;
        Poly* rep = grown(rep_, elems);
        const Fr zero{};
        rep->upload(&zero, 1);
        uint32_t* verdict = static_cast<uint32_t*>(rep->at(0));
        auto at = [&](size_t i) { return static_cast<char*>(rep->at(1)) + 8 * W * i; };
        upload(cells_, b.cells, 32 * N);
        if (R) {
            upload(rat_idx_, b.rational_index, 8 * R);
            upload(rat_den_, b.rational_den, 32 * R);
        }
        ctx.check(h2b_apply_rational_dev(c, cells_->at(), N, R ? rat_idx_->at() : nullptr, R ? rat_den_->at() : nullptr, R, verdict));
        const uint64_t* bp = out.break_points.empty() ? nullptr : out.break_points.data();
        ctx.check(h2b_assign_columns_dev(c, cells_->at(), N, bp, out.break_points.size(), k, A, adv->at()));
        upload(sel_, b.selectors, N);
        ctx.check(h2b_mock_selectors_dev(c, sel_->at(), N, bp, out.break_points.size(), k, A, q->at()));
        upload(lk_idx_, b.lookup_index, 8 * b.n_lookup);
        if (L)
            ctx.check(h2b_assign_lookups_indexed_dev(c, cells_->at(), N, lk_idx_->at(), b.n_lookup, k, L, adv->at(A * n), verdict + 1));
        if (selector_lookup) {
            ctx.check(h2b_mock_lookup_selector_dev(c, lk_idx_->at(), b.n_lookup, N, max_rows, k, q_lookup->at(), verdict + 2));
            ctx.check(h2b_fr_mul_elementwise_dev(c, q_lookup->at(), adv->at(), n, input->at()));
        }
        upload(eq_, b.advice_equalities, 16 * M);
        ctx.check(h2b_check_equalities_dev(c, cells_->at(), N, eq_->at(), M, max_report, at(A + n_lookups), verdict + 3));
        upload(const_, b.constants, 32 * Mc);
        upload(const_idx_, b.constant_index, 8 * Mc);
        ctx.check(h2b_check_constants_dev(c, cells_->at(), N, const_->at(), const_idx_->at(), Mc, max_report, at(A + n_lookups + 1), verdict + 4));
        ctx.check(h2b_count_distinct_dev(c, const_->at(), Mc, verdict + 5));
        for (size_t j = 0; j < A; j++) {
            const void* fx[1] = {q->at(j * n)};
            const void* ad[1] = {adv->at(j * n)};
            const h2b_graph g = bind(fx, ad);
            ctx.check(h2b_check_graph_dev(c, &g, k, u, max_report, at(j)));
        }
        for (size_t t = 0; t < n_lookups; t++)
            ctx.check(h2b_check_lookup_dev(c, L ? adv->at((A + t) * n) : input->at(), table->at(), k, u, max_report, at(A + t)));
        const std::vector<Fr> raw = rep->download(0, elems);
        const uint32_t* v = reinterpret_cast<const uint32_t*>(raw[0].data());
        if (v[0] & 1) throw Error(H2B_ERR_ARG, "MockProver: a Rational index is >= the witness length");
        if (v[0] & 2) throw Error(H2B_ERR_ARG, "MockProver: the Rational indices do not strictly increase");
        // in the order of the keygen pass: the lookups, then assign_raw (constants placed first, then the equalities resolved)
        if ((v[1] | v[2]) & 1) throw Error(H2B_ERR_ARG, "virtual cell not assigned");
        if (v[2] & 2) throw Error(H2B_ERR_ARG, "range lookup assigned to an unusable row");
        if (v[5] > u)
            throw Error(H2B_ERR_ARG, "NotEnoughRowsAvailable { current_k: " + std::to_string(k) + " }: " + std::to_string(v[5]) +
                                         " distinct constants for the " + std::to_string(u) + " usable rows of the constants column");
        if ((v[3] | v[4]) & 1) throw Error(H2B_ERR_ARG, "virtual cell not assigned");
        const uint64_t* w = raw[1].data();
        auto item = [&](size_t i) {
            const uint64_t* r = w + W * i;
            out.satisfied = out.satisfied && r[0] == 0;
            return std::pair<uint64_t, std::vector<uint64_t>>{r[0], std::vector<uint64_t>(r + 1, r + 1 + std::min<uint64_t>(r[0], max_report))};
        };
        for (size_t j = 0; j < A; j++) out.gates.push_back(item(j));
        for (size_t t = 0; t < n_lookups; t++) out.lookups.push_back(item(A + t));
        out.equalities = item(A + n_lookups);
        out.constants = item(A + n_lookups + 1);
        for (uint64_t i : out.equalities.second)
            out.equality_cells.push_back({raw_cell(out.break_points, b.advice_equalities[2 * i]), raw_cell(out.break_points, b.advice_equalities[2 * i + 1])});
        for (uint64_t i : out.constants.second) out.constant_cells.push_back(raw_cell(out.break_points, b.constant_index[i]));
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
    uint32_t k;
    size_t n = 0, u = 0, A, L;
    bool selector_lookup;
    uint32_t lookup_bits;
    size_t max_rows, n_lookups = 0;

private:
    // bytes from the host into a buffer reallocated only when a run needs more than any run before it
    void upload(PolyPtr& p, const void* host, size_t bytes) {
        const size_t full = bytes / 32, tail = bytes % 32;
        if (!p || p->len() < full + 1) p = std::make_unique<Poly>(ctx, full + 1);
        if (full) p->upload(static_cast<const Fr*>(host), full);
        if (tail) {
            Fr last{};
            std::memcpy(last.data(), static_cast<const char*>(host) + 32 * full, tail);
            p->upload(&last, 1, full);
        }
    }
    Poly* grown(PolyPtr& p, size_t m) {
        if (!p || p->len() < m) p = std::make_unique<Poly>(ctx, m);
        return p.get();
    }
    h2b_graph bind(const void* const* fixed, const void* const* advice) const {
        h2b_graph g{};
        g.program = program.data();
        g.program_words = program.size();
        g.n_calculations = uint32_t(ev.calculations.size());
        g.result = gate.word();
        g.constants = reinterpret_cast<const uint64_t*>(ev.constants.data());
        g.n_constants = ev.constants.size();
        g.rotations = ev.rotations.data();
        g.n_rotations = ev.rotations.size();
        g.fixed = fixed;
        g.n_fixed = 1;
        g.advice = advice;
        g.n_advice = 1;
        return g;
    }

    GraphEvaluator ev;
    ValueSource gate{};
    std::vector<uint32_t> program;
    PolyPtr adv, q, q_lookup, input, table;
    PolyPtr cells_, rat_idx_, rat_den_, sel_, lk_idx_, eq_, const_, const_idx_, rep_;
};

}  // namespace h2b
