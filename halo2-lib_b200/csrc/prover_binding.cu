// prover_binding.cu — the private C binding of the resident prover (include/h2b200_prover.hpp) that halo2-lib_b200/prover.py
// calls through ctypes.  The calls are the Python package's binding, not product ABI: include/h2b200.h does not declare them.
// Host code only.  No exception leaves this file: every call maps failures to a status code + h2b_last_error().
#include <algorithm>
#include <array>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "h2b_internal.cuh"

// the header's inline code stays private to the library: programs that include the header never bind to this copy
#pragma GCC visibility push(hidden)
#include "../../include/h2b200_prover.hpp"
#include "../../include/h2b200_mock.hpp"
#include "../../include/h2b200_keygen.hpp"

namespace h2bp {
using namespace h2b;

struct BoundCircuit {
    Context ctx;
    std::unique_ptr<ProverCircuit> cs;  // built against ctx (a circuit keeps a reference to its context)
    explicit BoundCircuit(h2b_ctx* c) : ctx(c) {}
};
struct BoundMock {
    Context ctx;
    MockProver mock;
    BoundMock(h2b_ctx* c, uint32_t k, size_t A, size_t L, bool sel, uint32_t lookup_bits, size_t max_rows, size_t I, size_t F)
        : ctx(c), mock(ctx, k, A, L, sel, lookup_bits, max_rows, I, F) {}
};
struct BoundSession {
    Context ctx;
    ParamsKZG params;
    ProverSession sess;
    BoundSession(h2b_ctx* c, h2b_srs* srs, uint32_t k, size_t srs_count, const ProverCircuit& cs)
        : ctx(c), params(ctx, k, srs, srs_count), sess(ctx, params, cs) {}
};

// Runs `body` and translates every failure.  The context lock is taken only to store the message: the prover calls the public
// entry points, which take that (non-recursive) lock themselves.
template <class Fn>
int run(h2b_ctx* ctx, Fn&& body) {
    if (!ctx) return H2B_ERR_ARG;
    int code;
    std::string msg;
    try {
        body();
        return H2B_OK;
    } catch (const Error& e) {
        code = e.code;
        msg = e.what();
        const std::string prefix = "h2b200 error " + std::to_string(e.code) + ": ";
        if (msg.compare(0, prefix.size(), prefix) == 0) msg.erase(0, prefix.size());
    } catch (const std::bad_alloc&) {
        code = H2B_ERR_OOM;
        msg = "host allocation failed";
    } catch (const std::exception& e) {
        code = H2B_ERR_CUDA;
        msg = e.what();
    } catch (...) {
        code = H2B_ERR_CUDA;
        msg = "unknown failure";
    }
    std::lock_guard<std::mutex> lock(ctx->mu);
    ctx->err = msg;
    return code;
}

std::string join(const std::vector<std::string>& v) {
    std::string s;
    for (auto& x : v) s += (s.empty() ? "" : ",") + x;
    return s;
}
void write_text(const std::string& s, char* out, size_t cap) {
    if (!out || s.size() + 1 > cap) throw Error(H2B_ERR_ARG, "name buffer too small");
    std::memcpy(out, s.c_str(), s.size() + 1);
}
// one report as max_report + 1 words: the failure count, then the rows, zero-padded
uint64_t* write_report(uint64_t* p, const ReportItem& e, size_t max_report) {
    std::fill(p, p + max_report + 1, 0);
    p[0] = e.first;
    std::copy(e.second.begin(), e.second.end(), p + 1);
    return p + max_report + 1;
}
void write_column(const NamedColumn& c, h2b_poly** poly, size_t* offset, size_t* rows) {
    if (!poly || !offset || !rows) throw Error(H2B_ERR_ARG, "null output");
    *poly = c.col.poly->raw();
    *offset = c.col.offset;
    *rows = c.rows;
}
}  // namespace h2bp
using namespace h2b;
using namespace h2bp;

// callbacks: 0 = success; anything else aborts the proof with H2B_ERR_ARG
typedef int (*h2bp_blind_fn)(void* user, size_t rows, uint64_t* out);              // rows x 4 limbs of blinding scalars
typedef int (*h2bp_allreduce_fn)(void* user, void* d_points, size_t m);             // see ProverSession::shard
typedef int (*h2bp_commit_fn)(void* user, int basis, const uint64_t* rows, size_t n);  // see ProverSession::observer

#define H2BP_API extern "C" __attribute__((visibility("default")))

// fixed: n_fixed named columns (at least the circuit's fixed_names), sigma: one per permutation column; 2^k rows each; I instance
// columns, F constants columns; compress_selectors: halo2's keygen_vk layout (ProverCircuit)
H2BP_API int h2bp_circuit_create(h2b_ctx* ctx, uint32_t k, size_t A, size_t L, int selector_lookup, size_t I, size_t F, const char* const* fixed_names,
                                 const uint64_t* const* fixed, size_t n_fixed, const uint64_t* const* sigma, size_t n_sigma,
                                 BoundCircuit** out, int compress_selectors) {
    return run(ctx, [&] {
        if (!out || (n_fixed && (!fixed_names || !fixed)) || (n_sigma && !sigma)) throw Error(H2B_ERR_ARG, "circuit_create: null argument");
        std::map<std::string, const Fr*> f;
        for (size_t i = 0; i < n_fixed; i++) f[fixed_names[i]] = reinterpret_cast<const Fr*>(fixed[i]);
        std::vector<const Fr*> s;
        for (size_t i = 0; i < n_sigma; i++) s.push_back(reinterpret_cast<const Fr*>(sigma[i]));
        auto b = std::make_unique<BoundCircuit>(ctx);
        b->cs = std::make_unique<ProverCircuit>(b->ctx, k, A, L, selector_lookup != 0, f, s, I, F, compress_selectors != 0);
        *out = b.release();
    });
}
H2BP_API void h2bp_circuit_free(BoundCircuit* b) { delete b; }

// shape: degree, chunk, ext_k, bf, u, n_sets, n_lookups, selector_lookup; names: "adv=..\nperm=..\nfixed=..\nsigma=..\nconst=..
// \nqueries=..\nselectors=.." (comma-separated; fixed: the fixed columns in column order, queries: in query order; const: the
// constants columns, empty when F = 0; selectors: name:column:root:len per selector)
H2BP_API int h2bp_circuit_info(BoundCircuit* b, uint64_t* shape, char* names, size_t cap) {
    return run(b ? b->ctx.raw() : nullptr, [&] {
        const ProverCircuit& cs = *b->cs;
        const uint64_t v[8] = {cs.degree, cs.chunk, cs.ext_k, cs.bf, cs.u, cs.n_sets, cs.n_lookups, cs.selector_lookup};
        if (!shape) throw Error(H2B_ERR_ARG, "circuit_info: null shape");
        std::copy(v, v + 8, shape);
        std::vector<std::string> sel;
        for (auto& [nm, a] : cs.layout.selectors) sel.push_back(nm + ":" + a.column + ":" + std::to_string(a.root) + ":" + std::to_string(a.len));
        write_text("adv=" + join(cs.adv_names) + "\nperm=" + join(cs.perm_cols) + "\nfixed=" + join(cs.layout.fixed_columns) + "\nsigma=" +
                       join(cs.sigma_names) + "\nconst=" + join(cs.const_names) + "\nqueries=" + join(cs.layout.fixed_queries) +
                       "\nselectors=" + join(sel),
                   names, cap);
    });
}
H2BP_API int h2bp_circuit_column(BoundCircuit* b, const char* table, const char* name, h2b_poly** poly, size_t* offset, size_t* rows) {
    return run(b ? b->ctx.raw() : nullptr, [&] { write_column(b->cs->column(table ? table : "", name ? name : ""), poly, offset, rows); });
}

// srs: the caller's SRS handle (its shard holds srs_count points); both handles must outlive the session
H2BP_API int h2bp_session_create(h2b_ctx* ctx, h2b_srs* srs, uint32_t k, size_t srs_count, BoundCircuit* cs, BoundSession** out) {
    return run(ctx, [&] {
        if (!srs || !cs || !out) throw Error(H2B_ERR_ARG, "session_create: null argument");
        *out = new BoundSession(ctx, srs, k, srs_count, *cs->cs);
    });
}
H2BP_API void h2bp_session_free(BoundSession* b) { delete b; }

// counts: commitments per proof, evaluations per proof; names: the evaluations' "column:rotation", comma-separated, in order
H2BP_API int h2bp_session_info(BoundSession* b, uint64_t* counts, char* names, size_t cap) {
    return run(b ? b->ctx.raw() : nullptr, [&] {
        const auto q = b->sess.queries();
        std::vector<std::string> nm;
        for (auto& e : q) nm.push_back(e.name + ":" + std::to_string(e.rot));
        if (!counts) throw Error(H2B_ERR_ARG, "session_info: null counts");
        counts[0] = b->sess.commitments_per_proof();
        counts[1] = q.size();
        write_text(join(nm), names, cap);
    });
}
H2BP_API int h2bp_session_column(BoundSession* b, const char* table, const char* name, h2b_poly** poly, size_t* offset, size_t* rows) {
    return run(b ? b->ctx.raw() : nullptr, [&] { write_column(b->sess.column(table ? table : "", name ? name : ""), poly, offset, rows); });
}
H2BP_API int h2bp_session_shard(BoundSession* b, size_t begin, size_t n_loc, h2bp_allreduce_fn fn, void* user) {
    return run(b ? b->ctx.raw() : nullptr, [&] {
        ProverSession::AllReduce ar;
        if (fn)
            ar = [fn, user](void* d, size_t m) {
                if (fn(user, d, m)) throw Error(H2B_ERR_ARG, "the all-reduce callback failed");
            };
        b->sess.shard(begin, n_loc, std::move(ar));
    });
}

// one proof.  random_poly: 2^k elements (pinned); observer may be null.  Out: commitments (affine, 12 limbs each),
// evaluations (4 limbs each), the challenges theta beta gamma y x (Montgomery, 4 limbs each), bytes = [h2d, d2h]
H2BP_API int h2bp_prove(BoundSession* b, const WitnessView* w, const uint64_t* random_poly, h2bp_blind_fn blind, void* blind_user,
                        h2bp_commit_fn observer, void* observer_user, uint64_t* commitments, uint64_t* evals, uint64_t* challenges,
                        uint64_t* bytes) {
    return run(b ? b->ctx.raw() : nullptr, [&] {
        if (!w || !blind || !commitments || !evals || !challenges || !bytes) throw Error(H2B_ERR_ARG, "prove: null argument");
        ProverSession& s = b->sess;
        s.observer = nullptr;
        if (observer)
            s.observer = [observer, observer_user](int basis, const std::vector<Fr>& rows) {
                if (observer(observer_user, basis, rows[0].data(), rows.size())) throw Error(H2B_ERR_ARG, "the commit observer failed");
            };
        auto source = [&](size_t rows) {
            std::vector<Fr> out(rows);
            if (blind(blind_user, rows, out[0].data())) throw Error(H2B_ERR_ARG, "the blinding callback failed");
            return out;
        };
        const Proof pr = s.create_proof(*w, reinterpret_cast<const Fr*>(random_poly), source);
        std::memcpy(commitments, pr.commitments.data(), pr.commitments.size() * sizeof(G1));
        for (size_t i = 0; i < pr.evals.size(); i++) std::memcpy(evals + 4 * i, pr.evals[i].second.data(), 32);
        const Fr* ch[5] = {&pr.theta, &pr.beta, &pr.gamma, &pr.y, &pr.x};
        for (int i = 0; i < 5; i++) std::memcpy(challenges + 4 * i, ch[i]->data(), 32);
        bytes[0] = pr.h2d_bytes;
        bytes[1] = pr.d2h_bytes;
    });
}

// one proof in halo2's form (ProverSession::create_proof_halo2): vk_repr (Montgomery, 4 limbs) absorbed first; the proof bytes
// go to `proof` (capacity `cap` bytes), their number to *len
H2BP_API int h2bp_prove_halo2(BoundSession* b, const WitnessView* w, const uint64_t* random_poly, h2bp_blind_fn blind, void* blind_user,
                              const uint64_t* vk_repr, uint8_t* proof, size_t cap, size_t* len) {
    return run(b ? b->ctx.raw() : nullptr, [&] {
        if (!w || !blind || !vk_repr || !proof || !len) throw Error(H2B_ERR_ARG, "prove_halo2: null argument");
        ProverSession& s = b->sess;
        s.observer = nullptr;
        auto source = [&](size_t rows) {
            std::vector<Fr> out(rows);
            if (blind(blind_user, rows, out[0].data())) throw Error(H2B_ERR_ARG, "the blinding callback failed");
            return out;
        };
        Fr repr;
        std::memcpy(repr.data(), vk_repr, 32);
        const std::vector<uint8_t> bytes = s.create_proof_halo2(*w, reinterpret_cast<const Fr*>(random_poly), source, repr);
        if (bytes.size() > cap) throw Error(H2B_ERR_ARG, "prove_halo2: the proof needs " + std::to_string(bytes.size()) + " bytes");
        std::memcpy(proof, bytes.data(), bytes.size());
        *len = bytes.size();
    });
}

// the constraint check.  report: max_report + 1 words per gate column, lookup and permutation column (in that order, instance
// columns last): the failure count, then the first min(count, max_report) failing rows ascending
H2BP_API int h2bp_check(BoundSession* b, const WitnessView* w, size_t max_report, uint64_t* report) {
    return run(b ? b->ctx.raw() : nullptr, [&] {
        if (!w || !report) throw Error(H2B_ERR_ARG, "check: null argument");
        const CheckReport r = b->sess.check(*w, max_report);
        uint64_t* p = report;
        for (auto* part : {&r.gates, &r.lookups, &r.copies})
            for (auto& e : *part) p = write_report(p, e, max_report);
    });
}

// MockProver of a builder (include/h2b200_mock.hpp), I instance columns, F constants columns.  n_lookups: the number of lookup
// reports (L, 1 for the selector lookup, or 0)
H2BP_API int h2bp_mock_create(h2b_ctx* ctx, uint32_t k, size_t A, size_t L, int selector_lookup, uint32_t lookup_bits, size_t max_rows, size_t I,
                              size_t F, BoundMock** out, uint64_t* n_lookups) {
    return run(ctx, [&] {
        if (!out || !n_lookups) throw Error(H2B_ERR_ARG, "mock_create: null argument");
        *out = new BoundMock(ctx, k, A, L, selector_lookup != 0, lookup_bits, max_rows, I, F);
        *n_lookups = (*out)->mock.n_lookups;
    });
}
H2BP_API void h2bp_mock_free(BoundMock* b) { delete b; }
H2BP_API int h2bp_mock_column(BoundMock* b, const char* name, h2b_poly** poly, size_t* offset, size_t* rows) {
    return run(b ? b->ctx.raw() : nullptr, [&] { write_column(b->mock.column(name ? name : ""), poly, offset, rows); });
}

// one run.  break_points: A - 1 words (the count in *n_break_points); report: max_report + 1 words per gate column, lookup, then
// the advice equalities, the constant equalities and each instance column (as h2bp_check); cells: max_report x (column, row,
// column, row) of the reported advice equalities, then max_report x (column, row) of the reported constant equalities, then
// the same for the reported rows of each instance column; *distinct_constants: the number of distinct constants
H2BP_API int h2bp_mock_run(BoundMock* b, const BuilderView* v, size_t max_report, uint64_t* break_points, uint64_t* n_break_points,
                           uint64_t* report, uint64_t* cells, uint64_t* distinct_constants) {
    return run(b ? b->ctx.raw() : nullptr, [&] {
        if (!v || !n_break_points || !report || !cells || !distinct_constants || (b->mock.A > 1 && !break_points))
            throw Error(H2B_ERR_ARG, "mock_run: null argument");
        const MockReport r = b->mock.run(*v, max_report);
        *distinct_constants = r.distinct_constants;
        *n_break_points = r.break_points.size();
        std::copy(r.break_points.begin(), r.break_points.end(), break_points);
        uint64_t* p = report;
        for (auto* part : {&r.gates, &r.lookups})
            for (auto& e : *part) p = write_report(p, e, max_report);
        p = write_report(write_report(p, r.equalities, max_report), r.constants, max_report);
        for (auto& e : r.instances) p = write_report(p, e, max_report);
        std::fill(cells, cells + (6 + 2 * r.instances.size()) * max_report, 0);
        for (size_t i = 0; i < r.equality_cells.size(); i++) {
            const auto& [x, y] = r.equality_cells[i];
            const uint64_t w[4] = {x.column, x.row, y.column, y.row};
            std::copy(w, w + 4, cells + 4 * i);
        }
        for (size_t i = 0; i < r.constant_cells.size(); i++) {
            cells[4 * max_report + 2 * i] = r.constant_cells[i].column;
            cells[4 * max_report + 2 * i + 1] = r.constant_cells[i].row;
        }
        for (size_t m = 0; m < r.instance_cells.size(); m++)
            for (size_t i = 0; i < r.instance_cells[m].size(); i++) {
                cells[(6 + 2 * m) * max_report + 2 * i] = r.instance_cells[m][i].column;
                cells[(6 + 2 * m) * max_report + 2 * i + 1] = r.instance_cells[m][i].row;
            }
    });
}

// keygen of a builder (include/h2b200_keygen.hpp).  Out: the circuit (freed with h2bp_circuit_free); break_points (A - 1 words,
// the count in *n_break_points); vk: 12 limbs per commitment, the fixed columns in the circuit's fixed_names order, then the sigma
// columns (F + A + L + v->n_instance_columns); times: the five phases of KeygenTimes in ms (may be null); F constants columns;
// compress_selectors: halo2's keygen_vk layout (the vk's fixed commitments in the circuit's column order)
H2BP_API int h2bp_keygen(h2b_ctx* ctx, h2b_srs* srs, uint32_t k, size_t srs_count, size_t A, size_t L, int selector_lookup, uint32_t lookup_bits,
                         size_t max_rows, size_t F, const BuilderView* v, BoundCircuit** out, uint64_t* break_points, uint64_t* n_break_points, uint64_t* vk,
                         double* times, int compress_selectors) {
    return run(ctx, [&] {
        if (!srs || !v || !out || !n_break_points || !vk || (A > 1 && !break_points)) throw Error(H2B_ERR_ARG, "keygen: null argument");
        auto b = std::make_unique<BoundCircuit>(ctx);
        const ParamsKZG params(b->ctx, k, srs, srs_count);
        KeygenTimes t;
        KeygenResult r = keygen(b->ctx, params, k, A, L, selector_lookup != 0, lookup_bits, max_rows, *v, &t, F, compress_selectors != 0);
        b->cs = std::move(r.pk);
        *n_break_points = r.break_points.size();
        std::copy(r.break_points.begin(), r.break_points.end(), break_points);
        size_t i = 0;
        for (auto& f : r.vk.fixed) std::memcpy(vk + 12 * i++, f.second.x.data(), sizeof(G1));
        for (auto& p : r.vk.permutation) std::memcpy(vk + 12 * i++, p.x.data(), sizeof(G1));
        if (times) {
            const double w[5] = {t.copies, t.forest, t.sigma, t.pk, t.vk};
            std::copy(w, w + 5, times);
        }
        *out = b.release();
    });
}

#pragma GCC visibility pop
