// h2b200_keygen.hpp — keygen_vk + keygen_pk for a halo2-base builder in its keygen form, on the device: the break points, the
// fixed columns (q_j, q_lookup, the table, the constants columns c, c1..), sigma bit-exact to what halo2's permutation Assembly
// builds from halo2-base's copy calls, the proving key as a ProverCircuit and the verifying key's commitments.  DESIGN.md §4.8,
// §4.11.
//
// The builder comes as MockProver takes it (BuilderView, include/h2b200_mock.hpp); keygen reads no witness values: `cells` and
// the rational pairs are ignored, `n_cells` is used.  The copy calls of BaseCircuitBuilder::synthesize, in order:
//   1. the break copies of assign_with_constraints: (a{j+1}, 0) ~ (a_j, bp_j), j = 0, 1, ..;
//   2. L > 0: LookupAnyManager::assign_raw's copies raw(lookup_index[i]) ~ (l{i mod L}, i / L), i = 0, 1, ..;
//   3. CopyConstraintManager::assign_raw: the advice equalities sorted by (a, b), then the constant equalities sorted by
//      (constant, cell) as (the constant's cell) ~ raw(cell), the distinct constants placed left to right, then top to bottom
//      over the F constants columns in that order: distinct constant d at row d div F of column d mod F (c, c1, ..);
//   4. after the region, BaseCircuitBuilder::assign_instances: raw(instance_index_m[r]) ~ (i_m, r) for each instance column m
//      (b.n_instance_columns of them) in order and r = 0, 1, .. (an index >= N: "instance not assigned"; r >= u: halo2's
//      NotEnoughRowsAvailable).
// So the builder's own order of its equalities does not change the keys.  Errors: halo2-base's panics as MockProver raises them.
// F (BaseCircuitParams::num_fixed) may be 0 when the builder has no constant equalities.
#pragma once
#include <chrono>

#include "h2b200_mock.hpp"

namespace h2b {

// affine commitments (z = 1; the identity all zero) of the Lagrange columns, as ProverSession commits them
struct VerifyingKey {
    std::vector<std::pair<std::string, G1>> fixed;  // the circuit's column order (its layout.fixed_columns)
    std::vector<G1> permutation;                    // one per permutation column, perm_cols order (instance columns last)
};

// milliseconds per phase of one keygen call (each phase ends with the stream synchronised)
struct KeygenTimes {
    double copies = 0;  // uploads, fixed columns, the copy list and its sorts
    double forest = 0;  // spanning forest and walk: the sigma map
    double sigma = 0;   // sigma values
    double pk = 0;      // the proving key's coefficient and extended-coset forms
    double vk = 0;      // the commitments
};

struct KeygenResult {
    std::vector<uint64_t> break_points;
    std::unique_ptr<ProverCircuit> pk;
    VerifyingKey vk;
};

// params: the SRS of the 2^k domain (its Lagrange bases commit the vk); max_rows as for MockProver (<= 2^k - 7); F constants columns;
// compress_selectors: keygen_vk's selector compression (h2b200_selectors.hpp, timed in `pk`): the vk's fixed commitments are then
// halo2's columns in halo2's column order, [table], c.., s0, s1..
inline KeygenResult keygen(const Context& ctx, const ParamsKZG& params, uint32_t k, size_t A, size_t L, bool selector_lookup, uint32_t lookup_bits,
                           size_t max_rows, const BuilderView& b, KeygenTimes* times = nullptr, size_t F = 1, bool compress_selectors = false) {
    using clock = std::chrono::steady_clock;
    auto t0 = clock::now();
    auto lap = [&](double KeygenTimes::*field) {
        const auto t = clock::now();
        if (times) times->*field = std::chrono::duration<double, std::milli>(t - t0).count();
        t0 = t;
    };
    const CircuitShape s = builder_shape("keygen", k, A, L, selector_lookup, lookup_bits, max_rows, b.n_instance_columns, F);
    const size_t n = s.n, N = b.n_cells, M = b.n_advice_equalities, Mc = b.n_constant_equalities, NL = b.n_lookup;
    h2b_ctx* c = ctx.raw();
    KeygenResult out;
    out.break_points = builder_break_points(s, "keygen", max_rows, b, false);
    const size_t I = s.I, nbp = out.break_points.size(), npc = s.perm_cols.size(), E0 = nbp + (L ? NL : 0) + M + Mc;
    size_t E = E0;
    for (size_t m = 0; m < I; m++) E += b.n_instance[m];
    PolyPtr sel_d, lk_d, eq_d, const_d, const_idx_d;
    upload_bytes(ctx, sel_d, b.selectors, N);
    upload_bytes(ctx, lk_d, b.lookup_index, 8 * NL);
    upload_bytes(ctx, eq_d, b.advice_equalities, 16 * M);
    upload_bytes(ctx, const_d, b.constants, 32 * Mc);
    upload_bytes(ctx, const_idx_d, b.constant_index, 8 * Mc);
    // the fixed columns in the circuit's order: q0.., [q_lookup], [table], c, c1.. (the F constants columns last, one block)
    const size_t nf = s.fixed_names.size();
    Poly fixed(ctx, nf * n), status(ctx, 1);
    auto col = [&](size_t i) { return static_cast<Fr*>(fixed.at(i * n)); };
    const uint64_t* bp = nbp ? out.break_points.data() : nullptr;
    ctx.check(h2b_mock_selectors_dev(c, sel_d->at(), N, bp, nbp, k, A, fixed.at()));
    uint32_t* st = static_cast<uint32_t*>(status.at());
    uint32_t v[2] = {0, 0};
    if (s.selector_lookup) {
        ctx.check(h2b_mock_lookup_selector_dev(c, lk_d->at(), NL, N, max_rows, k, col(A), st));
        std::memcpy(v, status.download(0, 1)[0].data(), 8);
        builder_panics(s, v[0] & 1, v[0] & 2, 0, false);
    }
    if (s.n_lookups) ctx.check(h2b_poly_upload(c, fixed.raw(), (nf - F - 1) * n, lookup_table(n, lookup_bits)[0].data(), n));
    Poly edges(ctx, (8 * E + 31) / 32 + 1);
    ctx.check(h2b_keygen_copies_nf_dev(c, N, bp, nbp, k, F, A, L, lk_d->at(), L ? NL : 0, eq_d->at(), M, const_d->at(), const_idx_d->at(), Mc,
                                       F ? col(nf - F) : nullptr, edges.at(), st));
    std::memcpy(v, status.download(0, 1)[0].data(), 8);
    builder_panics(s, v[0] & 1, false, v[1], v[0] & 2);
    if (I) {  // the instance copies, after the region's
        std::vector<uint64_t> idx;
        for (size_t m = 0; m < I; m++) idx.insert(idx.end(), b.instance_index[m], b.instance_index[m] + b.n_instance[m]);
        PolyPtr idx_d;
        upload_bytes(ctx, idx_d, idx.data(), 8 * idx.size());
        Poly inst_status(ctx, (I + 7) / 8);
        ctx.check(h2b_keygen_instance_edges_nf_dev(c, N, bp, nbp, k, F, A, L, s.u, I, b.n_instance, idx_d->at(),
                                                   static_cast<char*>(edges.at()) + 8 * E0, static_cast<uint32_t*>(inst_status.at())));
        const std::vector<Fr> w = inst_status.download(0, inst_status.len());
        const uint32_t* iv = reinterpret_cast<const uint32_t*>(w[0].data());
        for (size_t m = 0; m < I; m++) {  // the first failing cell in assign_instances' order
            if (iv[m] & 1) throw Error(H2B_ERR_ARG, "instance not assigned");
            if (iv[m] & 2)
                throw Error(H2B_ERR_ARG, "NotEnoughRowsAvailable { current_k: " + std::to_string(k) + " }: instance column i" + std::to_string(m) +
                                             " has " + std::to_string(b.n_instance[m]) + " cells for its " + std::to_string(s.u) + " usable rows");
        }
    }
    lap(&KeygenTimes::copies);
    Poly map(ctx, (npc * n + 7) / 8), sigma(ctx, npc * n);
    ctx.check(h2b_keygen_sigma_map_dev(c, edges.at(), E, npc, k, map.at()));
    lap(&KeygenTimes::forest);
    ctx.check(h2b_keygen_sigma_values_dev(c, map.at(), npc, k, sigma.at()));
    lap(&KeygenTimes::sigma);
    std::map<std::string, const Fr*> fx;
    for (size_t i = 0; i < nf; i++) fx[s.fixed_names[i]] = col(i);
    std::vector<const Fr*> sg;
    for (size_t i = 0; i < npc; i++) sg.push_back(static_cast<const Fr*>(sigma.at(i * n)));
    out.pk = std::make_unique<ProverCircuit>(ProverCircuit::OnDevice{}, ctx, k, A, L, selector_lookup, fx, sg, I, F, compress_selectors);
    lap(&KeygenTimes::pk);
    // the vk: every fixed column (compressed: the circuit's, in its column order), then every sigma column, committed in Lagrange
    // form, up to 16 MSMs per batch
    const std::vector<std::string>& fixed_order = compress_selectors ? out.pk->layout.fixed_columns : s.fixed_names;
    const size_t nvf = fixed_order.size();
    std::vector<const void*> cols;
    for (size_t i = 0; i < nvf; i++) cols.push_back(compress_selectors ? out.pk->lagr.at(fixed_order[i])->at() : col(i));
    for (size_t i = 0; i < npc; i++) cols.push_back(sigma.at(i * n));
    std::vector<G1> pts(cols.size());
    Poly d_out(ctx, 48);
    for (size_t lo = 0; lo < cols.size(); lo += 16) {
        const size_t m = std::min<size_t>(16, cols.size() - lo);
        const std::vector<int> basis(m, H2B_BASIS_LAGRANGE);
        ctx.check(h2b_msm_g1_batch_dev(c, params.raw(), basis.data(), cols.data() + lo, m, n, d_out.at()));
        ctx.check(h2b_poly_download(c, d_out.raw(), 0, pts[lo].x.data(), m * 3));
        g1_normalize_host_batch(pts.data() + lo, m);
    }
    for (size_t i = 0; i < nvf; i++) out.vk.fixed.push_back({fixed_order[i], pts[i]});
    out.vk.permutation.assign(pts.begin() + nvf, pts.end());
    lap(&KeygenTimes::vk);
    return out;
}

}  // namespace h2b
