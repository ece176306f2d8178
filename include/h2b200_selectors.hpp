// h2b200_selectors.hpp — halo2's selector compression (keygen_vk = keygen_vk_custom(.., compress_selectors = true), recalled from
// halo2-axiom 0.5.3 plonk/circuit/compress_selectors.rs and ConstraintSystem::compress_selectors; DESIGN.md §2 conventions 11-14,
// §4.13) for the circuit halo2-base builds: which selectors share a fixed column, with which root, and the order in which the
// fixed columns are committed (the vk) and queried (the evaluations and openings).  ProverCircuit (include/h2b200_prover.hpp)
// holds the layout of its circuit; nothing else derives it.
//
//   process      convention 12 restated literally from the degrees, max_degree and the conflict matrix: every degree-0
//                selector (complex, or in no gate) gets a column of its own in selector order; then each simple selector not yet
//                placed starts a combination with d = deg - 1, and later selectors j join it greedily (stop when d + len =
//                max_degree; skip j when placed or active on a row where a member is; join when max(d, deg_j - 1) + len + 1 <=
//                max_degree).  Member m of a combination gets root m + 1; its column holds the root where it is active.
//   substitution member with root r of a combination of len: q -> S * prod_{t = 1..len, t != r} (t - S), not normalised.
//   conflicts    h2b_selector_conflicts_dev (csrc/selectors.cu): the pairs active on a common row, on the device.
#pragma once
#include <map>
#include <string>
#include <vector>

#include "h2b200.hpp"

namespace h2b {

// where one selector went: its column, its root there and the length of its combination (1, 1 for an uncompressed selector)
struct SelectorAssignment {
    std::string column;
    size_t root = 1, len = 1;
};

// the fixed side of a circuit as halo2 lays it out
struct SelectorLayout {
    bool compressed = false;
    std::vector<std::string> fixed_columns;  // column order: the vk's fixed commitments
    std::vector<std::string> fixed_queries;  // query order: the fixed evaluations and opening queries
    std::map<std::string, SelectorAssignment> selectors;
    // per combination column (compressed only), in allocation order: (selector name, root) in join order
    std::vector<std::pair<std::string, std::vector<std::pair<std::string, size_t>>>> combinations;
};

// convention 12: the combinations, each the selector indices in join order, in the order their columns are allocated.
// degree[i]: the largest degree of a gate polynomial whose simple selector is i (0: complex or in no gate); conflicts: S x S,
// conflicts[i S + j] != 0 when i and j are active on a common row (the diagonal is not read)
inline std::vector<std::vector<size_t>> compress_selectors_process(const std::vector<size_t>& degree, size_t max_degree,
                                                                   const std::vector<uint8_t>& conflicts) {
    const size_t S = degree.size();
    if (conflicts.size() != S * S) throw Error(H2B_ERR_ARG, "compress_selectors: the conflict matrix must be S x S");
    std::vector<std::vector<size_t>> out;
    for (size_t i = 0; i < S; i++)
        if (degree[i] == 0) out.push_back({i});
    std::vector<bool> added(S, false);
    for (size_t i = 0; i < S; i++) {
        if (degree[i] == 0 || added[i]) continue;
        if (degree[i] > max_degree) throw Error(H2B_ERR_ARG, "compress_selectors: a selector's degree exceeds max_degree");
        added[i] = true;
        size_t d = degree[i] - 1;
        std::vector<size_t> comb{i};
        for (size_t j = i + 1; j < S; j++) {
            if (d + comb.size() == max_degree) break;
            if (degree[j] == 0 || added[j]) continue;
            bool excluded = false;
            for (size_t m : comb) excluded = excluded || conflicts[j * S + m];
            if (excluded) continue;
            const size_t nd = std::max(d, degree[j] - 1);
            if (nd + comb.size() + 1 > max_degree) continue;
            d = nd;
            comb.push_back(j);
            added[j] = true;
        }
        out.push_back(std::move(comb));
    }
    return out;
}

// the layout without compression: the circuit's own fixed columns in one order for everything, every selector its own column
inline SelectorLayout uncompressed_layout(const std::vector<std::string>& fixed_names, const std::vector<std::string>& selectors) {
    SelectorLayout y;
    y.fixed_columns = y.fixed_queries = fixed_names;
    for (auto& s : selectors) y.selectors[s] = {s, 1, 1};
    return y;
}

// convention 13: the combination columns s0, s1.. appended after the circuit's fixed columns (columns: in column order; queries:
// in query order), one Rotation::cur() query each, in allocation order
inline SelectorLayout compressed_layout(const std::vector<std::string>& columns, const std::vector<std::string>& queries,
                                        const std::vector<std::string>& selectors, const std::vector<std::vector<size_t>>& combos) {
    SelectorLayout y;
    y.compressed = true;
    y.fixed_columns = columns;
    y.fixed_queries = queries;
    for (size_t c = 0; c < combos.size(); c++) {
        const std::string name = "s" + std::to_string(c);
        y.fixed_columns.push_back(name);
        y.fixed_queries.push_back(name);
        std::vector<std::pair<std::string, size_t>> members;
        for (size_t m = 0; m < combos[c].size(); m++) {
            const std::string& sel = selectors.at(combos[c][m]);
            y.selectors[sel] = {name, m + 1, combos[c].size()};
            members.push_back({sel, m + 1});
        }
        y.combinations.push_back({name, std::move(members)});
    }
    return y;
}

// the conflict matrix of S selector columns (device pointers, 2^k Lagrange values each, every one 0 or 1) on the device
inline std::vector<uint8_t> selector_conflicts_dev(const Context& ctx, const std::vector<const void*>& d_selectors, uint32_t k) {
    std::vector<uint8_t> m(d_selectors.size() * d_selectors.size());
    if (!d_selectors.empty()) ctx.check(h2b_selector_conflicts_dev(ctx.raw(), d_selectors.data(), d_selectors.size(), k, m.data()));
    return m;
}

}  // namespace h2b
