// Runs MockProver on a halo2-base builder through the C++ front end (include/h2b200_mock.hpp) on an instance the Python test
// wrote to a directory, in both witness forms, and writes the reports back for a byte comparison with halo2_lib_b200.MockProver
// (tests/test_gpu_mock_prover.py::test_cpp_mock_prover_matches_python).
//
// Directory layout (little-endian; Fr elements are 32 bytes of Montgomery limbs, indices are u64):
//   manifest.txt   k A L selector_lookup lookup_bits max_rows n_cells n_rational n_advice_eq n_constant_eq n_lookup max_report
//   cells.bin      the evaluated witness;  witness.bin, rational_index.bin, rational_den.bin: the halo2-base form of it
//   selectors.bin  one byte per cell;  eq.bin: (a, b) pairs;  consts.bin, const_index.bin;  lookups.bin
// Output: report.bin = for the evaluated form, the halo2-base form, and the halo2-base form again after a rejected run:
//   [n_break_points][break points] then for every gate, lookup, the advice and the constant equalities [count][n][items...],
//   then (column, row, column, row) per reported advice equality and (column, row) per reported constant equality
#include <cstdio>
#include <fstream>
#include <iostream>

#include "../../include/h2b200_mock.hpp"

using namespace h2b;

template <class T>
static std::vector<T> read_file(const std::string& path, size_t count) {
    std::vector<T> v(count);
    if (!count) return v;
    std::ifstream f(path, std::ios::binary);
    if (!f) throw std::runtime_error("cannot open " + path);
    f.read(reinterpret_cast<char*>(v.data()), std::streamsize(count * sizeof(T)));
    if (size_t(f.gcount()) != count * sizeof(T)) throw std::runtime_error("short read: " + path);
    return v;
}

static void write_report(std::ofstream& out, const MockReport& r) {
    std::vector<uint64_t> w{r.break_points.size()};
    w.insert(w.end(), r.break_points.begin(), r.break_points.end());
    std::vector<const std::pair<uint64_t, std::vector<uint64_t>>*> items;
    for (auto& e : r.gates) items.push_back(&e);
    for (auto& e : r.lookups) items.push_back(&e);
    items.push_back(&r.equalities);
    items.push_back(&r.constants);
    for (auto* e : items) {
        w.push_back(e->first);
        w.push_back(e->second.size());
        w.insert(w.end(), e->second.begin(), e->second.end());
    }
    for (auto& [a, b] : r.equality_cells) w.insert(w.end(), {a.column, a.row, b.column, b.row});
    for (auto& a : r.constant_cells) w.insert(w.end(), {a.column, a.row});
    out.write(reinterpret_cast<const char*>(w.data()), std::streamsize(8 * w.size()));
}

int main(int argc, char** argv) {
    if (argc < 2) {
        std::fprintf(stderr, "usage: mock_prover_test <dir>\n");
        return 2;
    }
    const std::string dir = argv[1];
    try {
        std::ifstream mf(dir + "/manifest.txt");
        uint32_t k, bits;
        size_t A, L, max_rows, N, n_rat, n_eq, n_const, n_lk, max_report;
        int sel;
        mf >> k >> A >> L >> sel >> bits >> max_rows >> N >> n_rat >> n_eq >> n_const >> n_lk >> max_report;
        if (!mf) throw std::runtime_error("bad manifest");
        Context ctx(0);
        MockProver mock(ctx, k, A, L, sel != 0, bits, max_rows);
        const auto cells = read_file<Fr>(dir + "/cells.bin", N);
        const auto witness = read_file<Fr>(dir + "/witness.bin", N);
        const auto rat_idx = read_file<uint64_t>(dir + "/rational_index.bin", n_rat);
        const auto rat_den = read_file<Fr>(dir + "/rational_den.bin", n_rat);
        const auto selectors = read_file<uint8_t>(dir + "/selectors.bin", N);
        auto eq = read_file<uint64_t>(dir + "/eq.bin", 2 * n_eq);
        const auto consts = read_file<Fr>(dir + "/consts.bin", n_const);
        const auto const_idx = read_file<uint64_t>(dir + "/const_index.bin", n_const);
        const auto lookups = read_file<uint64_t>(dir + "/lookups.bin", n_lk);
        BuilderView v;
        v.cells = cells.data();
        v.n_cells = N;
        v.selectors = selectors.data();
        v.advice_equalities = eq.data();
        v.n_advice_equalities = n_eq;
        v.constants = consts.data();
        v.constant_index = const_idx.data();
        v.n_constant_equalities = n_const;
        v.lookup_index = lookups.data();
        v.n_lookup = n_lk;
        std::ofstream out(dir + "/report.bin", std::ios::binary);
        write_report(out, mock.run(v, max_report));
        v.cells = witness.data();
        v.rational_index = rat_idx.data();
        v.rational_den = rat_den.data();
        v.n_rational = n_rat;
        write_report(out, mock.run(v, max_report));
        // an advice equality naming no cell is rejected, and the next run on the same context is right
        auto bad_eq = eq;
        bad_eq[1] = N;
        BuilderView bad = v;
        bad.advice_equalities = bad_eq.data();
        bool rejected = false;
        try {
            mock.run(bad, max_report);
        } catch (const Error& e) {
            rejected = std::string(e.what()).find("virtual cell not assigned") != std::string::npos;
        }
        if (!rejected) throw std::runtime_error("an advice equality naming no cell was not rejected");
        write_report(out, mock.run(v, max_report));
        return 0;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "mock prover FAILED: %s\n", e.what());
        return 1;
    }
}
