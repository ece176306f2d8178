// Runs the constraint check through the C++ host side (include/h2b200_prover.hpp, ProverSession::check) on an instance the
// Python test wrote to a directory, in both witness forms, and writes the reports back for a comparison with
// halo2-lib_b200/prover.py (tests/test_gpu_check.py::test_cpp_check_matches_python).
//
// Directory layout (little-endian; Fr elements are 32 bytes of Montgomery limbs, indices are u64):
//   manifest.txt            k A L selector_lookup n_eval n_lookup_cells n_witness n_breaks n_rational n_lookup_index max_report
//   fixed_<name>.bin, sigma_<i>.bin     the circuit
//   eval.bin, lookup.bin    the evaluated witness and the looked-up values
//   witness.bin, rational_index.bin, rational_den.bin, lookup_index.bin   the halo2-base form of the same witness
//   breaks.bin              u64 break points
// Output: report.bin = for each form, for every gate, lookup and permutation column: [count u64][n_rows u64][rows u64...]
#include <cstdio>
#include <fstream>
#include <iostream>

#include "../../include/h2b200_prover.hpp"

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

static void write_report(std::ofstream& out, const CheckReport& r) {
    for (auto* items : {&r.gates, &r.lookups, &r.copies})
        for (auto& [count, rows] : *items) {
            const uint64_t nr = rows.size();
            out.write(reinterpret_cast<const char*>(&count), 8);
            out.write(reinterpret_cast<const char*>(&nr), 8);
            out.write(reinterpret_cast<const char*>(rows.data()), std::streamsize(8 * nr));
        }
}

int main(int argc, char** argv) {
    if (argc < 2) {
        std::fprintf(stderr, "usage: prover_check_test <dir>\n");
        return 2;
    }
    const std::string dir = argv[1];
    try {
        std::ifstream mf(dir + "/manifest.txt");
        uint32_t k;
        size_t A, L, n_eval, n_lkc, n_wit, n_bp, n_rat, n_lk, max_report;
        int sel;
        mf >> k >> A >> L >> sel >> n_eval >> n_lkc >> n_wit >> n_bp >> n_rat >> n_lk >> max_report;
        if (!mf) throw std::runtime_error("bad manifest");
        const size_t n = size_t(1) << k;
        Context ctx(0);
        std::map<std::string, std::vector<Fr>> fixed;
        std::vector<std::string> names;
        for (size_t j = 0; j < A; j++) names.push_back("q" + std::to_string(j));
        const bool selector = sel && L == 0;
        if (selector) names.push_back("q_lookup");
        if (L || selector) names.push_back("table");
        names.push_back("c");
        for (auto& nm : names) fixed[nm] = read_file<Fr>(dir + "/fixed_" + nm + ".bin", n);
        std::vector<std::vector<Fr>> sigma;
        for (size_t i = 0; i < 1 + A + L; i++) sigma.push_back(read_file<Fr>(dir + "/sigma_" + std::to_string(i) + ".bin", n));
        ProverCircuit cs(ctx, k, A, L, sel != 0, fixed, sigma);
        ParamsKZG params(ctx, k, {}, std::vector<G1Affine>(n, G1Affine{}));  // a check commits nothing: identity bases do
        ProverSession sess(ctx, params, cs);
        const auto breaks = read_file<uint64_t>(dir + "/breaks.bin", n_bp);
        const auto eval = read_file<Fr>(dir + "/eval.bin", n_eval);
        const auto lookup = read_file<Fr>(dir + "/lookup.bin", n_lkc);
        AssignedWitness form;
        const auto witness = read_file<Fr>(dir + "/witness.bin", n_wit);
        form.rational_index = read_file<uint64_t>(dir + "/rational_index.bin", n_rat);
        form.rational_den = read_file<Fr>(dir + "/rational_den.bin", n_rat);
        form.lookup_index = read_file<uint64_t>(dir + "/lookup_index.bin", n_lk);
        std::ofstream out(dir + "/report.bin", std::ios::binary);
        write_report(out, sess.check(eval, breaks, lookup, nullptr, max_report));
        write_report(out, sess.check(witness, breaks, {}, &form, max_report));
        // a Rational index out of range is rejected, and the session checks correctly afterwards
        AssignedWitness bad = form;
        bad.rational_index.push_back(n_wit);
        bad.rational_den.push_back(Fr{});
        bool rejected = false;
        try {
            sess.check(witness, breaks, {}, &bad, max_report);
        } catch (const Error&) {
            rejected = true;
        }
        if (!rejected) throw std::runtime_error("an out-of-range Rational index was accepted");
        write_report(out, sess.check(witness, breaks, {}, &form, max_report));
        return 0;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "prover check FAILED: %s\n", e.what());
        return 1;
    }
}
