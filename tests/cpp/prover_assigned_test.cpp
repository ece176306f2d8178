// Runs ONE resident proof through the C++ host side (include/h2b200_prover.hpp) from halo2-base's own witness form —
// Rational cells as (index, denominator) pairs, looked-up cells as virtual-column indices — on an instance the Python test
// wrote to a directory, and writes the proof back for a byte-for-byte comparison with halo2-lib_b200/prover.py
// (tests/test_gpu_assigned_witness.py::test_cpp_prover_from_assigned_witness_matches_python).
//
// Directory layout (little-endian; Fr elements are 32 bytes of Montgomery limbs, indices are u64):
//   manifest.txt            k A L selector_lookup n_witness n_breaks n_rational n_lookup n_blind
//   fixed_<name>.bin, sigma_<i>.bin, random.bin, blind.bin, bases_m.bin, bases_l.bin   as for prover_mirror_test
//   witness.bin             the virtual column, n in place of every Rational(n, d) cell
//   breaks.bin              u64 break points
//   rational_index.bin      u64, rational_den.bin  Fr: the Rational pairs
//   lookup_index.bin        u64: the looked-up cells in assign_raw order
// Output: proof.bin = [n_commitments u64][commitments 96 B each][n_evals u64][evals 32 B each][theta beta gamma y x]
//         and on stdout the bytes that went up.
#include <cstdio>
#include <fstream>
#include <iostream>

#include "../../include/h2b200_prover.hpp"

using namespace h2b;

template <class T>
static std::vector<T> read_file(const std::string& path, size_t count) {
    std::vector<T> v(count);
    std::ifstream f(path, std::ios::binary);
    if (!f) throw std::runtime_error("cannot open " + path);
    f.read(reinterpret_cast<char*>(v.data()), std::streamsize(count * sizeof(T)));
    if (size_t(f.gcount()) != count * sizeof(T)) throw std::runtime_error("short read: " + path);
    return v;
}

int main(int argc, char** argv) {
    if (argc < 2) {
        std::fprintf(stderr, "usage: prover_assigned_test <dir>\n");
        return 2;
    }
    const std::string dir = argv[1];
    try {
        std::ifstream mf(dir + "/manifest.txt");
        uint32_t k;
        size_t A, L, n_wit, n_bp, n_rat, n_lk, n_blind;
        int sel;
        mf >> k >> A >> L >> sel >> n_wit >> n_bp >> n_rat >> n_lk >> n_blind;
        if (!mf) throw std::runtime_error("bad manifest");
        const size_t n = size_t(1) << k;
        Context ctx(0);
        ParamsKZG params(ctx, k, read_file<G1Affine>(dir + "/bases_m.bin", n), read_file<G1Affine>(dir + "/bases_l.bin", n));
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
        ProverSession sess(ctx, params, cs);
        const auto witness = read_file<Fr>(dir + "/witness.bin", n_wit);
        const auto breaks = read_file<uint64_t>(dir + "/breaks.bin", n_bp);
        AssignedWitness form;
        form.rational_index = read_file<uint64_t>(dir + "/rational_index.bin", n_rat);
        form.rational_den = read_file<Fr>(dir + "/rational_den.bin", n_rat);
        form.lookup_index = read_file<uint64_t>(dir + "/lookup_index.bin", n_lk);
        const auto rnd = read_file<Fr>(dir + "/random.bin", n);
        const auto blind = read_file<Fr>(dir + "/blind.bin", n_blind);
        size_t pos = 0;
        auto source = [&](size_t rows) {
            if (pos + rows > blind.size()) throw std::runtime_error("blind.bin exhausted");
            std::vector<Fr> b(blind.begin() + pos, blind.begin() + pos + rows);
            pos += rows;
            return b;
        };
        // a Rational index out of range is rejected, and the session proves correctly afterwards
        AssignedWitness bad = form;
        bad.rational_index.push_back(n_wit);
        bad.rational_den.push_back(Fr{});
        bool rejected = false;
        try {
            sess.create_proof(witness, breaks, {}, rnd, source, &bad);
        } catch (const Error&) {
            rejected = true;
        }
        if (!rejected) throw std::runtime_error("an out-of-range Rational index was accepted");
        pos = 0;
        const Proof pr = sess.create_proof(witness, breaks, {}, rnd, source, &form);
        if (pos != blind.size()) throw std::runtime_error("blinding rows consumed: " + std::to_string(pos) + " of " + std::to_string(blind.size()));
        std::ofstream out(dir + "/proof.bin", std::ios::binary);
        const uint64_t nc = pr.commitments.size(), ne = pr.evals.size();
        out.write(reinterpret_cast<const char*>(&nc), 8);
        out.write(reinterpret_cast<const char*>(pr.commitments.data()), std::streamsize(nc * sizeof(G1)));
        out.write(reinterpret_cast<const char*>(&ne), 8);
        for (auto& e : pr.evals) out.write(reinterpret_cast<const char*>(e.second.data()), 32);
        for (const Fr* c : {&pr.theta, &pr.beta, &pr.gamma, &pr.y, &pr.x}) out.write(reinterpret_cast<const char*>(c->data()), 32);
        std::printf("h2d_bytes %zu\n", pr.h2d_bytes);
        return 0;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "prover assigned FAILED: %s\n", e.what());
        return 1;
    }
}
