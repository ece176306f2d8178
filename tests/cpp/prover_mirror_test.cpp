// Runs ONE resident proof through the C++ front end of the compiled prover (include/h2b200_prover.hpp over std::vector
// inputs) on an instance that the Python test wrote to a directory, and writes the proof back for a byte-for-byte comparison
// with the Python binding (tests/test_gpu_prover.py::test_cpp_prover_matches_python).  No arithmetic is checked here: the
// Python proof is the one the protocol-level checks run on; this binary shows that both front ends pass the same inputs.
//
// Directory layout (little-endian u64 limbs, Montgomery form, 32 bytes per element):
//   manifest.txt            k A L selector_lookup n_witness n_breaks n_lookup n_blind
//   fixed_<name>.bin        2^k elements per fixed column;  sigma_<i>.bin  per permutation column
//   witness.bin, breaks.bin (u64 each), lookup.bin, random.bin (2^k), blind.bin (the blinding rows in the order of use)
//   bases_m.bin, bases_l.bin   2^k affine points (64 bytes each): the SRS
// Output: proof.bin = [n_commitments u64][commitments 96 B each][n_evals u64][evals 32 B each][theta beta gamma y x]
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <sstream>

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
        std::fprintf(stderr, "usage: prover_mirror_test <dir>\n");
        return 2;
    }
    const std::string dir = argv[1];
    try {
        std::ifstream mf(dir + "/manifest.txt");
        uint32_t k;
        size_t A, L, n_wit, n_bp, n_lk, n_blind;
        int sel;
        mf >> k >> A >> L >> sel >> n_wit >> n_bp >> n_lk >> n_blind;
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
        const auto lookup = read_file<Fr>(dir + "/lookup.bin", n_lk);
        const auto rnd = read_file<Fr>(dir + "/random.bin", n);
        const auto blind = read_file<Fr>(dir + "/blind.bin", n_blind);
        size_t pos = 0;
        auto source = [&](size_t rows) {
            if (pos + rows > blind.size()) throw std::runtime_error("blind.bin exhausted");
            std::vector<Fr> b(blind.begin() + pos, blind.begin() + pos + rows);
            pos += rows;
            return b;
        };
        Proof pr;
        for (int rep = 0; rep < 2; rep++) {  // twice on one session: the working set is reused
            pos = 0;
            pr = sess.create_proof(witness, breaks, lookup, rnd, source);
        }
        if (pos != blind.size()) throw std::runtime_error("blinding rows consumed: " + std::to_string(pos) + " of " + std::to_string(blind.size()));
        std::ofstream out(dir + "/proof.bin", std::ios::binary);
        const uint64_t nc = pr.commitments.size(), ne = pr.evals.size();
        out.write(reinterpret_cast<const char*>(&nc), 8);
        out.write(reinterpret_cast<const char*>(pr.commitments.data()), std::streamsize(nc * sizeof(G1)));
        out.write(reinterpret_cast<const char*>(&ne), 8);
        for (auto& e : pr.evals) out.write(reinterpret_cast<const char*>(e.second.data()), 32);
        for (const Fr* c : {&pr.theta, &pr.beta, &pr.gamma, &pr.y, &pr.x}) out.write(reinterpret_cast<const char*>(c->data()), 32);
        std::printf("prover mirror: %zu commitments, %zu evaluations, %zu bytes up, %zu bytes down\n", size_t(nc), size_t(ne), pr.h2d_bytes, pr.d2h_bytes);
        return 0;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "prover mirror FAILED: %s\n", e.what());
        return 1;
    }
}
