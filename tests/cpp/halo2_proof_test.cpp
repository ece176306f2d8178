// halo2's proof bytes through the C++ front end: ProverCircuit from the fixed and sigma columns, ProverSession over params from
// host bases, and ProverSession::create_proof_halo2 with the caller's vk_repr and blinding stream, on an instance the Python test
// wrote to a directory.  The proof bytes go back for a byte comparison with the Python front end and the committed golden proof
// (tests/test_gpu_halo2_proof.py::test_cpp_front_end_matches_python).
//
// Directory layout (little-endian; Fr elements are 32 bytes of Montgomery limbs, indices are u64, points 64 bytes):
//   manifest.txt   k A L selector_lookup I F n_cells n_break_points n_lookup n_public n_blind
//   fixed_names.txt (the circuit's fixed columns, space-separated), fixed_<name>.bin and sigma<c>.bin (2^k values each),
//   cells.bin, break_points.bin, lookup.bin (the looked-up values), pub<m>.bin (n_public values per instance column), rnd.bin
//   (2^k), g.bin, gl.bin (2^k affine points each), vk_repr.bin (one Fr), blind.bin (n_blind Fr: the blinding rows, consumed in
//   the order the prover asks for them)
// Output: out.bin = the proof bytes.
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

int main(int argc, char** argv) {
    if (argc < 2) {
        std::fprintf(stderr, "usage: halo2_proof_test <dir>\n");
        return 2;
    }
    const std::string dir = argv[1];
    try {
        std::ifstream mf(dir + "/manifest.txt");
        uint32_t k;
        size_t A, L, I, F, N, nbp, n_lk, n_pub, n_blind;
        int sel;
        mf >> k >> A >> L >> sel >> I >> F >> N >> nbp >> n_lk >> n_pub >> n_blind;
        if (!mf) throw std::runtime_error("bad manifest");
        const size_t n = size_t(1) << k;
        Context ctx(0);
        const ParamsKZG params(ctx, k, read_file<G1Affine>(dir + "/g.bin", n), read_file<G1Affine>(dir + "/gl.bin", n));
        std::map<std::string, std::vector<Fr>> fixed;
        std::ifstream nf(dir + "/fixed_names.txt");
        for (std::string nm; nf >> nm;) fixed[nm] = read_file<Fr>(dir + "/fixed_" + nm + ".bin", n);
        std::vector<std::vector<Fr>> sigma;
        for (size_t c = 0; c < F + A + L + I; c++) sigma.push_back(read_file<Fr>(dir + "/sigma" + std::to_string(c) + ".bin", n));
        const ProverCircuit cs(ctx, k, A, L, sel != 0, fixed, sigma, I, F);
        const auto cells = read_file<Fr>(dir + "/cells.bin", N);
        const auto bps = read_file<uint64_t>(dir + "/break_points.bin", nbp);
        const auto lookup = read_file<Fr>(dir + "/lookup.bin", n_lk);
        const auto rnd = read_file<Fr>(dir + "/rnd.bin", n);
        const auto repr = read_file<Fr>(dir + "/vk_repr.bin", 1);
        const auto blinds = read_file<Fr>(dir + "/blind.bin", n_blind);
        std::vector<std::vector<Fr>> pub;
        std::vector<const Fr*> pub_p;
        const std::vector<size_t> counts(I, n_pub);
        for (size_t m = 0; m < I; m++) pub.push_back(read_file<Fr>(dir + "/pub" + std::to_string(m) + ".bin", n_pub));
        for (auto& p : pub) pub_p.push_back(p.data());
        ProverSession sess(ctx, params, cs);
        WitnessView w;
        w.cells = cells.data();
        w.n_cells = N;
        w.break_points = nbp ? bps.data() : nullptr;
        w.n_break_points = nbp;
        w.lookup_cells = n_lk ? lookup.data() : nullptr;
        w.n_lookup = n_lk;
        w.instance = pub_p.data();
        w.n_instance = counts.data();
        w.n_instance_columns = I;
        size_t next = 0;
        const std::vector<uint8_t> proof = sess.create_proof_halo2(w, rnd.data(), [&](size_t rows) {
            if (next + rows > blinds.size()) throw std::runtime_error("the blinding stream is too short");
            std::vector<Fr> b(blinds.begin() + next, blinds.begin() + next + rows);
            next += rows;
            return b;
        }, repr[0]);
        std::ofstream out(dir + "/out.bin", std::ios::binary);
        out.write(reinterpret_cast<const char*>(proof.data()), std::streamsize(proof.size()));
        return 0;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "halo2 proof test FAILED: %s\n", e.what());
        return 1;
    }
}
