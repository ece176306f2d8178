// Several constants columns through the C++ front end: keygen of a halo2-base builder with F constants columns and instance
// columns (include/h2b200_keygen.hpp), MockProver with F constants columns on cells with one broken constant
// (include/h2b200_mock.hpp), and a resident proof on the keygen circuit with the public values (include/h2b200_prover.hpp), on a
// builder the Python test wrote to a directory.  The outputs go back for a byte comparison with the Python front end
// (tests/test_gpu_constants.py::test_cpp_front_end_matches_python).
//
// Directory layout (little-endian; Fr elements are 32 bytes of Montgomery limbs, indices are u64, points 64 bytes):
//   manifest.txt   k A L selector_lookup lookup_bits max_rows n_cells n_advice_eq n_constant_eq n_lookup I count max_report F
//   cells.bin, bad_cells.bin (one tied cell changed), selectors.bin (one byte per cell), eq.bin ((a, b) pairs), consts.bin,
//   const_index.bin, lookups.bin, inst<m>.bin (count indices), pub<m>.bin (count values), rnd.bin (2^k), g.bin, gl.bin (2^k
//   affine points each)
// Output: out.bin = [n_break_points][break points], the vk's fixed then permutation commitments (12 limbs each); MockProver's
//   constants report [count][n][indices..], its raw cells (column, row) and [distinct_constants]; the proof's commitments (12
//   limbs each), evaluations (4 limbs each) and challenges theta beta gamma y x.  The blinding rows are 1, 2, 3, .. in the order
//   the prover asks for them.
#include <cstdio>
#include <fstream>
#include <iostream>

#include "../../include/h2b200_keygen.hpp"

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

template <class T>
static void put(std::ofstream& out, const T* p, size_t count) {
    out.write(reinterpret_cast<const char*>(p), std::streamsize(count * sizeof(T)));
}

int main(int argc, char** argv) {
    if (argc < 2) {
        std::fprintf(stderr, "usage: constants_test <dir>\n");
        return 2;
    }
    const std::string dir = argv[1];
    try {
        std::ifstream mf(dir + "/manifest.txt");
        uint32_t k, bits;
        size_t A, L, max_rows, N, n_eq, n_const, n_lk, I, count, max_report, F;
        int sel;
        mf >> k >> A >> L >> sel >> bits >> max_rows >> N >> n_eq >> n_const >> n_lk >> I >> count >> max_report >> F;
        if (!mf) throw std::runtime_error("bad manifest");
        const size_t n = size_t(1) << k;
        Context ctx(0);
        const ParamsKZG params(ctx, k, read_file<G1Affine>(dir + "/g.bin", n), read_file<G1Affine>(dir + "/gl.bin", n));
        const auto cells = read_file<Fr>(dir + "/cells.bin", N);
        const auto bad_cells = read_file<Fr>(dir + "/bad_cells.bin", N);
        const auto selectors = read_file<uint8_t>(dir + "/selectors.bin", N);
        const auto eq = read_file<uint64_t>(dir + "/eq.bin", 2 * n_eq);
        const auto consts = read_file<Fr>(dir + "/consts.bin", n_const);
        const auto const_idx = read_file<uint64_t>(dir + "/const_index.bin", n_const);
        const auto lookups = read_file<uint64_t>(dir + "/lookups.bin", n_lk);
        const auto rnd = read_file<Fr>(dir + "/rnd.bin", n);
        std::vector<std::vector<uint64_t>> idx;
        std::vector<std::vector<Fr>> pub;
        std::vector<const uint64_t*> idx_p;
        std::vector<const Fr*> pub_p;
        const std::vector<size_t> counts(I, count);
        for (size_t m = 0; m < I; m++) {
            idx.push_back(read_file<uint64_t>(dir + "/inst" + std::to_string(m) + ".bin", count));
            pub.push_back(read_file<Fr>(dir + "/pub" + std::to_string(m) + ".bin", count));
        }
        for (size_t m = 0; m < I; m++) {
            idx_p.push_back(idx[m].data());
            pub_p.push_back(pub[m].data());
        }
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
        v.instance_index = idx_p.data();
        v.n_instance = counts.data();
        v.n_instance_columns = I;
        std::ofstream out(dir + "/out.bin", std::ios::binary);
        // keygen
        KeygenResult kg = keygen(ctx, params, k, A, L, sel != 0, bits, max_rows, v, nullptr, F);
        const uint64_t nbp = kg.break_points.size();
        put(out, &nbp, 1);
        put(out, kg.break_points.data(), nbp);
        for (auto& f : kg.vk.fixed) put(out, &f.second, 1);
        put(out, kg.vk.permutation.data(), kg.vk.permutation.size());
        // MockProver on the cells with a broken constant
        MockProver mock(ctx, k, A, L, sel != 0, bits, max_rows, I, F);
        v.cells = bad_cells.data();
        v.instance_values = pub_p.data();
        const MockReport r = mock.run(v, max_report);
        const uint64_t head[2] = {r.constants.first, r.constants.second.size()};
        put(out, head, 2);
        put(out, r.constants.second.data(), r.constants.second.size());
        for (auto& c : r.constant_cells) {
            const uint64_t w[2] = {c.column, c.row};
            put(out, w, 2);
        }
        put(out, &r.distinct_constants, 1);
        // a proof with the public values
        ProverSession sess(ctx, params, *kg.pk);
        WitnessView w;
        w.cells = cells.data();
        w.n_cells = N;
        w.break_points = nbp ? kg.break_points.data() : nullptr;
        w.n_break_points = nbp;
        if (L) {
            w.lookup_index = lookups.data();
            w.n_lookup = n_lk;
        }
        w.instance = pub_p.data();
        w.n_instance = counts.data();
        w.n_instance_columns = I;
        uint64_t next = 1;
        const Proof pr = sess.create_proof(w, rnd.data(), [&](size_t rows) {
            std::vector<Fr> b(rows, Fr{});
            for (auto& x : b) x[0] = next++;
            return b;
        });
        put(out, pr.commitments.data(), pr.commitments.size());
        for (auto& e : pr.evals) put(out, &e.second, 1);
        for (const Fr* c : {&pr.theta, &pr.beta, &pr.gamma, &pr.y, &pr.x}) put(out, c, 1);
        return 0;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "constants test FAILED: %s\n", e.what());
        return 1;
    }
}
