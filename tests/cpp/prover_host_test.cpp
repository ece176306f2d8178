// CPU-only checks of the host pieces of include/h2b200_prover.hpp (Blake2b transcript, 254-bit host arithmetic, the
// normalisation of commitments): prints
// values that tests/test_cpp_mirror.py recomputes with hashlib and Python integers.
#include <cstdio>

#include "../../include/h2b200_prover.hpp"

using namespace h2b;

static void hex(const char* label, const void* p, size_t n) {
    std::printf("%s ", label);
    for (size_t i = 0; i < n; i++) std::printf("%02x", static_cast<const uint8_t*>(p)[i]);
    std::printf("\n");
}

int main() {
    {
        Blake2b b;
        hex("blake_empty", b.digest().data(), 64);
        b.update("abc", 3);
        hex("blake_abc", b.digest().data(), 64);
    }
    uint8_t pat[300];
    for (int i = 0; i < 300; i++) pat[i] = uint8_t(i * 7 + 3);
    {
        Blake2b b;
        b.update(pat, 96);
        b.update(pat + 96, 32);
        hex("blake_128", b.digest().data(), 64);  // exactly one full block: must be compressed as the LAST block
        b.update(pat + 128, 172);
        hex("blake_300", b.digest().data(), 64);
    }
    Transcript tr;
    tr.absorb(pat, 96);
    const Fr c1 = tr.squeeze();
    tr.absorb(pat + 96, 200);
    const Fr c2 = tr.squeeze(), c3 = tr.squeeze();
    hex("squeeze1", c1.data(), 32);
    hex("squeeze2", c2.data(), 32);
    hex("squeeze3", c3.data(), 32);
    hex("mul", HostFr::mul(c1, c2).data(), 32);
    hex("add", HostFr::add(c1, c2).data(), 32);
    hex("pow", HostFr::pow(c3, 1234567).data(), 32);
    hex("omega5", HostFr::omega(5).data(), 32);
    hex("omega19", HostFr::omega(19).data(), 32);
    uint8_t wide[64];
    for (int i = 0; i < 64; i++) wide[i] = 0xff;
    hex("wide_ff", HostFr::from_wide_bytes(wide).data(), 32);
    const G1 pt{c1, c2, c3}, nz = g1_normalize_host(pt), id = g1_normalize_host(G1{c1, c2, Fq{0, 0, 0, 0}});
    hex("normalize", &nz, 96);
    hex("normalize_identity", &id, 96);
    G1 batch[3] = {pt, G1{c2, c3, Fq{0, 0, 0, 0}}, G1{c3, c1, c2}};  // one inversion for the batch, the identity in the middle
    g1_normalize_host_batch(batch, 3);
    for (int i = 0; i < 3; i++) hex(("batch" + std::to_string(i)).c_str(), &batch[i], 96);
    return 0;
}
