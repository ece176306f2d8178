// The host field arithmetic of include/h2b200_prover.hpp (HostField<Fr / Fq>, HostFr::from_wide_bytes, HostFr::omega,
// g1_normalize_host_batch) on operands read from stdin, one request per line; tests/test_host_field_edges.py writes the
// requests and checks every answer against plain Python integers.  Field elements are 64 hex digits (the integer held
// in the 4 x 64-bit limbs, most significant digit first); `q` / `r` picks the field.
//     mul F a b | add F a b | pow F a e | inv F a | canon F c     -> one element
//     wide <128 hex digits: 64 bytes in memory order>               -> one element of Fr
//     omega k                                                       -> one element of Fr
//     norm m x0 y0 z0 ... x{m-1} y{m-1} z{m-1}                      -> 3m elements of Fq (the batch, normalised)
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>

#include "../../include/h2b200_prover.hpp"

using namespace h2b;
using E = std::array<uint64_t, 4>;

static E parse(const std::string& s) {
    E e{};
    for (int i = 0; i < 4; i++) e[3 - i] = std::stoull(s.substr(16 * i, 16), nullptr, 16);
    return e;
}

static void put(const E& e) { std::printf(" %016llx%016llx%016llx%016llx", (unsigned long long)e[3], (unsigned long long)e[2], (unsigned long long)e[1], (unsigned long long)e[0]); }

template <class F>
static E field_op(const std::string& op, std::istringstream& in) {
    std::string a, b;
    in >> a;
    if (op == "mul" || op == "add") {
        in >> b;
        return op == "mul" ? F::mul(parse(a), parse(b)) : F::add(parse(a), parse(b));
    }
    if (op == "pow") {
        in >> b;
        return F::pow(parse(a), std::stoull(b, nullptr, 16));
    }
    if (op == "inv") return F::inv(parse(a));
    if (op == "canon") {
        const E c = parse(a);
        return F::from_canonical(c.data());
    }
    throw std::runtime_error("unknown op " + op);
}

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op;
        in >> op;
        std::printf("%s", op.c_str());
        if (op == "wide") {
            std::string h;
            in >> h;
            uint8_t d[64];
            for (int i = 0; i < 64; i++) d[i] = uint8_t(std::stoul(h.substr(2 * i, 2), nullptr, 16));
            put(HostFr::from_wide_bytes(d));
        } else if (op == "omega") {
            uint32_t k;
            in >> k;
            put(HostFr::omega(k));
        } else if (op == "norm") {
            size_t m;
            in >> m;
            std::vector<G1> pts(m);
            for (auto& p : pts) {
                std::string x, y, z;
                in >> x >> y >> z;
                p = G1{parse(x), parse(y), parse(z)};
            }
            g1_normalize_host_batch(pts.data(), m);
            for (const auto& p : pts) {
                put(p.x);
                put(p.y);
                put(p.z);
            }
        } else {
            std::string f;
            in >> f;
            put(f == "q" ? field_op<HostFq>(op, in) : field_op<HostFr>(op, in));
        }
        std::printf("\n");
    }
    return 0;
}
