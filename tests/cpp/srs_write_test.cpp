// halo2-lib's params through the C++ front end (include/h2b200.hpp): setup_seeded, write, downsize, read_downsized and gen_srs
// write their bytes to a directory for a byte comparison with the Python front end
// (tests/test_gpu_srs_write.py::test_cpp_front_end_matches_python).
// Output files: k4_processed.bin, k4_raw.bin             setup_seeded(4).write(Processed / RawBytes)
//               down_12_8.bin                          setup_seeded(12), downsize(8), write(RawBytes)
//               image_12_8.bin                         read_downsized(setup_seeded(12).write(Processed), 8).write(Processed)
//               params/kzg_bn254_6.srs                 created by gen_srs(6, <dir>/params); then read back by a second call
#include <cstdio>
#include <fstream>
#include <iostream>

#include "../../include/h2b200.hpp"

using namespace h2b;

static void save(const std::string& path, const std::vector<uint8_t>& b) {
    std::ofstream f(path, std::ios::binary);
    f.write(reinterpret_cast<const char*>(b.data()), std::streamsize(b.size()));
}

int main(int argc, char** argv) {
    if (argc < 2) {
        std::fprintf(stderr, "usage: srs_write_test <dir>\n");
        return 2;
    }
    const std::string dir = argv[1];
    try {
        Context ctx(0);
        {
            ParamsKZG p = ParamsKZG::setup_seeded(ctx, 4);
            save(dir + "/k4_processed.bin", p.write(SerdeFormat::Processed));
            save(dir + "/k4_raw.bin", p.write(SerdeFormat::RawBytes));
        }
        {
            ParamsKZG p = ParamsKZG::setup_seeded(ctx, 12);
            const std::vector<uint8_t> image = p.write();
            p.downsize(8);
            save(dir + "/down_12_8.bin", p.write(SerdeFormat::RawBytes));
            ParamsKZG q = ParamsKZG::read_downsized(ctx, image, 8);
            save(dir + "/image_12_8.bin", q.write(SerdeFormat::Processed));
        }
        {
            ParamsKZG created = gen_srs(ctx, 6, dir + "/params");
            ParamsKZG read = gen_srs(ctx, 6, dir + "/params");
            if (read.k() != 6 || read.g2_processed() != created.g2_processed()) throw Error(H2B_ERR_ARG, "gen_srs: read back differs");
            bool threw = false;
            try {
                read.write();
            } catch (const Error& e) {
                threw = e.code == H2B_ERR_ARG;
            }
            if (!threw) throw Error(H2B_ERR_ARG, "write on params read from an image must fail");
        }
        std::cout << "all checks passed" << std::endl;
    } catch (const std::exception& e) {
        std::cerr << e.what() << std::endl;
        return 1;
    }
    return 0;
}
