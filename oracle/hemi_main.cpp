// ORACLE — TEST INFRASTRUCTURE ONLY. Never linked into or called from the product path.
//
// `modkit_oracle_hemi pileup-hemi [flags] <in.bam> -r <ref.fa> [-o out.bed]`: the CPU restatement of `modkit pileup-hemi`
// (hemi.hpp), a binary of its own beside modkit_oracle. Built on demand by tests/test_hemi_cpu.py (fixture hemi_oracle_exe):
//     g++ -O2 -std=c++17 -ffp-contract=off -pthread oracle/hemi_main.cpp -o oracle/_build/modkit_oracle_hemi -lz
#include "hemi.hpp"

int main(int argc, char** argv) {
    try {
        if (argc < 2 || std::string(argv[1]) != "pileup-hemi") throw std::runtime_error("usage: modkit_oracle_hemi pileup-hemi [flags] <in.bam> -r <ref.fa> [-o out.bed]");
        return orc::hemi_main(argc, argv);
    } catch (const std::exception& e) {
        fprintf(stderr, "> Error! %s\n", e.what());
        return 1;
    }
}
