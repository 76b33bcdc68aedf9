// kb2_muvera_proj.cpp — the MUVERA projections (kb2_muvera.cuh), in a host translation unit of their own.
// The library is built with -mfma, and GCC then contracts a * b + c into fused multiply-adds, also inside
// std::normal_distribution: its draws would differ from the reference's (built without FMA) in the last bit.  Every
// function of this file, the standard library's templates instantiated here included, is compiled without contraction.
#pragma GCC optimize("fp-contract=off")
#include <cstdint>
#include <random>
#include <vector>

namespace kb2 {

// [R][P][d] projections, row-major per repeat: repeat r draws P * d values in order from N(0, 1) over mt19937(S + r)
std::vector<float>
muvera_projections(int P, int R, int S, int d) {
    std::vector<float> h((size_t)R * P * d);
    for (int r = 0; r < R; r++) {
        std::mt19937 rng((uint32_t)((int64_t)S + r));   // the reference's int32 seed + r, taken modulo 2^32
        std::normal_distribution<float> nd(0.0f, 1.0f);
        for (size_t i = 0; i < (size_t)P * d; i++) h[(size_t)r * P * d + i] = nd(rng);
    }
    return h;
}

}  // namespace kb2
