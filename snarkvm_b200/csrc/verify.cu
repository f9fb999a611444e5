// Validation of G1 points that reach the verifier from outside (Affine::check: curves/src/templates/short_weierstrass_jacobian/
// affine.rs, is_on_curve and is_in_correct_subgroup_assuming_on_curve of curves/src/bls12_377/g1.rs:98-106).
//
//   k_g1_validate   one thread per point: coordinates below q, y² = x³ + 1, then [x²]·φ(P) + P = O with φ(x, y) = (PHI·x, y)
//
// The subgroup test is the reference's: x² (x = 0x8508c00000000001, the BLS parameter) is 127 bits, so the chain is 126 doublings
// and one mixed addition per set bit of x² in XYZZ coordinates, then one mixed addition of P.
#include "ec.cuh"
#include "msm.cuh"
#include "../../include/snarkvm_b200.h"

namespace b200 {
namespace {

// PHI of curves/src/bls12_377/g1.rs, a primitive cube root of unity in Fq (Montgomery limbs)
__constant__ uint32_t G1_PHI[12] = {0xa5847973u, 0xdacd106du, 0xbac2a79au, 0xd8fe2454u, 0xfd832edcu, 0x1ada4fd6u,
                                    0x9d150908u, 0xfb986844u, 0xea32285eu, 0xd63eb8aeu, 0x6f873fd0u, 0x0167d6a3u};
// x² = 0x452217cc900000010a11800000000001 for the BLS parameter x
constexpr uint64_t X_SQUARE_HI = 0x452217cc90000001ull, X_SQUARE_LO = 0x0a11800000000001ull;
constexpr int X_SQUARE_BITS = 127;

__global__ void __launch_bounds__(128) k_g1_validate(int32_t* __restrict__ status, const uint8_t* __restrict__ points, size_t n,
                                                     size_t stride) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const AffinePoint p = load_affine(points, stride, i);
    int32_t s = SNARKVM_B200_G1_VALID;
    if (!p.inf) {
        if (!fq_is_canonical(p.x) || !fq_is_canonical(p.y)) {
            s = SNARKVM_B200_G1_NOT_CANONICAL;
        } else if (p.y.sqr() != p.x.sqr() * p.x + Fq::one()) {
            s = SNARKVM_B200_G1_NOT_ON_CURVE;
        } else {
            Fq phi;
#pragma unroll
            for (int k = 0; k < 12; k++) phi.v[k] = G1_PHI[k];
            AffinePoint q = p;
            q.x = p.x * phi;
            XYZZ acc = XYZZ::from_affine(q);                              // the leading bit of x²
            for (int b = X_SQUARE_BITS - 2; b >= 0; b--) {
                acc.dbl();
                const uint64_t word = b >= 64 ? X_SQUARE_HI : X_SQUARE_LO;
                if ((word >> (b & 63)) & 1ull) acc.add_affine(q, false);
            }
            acc.add_affine(p, false);
            if (!acc.is_inf()) s = SNARKVM_B200_G1_NOT_IN_SUBGROUP;
        }
    }
    status[i] = s;
}

}  // namespace
}  // namespace b200

extern "C" int snarkvm_b200_g1_validate_device(int32_t* d_status, const void* d_points, size_t n, size_t stride, void* stream) {
    using namespace b200;
    if (n == 0) return 0;
    if (!d_status || !d_points || stride < 104 || stride % 8 || ((uintptr_t)d_points & 7) || ((uintptr_t)d_status & 3) ||
        n > ((size_t)1 << 31))
        return (int)cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    k_g1_validate<<<blocks, 128, 0, (cudaStream_t)stream>>>(d_status, (const uint8_t*)d_points, n, stride);
    count_launch();
    return (int)cudaGetLastError();
}
