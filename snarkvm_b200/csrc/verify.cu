// G1 points that reach the verifier from outside: validation (Affine::check: curves/src/templates/short_weierstrass_jacobian/
// affine.rs, is_on_curve and is_in_correct_subgroup_assuming_on_curve of curves/src/bls12_377/g1.rs:98-106) and the byte forms
// (CanonicalSerialize / CanonicalDeserialize of Affine<G1>, curves/src/templates/macros.rs:67-144, SWFlags of
// utilities/src/serialize/flags.rs).
//
//   k_g1_validate      one thread per point: coordinates below q, y² = x³ + 1, then [x²]·φ(P) + P = O with φ(x, y) = (PHI·x, y)
//   k_g1_deserialize   one thread per point: 48 compressed or 96 uncompressed bytes → Affine image and status; a compressed point's
//                      y is the square root of x³ + 1 (Tonelli–Shanks) whose sign the PositiveY flag picks
//   k_g1_serialize     one thread per point: normalised projective image → the compressed or uncompressed bytes
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

// Affine::check of one point: the status of the first test that fails (infinity is valid)
FF_DEV int32_t g1_check(const AffinePoint& p) {
    if (p.inf) return SNARKVM_B200_G1_VALID;
    if (!fq_is_canonical(p.x) || !fq_is_canonical(p.y)) return SNARKVM_B200_G1_NOT_CANONICAL;
    if (p.y.sqr() != p.x.sqr() * p.x + Fq::one()) return SNARKVM_B200_G1_NOT_ON_CURVE;
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
    return acc.is_inf() ? SNARKVM_B200_G1_VALID : SNARKVM_B200_G1_NOT_IN_SUBGROUP;
}

__global__ void __launch_bounds__(128) k_g1_validate(int32_t* __restrict__ status, const uint8_t* __restrict__ points, size_t n,
                                                     size_t stride) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    status[i] = g1_check(load_affine(points, stride, i));
}

// q − 1 = 2^46·t with t odd (FqParameters::TWO_ADICITY, T).  TS_ROOT = TWO_ADIC_ROOT_OF_UNITY (Montgomery limbs, = GENERATOR^t, a
// primitive 2^46-th root of unity); TS_EXP = (t − 1)/2 (330 bits); Q_HALF = (q − 1)/2, canonical: y > −y ⇔ y > Q_HALF.
constexpr int TWO_ADICITY = 46;
__constant__ uint32_t TS_ROOT[12] = {0x744e6e0fu, 0x1c104955u, 0x898dd1afu, 0xf1bd15c3u, 0x9a7f3950u, 0x76da7816u,
                                     0xe367c337u, 0xee086c1fu, 0xcbc1b61fu, 0xf95564f4u, 0x4ef58c54u, 0x00f3c141u};
__constant__ uint32_t Q_HALF[12] = {0x00000000u, 0x42846000u, 0x18000000u, 0x0b85aea2u, 0xdd04a400u, 0x8f79b117u,
                                    0x807a89c7u, 0x8d116cf9u, 0x3650a49du, 0x631d82e0u, 0x0be28875u, 0x00d71d23u};
__constant__ uint32_t TS_EXP[11] = {0x00010a11u, 0xba886000u, 0x90002e16u, 0xc45f7412u, 0x271e3de6u, 0xb3e601eau,
                                     0x92763445u, 0x0b80d942u, 0x21d58c76u, 0x748c2f8au, 0x0000035cu};

// Tonelli–Shanks: a square root of the Montgomery image a, or false when a is no square.  Any root serves: the caller picks the
// sign.  With b = a^t of order 2^k, each round multiplies b by an element of order 2^k, so k falls; a non-residue has k = 46.
__device__ __noinline__ bool fq_sqrt(Fq a, Fq* root) {
    if (a.is_zero()) { *root = a; return true; }
    const Fq one = Fq::one();
    Fq w = a.pow_const<11>(TS_EXP);                               // a^((t − 1)/2)
    Fq x = a * w;                                                 // a^((t + 1)/2)
    Fq b = x * w;                                                 // a^t
    Fq z;
#pragma unroll
    for (int k = 0; k < 12; k++) z.v[k] = TS_ROOT[k];
    int v = TWO_ADICITY;
    while (b != one) {
        int k = 0;
        Fq b2k = b;
        while (b2k != one && k < v) { b2k = b2k.sqr(); k++; }
        if (k == v) return false;
        Fq c = z;                                                 // z^(2^(v − k − 1)), of order 2^(k + 1)
        for (int j = 0; j < v - k - 1; j++) c = c.sqr();
        z = c.sqr();
        b = b * z;
        x = x * c;
        v = k;
    }
    *root = x;
    return true;
}

// 48 little-endian bytes → raw limbs; `top_mask` clears flag bits of the last byte
FF_DEV Fq fq_from_bytes(const uint8_t* p, uint8_t top_mask) {
    Fq r;
#pragma unroll
    for (int k = 0; k < 12; k++) {
        uint32_t b3 = p[4 * k + 3];
        if (k == 11) b3 &= top_mask;
        r.v[k] = (uint32_t)p[4 * k] | ((uint32_t)p[4 * k + 1] << 8) | ((uint32_t)p[4 * k + 2] << 16) | (b3 << 24);
    }
    return r;
}

FF_DEV void fq_to_bytes(uint8_t* p, const Fq& a, uint8_t flags) {
#pragma unroll
    for (int k = 0; k < 12; k++) {
        p[4 * k] = (uint8_t)a.v[k];
        p[4 * k + 1] = (uint8_t)(a.v[k] >> 8);
        p[4 * k + 2] = (uint8_t)(a.v[k] >> 16);
        p[4 * k + 3] = (uint8_t)(a.v[k] >> 24) | (k == 11 ? flags : 0);
    }
}

// the canonical value of a Montgomery image is above (q − 1)/2, i.e. y > −y as the reference orders field elements
FF_DEV bool fq_above_half(const Fq& a) {
    const Fq c = a.from_mont();
    (void)ptx_sub_cc(Q_HALF[0], c.v[0]);
#pragma unroll
    for (int k = 1; k < 12; k++) (void)ptx_subc_cc(Q_HALF[k], c.v[k]);
    return ptx_subc(0u, 0u) != 0u;                                // borrow of Q_HALF − c
}

constexpr uint8_t FLAG_POSITIVE_Y = 0x80, FLAG_INFINITY = 0x40;

__global__ void __launch_bounds__(128) k_g1_deserialize(uint8_t* __restrict__ points, int32_t* __restrict__ status,
                                                        const uint8_t* __restrict__ bytes, size_t n, int compressed, int validate) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    AffinePoint p;
    p.x = Fq::zero(); p.y = Fq::zero(); p.inf = false;            // the image of bytes that decode to no point
    int32_t s = SNARKVM_B200_G1_VALID;
    bool decoded = false;
    if (compressed) {
        const uint8_t* src = bytes + i * 48;
        const uint8_t flags = src[47] & 0xC0;
        const Fq x = fq_from_bytes(src, 0x3F);
        if (flags == 0xC0) {
            s = SNARKVM_B200_G1_BAD_FLAGS;
        } else if (!fq_is_canonical(x)) {
            s = SNARKVM_B200_G1_NOT_CANONICAL;
        } else if (flags == FLAG_INFINITY) {
            decoded = true;                                       // Affine::zero() = (0, 1, infinity), whatever x was
            p.y = Fq::one(); p.inf = true;
        } else {
            const Fq xm = x.to_mont();
            Fq y;
            if (!fq_sqrt(xm.sqr() * xm + Fq::one(), &y)) {
                s = SNARKVM_B200_G1_NOT_ON_CURVE;                 // no point of the curve has this x
            } else {
                // from_x_coordinate: the larger root of the two when PositiveY is set, the smaller otherwise
                if (fq_above_half(y) != (flags == FLAG_POSITIVE_Y)) y = y.neg();
                p.x = xm; p.y = y;
                decoded = true;
            }
        }
    } else {
        const uint8_t* src = bytes + i * 96;
        const uint8_t flags = src[95] & 0xC0;
        const Fq x = fq_from_bytes(src, 0xFF), y = fq_from_bytes(src + 48, 0x3F);
        if (src[47] & 0x80) {
            s = SNARKVM_B200_G1_BAD_FLAGS;                        // x carries no flags (EmptyFlags)
        } else if (!fq_is_canonical(x)) {
            s = SNARKVM_B200_G1_NOT_CANONICAL;
        } else if (flags == 0xC0) {
            s = SNARKVM_B200_G1_BAD_FLAGS;
        } else if (!fq_is_canonical(y)) {
            s = SNARKVM_B200_G1_NOT_CANONICAL;
        } else if (flags == FLAG_INFINITY) {
            decoded = true;
            p.y = Fq::one(); p.inf = true;
        } else {
            p.x = x.to_mont(); p.y = y.to_mont();                 // Affine::new: no curve test unless validate
            decoded = true;
        }
    }
    if (decoded && validate) s = g1_check(p);
    store_affine(points, 104, i, p);
    status[i] = s;
}

__global__ void __launch_bounds__(128) k_g1_serialize(uint8_t* __restrict__ bytes, const uint8_t* __restrict__ projective, size_t n,
                                                      int compressed) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* src = projective + i * 144;
    const Fq X = load_fq_u64(src), Y = load_fq_u64(src + 48), Z = load_fq_u64(src + 96);
    Fq x = Fq::zero(), y = Fq::zero();
    uint8_t flags = FLAG_INFINITY;
    if (!Z.is_zero()) {                                           // normalised: Z = one, (X, Y) = (x, y)
        x = X.from_mont();
        y = Y.from_mont();
        flags = compressed && fq_above_half(Y) ? FLAG_POSITIVE_Y : 0;
    } else {
        y.v[0] = 1u;                                              // Affine::zero() = (0, 1)
    }
    if (compressed) {
        fq_to_bytes(bytes + i * 48, x, flags);
    } else {
        fq_to_bytes(bytes + i * 96, x, 0);
        fq_to_bytes(bytes + i * 96 + 48, y, flags);
    }
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

extern "C" int snarkvm_b200_g1_deserialize_device(void* d_points, int32_t* d_status, const void* d_bytes, size_t n, int compressed,
                                                  int validate, void* stream) {
    using namespace b200;
    if (n == 0) return 0;
    if (!d_points || !d_status || !d_bytes || ((uintptr_t)d_points & 7) || ((uintptr_t)d_status & 3) || n > ((size_t)1 << 31))
        return (int)cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    k_g1_deserialize<<<blocks, 128, 0, (cudaStream_t)stream>>>((uint8_t*)d_points, d_status, (const uint8_t*)d_bytes, n,
                                                               compressed ? 1 : 0, validate ? 1 : 0);
    count_launch();
    return (int)cudaGetLastError();
}

extern "C" int snarkvm_b200_g1_serialize_device(void* d_bytes, const void* d_projective, size_t n, int compressed, void* stream) {
    using namespace b200;
    if (n == 0) return 0;
    if (!d_bytes || !d_projective || ((uintptr_t)d_projective & 7) || n > ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    k_g1_serialize<<<blocks, 128, 0, (cudaStream_t)stream>>>((uint8_t*)d_bytes, (const uint8_t*)d_projective, n, compressed ? 1 : 0);
    count_launch();
    return (int)cudaGetLastError();
}
