// G1 points that reach the verifier from outside: validation (Affine::check: curves/src/templates/short_weierstrass_jacobian/
// affine.rs, is_on_curve and is_in_correct_subgroup_assuming_on_curve of curves/src/bls12_377/g1.rs:98-106) and the byte forms
// (CanonicalSerialize / CanonicalDeserialize of Affine<G1>, curves/src/templates/macros.rs:67-144, SWFlags of
// utilities/src/serialize/flags.rs; ToBytes / FromBytes of Affine, short_weierstrass_jacobian/affine.rs:293-313).  The same for G2
// (Valid for Affine<G2>: is_on_curve and [r]·P = O, curves/src/bls12_377/g2.rs:120-124; Fp2 with flags, fields/src/fp2.rs:427-457,
// ordered c1 first, :241-250).  Also the Fr records of a proving key's byte form (matrix entries and evaluations, CanonicalSerialize
// of Circuit) and its matrix row walk.
//
//   k_g1_validate      one thread per point: coordinates below q, y² = x³ + 1, then [x²]·φ(P) + P = O with φ(x, y) = (PHI·x, y)
//   k_g1_deserialize   one thread per point: 48 compressed, 96 uncompressed or 97 ToBytes bytes → Affine image and status; a
//                      compressed point's y is the square root of x³ + 1 (Tonelli–Shanks) whose sign the PositiveY flag picks
//   k_g1_serialize     one thread per point: normalised projective image → the compressed or uncompressed bytes, or Affine image →
//                      the 97 ToBytes bytes
//   k_g2_validate      one thread per point: coordinates below q, y² = x³ + B', then [r]·P = O
//   k_g2_deserialize   one thread per point: 96 compressed or 192 uncompressed bytes → Affine<G2> image and status; a compressed
//                      point's y is a square root of x³ + B' in Fq2 (by the norm, on Tonelli–Shanks in Fq), signed by PositiveY
//   k_g2_serialize     one thread per point: Affine<G2> image → the compressed or uncompressed bytes
//   k_fr_records       one thread per record of every segment: canonical Fr (and column) → Montgomery Fr (and int32 column)
//   k_test_sqrt        one thread per element: fq_sqrt or fq2_sqrt as the decoders call them, for the tests
//
// The G1 subgroup test is the reference's: x² (x = 0x8508c00000000001, the BLS parameter) is 127 bits, so the chain is 126
// doublings and one mixed addition per set bit of x² in XYZZ coordinates, then one mixed addition of P.  The G2 test is the
// reference's too, mul_bits by r: 252 doublings and 87 mixed additions of P in XYZZ coordinates over Fq2.
#include <cstring>
#include <vector>

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
                                                        const uint8_t* __restrict__ bytes, size_t n, int form, int validate) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    AffinePoint p;
    p.x = Fq::zero(); p.y = Fq::zero(); p.inf = false;            // the image of bytes that decode to no point
    int32_t s = SNARKVM_B200_G1_VALID;
    bool decoded = false;
    if (form == SNARKVM_B200_G1_FORM_TO_BYTES) {
        // FromBytes for Affine: x, y (Fq::read_le: below q), the infinity flag (bool::read_le: 0 or 1), then the only test the
        // reference makes, `infinity != x.is_zero() && y.is_one()` refused; Affine::new keeps x and y, infinity included
        const uint8_t* src = bytes + i * 97;
        const Fq x = fq_from_bytes(src, 0xFF), y = fq_from_bytes(src + 48, 0xFF);
        const uint8_t inf = src[96];
        Fq one_raw = Fq::zero();
        one_raw.v[0] = 1u;
        if (!fq_is_canonical(x) || !fq_is_canonical(y)) {
            s = SNARKVM_B200_G1_NOT_CANONICAL;
        } else if (inf > 1 || ((inf == 1) != x.is_zero() && y == one_raw)) {
            s = SNARKVM_B200_G1_BAD_FLAGS;
        } else {
            p.x = x.to_mont(); p.y = y.to_mont(); p.inf = inf == 1;
            decoded = true;
        }
    } else if (form == SNARKVM_B200_G1_FORM_COMPRESSED) {
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
                                                      int form) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (form == SNARKVM_B200_G1_FORM_TO_BYTES) {                  // ToBytes of the Affine image: x, y as held, the infinity byte
        const AffinePoint a = load_affine(projective, 104, i);
        uint8_t* dst = bytes + i * 97;
        fq_to_bytes(dst, a.x.from_mont(), 0);
        fq_to_bytes(dst + 48, a.y.from_mont(), 0);
        dst[96] = a.inf ? 1 : 0;
        return;
    }
    const bool compressed = form == SNARKVM_B200_G1_FORM_COMPRESSED;
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

// b1 of G2's WEIERSTRASS_B = (0, b1) (curves/src/bls12_377/g2.rs, as G2_B1 of pairing.cu), Montgomery limbs.  b1 = −1/5, which
// the square root below also uses: −5 is the non-residue that defines Fq2.
__constant__ uint32_t G2_B1[12] = {0x66666685u, 0x80722666u, 0x899999a9u, 0x8df55926u, 0xd64f34cfu, 0x7fe4561au,
                                   0xb6e4f01bu, 0xb95da6d8u, 0xfc142743u, 0x4b747cccu, 0x70f49f43u, 0x0039c3fau};
// 1/2 (Montgomery limbs)
__constant__ uint32_t FQ_HALF[12] = {0xffffffb4u, 0x8166ffffu, 0xbfffffd8u, 0x28a04fc1u, 0xc53e9ff9u, 0xcfbed9d4u,
                                     0xb73e3182u, 0x3da74bdbu, 0xc01e4274u, 0x267a4adfu, 0xf17efa4du, 0x0046b330u};
// r = 0x12ab655e9a2ca55660b44d1e5c37b00159aa76fed00000010a11800000000001 (FrParameters::MODULUS), 253 bits, 88 of them set
__constant__ uint64_t R_WORDS[4] = {0x0a11800000000001ull, 0x59aa76fed0000001ull, 0x60b44d1e5c37b001ull, 0x12ab655e9a2ca556ull};
constexpr int R_BITS = 253;

FF_DEV Fq fq_from_const(const uint32_t (&t)[12]) {
    Fq r;
#pragma unroll
    for (int k = 0; k < 12; k++) r.v[k] = t[k];
    return r;
}

// x³ + B'
FF_DEV Fq2 g2_curve_rhs(const Fq2& x) {
    Fq2 r = x.sqr() * x;
    r.c1 = r.c1 + fq_from_const(G2_B1);
    return r;
}

// y > −y in the reference's order on Fp2: c1 decides unless it is zero (then c1 = −c1), and c0 decides after it
FF_DEV bool fq2_above_half(const Fq2& a) { return a.c1.is_zero() ? fq_above_half(a.c0) : fq_above_half(a.c1); }

// Fq2 for the [r]·P chain: the same arithmetic, with every Fq product an out-of-line call (Fp::mul_call, as FF_CALL_MUL makes
// them in msm_g2.cu), so that the accumulator stays in registers around the products
struct Fq2c {
    Fq2 a;
    static constexpr int WORDS = Fq2::WORDS;
    FF_DEV static Fq2c of(const Fq2& v) { Fq2c r; r.a = v; return r; }
    FF_DEV static Fq2c zero() { return of(Fq2::zero()); }
    FF_DEV static Fq2c one() { return of(Fq2::one()); }
    FF_DEV bool is_zero() const { return a.is_zero(); }
    FF_DEV Fq2c neg() const { return of(a.neg()); }
    FF_DEV Fq2c dbl() const { return of(a.dbl()); }
    FF_DEV friend Fq2c operator+(const Fq2c& x, const Fq2c& y) { return of(x.a + y.a); }
    FF_DEV friend Fq2c operator-(const Fq2c& x, const Fq2c& y) { return of(x.a - y.a); }
    FF_DEV friend Fq2c operator*(const Fq2c& x, const Fq2c& y) {
        const Fq v0 = Fq::mul_call(x.a.c0, y.a.c0), v1 = Fq::mul_call(x.a.c1, y.a.c1);
        Fq2c r;
        r.a.c1 = Fq::mul_call(x.a.c0 + x.a.c1, y.a.c0 + y.a.c1) - v0 - v1;
        r.a.c0 = v0 - Fq2::times5(v1);
        return r;
    }
    FF_DEV Fq2c sqr() const {
        const Fq t = Fq::mul_call(a.c0, a.c1);
        Fq2c r;
        r.a.c0 = Fq::mul_call(a.c0 + a.c1, a.c0 - Fq2::times5(a.c1)) + t.dbl().dbl();
        r.a.c1 = t.dbl();
        return r;
    }
};
using ChainF = Fq2c;

// one coordinate of an Affine<G2> image, read from global memory where it is used: an asm load, which the compiler neither hoists
// out of the chain nor forwards from the decoder's store, so P is not held in registers across the chain
FF_DEV Fq fq_load_at_use(const uint8_t* p) {
    Fq r;
#pragma unroll
    for (int k = 0; k < 6; k++)
        asm volatile("ld.global.v2.u32 {%0, %1}, [%2];" : "=r"(r.v[2 * k]), "=r"(r.v[2 * k + 1]) : "l"(p + 8 * k));
    return r;
}
FF_DEV AffineT<ChainF> g2_load_at_use(const uint8_t* img) {
    AffineT<ChainF> a;
    Fq2 x, y;
    x.c0 = fq_load_at_use(img); x.c1 = fq_load_at_use(img + 48);
    y.c0 = fq_load_at_use(img + 96); y.c1 = fq_load_at_use(img + 144);
    a.x = Fq2c::of(x); a.y = Fq2c::of(y); a.inf = false;
    return a;
}

// The chain's group law on XyzzT over Fq2: dbl-2008-s-1 and madd-2008-s as XyzzT::dbl / add_affine compute them, with the
// products reordered so that each temporary dies early (ZZ and ZZZ are updated as soon as their factor exists).  In XyzzT's own
// order eight Fq2 values (192 registers) are live at once and the chain spills; in this order it does not.
FF_DEV void g2_chain_dbl(XyzzT<ChainF>& a) {
    if (a.is_inf()) return;
    const ChainF U = a.Y.dbl();
    const ChainF V = U.sqr();
    const ChainF W = U * V;
    a.ZZ = V * a.ZZ;
    a.ZZZ = W * a.ZZZ;
    const ChainF S = a.X * V;
    a.Y = W * a.Y;                                                // W·Y, subtracted below
    const ChainF XX = a.X.sqr();
    const ChainF M = XX.dbl() + XX;
    a.X = M.sqr() - S.dbl();
    a.Y = M * (S - a.X) - a.Y;
}

// acc + P for the image at `img`; P's coordinates are read where they are used
FF_DEV void g2_chain_add(XyzzT<ChainF>& a, const uint8_t* img) {
    if (a.is_inf()) { a = XyzzT<ChainF>::from_affine(g2_load_at_use(img)); return; }
    ChainF P, R;
    {
        const AffineT<ChainF> q = g2_load_at_use(img);
        P = q.x * a.ZZ - a.X;
        R = q.y * a.ZZZ - a.Y;
    }
    if (P.is_zero()) {
        if (R.is_zero()) { a = XyzzT<ChainF>::from_affine(g2_load_at_use(img)); g2_chain_dbl(a); }   // acc = P: 2·P
        else a = XyzzT<ChainF>::infinity();                                                         // acc = −P
        return;
    }
    const ChainF PP = P.sqr();
    const ChainF PPP = P * PP;
    a.ZZ = a.ZZ * PP;
    a.ZZZ = a.ZZZ * PPP;
    const ChainF Q = a.X * PP;
    a.Y = a.Y * PPP;                                              // Y·PPP, subtracted below
    a.X = R.sqr() - PPP - Q.dbl();
    a.Y = R * (Q - a.X) - a.Y;
}

// Valid for Affine<G2> of the Affine<G2> image at `img` (global memory): the status of the first test that fails (infinity is
// valid).  The chain is complete: the mixed addition doubles when it meets P and returns O when it meets −P, so off-subgroup
// points run it as well.
__device__ __noinline__ int32_t g2_check(const uint8_t* img) {
    if (img[192]) return SNARKVM_B200_G1_VALID;
    {
        Fq2 x, y;
        x.c0 = fq_load_at_use(img); x.c1 = fq_load_at_use(img + 48);
        y.c0 = fq_load_at_use(img + 96); y.c1 = fq_load_at_use(img + 144);
        if (!fq_is_canonical(x.c0) || !fq_is_canonical(x.c1) || !fq_is_canonical(y.c0) || !fq_is_canonical(y.c1))
            return SNARKVM_B200_G1_NOT_CANONICAL;
        if (y.sqr() != g2_curve_rhs(x)) return SNARKVM_B200_G1_NOT_ON_CURVE;
    }
    XyzzT<ChainF> acc = XyzzT<ChainF>::from_affine(g2_load_at_use(img));   // the leading bit of r
    for (int b = R_BITS - 2; b >= 0; b--) {
        g2_chain_dbl(acc);
        if ((R_WORDS[b >> 6] >> (b & 63)) & 1ull) g2_chain_add(acc, img);
    }
    return acc.is_inf() ? SNARKVM_B200_G1_VALID : SNARKVM_B200_G1_NOT_IN_SUBGROUP;
}

__global__ void __launch_bounds__(128) k_g2_validate(int32_t* __restrict__ status, const uint8_t* __restrict__ points, size_t n,
                                                     size_t stride) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    status[i] = g2_check(points + i * stride);
}

// A square root of a = a0 + a1·u in Fq2 (u² = −5), or false when a is no square.  a is a square iff its norm a0² + 5·a1² is one
// in Fq.  With a1 ≠ 0 and n = √(a0² + 5·a1²), exactly one of t = (a0 ± n)/2 is a square in Fq (their product −5·a1²/4 is not), and
// (c0 + c1·u)² = a for c0 = √t, c1 = a1/(2·c0).  With a1 = 0 the root is √a0, or √(−a0/5)·u when a0 is no square.  Any root
// serves: the caller picks the sign.
__device__ __noinline__ bool fq2_sqrt(Fq2 a, Fq2* root) {
    Fq2 r;
    if (a.c1.is_zero()) {
        r.c1 = Fq::zero();
        if (!fq_sqrt(a.c0, &r.c0)) {
            r.c0 = Fq::zero();
            if (!fq_sqrt(a.c0 * fq_from_const(G2_B1), &r.c1)) return false;      // a0·b1 = −a0/5: a square when a0 is not
        }
    } else {
        Fq n;
        if (!fq_sqrt(a.c0.sqr() + Fq2::times5(a.c1.sqr()), &n)) return false;
        const Fq half = fq_from_const(FQ_HALF);
        if (!fq_sqrt((a.c0 + n) * half, &r.c0) && !fq_sqrt((a.c0 - n) * half, &r.c0)) return false;
        r.c1 = a.c1 * r.c0.dbl().inverse();
    }
    *root = r;
    return true;
}

// CanonicalDeserialize of Affine<G2>: the coordinates are read in order (x.c0, x.c1, then y.c0, y.c1 when uncompressed), each
// refused for bit 7 of its last byte (EmptyFlags) and then for a value not below q; the last one carries the SWFlags in its top two
// bits instead, refused when both are set.
__global__ void __launch_bounds__(128) k_g2_deserialize(uint8_t* __restrict__ points, int32_t* __restrict__ status,
                                                        const uint8_t* __restrict__ bytes, size_t n, int compressed, int validate) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int ncoords = compressed ? 2 : 4;
    const uint8_t* src = bytes + i * 48 * ncoords;
    const uint8_t flags = src[48 * ncoords - 1] & 0xC0;
    AffineT<Fq2> p;
    p.x = Fq2::zero(); p.y = Fq2::zero(); p.inf = false;          // the image of bytes that decode to no point
    Fq c[4];
    int32_t s = SNARKVM_B200_G1_VALID;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (k >= ncoords || s != SNARKVM_B200_G1_VALID) break;
        const bool last = k == ncoords - 1;
        if (last ? flags == 0xC0 : (src[48 * k + 47] & 0x80) != 0) {
            s = SNARKVM_B200_G1_BAD_FLAGS;
        } else {
            c[k] = fq_from_bytes(src + 48 * k, last ? 0x3F : 0xFF);
            if (!fq_is_canonical(c[k])) s = SNARKVM_B200_G1_NOT_CANONICAL;
        }
    }
    bool decoded = false;
    if (s != SNARKVM_B200_G1_VALID) {
    } else if (flags == FLAG_INFINITY) {
        decoded = true;                                           // Affine::zero() = (0, 1, infinity), whatever the coordinates were
        p.y = Fq2::one(); p.inf = true;
    } else if (compressed) {
        Fq2 x, y;
        x.c0 = c[0].to_mont(); x.c1 = c[1].to_mont();
        if (!fq2_sqrt(g2_curve_rhs(x), &y)) {
            s = SNARKVM_B200_G1_NOT_ON_CURVE;                     // no point of the curve has this x
        } else {
            // from_x_coordinate: the larger root of the two when PositiveY is set, the smaller otherwise
            if (fq2_above_half(y) != (flags == FLAG_POSITIVE_Y)) y = y.neg();
            p.x = x; p.y = y;
            decoded = true;
        }
    } else {
        p.x.c0 = c[0].to_mont(); p.x.c1 = c[1].to_mont();         // Affine::new: no curve test unless validate
        p.y.c0 = c[2].to_mont(); p.y.c1 = c[3].to_mont();
        decoded = true;
    }
    store_affine_g2(points, 200, i, p);
    if (decoded && validate) s = g2_check(points + i * 200);
    status[i] = s;
}

__global__ void __launch_bounds__(128) k_g2_serialize(uint8_t* __restrict__ bytes, const uint8_t* __restrict__ points, size_t n,
                                                      int compressed) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const AffineT<Fq2> a = load_affine_g2(points, 200, i);
    Fq2 x = Fq2::zero(), y = Fq2::zero();
    uint8_t flags = FLAG_INFINITY;
    if (!a.inf) {
        x.c0 = a.x.c0.from_mont(); x.c1 = a.x.c1.from_mont();
        y.c0 = a.y.c0.from_mont(); y.c1 = a.y.c1.from_mont();
        flags = compressed && fq2_above_half(a.y) ? FLAG_POSITIVE_Y : 0;
    } else {
        y.c0.v[0] = 1u;                                           // Affine::zero() = (0, 1)
    }
    if (compressed) {
        uint8_t* dst = bytes + i * 96;
        fq_to_bytes(dst, x.c0, 0);
        fq_to_bytes(dst + 48, x.c1, flags);
    } else {
        uint8_t* dst = bytes + i * 192;
        fq_to_bytes(dst, x.c0, 0);
        fq_to_bytes(dst + 48, x.c1, 0);
        fq_to_bytes(dst + 96, y.c0, 0);
        fq_to_bytes(dst + 144, y.c1, flags);
    }
}

// A run of Fr records in a proving key's bytes.  Thread g takes record g − first of its segment: record e sits at src + stride·e,
// or — a matrix entry, row_ptr set — at src + 16 + 8·row(e) + 40·e (the u64 row count, then per row a u64 length and the row's
// entries).  The row is searched in [0, nrows), so a row_ptr that disagrees with the section cannot move a read past the extent
// the host checked.  The first bad record of a segment wins an atomicMin of (e << 2 | reason).
struct FrRecordSeg {
    uint64_t first, src, count;
    uint32_t stride, nrows;
    const uint32_t* row_ptr;
    uint32_t* out;
    int32_t* cols;
    uint64_t num_cols;
};
constexpr unsigned long long FR_RECORD_NOT_CANONICAL = 1, FR_RECORD_BAD_COLUMN = 2;

FF_DEV bool fr_is_canonical(const Fr& a) {
    (void)ptx_sub_cc(a.v[0], FrParams::mod(0));
#pragma unroll
    for (int k = 1; k < 8; k++) (void)ptx_subc_cc(a.v[k], FrParams::mod(k));
    return ptx_subc(0u, 0u) != 0u;
}

__global__ void __launch_bounds__(256) k_fr_records(const FrRecordSeg* __restrict__ segs, uint32_t nsegs, uint64_t total,
                                                    const uint8_t* __restrict__ blob, unsigned long long* __restrict__ bad) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    uint32_t lo = 0, hi = nsegs;                                  // the last segment whose `first` is ≤ g
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (segs[mid].first <= g) lo = mid; else hi = mid;
    }
    const FrRecordSeg& sg = segs[lo];
    const uint64_t e = g - sg.first;
    uint64_t at = sg.src + (uint64_t)sg.stride * e;
    if (sg.row_ptr) {
        uint32_t rlo = 0, rhi = sg.nrows;                         // the last row whose start is ≤ e
        while (rhi - rlo > 1) {
            const uint32_t mid = rlo + (rhi - rlo) / 2;
            if (__ldg(sg.row_ptr + mid) <= e) rlo = mid; else rhi = mid;
        }
        at = sg.src + 16 + 8 * (uint64_t)rlo + 40 * e;
    }
    const uint8_t* p = blob + at;
    Fr v;
#pragma unroll
    for (int k = 0; k < 8; k++)
        v.v[k] = (uint32_t)p[4 * k] | ((uint32_t)p[4 * k + 1] << 8) | ((uint32_t)p[4 * k + 2] << 16) | ((uint32_t)p[4 * k + 3] << 24);
    unsigned long long reason = 0;
    if (!fr_is_canonical(v)) {
        reason = FR_RECORD_NOT_CANONICAL;
        v = Fr::zero();
    }
    if (sg.cols) {
        uint64_t c = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) c |= (uint64_t)p[32 + k] << (8 * k);
        if (c >= sg.num_cols && !reason) reason = FR_RECORD_BAD_COLUMN;
        sg.cols[e] = c < sg.num_cols ? (int32_t)c : 0;
    }
    v.to_mont().store(sg.out + 8 * e);
    if (reason) atomicMin(bad + lo, (e << 2) | reason);
}

// Element-wise square roots for the tests (snarkvm_b200_test_sqrt_device): the decoders' own out-of-line fq_sqrt / fq2_sqrt, one
// thread per element; an element without a root gets a zero root
__global__ void __launch_bounds__(128) k_test_sqrt(uint32_t* __restrict__ out, int32_t* __restrict__ ok, const uint32_t* __restrict__ in,
                                                   size_t n, int field) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool s;
    if (field == SNARKVM_B200_FIELD_FQ) {
        Fq r = Fq::zero();
        s = fq_sqrt(Fq::load(in + 12 * i), &r);
        (s ? r : Fq::zero()).store(out + 12 * i);
    } else {
        Fq2 a, r = Fq2::zero();
        a.c0 = Fq::load(in + 24 * i); a.c1 = Fq::load(in + 24 * i + 12);
        s = fq2_sqrt(a, &r);
        if (!s) r = Fq2::zero();
        r.c0.store(out + 24 * i); r.c1.store(out + 24 * i + 12);
    }
    ok[i] = s ? 1 : 0;
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

extern "C" int snarkvm_b200_g1_deserialize_device(void* d_points, int32_t* d_status, const void* d_bytes, size_t n, int form,
                                                  int validate, void* stream) {
    using namespace b200;
    if (n == 0) return 0;
    if (!d_points || !d_status || !d_bytes || ((uintptr_t)d_points & 7) || ((uintptr_t)d_status & 3) || n > ((size_t)1 << 31) ||
        form < SNARKVM_B200_G1_FORM_UNCOMPRESSED || form > SNARKVM_B200_G1_FORM_TO_BYTES)
        return (int)cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    k_g1_deserialize<<<blocks, 128, 0, (cudaStream_t)stream>>>((uint8_t*)d_points, d_status, (const uint8_t*)d_bytes, n, form,
                                                               validate ? 1 : 0);
    count_launch();
    return (int)cudaGetLastError();
}

extern "C" int snarkvm_b200_g1_serialize_device(void* d_bytes, const void* d_points, size_t n, int form, void* stream) {
    using namespace b200;
    if (n == 0) return 0;
    if (!d_bytes || !d_points || ((uintptr_t)d_points & 7) || n > ((size_t)1 << 31) || form < SNARKVM_B200_G1_FORM_UNCOMPRESSED ||
        form > SNARKVM_B200_G1_FORM_TO_BYTES)
        return (int)cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    k_g1_serialize<<<blocks, 128, 0, (cudaStream_t)stream>>>((uint8_t*)d_bytes, (const uint8_t*)d_points, n, form);
    count_launch();
    return (int)cudaGetLastError();
}

extern "C" int snarkvm_b200_g2_validate_device(int32_t* d_status, const void* d_points, size_t n, size_t stride, void* stream) {
    using namespace b200;
    if (n == 0) return 0;
    if (!d_status || !d_points || stride < 200 || stride % 8 || ((uintptr_t)d_points & 7) || ((uintptr_t)d_status & 3) ||
        n > ((size_t)1 << 31))
        return (int)cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    k_g2_validate<<<blocks, 128, 0, (cudaStream_t)stream>>>(d_status, (const uint8_t*)d_points, n, stride);
    count_launch();
    return (int)cudaGetLastError();
}

extern "C" int snarkvm_b200_g2_deserialize_device(void* d_points, int32_t* d_status, const void* d_bytes, size_t n, int compressed,
                                                  int validate, void* stream) {
    using namespace b200;
    if (n == 0) return 0;
    if (!d_points || !d_status || !d_bytes || ((uintptr_t)d_points & 7) || ((uintptr_t)d_status & 3) || n > ((size_t)1 << 31))
        return (int)cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    k_g2_deserialize<<<blocks, 128, 0, (cudaStream_t)stream>>>((uint8_t*)d_points, d_status, (const uint8_t*)d_bytes, n,
                                                               compressed ? 1 : 0, validate ? 1 : 0);
    count_launch();
    return (int)cudaGetLastError();
}

extern "C" int snarkvm_b200_g2_serialize_device(void* d_bytes, const void* d_points, size_t n, int compressed, void* stream) {
    using namespace b200;
    if (n == 0) return 0;
    if (!d_bytes || !d_points || ((uintptr_t)d_points & 7) || n > ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    k_g2_serialize<<<blocks, 128, 0, (cudaStream_t)stream>>>((uint8_t*)d_bytes, (const uint8_t*)d_points, n, compressed ? 1 : 0);
    count_launch();
    return (int)cudaGetLastError();
}

extern "C" int snarkvm_b200_test_sqrt_device(int field, void* d_out, int32_t* d_ok, const void* d_in, size_t n, void* stream) {
    using namespace b200;
    if (field != SNARKVM_B200_FIELD_FQ && field != SNARKVM_B200_FIELD_FQ2) return (int)cudaErrorInvalidValue;
    if (n == 0) return 0;
    if (!d_out || !d_ok || !d_in || ((uintptr_t)d_out & 15) || ((uintptr_t)d_in & 15) || ((uintptr_t)d_ok & 3) || n > ((size_t)1 << 31))
        return (int)cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    k_test_sqrt<<<blocks, 128, 0, (cudaStream_t)stream>>>((uint32_t*)d_out, d_ok, (const uint32_t*)d_in, n, field);
    count_launch();
    return (int)cudaGetLastError();
}

extern "C" int snarkvm_b200_fr_records_decode_device(const void* d_blob, size_t blob_bytes, const snarkvm_b200_fr_records_segment_t* segs,
                                                     size_t count, uint64_t* bad_record, void* stream) {
    using namespace b200;
    if (count == 0) return 0;
    if (!d_blob || !segs || !bad_record || count >= ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    std::vector<FrRecordSeg> table(count);
    uint64_t total = 0;
    for (size_t i = 0; i < count; i++) {
        const snarkvm_b200_fr_records_segment_t& s = segs[i];
        FrRecordSeg& t = table[i];
        const bool matrix = s.d_row_ptr != nullptr;
        if ((s.stride != 32 && s.stride != 40) || (s.count && !s.d_out) || ((uintptr_t)s.d_out & 15) || s.count >= ((uint64_t)1 << 32))
            return (int)cudaErrorInvalidValue;
        if ((s.stride == 40) != (s.d_cols != nullptr) || (matrix && (s.stride != 40 || s.nrows == 0 || s.nrows >= ((uint64_t)1 << 32))) ||
            ((uintptr_t)s.d_cols & 3) || (s.d_cols && s.num_cols > ((uint64_t)1 << 31)))
            return (int)cudaErrorInvalidValue;
        // the extent every read of the segment stays inside
        const uint64_t extent = matrix ? 8 + 8 * s.nrows + 40 * s.count : (uint64_t)s.stride * s.count;
        if (s.offset > blob_bytes || extent > blob_bytes - s.offset) return (int)cudaErrorInvalidValue;
        t = FrRecordSeg{total, s.offset, s.count, s.stride, (uint32_t)s.nrows, (const uint32_t*)s.d_row_ptr, (uint32_t*)s.d_out,
                        (int32_t*)s.d_cols, s.num_cols};
        total += s.count;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const size_t nbad = (count * sizeof(unsigned long long) + 255) & ~(size_t)255;
    uint8_t* scratch = nullptr;
    cudaError_t e = pool_alloc(&scratch, nbad + count * sizeof(FrRecordSeg), st);
    if (e != cudaSuccess) return (int)e;
    unsigned long long* d_bad = (unsigned long long*)scratch;
    FrRecordSeg* d_table = (FrRecordSeg*)(scratch + nbad);
    int rc = (int)cudaMemsetAsync(d_bad, 0xFF, count * sizeof(unsigned long long), st);
    if (rc == 0) rc = (int)cudaMemcpyAsync(d_table, table.data(), count * sizeof(FrRecordSeg), cudaMemcpyHostToDevice, st);
    if (rc == 0 && total) {
        k_fr_records<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d_table, (uint32_t)count, total, (const uint8_t*)d_blob, d_bad);
        count_launch();
        rc = (int)cudaGetLastError();
    }
    if (rc == 0) rc = (int)cudaMemcpyAsync(bad_record, d_bad, count * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(scratch, st);
    if (rc == 0) rc = (int)cudaStreamSynchronize(st);
    return rc;
}

// The row headers of one matrix section, walked on the host: a chain of lengths, each locating the next.  Bounds-checked against
// the bytes the caller holds, so a length cannot carry the walk past them.
extern "C" int snarkvm_b200_matrix_row_walk(const void* rows, size_t bytes, uint64_t nrows, uint64_t nnz, int32_t* row_ptr,
                                            int64_t* bad_row) {
    if (bad_row) *bad_row = -1;
    if (!row_ptr || (nrows && !rows) || nnz >= ((uint64_t)1 << 31)) return (int)cudaErrorInvalidValue;
    const uint8_t* p = (const uint8_t*)rows;
    uint64_t at = 0, total = 0;
    row_ptr[0] = 0;
    for (uint64_t i = 0; i < nrows; i++) {
        uint64_t len = 0;
        if (bytes - at < 8) { if (bad_row) *bad_row = (int64_t)i; return (int)cudaErrorInvalidValue; }
        std::memcpy(&len, p + at, 8);
        at += 8;
        if (len > (bytes - at) / 40 || len > nnz - total) { if (bad_row) *bad_row = (int64_t)i; return (int)cudaErrorInvalidValue; }
        at += 40 * len;
        total += len;
        row_ptr[i + 1] = (int32_t)total;
    }
    if (total != nnz) { if (bad_row) *bad_row = (int64_t)nrows; return (int)cudaErrorInvalidValue; }
    return 0;
}
