// BLS12-377 pairing (curves/src/templates/bls12/{bls12.rs, g2.rs}; X = 0x8508c00000000001, X not negative, twist type D).
//
//   G2Prepared::from_affine  →  k_g2_prepare      one thread per G2 point: 63 doubling and 6 addition steps in homogeneous
//                                                 projective coordinates, 69 coefficient triples (3 Fq2) written to HBM
//   miller_loop              →  k_miller_pairs    one thread per (G1, prepared G2) pair: the pair's own Miller loop
//   final_exponentiation     →  k_pairing_checks  one thread per check: the product of its pairs' Miller values, then one final
//                                                 exponentiation (eprint 2016/130, Table 1, as the reference)
//
// The reference's multi-pair miller_loop shares one squaring chain among the pairs.  Squaring distributes over a product in Fq12,
// so the product of the pairs' separate loops is the same Fq12 element, bit for bit (every Fq is kept reduced); the pairs of a
// check then run on separate threads and the check only multiplies.  Pairs with a G1 or G2 point at infinity contribute one, as
// the reference drops them from the loop; a check whose pairs all do is the empty product and its result is one.
//
// A prepared point is 69 × 3 Fq2 (288 B per triple: c0, c1, c2) = 19872 B, then its infinity flag (u32) and 28 zero bytes: 19904 B.
#include "msm.cuh"

#define FF_CALL_MUL 1
#include "tower.cuh"
#include "pairing.cuh"
#include "../../include/snarkvm_b200.h"   // the test ops

namespace b200 {

static constexpr uint64_t BLS_X = 0x8508c00000000001ull;
static constexpr int COEFF_TRIPLES = 69;
static constexpr size_t TRIPLE_BYTES = 3 * 96;
static constexpr size_t PREP_FLAG = COEFF_TRIPLES * TRIPLE_BYTES;          // 19872
static constexpr size_t PREP_BYTES = PREP_FLAG + 32;                        // 19904
static constexpr uint32_t NO_BAD = 0xffffffffu;

// the c1 of G2's WEIERSTRASS_B = (0, b1) (curves/src/bls12_377/g2.rs), Montgomery limbs
__constant__ uint32_t G2_B1[12] = {0x66666685u, 0x80722666u, 0x899999a9u, 0x8df55926u, 0xd64f34cfu, 0x7fe4561au,
                                   0xb6e4f01bu, 0xb95da6d8u, 0xfc142743u, 0x4b747cccu, 0x70f49f43u, 0x0039c3fau};

struct G2Hom { Fq2 x, y, z; };

// (0, b1)·a = (−5·b1·a1, b1·a0)
FF_DEV Fq2 mul_by_g2_b(const Fq2& a) {
    const Fq b1 = fq_const(G2_B1);
    Fq2 r; r.c0 = Fq2::times5(a.c1 * b1).neg(); r.c1 = a.c0 * b1;
    return r;
}

FF_DEV void store_triple(uint8_t* p, const Fq2& c0, const Fq2& c1, const Fq2& c2) { c0.store(p); c1.store(p + 96); c2.store(p + 192); }

// g2.rs doubling_step, twist D: (−h, 3·j, i)
FF_DEV void doubling_step(G2Hom& r, const Fq& two_inv, uint8_t* out) {
    const Fq2 a = fq2_mul_by_fp(r.x * r.y, two_inv);
    const Fq2 b = r.y.sqr();
    const Fq2 c = r.z.sqr();
    const Fq2 e = mul_by_g2_b(c.dbl() + c);
    const Fq2 f = e.dbl() + e;
    const Fq2 g = fq2_mul_by_fp(b + f, two_inv);
    const Fq2 h = (r.y + r.z).sqr() - (b + c);
    const Fq2 i = e - b;
    const Fq2 j = r.x.sqr();
    const Fq2 e_sq = e.sqr();
    r.x = a * (b - f);
    r.y = g.sqr() - (e_sq.dbl() + e_sq);
    r.z = b * h;
    store_triple(out, h.neg(), j.dbl() + j, i);
}

// g2.rs addition_step, twist D: (λ, −θ, j)
FF_DEV void addition_step(G2Hom& r, const Fq2& qx, const Fq2& qy, uint8_t* out) {
    const Fq2 theta = r.y - qy * r.z;
    const Fq2 lambda = r.x - qx * r.z;
    const Fq2 c = theta.sqr();
    const Fq2 d = lambda.sqr();
    const Fq2 e = lambda * d;
    const Fq2 f = r.z * c;
    const Fq2 g = r.x * d;
    const Fq2 h = e + f - g.dbl();
    const Fq2 ry = r.y;
    r.x = lambda * h;
    r.y = theta * (g - h) - e * ry;
    r.z = r.z * e;
    const Fq2 j = theta * qx - lambda * qy;
    store_triple(out, lambda, theta.neg(), j);
}

// one thread per G2 Affine image (x.c0 x.c1 y.c0 y.c1 infinity, `stride` bytes apart, 8-byte aligned); *bad_min receives the lowest
// index whose coordinates are not below q
__global__ void __launch_bounds__(128) k_g2_prepare(const uint8_t* __restrict__ points, size_t n, size_t stride, uint8_t* __restrict__ out,
                                                    uint32_t* __restrict__ bad_min) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* p = points + i * stride;
    Fq2 qx, qy;
    qx.c0 = load_fq_u64(p); qx.c1 = load_fq_u64(p + 48);
    qy.c0 = load_fq_u64(p + 96); qy.c1 = load_fq_u64(p + 144);
    const bool inf = __ldg(p + 192) != 0;
    if (!fq_is_canonical(qx.c0) || !fq_is_canonical(qx.c1) || !fq_is_canonical(qy.c0) || !fq_is_canonical(qy.c1)) {
        atomicMin(bad_min, (uint32_t)i);
        return;
    }
    uint8_t* o = out + i * PREP_BYTES;
    reinterpret_cast<uint4*>(o + PREP_FLAG)[0] = make_uint4(inf ? 1u : 0u, 0u, 0u, 0u);
    reinterpret_cast<uint4*>(o + PREP_FLAG)[1] = make_uint4(0u, 0u, 0u, 0u);
    if (inf) {                                    // G2Prepared { ell_coeffs: [], infinity: true }: no coefficients
#pragma unroll 1
        for (size_t k = 0; k < PREP_FLAG / 16; k++) reinterpret_cast<uint4*>(o)[k] = make_uint4(0u, 0u, 0u, 0u);
        return;
    }
    const Fq two_inv = Fq::one().half();
    G2Hom r{qx, qy, Fq2::one()};
    int j = 0;
#pragma unroll 1
    for (int b = 62; b >= 0; b--) {
        doubling_step(r, two_inv, o + (size_t)j++ * TRIPLE_BYTES);
        if ((BLS_X >> b) & 1ull) addition_step(r, qx, qy, o + (size_t)j++ * TRIPLE_BYTES);
    }
}

// bls12.rs ell, twist D: f · mul_by_034(c0·p.y, c1·p.x, c2)
FF_DEV Fq12 ell(const Fq12& f, const uint8_t* triple, const AffinePoint& p) {
    const Fq2 c0 = fq2_mul_by_fp(Fq2::load(triple), p.y);
    const Fq2 c1 = fq2_mul_by_fp(Fq2::load(triple + 96), p.x);
    const Fq2 c2 = Fq2::load(triple + 192);
    return fq12_mul_by_034(f, c0, c1, c2);
}

__device__ __noinline__ Fq12 miller_loop(const AffinePoint& p, const uint8_t* prep) {
    Fq12 f = Fq12::one();
    int j = 0;
#pragma unroll 1
    for (int b = 62; b >= 0; b--) {
        f = fq12_sqr(f);
        f = ell(f, prep + (size_t)j++ * TRIPLE_BYTES, p);
        if ((BLS_X >> b) & 1ull) f = ell(f, prep + (size_t)j++ * TRIPLE_BYTES, p);
    }
    return f;
}

// cyclotomic_exp by X (X_IS_NEGATIVE = false: no conjugation).  The reference starts from one and squares it at the top bit; the
// square of one is one, so starting from f at the top bit is the same element.
__device__ __noinline__ Fq12 exp_by_x(const Fq12& f) {
    Fq12 res = f;
#pragma unroll 1
    for (int b = 62; b >= 0; b--) {
        res = fq12_cyclotomic_square(res);
        if ((BLS_X >> b) & 1ull) res = fq12_mul(res, f);
    }
    return res;
}

// bls12.rs final_exponentiation: the easy part f^((q⁶ − 1)(q² + 1)), then eprint 2016/130 Table 1 (3·(q⁴ − q² + 1)/r)
__device__ __noinline__ Fq12 final_exponentiation(const Fq12& f) {
    Fq12 r = fq12_mul(f.conjugate(), fq12_inverse(f));
    r = fq12_mul(fq12_frobenius_map(r, 2), r);
    Fq12 y0 = fq12_cyclotomic_square(r).conjugate();
    Fq12 y5 = exp_by_x(r);
    Fq12 y1 = fq12_cyclotomic_square(y5);
    Fq12 y3 = fq12_mul(y0, y5);
    y0 = exp_by_x(y3);
    const Fq12 y2 = exp_by_x(y0);
    Fq12 y4 = fq12_mul(exp_by_x(y2), y1);
    y1 = exp_by_x(y4);
    y1 = fq12_mul(fq12_mul(y1, y3.conjugate()), r);
    y0 = fq12_frobenius_map(fq12_mul(y0, r), 3);
    y4 = fq12_frobenius_map(fq12_mul(y4, r.conjugate()), 1);
    y5 = fq12_frobenius_map(fq12_mul(y5, y2), 2);
    return fq12_mul(fq12_mul(fq12_mul(y5, y0), y4), y1);
}

// one thread per pair: its Miller value (one when either point is at infinity) → miller[t]; a coordinate ≥ q or a G2 index out of
// range names the pair's check in *bad_min (the last check whose first pair is ≤ t: a binary search over check_start)
__global__ void __launch_bounds__(128) k_miller_pairs(const uint8_t* __restrict__ g1, size_t g1_stride, const uint32_t* __restrict__ g2_index,
                                                      uint32_t npairs, const uint8_t* __restrict__ prepared, uint32_t nprepared,
                                                      const uint32_t* __restrict__ check_start, uint32_t nchecks, uint32_t* __restrict__ miller,
                                                      uint32_t* __restrict__ bad_min) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= npairs) return;
    const AffinePoint p = load_affine(g1, g1_stride, t);
    const uint32_t q = g2_index[t];
    Fq12 f = Fq12::one();
    if (!fq_is_canonical(p.x) || !fq_is_canonical(p.y) || q >= nprepared) {
        uint32_t lo = 0, hi = nchecks;
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (check_start[mid] <= t) lo = mid; else hi = mid; }
        atomicMin(bad_min, lo);
    } else if (!p.inf) {
        const uint8_t* prep = prepared + (size_t)q * PREP_BYTES;
        if (*reinterpret_cast<const uint32_t*>(prep + PREP_FLAG) == 0u) f = miller_loop(p, prep);
    }
    f.store(miller + (size_t)t * Fq12::WORDS);
}

// one thread per check c over pairs [check_start[c], check_start[c + 1]): product of the Miller values, final exponentiation
__global__ void __launch_bounds__(128) k_pairing_checks(const uint32_t* __restrict__ miller, const uint32_t* __restrict__ check_start,
                                                        uint32_t nchecks, uint32_t npairs, uint32_t* __restrict__ gt,
                                                        uint32_t* __restrict__ is_one, uint32_t* __restrict__ bad_min) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchecks) return;
    const uint32_t s = check_start[c], e = check_start[c + 1];
    if (s > e || e > npairs || (c == 0 && s != 0) || (c + 1 == nchecks && e != npairs)) { atomicMin(bad_min, c); return; }
    Fq12 f = Fq12::one();
#pragma unroll 1
    for (uint32_t i = s; i < e; i++) f = fq12_mul(f, Fq12::load(miller + (size_t)i * Fq12::WORDS));
    f = final_exponentiation(f);
    f.store(gt + (size_t)c * Fq12::WORDS);
    is_one[c] = f.is_one() ? 1u : 0u;
}

// scratch of one call: the bad word, then (optionally) the Miller values; reads the bad word back with the one synchronisation
static int finish(int rc, uint8_t* scratch, const uint32_t* d_bad, int64_t* bad_out, cudaStream_t stream) {
    uint32_t h_bad = NO_BAD;
    if (rc == 0) rc = (int)cudaMemcpyAsync(&h_bad, d_bad, 4, cudaMemcpyDeviceToHost, stream);
    cudaFreeAsync(scratch, stream);
    if (rc == 0) rc = (int)cudaStreamSynchronize(stream);
    if (rc != 0) return rc;
    if (h_bad != NO_BAD) {
        if (bad_out) *bad_out = (int64_t)h_bad;
        return (int)cudaErrorInvalidValue;
    }
    return 0;
}

int g2_prepare_device(void* d_prepared, const void* d_points, size_t npoints, size_t stride, int64_t* bad_point, cudaStream_t stream) {
    if (bad_point) *bad_point = -1;
    if (npoints == 0) return 0;
    if (!d_prepared || !d_points || stride < 200 || (stride & 7) || npoints >= NO_BAD) return (int)cudaErrorInvalidValue;
    uint8_t* scratch = nullptr;
    cudaError_t e = pool_alloc(&scratch, 256, stream);
    if (e != cudaSuccess) return (int)e;
    uint32_t* d_bad = (uint32_t*)scratch;
    int rc = (int)cudaMemsetAsync(d_bad, 0xff, 4, stream);
    if (rc == 0) {
        k_g2_prepare<<<(unsigned)((npoints + 127) / 128), 128, 0, stream>>>((const uint8_t*)d_points, npoints, stride, (uint8_t*)d_prepared, d_bad);
        count_launch();
        rc = (int)cudaGetLastError();
    }
    return finish(rc, scratch, d_bad, bad_point, stream);
}

int pairing_products_device(void* d_gt, uint32_t* d_is_one, void* d_miller, const void* d_g1, size_t g1_stride, const uint32_t* d_g2_index,
                            size_t npairs, const void* d_prepared, size_t nprepared, const uint32_t* d_check_start, size_t nchecks,
                            int64_t* bad_check, cudaStream_t stream) {
    if (bad_check) *bad_check = -1;
    if (nchecks == 0) return npairs == 0 ? 0 : (int)cudaErrorInvalidValue;
    if (!d_gt || !d_is_one || !d_check_start || nchecks >= ((size_t)1 << 31) || npairs >= ((size_t)1 << 31) || nprepared >= NO_BAD)
        return (int)cudaErrorInvalidValue;
    if (npairs > 0 && (!d_g1 || !d_g2_index || !d_prepared || g1_stride < 104 || (g1_stride & 7))) return (int)cudaErrorInvalidValue;
    const size_t miller_bytes = d_miller ? 0 : npairs * Fq12::WORDS * 4;
    uint8_t* scratch = nullptr;
    cudaError_t e = pool_alloc(&scratch, 256 + miller_bytes, stream);
    if (e != cudaSuccess) return (int)e;
    uint32_t* d_bad = (uint32_t*)scratch;
    uint32_t* miller = d_miller ? (uint32_t*)d_miller : (uint32_t*)(scratch + 256);
    int rc = (int)cudaMemsetAsync(d_bad, 0xff, 4, stream);
    if (rc == 0 && npairs > 0) {
        k_miller_pairs<<<(unsigned)((npairs + 127) / 128), 128, 0, stream>>>((const uint8_t*)d_g1, g1_stride, d_g2_index, (uint32_t)npairs,
                                                                            (const uint8_t*)d_prepared, (uint32_t)nprepared, d_check_start,
                                                                            (uint32_t)nchecks, miller, d_bad);
        count_launch();
        rc = (int)cudaGetLastError();
    }
    if (rc == 0) {
        k_pairing_checks<<<(unsigned)((nchecks + 127) / 128), 128, 0, stream>>>(miller, d_check_start, (uint32_t)nchecks, (uint32_t)npairs,
                                                                               (uint32_t*)d_gt, d_is_one, d_bad);
        count_launch();
        rc = (int)cudaGetLastError();
    }
    return finish(rc, scratch, d_bad, bad_check, stream);
}

// ---- element-wise tests of the tower and the line steps (snarkvm_b200_test_tower_op_device) -------------------------------------
// Compiled here so that they call the same doubling_step, addition_step, ell, exp_by_x and final_exponentiation, and the same
// out-of-line Fq products, as the kernels above.  Operands and results: Montgomery words, one element per thread.
namespace {

FF_DEV Fq6 t6_load(const uint32_t* p) { Fq6 r; r.c0 = Fq2::load(p); r.c1 = Fq2::load(p + 24); r.c2 = Fq2::load(p + 48); return r; }
FF_DEV void t6_store(uint32_t* p, const Fq6& x) { x.c0.store(p); x.c1.store(p + 24); x.c2.store(p + 48); }

__global__ void __launch_bounds__(128) k_test_fq6_op(int op, int k, uint32_t* __restrict__ out, const uint32_t* __restrict__ a,
                                                     const uint32_t* __restrict__ b, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fq6 x = t6_load(a + i * Fq6::WORDS);
    Fq6 r;
    switch (op) {
        case SNARKVM_B200_OP_FQ6_MUL: r = x * t6_load(b + i * Fq6::WORDS); break;
        case SNARKVM_B200_OP_FQ6_SQR: r = x.sqr(); break;
        case SNARKVM_B200_OP_FQ6_MUL_BY_01: r = x.mul_by_01(Fq2::load(b + i * 48), Fq2::load(b + i * 48 + 24)); break;
        case SNARKVM_B200_OP_FQ6_MUL_BY_NONRESIDUE: r = x.mul_by_nonresidue(); break;
        case SNARKVM_B200_OP_FQ6_INVERSE: r = x.inverse(); break;
        default: r = x.frobenius_map(k); break;
    }
    t6_store(out + i * Fq6::WORDS, r);
}

__global__ void __launch_bounds__(128) k_test_fq12_op(int op, int k, uint32_t* __restrict__ out, const uint32_t* __restrict__ a,
                                                      const uint32_t* __restrict__ b, const uint32_t* __restrict__ c, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fq12 x = Fq12::load(a + i * Fq12::WORDS);
    if (op == SNARKVM_B200_OP_FQ12_IS_ONE) { out[i] = x.is_one() ? 1u : 0u; return; }
    Fq12 r;
    switch (op) {
        case SNARKVM_B200_OP_FQ12_MUL: r = fq12_mul(x, Fq12::load(b + i * Fq12::WORDS)); break;
        case SNARKVM_B200_OP_FQ12_SQR: r = fq12_sqr(x); break;
        case SNARKVM_B200_OP_FQ12_MUL_BY_034: {
            const uint32_t* y = b + i * 72;
            r = fq12_mul_by_034(x, Fq2::load(y), Fq2::load(y + 24), Fq2::load(y + 48));
            break;
        }
        case SNARKVM_B200_OP_FQ12_CYCLOTOMIC_SQUARE: r = fq12_cyclotomic_square(x); break;
        case SNARKVM_B200_OP_FQ12_INVERSE: r = fq12_inverse(x); break;
        case SNARKVM_B200_OP_FQ12_CONJUGATE: r = x.conjugate(); break;
        case SNARKVM_B200_OP_FQ12_FROBENIUS: r = fq12_frobenius_map(x, k); break;
        case SNARKVM_B200_OP_FQ12_EXP_BY_X: r = exp_by_x(x); break;
        case SNARKVM_B200_OP_FQ12_FINAL_EXPONENTIATION: r = final_exponentiation(x); break;
        default: {                                                               // ELL
            AffinePoint p;
            p.x = Fq::load(c + i * 24); p.y = Fq::load(c + i * 24 + 12); p.inf = false;
            r = ell(x, reinterpret_cast<const uint8_t*>(b + i * 72), p);
        }
    }
    r.store(out + i * Fq12::WORDS);
}

__global__ void __launch_bounds__(128) k_test_line_step(int op, uint32_t* __restrict__ out, const uint32_t* __restrict__ a,
                                                        const uint32_t* __restrict__ b, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t* s = a + i * 72;
    G2Hom r{Fq2::load(s), Fq2::load(s + 24), Fq2::load(s + 48)};
    uint32_t* o = out + i * 144;
    if (op == SNARKVM_B200_OP_G2_DOUBLING_STEP) doubling_step(r, Fq::one().half(), reinterpret_cast<uint8_t*>(o + 72));
    else addition_step(r, Fq2::load(b + i * 48), Fq2::load(b + i * 48 + 24), reinterpret_cast<uint8_t*>(o + 72));
    r.x.store(o); r.y.store(o + 24); r.z.store(o + 48);
}

}  // namespace

int test_tower_op_device(int op, int k, void* d_out, const void* d_a, const void* d_b, const void* d_c, size_t n, cudaStream_t stream) {
    const bool frob6 = op == SNARKVM_B200_OP_FQ6_FROBENIUS, frob12 = op == SNARKVM_B200_OP_FQ12_FROBENIUS;
    if (op < SNARKVM_B200_OP_FQ6_MUL || op > SNARKVM_B200_OP_G2_ADDITION_STEP) return (int)cudaErrorInvalidValue;
    if (k < 0 || k >= (frob6 ? 6 : frob12 ? 12 : 1)) return (int)cudaErrorInvalidValue;
    if (n == 0) return 0;
    const bool needs_b = op == SNARKVM_B200_OP_FQ6_MUL || op == SNARKVM_B200_OP_FQ6_MUL_BY_01 || op == SNARKVM_B200_OP_FQ12_MUL ||
                         op == SNARKVM_B200_OP_FQ12_MUL_BY_034 || op == SNARKVM_B200_OP_FQ12_ELL || op == SNARKVM_B200_OP_G2_ADDITION_STEP;
    if (!d_out || !d_a || (needs_b && !d_b) || (op == SNARKVM_B200_OP_FQ12_ELL && !d_c) || n > ((size_t)1 << 26))
        return (int)cudaErrorInvalidValue;
    if (((uintptr_t)d_out | (uintptr_t)d_a | (uintptr_t)d_b | (uintptr_t)d_c) & 15) return (int)cudaErrorInvalidValue;  // 16-B loads
    uint32_t* out = (uint32_t*)d_out;
    const uint32_t *a = (const uint32_t*)d_a, *b = (const uint32_t*)d_b, *c = (const uint32_t*)d_c;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    if (op <= SNARKVM_B200_OP_FQ6_FROBENIUS) k_test_fq6_op<<<blocks, 128, 0, stream>>>(op, k, out, a, b, n);
    else if (op <= SNARKVM_B200_OP_FQ12_ELL) k_test_fq12_op<<<blocks, 128, 0, stream>>>(op, k, out, a, b, c, n);
    else k_test_line_step<<<blocks, 128, 0, stream>>>(op, out, a, b, n);
    count_launch();
    return (int)cudaGetLastError();
}

}  // namespace b200

// the field-arithmetic test kernels, compiled here with this translation unit's own mul_call / sqr_call
#define FIELD_TEST_ENTRY test_field_op_pairing
#include "testops.cuh"
