// The BLS12-377 extension tower above Fq2 on the device: Fq6 = Fq2[v]/(v³ − u) and Fq12 = Fq6[w]/(w² − v)
// (fields/src/fp6_3over2.rs, fp12_2over3over2.rs; curves/src/bls12_377/fq6.rs: NONRESIDUE = u, fq12.rs).
//
// In memory an Fq6 is c0 c1 c2 and an Fq12 is c0 c1, so an Fq12 is twelve Montgomery Fq in the reference's order
// c0.c0.c0, c0.c0.c1, c0.c1.c0, … c1.c2.c1: 144 words, 576 bytes — the reference's `Fp12` image.  Every Fq is kept fully reduced
// (ff.cuh), so any correct formula stores the same bytes as the reference's; the schedules below are the reference's anyway.
//
// The Frobenius coefficients u^((q^k − 1)/3), u^((2q^k − 2)/3) (Fq6) and u^((q^k − 1)/6) (Fq12) all lie in Fq for BLS12-377, so
// only their c0 is kept (Montgomery limbs; tests/test_pairing_oracle.py checks these tables against the oracle, which computes them
// from their definitions, and the oracle against the reference's numbers).
//
// The Fq12 operations are out of line: a Miller loop or a final exponentiation calls each of them dozens of times, and inlining
// 54 Fq products per call would not fit the instruction cache.
#pragma once
#include "ec.cuh"

namespace b200 {

#define TOWER_CALL __device__ __noinline__

// u·(c0 + c1·u) = −5·c1 + c0·u
FF_DEV Fq2 fq2_mul_by_nonresidue(const Fq2& a) { Fq2 r; r.c0 = Fq2::times5(a.c1).neg(); r.c1 = a.c0; return r; }
FF_DEV Fq2 fq2_mul_by_fp(const Fq2& a, const Fq& s) { Fq2 r; r.c0 = a.c0 * s; r.c1 = a.c1 * s; return r; }
// Frobenius of Fq2: conjugation for odd powers (FROBENIUS_COEFF_FP2_C1 = [1, −1])
FF_DEV Fq2 fq2_frobenius(const Fq2& a, int k) { Fq2 r = a; if (k & 1) r.c1 = a.c1.neg(); return r; }

__constant__ uint32_t FROB_FP6_C1[6][12] = {
    {0xffffff68u, 0x02cdffffu, 0x7fffffb1u, 0x51409f83u, 0x8a7d3ff2u, 0x9f7db3a9u, 0x6e7c6305u, 0x7b4e97b7u, 0x803c84e8u, 0x4cf495bfu, 0xe2fdf49au, 0x008d6661u},
    {0xa58478dau, 0x5892506du, 0x0ac2a74bu, 0x13336694u, 0xcdf726cfu, 0x9b64a150u, 0x0a9c587eu, 0x5cc42609u, 0xfdcd640cu, 0x5cf848adu, 0x3ac02380u, 0x004702bfu},
    {0xa5847973u, 0xdacd106du, 0xbac2a79au, 0xd8fe2454u, 0xfd832edcu, 0x1ada4fd6u, 0x9d150908u, 0xfb986844u, 0xea32285eu, 0xd63eb8aeu, 0x6f873fd0u, 0x0167d6a3u},
    {0x00000099u, 0x823ac000u, 0xb000004fu, 0xc5cabdc0u, 0x2f8c080du, 0x7f75ae86u, 0x9278b089u, 0x9ed4423bu, 0xec64c452u, 0x79467000u, 0x34c71c50u, 0x0120d3e4u},
    {0x5a7b8727u, 0x2c766f92u, 0x253d58b5u, 0x03d7f6b0u, 0xec122131u, 0x838ec0deu, 0xf658bb10u, 0xbd5eb3e9u, 0x6ed3e52eu, 0x6942bd12u, 0xdd04ed6au, 0x01673786u},
    {0x5a7b868eu, 0xaa3baf92u, 0x753d5865u, 0x3e0d38efu, 0xbc861923u, 0x04191258u, 0x63e00a87u, 0x1e8a71aeu, 0x826f20dcu, 0xeffc4d11u, 0xa83dd119u, 0x004663a2u}};
__constant__ uint32_t FROB_FP6_C2[6][12] = {
    {0xffffff68u, 0x02cdffffu, 0x7fffffb1u, 0x51409f83u, 0x8a7d3ff2u, 0x9f7db3a9u, 0x6e7c6305u, 0x7b4e97b7u, 0x803c84e8u, 0x4cf495bfu, 0xe2fdf49au, 0x008d6661u},
    {0xa5847973u, 0xdacd106du, 0xbac2a79au, 0xd8fe2454u, 0xfd832edcu, 0x1ada4fd6u, 0x9d150908u, 0xfb986844u, 0xea32285eu, 0xd63eb8aeu, 0x6f873fd0u, 0x0167d6a3u},
    {0x5a7b8727u, 0x2c766f92u, 0x253d58b5u, 0x03d7f6b0u, 0xec122131u, 0x838ec0deu, 0xf658bb10u, 0xbd5eb3e9u, 0x6ed3e52eu, 0x6942bd12u, 0xdd04ed6au, 0x01673786u},
    {0xffffff68u, 0x02cdffffu, 0x7fffffb1u, 0x51409f83u, 0x8a7d3ff2u, 0x9f7db3a9u, 0x6e7c6305u, 0x7b4e97b7u, 0x803c84e8u, 0x4cf495bfu, 0xe2fdf49au, 0x008d6661u},
    {0xa5847973u, 0xdacd106du, 0xbac2a79au, 0xd8fe2454u, 0xfd832edcu, 0x1ada4fd6u, 0x9d150908u, 0xfb986844u, 0xea32285eu, 0xd63eb8aeu, 0x6f873fd0u, 0x0167d6a3u},
    {0x5a7b8727u, 0x2c766f92u, 0x253d58b5u, 0x03d7f6b0u, 0xec122131u, 0x838ec0deu, 0xf658bb10u, 0xbd5eb3e9u, 0x6ed3e52eu, 0x6942bd12u, 0xdd04ed6au, 0x01673786u}};
__constant__ uint32_t FROB_FP12_C1[12][12] = {
    {0xffffff68u, 0x02cdffffu, 0x7fffffb1u, 0x51409f83u, 0x8a7d3ff2u, 0x9f7db3a9u, 0x6e7c6305u, 0x7b4e97b7u, 0x803c84e8u, 0x4cf495bfu, 0xe2fdf49au, 0x008d6661u},
    {0xa3f7ca9eu, 0x6ec47a04u, 0x68c1fa44u, 0xa42e0cb9u, 0xfbd2bd23u, 0x578d5187u, 0xc79dd4bdu, 0x930eeb0au, 0x1e09a9eeu, 0xa24883deu, 0x8067d46fu, 0x00daa705u},
    {0xa58478dau, 0x5892506du, 0x0ac2a74bu, 0x13336694u, 0xcdf726cfu, 0x9b64a150u, 0x0a9c587eu, 0x5cc42609u, 0xfdcd640cu, 0x5cf848adu, 0x3ac02380u, 0x004702bfu},
    {0xd084771fu, 0x982c13d9u, 0x6da34a32u, 0xfd49de0cu, 0x83ab0e53u, 0x61a530d1u, 0x06dd9879u, 0xdf8fe441u, 0xd88472bcu, 0x40f29b58u, 0x99046d5du, 0x01587231u},
    {0xa5847973u, 0xdacd106du, 0xbac2a79au, 0xd8fe2454u, 0xfd832edcu, 0x1ada4fd6u, 0x9d150908u, 0xfb986844u, 0xea32285eu, 0xd63eb8aeu, 0x6f873fd0u, 0x0167d6a3u},
    {0x2c8cac81u, 0x296799d5u, 0x04e14feeu, 0x591bd153u, 0x87d85130u, 0x0a17df49u, 0x3f3fc3bcu, 0x4c80f936u, 0xba7ac8ceu, 0x9eaa177au, 0x189c98edu, 0x007dcb2cu},
    {0x00000099u, 0x823ac000u, 0xb000004fu, 0xc5cabdc0u, 0x2f8c080du, 0x7f75ae86u, 0x9278b089u, 0x9ed4423bu, 0xec64c452u, 0x79467000u, 0x34c71c50u, 0x0120d3e4u},
    {0x5c083563u, 0x164445fbu, 0xc73e05bcu, 0x72dd508au, 0xbe368adcu, 0xc76610a7u, 0x39573ed1u, 0x8713eee8u, 0x4e979f4cu, 0x23f281e2u, 0x975d3c7bu, 0x00d39340u},
    {0x5a7b8727u, 0x2c766f92u, 0x253d58b5u, 0x03d7f6b0u, 0xec122131u, 0x838ec0deu, 0xf658bb10u, 0xbd5eb3e9u, 0x6ed3e52eu, 0x6942bd12u, 0xdd04ed6au, 0x01673786u},
    {0x2f7b88e2u, 0xecdcac26u, 0xc25cb5cdu, 0x19c17f37u, 0x365e39acu, 0xbd4e315eu, 0xfa177b15u, 0x3a92f5b1u, 0x941cd67eu, 0x85486a67u, 0x7ec0a38du, 0x0055c814u},
    {0x5a7b868eu, 0xaa3baf92u, 0x753d5865u, 0x3e0d38efu, 0xbc861923u, 0x04191258u, 0x63e00a87u, 0x1e8a71aeu, 0x826f20dcu, 0xeffc4d11u, 0xa83dd119u, 0x004663a2u},
    {0xd3735380u, 0x5ba1262au, 0x2b1eb012u, 0xbdef8bf1u, 0x3230f6cfu, 0x14db82e6u, 0xc1b54fd3u, 0xcda1e0bcu, 0xb226806cu, 0x2790ee45u, 0xff2877fdu, 0x01306f19u}};

FF_DEV Fq fq_const(const uint32_t (&t)[12]) { Fq r;
#pragma unroll
    for (int i = 0; i < 12; i++) r.v[i] = t[i];
    return r; }

struct Fq6 {
    Fq2 c0, c1, c2;
    static constexpr int WORDS = 72;
    FF_DEV static Fq6 zero() { Fq6 r; r.c0 = Fq2::zero(); r.c1 = Fq2::zero(); r.c2 = Fq2::zero(); return r; }
    FF_DEV static Fq6 one() { Fq6 r; r.c0 = Fq2::one(); r.c1 = Fq2::zero(); r.c2 = Fq2::zero(); return r; }
    FF_DEV friend Fq6 operator+(const Fq6& a, const Fq6& b) { Fq6 r; r.c0 = a.c0 + b.c0; r.c1 = a.c1 + b.c1; r.c2 = a.c2 + b.c2; return r; }
    FF_DEV friend Fq6 operator-(const Fq6& a, const Fq6& b) { Fq6 r; r.c0 = a.c0 - b.c0; r.c1 = a.c1 - b.c1; r.c2 = a.c2 - b.c2; return r; }
    FF_DEV Fq6 neg() const { Fq6 r; r.c0 = c0.neg(); r.c1 = c1.neg(); r.c2 = c2.neg(); return r; }
    // ·v with v³ = u (Fp12::mul_fp6_by_nonresidue)
    FF_DEV Fq6 mul_by_nonresidue() const { Fq6 r; r.c0 = fq2_mul_by_nonresidue(c2); r.c1 = c0; r.c2 = c1; return r; }
    // Karatsuba, 6 Fq2 products (fp6_3over2.rs mul_assign)
    FF_DEV friend Fq6 operator*(const Fq6& a, const Fq6& b) {
        const Fq2 v0 = a.c0 * b.c0, v1 = a.c1 * b.c1, v2 = a.c2 * b.c2;
        Fq6 r;
        r.c0 = fq2_mul_by_nonresidue((a.c1 + a.c2) * (b.c1 + b.c2) - v1 - v2) + v0;
        r.c1 = (a.c0 + a.c1) * (b.c0 + b.c1) - v0 - v1 + fq2_mul_by_nonresidue(v2);
        r.c2 = (a.c0 + a.c2) * (b.c0 + b.c2) - v0 - v2 + v1;
        return r;
    }
    // CH-SQR2 (fp6_3over2.rs square_in_place)
    FF_DEV Fq6 sqr() const {
        const Fq2 s0 = c0.sqr(), s1 = (c0 * c1).dbl(), s2 = (c0 - c1 + c2).sqr(), s3 = (c1 * c2).dbl(), s4 = c2.sqr();
        Fq6 r;
        r.c0 = s0 + fq2_mul_by_nonresidue(s3);
        r.c1 = s1 + fq2_mul_by_nonresidue(s4);
        r.c2 = s1 + s2 + s3 - s0 - s4;
        return r;
    }
    // · (b0 + b1·v) (fp6_3over2.rs mul_by_01)
    FF_DEV Fq6 mul_by_01(const Fq2& b0, const Fq2& b1) const {
        const Fq2 a_a = c0 * b0, b_b = c1 * b1;
        Fq6 r;
        r.c0 = fq2_mul_by_nonresidue((c1 + c2) * b1 - b_b) + a_a;
        r.c1 = (b0 + b1) * (c0 + c1) - a_a - b_b;
        r.c2 = (c0 + c2) * b0 - a_a + b_b;
        return r;
    }
    FF_DEV Fq6 mul_by_fq2(const Fq2& s) const { Fq6 r; r.c0 = c0 * s; r.c1 = c1 * s; r.c2 = c2 * s; return r; }
    FF_DEV Fq6 mul_by_fp(const Fq& s) const { Fq6 r; r.c0 = fq2_mul_by_fp(c0, s); r.c1 = fq2_mul_by_fp(c1, s); r.c2 = fq2_mul_by_fp(c2, s); return r; }
    // fp6_3over2.rs inverse (through the Fq2 inverse, i.e. one Fermat inversion in Fq); zero ↦ zero
    FF_DEV Fq6 inverse() const {
        const Fq2 t0 = c0.sqr() - fq2_mul_by_nonresidue(c1 * c2);
        const Fq2 t1 = fq2_mul_by_nonresidue(c2.sqr()) - c0 * c1;
        const Fq2 t2 = c1.sqr() - c0 * c2;
        const Fq2 n = (c0 * t0 + fq2_mul_by_nonresidue(c2 * t1 + c1 * t2)).inverse();
        Fq6 r; r.c0 = t0 * n; r.c1 = t1 * n; r.c2 = t2 * n;
        return r;
    }
    FF_DEV Fq6 frobenius_map(int k) const {
        Fq6 r;
        r.c0 = fq2_frobenius(c0, k);
        r.c1 = fq2_mul_by_fp(fq2_frobenius(c1, k), fq_const(FROB_FP6_C1[k % 6]));
        r.c2 = fq2_mul_by_fp(fq2_frobenius(c2, k), fq_const(FROB_FP6_C2[k % 6]));
        return r;
    }
};

struct Fq12 {
    Fq6 c0, c1;
    static constexpr int WORDS = 144;
    FF_DEV static Fq12 one() { Fq12 r; r.c0 = Fq6::one(); r.c1 = Fq6::zero(); return r; }
    FF_DEV bool is_one() const {
        return c0.c0.c0 == Fq::one() && c0.c0.c1.is_zero() && c0.c1.is_zero() && c0.c2.is_zero() && c1.c0.is_zero() && c1.c1.is_zero() &&
               c1.c2.is_zero();
    }
    FF_DEV Fq12 conjugate() const { Fq12 r; r.c0 = c0; r.c1 = c1.neg(); return r; }
    FF_DEV static Fq12 load(const uint32_t* p) {
        Fq12 r;
        r.c0.c0 = Fq2::load(p); r.c0.c1 = Fq2::load(p + 24); r.c0.c2 = Fq2::load(p + 48);
        r.c1.c0 = Fq2::load(p + 72); r.c1.c1 = Fq2::load(p + 96); r.c1.c2 = Fq2::load(p + 120);
        return r;
    }
    FF_DEV void store(uint32_t* p) const {
        c0.c0.store(p); c0.c1.store(p + 24); c0.c2.store(p + 48);
        c1.c0.store(p + 72); c1.c1.store(p + 96); c1.c2.store(p + 120);
    }
};

// Karatsuba over w: 3 Fq6 products (fp12_2over3over2.rs mul_assign)
TOWER_CALL Fq12 fq12_mul(const Fq12& a, const Fq12& b) {
    const Fq6 v0 = a.c0 * b.c0, v1 = a.c1 * b.c1;
    Fq12 r;
    r.c1 = (a.c0 + a.c1) * (b.c0 + b.c1) - v0 - v1;
    r.c0 = v0 + v1.mul_by_nonresidue();
    return r;
}
// complex squaring, 2 Fq6 products (fp12_2over3over2.rs square_in_place)
TOWER_CALL Fq12 fq12_sqr(const Fq12& a) {
    const Fq6 ab = a.c0 * a.c1;
    Fq12 r;
    r.c0 = (a.c0 + a.c1.mul_by_nonresidue()) * (a.c0 + a.c1) - ab - ab.mul_by_nonresidue();
    r.c1 = ab + ab;
    return r;
}
// f · ((c0, 0, 0) + (c3, c4, 0)·w): the line value of a twist-D curve (fp12_2over3over2.rs mul_by_034)
TOWER_CALL Fq12 fq12_mul_by_034(const Fq12& f, const Fq2& c0, const Fq2& c3, const Fq2& c4) {
    const Fq6 a = f.c0.mul_by_fq2(c0);
    const Fq6 b = f.c1.mul_by_01(c3, c4);
    const Fq6 e = (f.c0 + f.c1).mul_by_01(c0 + c3, c4);
    Fq12 r;
    r.c1 = e - (a + b);
    r.c0 = a + b.mul_by_nonresidue();
    return r;
}
// Granger–Scott squaring, valid in the cyclotomic subgroup (fp12_2over3over2.rs cyclotomic_square)
FF_DEV void cyclotomic_pair(const Fq2& a, const Fq2& b, Fq2& t_even, Fq2& t_odd) {
    const Fq2 t = a * b;
    t_even = (a + b) * (a + fq2_mul_by_nonresidue(b)) - t - fq2_mul_by_nonresidue(t);
    t_odd = t.dbl();
}
TOWER_CALL Fq12 fq12_cyclotomic_square(const Fq12& f) {
    const Fq2 &z0 = f.c0.c0, &z4 = f.c0.c1, &z3 = f.c0.c2, &z2 = f.c1.c0, &z1 = f.c1.c1, &z5 = f.c1.c2;
    Fq2 t0, t1, t2, t3, t4, t5;
    cyclotomic_pair(z0, z1, t0, t1);
    cyclotomic_pair(z2, z3, t2, t3);
    cyclotomic_pair(z4, z5, t4, t5);
    Fq12 r;
    r.c0.c0 = (t0 - z0).dbl() + t0;
    r.c1.c1 = (t1 + z1).dbl() + t1;
    const Fq2 tmp = fq2_mul_by_nonresidue(t5);
    r.c1.c0 = (tmp + z2).dbl() + tmp;
    r.c0.c2 = (t4 - z3).dbl() + t4;
    r.c0.c1 = (t2 - z4).dbl() + t2;
    r.c1.c2 = (t3 + z5).dbl() + t3;
    return r;
}
// (c0 − c1·w) / (c0² − v·c1²) (fp12_2over3over2.rs inverse); zero ↦ zero
TOWER_CALL Fq12 fq12_inverse(const Fq12& a) {
    const Fq6 t = (a.c0.sqr() - a.c1.sqr().mul_by_nonresidue()).inverse();
    Fq12 r;
    r.c0 = a.c0 * t;
    r.c1 = (a.c1 * t).neg();
    return r;
}
TOWER_CALL Fq12 fq12_frobenius_map(const Fq12& a, int k) {
    Fq12 r;
    r.c0 = a.c0.frobenius_map(k);
    r.c1 = a.c1.frobenius_map(k).mul_by_fp(fq_const(FROB_FP12_C1[k % 12]));
    return r;
}

}  // namespace b200
