// BLS12-377 G1 group law on the device (curve y^2 = x^3 + 1, a = 0;
// curves/src/bls12_377/g1.rs:78-91).
//
// Input points use the reference's in-memory `Affine<P>` image
//   { x: Fq, y: Fq, infinity: bool }  — 104-byte stride, Montgomery Fq
//   (curves/src/templates/short_weierstrass_jacobian/affine.rs:41-46).
// Bucket accumulators use extended Jacobian "XYZZ" coordinates
//   x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2, infinity <=> ZZ == 0
// (EFD shortw/xyzz, a = 0: madd-2008-s 8M+2S, add-2008-s 12M+2S, dbl-2008-s-1).
// The group element computed is the same one the reference's Jacobian formulas
// (projective.rs:222-291, 302-339, 407-468) compute; only the final
// to_affine()-normalised image is compared, as in every reference test
// (algorithms/src/msm/variable_base/mod.rs:90-119).
#pragma once
#include "ff.cuh"

namespace b200 {

// Fq2 = Fq[u]/(u² + 5) (curves/src/bls12_377/fq2.rs:29-65: NONRESIDUE = −5; fields/src/fp2.rs): the base field of G2.
// In memory c0 then c1, 96 bytes — the reference's Fp2 { c0, c1 } image.
struct Fq2 {
    Fq c0, c1;
    static constexpr int WORDS = 24;
    FF_DEV static Fq2 zero() { Fq2 r; r.c0 = Fq::zero(); r.c1 = Fq::zero(); return r; }
    FF_DEV static Fq2 one() { Fq2 r; r.c0 = Fq::one(); r.c1 = Fq::zero(); return r; }
    FF_DEV bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    FF_DEV bool operator==(const Fq2& o) const { return c0 == o.c0 && c1 == o.c1; }
    FF_DEV bool operator!=(const Fq2& o) const { return !(*this == o); }
    FF_DEV friend Fq2 operator+(const Fq2& a, const Fq2& b) { Fq2 r; r.c0 = a.c0 + b.c0; r.c1 = a.c1 + b.c1; return r; }
    FF_DEV friend Fq2 operator-(const Fq2& a, const Fq2& b) { Fq2 r; r.c0 = a.c0 - b.c0; r.c1 = a.c1 - b.c1; return r; }
    FF_DEV Fq2 neg() const { Fq2 r; r.c0 = c0.neg(); r.c1 = c1.neg(); return r; }
    FF_DEV Fq2 dbl() const { Fq2 r; r.c0 = c0.dbl(); r.c1 = c1.dbl(); return r; }
    FF_DEV static Fq times5(const Fq& x) { Fq t = x.dbl().dbl(); return t + x; }
    // Karatsuba over the quadratic extension: 3 base-field multiplications (fp2.rs mul_assign)
    FF_DEV friend Fq2 operator*(const Fq2& a, const Fq2& b) {
        Fq v0 = a.c0 * b.c0, v1 = a.c1 * b.c1;
        Fq2 r;
        r.c1 = (a.c0 + a.c1) * (b.c0 + b.c1) - v0 - v1;
        r.c0 = v0 - times5(v1);                           // + u²·v1 with u² = −5
        return r;
    }
    // complex squaring: 2 base-field multiplications — (a0 + a1)(a0 − 5·a1) = a0² − 5·a1² − 4·a0·a1
    FF_DEV Fq2 sqr() const {
        Fq t = c0 * c1;
        Fq2 r;
        r.c0 = (c0 + c1) * (c0 - times5(c1)) + t.dbl().dbl();
        r.c1 = t.dbl();
        return r;
    }
    // (c0 − c1·u) / (c0² + 5·c1²); zero ↦ zero
    FF_DEV Fq2 inverse() const {
        Fq n = (c0.sqr() + times5(c1.sqr())).inverse();
        Fq2 r; r.c0 = c0 * n; r.c1 = (c1 * n).neg();
        return r;
    }
    FF_DEV static Fq2 load(const void* p) { Fq2 r; r.c0 = Fq::load(p); r.c1 = Fq::load((const uint32_t*)p + 12); return r; }
    FF_DEV void store(void* p) const { c0.store(p); c1.store((uint32_t*)p + 12); }
};

template <class F>
struct AffineT {
    F x, y;
    bool inf;
};
using AffinePoint = AffineT<Fq>;

// Reference layout: x[48] y[48] inf[1] pad.  The 104-byte stride is only 8-byte aligned
// (odd indices sit at 8 mod 16), so the gather uses 64-bit loads: 12 × LDG.64 per point.
FF_DEV Fq load_fq_u64(const uint8_t* p) {
    Fq r; const uint2* q = reinterpret_cast<const uint2*>(p);
#pragma unroll
    for (int i = 0; i < 6; i++) { uint2 t = __ldg(q + i); r.v[2 * i] = t.x; r.v[2 * i + 1] = t.y; }
    return r;
}
FF_DEV void store_fq_u64(uint8_t* p, const Fq& a) {
    uint2* q = reinterpret_cast<uint2*>(p);
#pragma unroll
    for (int i = 0; i < 6; i++) q[i] = make_uint2(a.v[2 * i], a.v[2 * i + 1]);
}
FF_DEV AffinePoint load_affine(const uint8_t* base, size_t stride, size_t i) {
    const uint8_t* p = base + i * stride;
    AffinePoint a;
    a.x = load_fq_u64(p);
    a.y = load_fq_u64(p + 48);
    a.inf = __ldg(p + 96) != 0;
    return a;
}
FF_DEV void store_affine(uint8_t* base, size_t stride, size_t i, const AffinePoint& a) {
    uint8_t* p = base + i * stride;
    store_fq_u64(p, a.x);
    store_fq_u64(p + 48, a.y);
    // infinity flag + padding as one 8-byte store (stride is a multiple of 8 ≥ 104)
    *reinterpret_cast<unsigned long long*>(p + 96) = a.inf ? 1ull : 0ull;
}

// Affine<G2>: x.c0 x.c1 y.c0 y.c1 (4 × 48 B) inf[1] pad, stride ≥ 200 and a multiple of 8
FF_DEV AffineT<Fq2> load_affine_g2(const uint8_t* base, size_t stride, size_t i) {
    const uint8_t* p = base + i * stride;
    AffineT<Fq2> a;
    a.x.c0 = load_fq_u64(p); a.x.c1 = load_fq_u64(p + 48);
    a.y.c0 = load_fq_u64(p + 96); a.y.c1 = load_fq_u64(p + 144);
    a.inf = __ldg(p + 192) != 0;
    return a;
}
FF_DEV void store_affine_g2(uint8_t* base, size_t stride, size_t i, const AffineT<Fq2>& a) {
    uint8_t* p = base + i * stride;
    store_fq_u64(p, a.x.c0); store_fq_u64(p + 48, a.x.c1);
    store_fq_u64(p + 96, a.y.c0); store_fq_u64(p + 144, a.y.c1);
    *reinterpret_cast<unsigned long long*>(p + 192) = a.inf ? 1ull : 0ull;
}

// a < q on the raw limbs: a coordinate image ≥ q is no field element
FF_DEV bool fq_is_canonical(const Fq& a) {
    (void)ptx_sub_cc(a.v[0], FqParams::mod(0));
#pragma unroll
    for (int i = 1; i < 12; i++) (void)ptx_subc_cc(a.v[i], FqParams::mod(i));
    return ptx_subc(0u, 0u) != 0u;
}

template <class F>
struct XyzzT {
    F X, Y, ZZ, ZZZ;
    static constexpr int WORDS = 4 * F::WORDS;

    FF_DEV static XyzzT infinity() { XyzzT r; r.X = F::zero(); r.Y = F::zero(); r.ZZ = F::zero(); r.ZZZ = F::zero(); return r; }
    FF_DEV bool is_inf() const { return ZZ.is_zero(); }

    FF_DEV static XyzzT from_affine(const AffineT<F>& p) {
        XyzzT r;
        if (p.inf) return infinity();
        r.X = p.x; r.Y = p.y; r.ZZ = F::one(); r.ZZZ = F::one();
        return r;
    }

    // dbl-2008-s-1 (a = 0)
    FF_DEV void dbl() {
        if (is_inf()) return;
        F U = Y.dbl();
        F V = U.sqr();
        F W = U * V;
        F S = X * V;
        F XX = X.sqr();
        F M = XX.dbl() + XX;
        F X3 = M.sqr() - S.dbl();
        F Y3 = M * (S - X3) - W * Y;
        X = X3; Y = Y3;
        ZZ = V * ZZ;
        ZZZ = W * ZZZ;
    }

    // mixed addition with an affine point whose y may be negated (signed-digit buckets).
    FF_DEV void add_affine(const AffineT<F>& q, bool negate) {
        if (q.inf) return;
        F qy = negate ? q.y.neg() : q.y;
        if (is_inf()) { X = q.x; Y = qy; ZZ = F::one(); ZZZ = F::one(); return; }
        F U2 = q.x * ZZ;
        F S2 = qy * ZZZ;
        F P = U2 - X;
        F R = S2 - Y;
        if (P.is_zero()) {
            if (R.is_zero()) {
                // same point: double the affine operand (mdbl-2008-s-1)
                F U = qy.dbl();
                F V = U.sqr();
                F W = U * V;
                F S = q.x * V;
                F XX = q.x.sqr();
                F M = XX.dbl() + XX;
                X = M.sqr() - S.dbl();
                Y = M * (S - X) - W * qy;
                ZZ = V; ZZZ = W;
            } else {
                *this = infinity();          // P + (-P)
            }
            return;
        }
        F PP = P.sqr();
        F PPP = P * PP;
        F Q = X * PP;
        F X3 = R.sqr() - PPP - Q.dbl();
        Y = R * (Q - X3) - Y * PPP;
        X = X3;
        ZZ = ZZ * PP;
        ZZZ = ZZZ * PPP;
    }

    // general addition (add-2008-s)
    FF_DEV void add(const XyzzT& o) {
        if (o.is_inf()) return;
        if (is_inf()) { *this = o; return; }
        F U1 = X * o.ZZ;
        F U2 = o.X * ZZ;
        F S1 = Y * o.ZZZ;
        F S2 = o.Y * ZZZ;
        F P = U2 - U1;
        F R = S2 - S1;
        if (P.is_zero()) {
            if (R.is_zero()) dbl(); else *this = infinity();
            return;
        }
        F PP = P.sqr();
        F PPP = P * PP;
        F Q = U1 * PP;
        F X3 = R.sqr() - PPP - Q.dbl();
        Y = R * (Q - X3) - S1 * PPP;
        X = X3;
        ZZ = ZZ * o.ZZ * PP;
        ZZZ = ZZZ * o.ZZZ * PPP;
    }

    // k·P for a small public multiplier (used by the bucket reduction: (lo-1)·running)
    FF_DEV XyzzT mul_u32(uint32_t k) const {
        XyzzT acc = infinity();
        bool started = false;
        for (int b = 31; b >= 0; b--) {
            if (started) acc.dbl();
            if ((k >> b) & 1u) { acc.add(*this); started = true; }
        }
        return acc;
    }

    FF_DEV AffineT<F> to_affine() const {
        AffineT<F> a;
        if (is_inf()) { a.x = F::zero(); a.y = F::one(); a.inf = true; return a; }   // Affine::zero(), affine.rs:57-59
        // x = X/ZZ, y = Y/ZZZ with one inversion: i = 1/(ZZ·ZZZ)
        F i = (ZZ * ZZZ).inverse();
        a.x = X * (i * ZZZ);
        a.y = Y * (i * ZZ);
        a.inf = false;
        return a;
    }

    FF_DEV static XyzzT load(const uint32_t* p) {
        XyzzT r; r.X = F::load(p); r.Y = F::load(p + F::WORDS); r.ZZ = F::load(p + 2 * F::WORDS); r.ZZZ = F::load(p + 3 * F::WORDS); return r;
    }
    FF_DEV void store(uint32_t* p) const { X.store(p); Y.store(p + F::WORDS); ZZ.store(p + 2 * F::WORDS); ZZZ.store(p + 3 * F::WORDS); }
};

using XYZZ = XyzzT<Fq>;
using XYZZ2 = XyzzT<Fq2>;           // G2 accumulators: 384 bytes
static constexpr int XYZZ_WORDS = 48;   // 192 bytes

}  // namespace b200
