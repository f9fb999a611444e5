// Host-side BLS12-377 Fq / Fq2 and G1 / G2 arithmetic used ONLY for the O(windows) tail of an MSM:
// summing the per-window bucket sums with Horner doublings and normalising the
// result (one inversion).  This mirrors where the reference's own CUDA plugin
// finishes on the host (algorithms/cuda/cuda/snarkvm.cu:290-295 adds the per-GPU
// partial points with point_t::dadd on the CPU).  ~253 doublings + ≤ 24 additions;
// all O(n) work stays on the GPU.  Independent of oracle/ (which is test-only).
#pragma once
#include <cstdint>
#include <cstring>
#if defined(__x86_64__)
#include <x86intrin.h>
#endif

namespace b200 { namespace host {

typedef unsigned __int128 u128;

struct Fq {
    uint64_t l[6];
};
static const uint64_t Q_MOD[6] = {0x8508c00000000001ull, 0x170b5d4430000000ull, 0x1ef3622fba094800ull,
                                  0x1a22d9f300f5138full, 0xc63b05c06ca1493bull, 0x01ae3a4617c510eaull};
static const uint64_t Q_R1[6] = {0x02cdffffffffff68ull, 0x51409f837fffffb1ull, 0x9f7db3a98a7d3ff2ull,
                                 0x7b4e97b76e7c6305ull, 0x4cf495bf803c84e8ull, 0x008d6661e2fdf49aull};
static const uint64_t Q_INV = 9586122913090633727ull;   // fq.rs:111

inline Fq fq_zero() { Fq r; memset(r.l, 0, 48); return r; }
inline Fq fq_one() { Fq r; memcpy(r.l, Q_R1, 48); return r; }
inline bool fq_is_zero(const Fq& a) { uint64_t t = 0; for (int i = 0; i < 6; i++) t |= a.l[i]; return t == 0; }
inline bool fq_eq(const Fq& a, const Fq& b) { return memcmp(a.l, b.l, 48) == 0; }
inline bool ge_mod(const uint64_t* t) {
    for (int i = 5; i >= 0; i--) { if (t[i] != Q_MOD[i]) return t[i] > Q_MOD[i]; }
    return true;
}
inline void sub_mod(uint64_t* t) {
    uint64_t br = 0;
    for (int i = 0; i < 6; i++) { u128 d = (u128)t[i] - Q_MOD[i] - br; t[i] = (uint64_t)d; br = (uint64_t)(d >> 64) & 1; }
}
// add / sub with carry intrinsics and a branch-free correction: the Jacobian doubling below has 13 of these next to 7 products
inline Fq fq_add(const Fq& a, const Fq& b) {
#if defined(__x86_64__)
    unsigned long long s[6], d[6];
    unsigned char c = 0, br = 0;
    for (int i = 0; i < 6; i++) c = _addcarry_u64(c, a.l[i], b.l[i], &s[i]);          // < 2q < 2^384: no carry out
    for (int i = 0; i < 6; i++) br = _subborrow_u64(br, s[i], Q_MOD[i], &d[i]);
    Fq r;
    for (int i = 0; i < 6; i++) r.l[i] = br ? s[i] : d[i];                            // borrow ⇔ sum < q
    return r;
#else
    Fq r; u128 c = 0;
    for (int i = 0; i < 6; i++) { c += (u128)a.l[i] + b.l[i]; r.l[i] = (uint64_t)c; c >>= 64; }
    if (ge_mod(r.l)) sub_mod(r.l);
    return r;
#endif
}
inline Fq fq_sub(const Fq& a, const Fq& b) {
#if defined(__x86_64__)
    unsigned long long d[6], e[6];
    unsigned char br = 0, c = 0;
    for (int i = 0; i < 6; i++) br = _subborrow_u64(br, a.l[i], b.l[i], &d[i]);
    for (int i = 0; i < 6; i++) c = _addcarry_u64(c, d[i], Q_MOD[i], &e[i]);
    Fq r;
    for (int i = 0; i < 6; i++) r.l[i] = br ? e[i] : d[i];
    return r;
#else
    Fq r; uint64_t br = 0;
    for (int i = 0; i < 6; i++) { u128 d = (u128)a.l[i] - b.l[i] - br; r.l[i] = (uint64_t)d; br = (uint64_t)(d >> 64) & 1; }
    if (br) { u128 c = 0; for (int i = 0; i < 6; i++) { c += (u128)r.l[i] + Q_MOD[i]; r.l[i] = (uint64_t)c; c >>= 64; } }
    return r;
#endif
}
inline Fq fq_dbl(const Fq& a) { return fq_add(a, a); }
// Montgomery product, operand scanning with the reduction row interleaved.  q has 7 spare bits in its top limb, so a row never
// carries out of six limbs (the "no-carry" CIOS the reference's fp_384.rs:771-899 uses as well); operands are always < q here.
// 27 % faster than the generic two-loop CIOS it replaced (76 → 56 ns on the build host) — the Horner tail of every MSM call is
// ≈ 3300 of these.
inline void fq_mul_row(uint64_t (&t)[6], const uint64_t* a, uint64_t bi) {
    u128 p = (u128)a[0] * bi + t[0];
    uint64_t c1 = (uint64_t)(p >> 64);
    const uint64_t lo = (uint64_t)p, k = lo * Q_INV;
    p = (u128)k * Q_MOD[0] + lo;
    uint64_t c2 = (uint64_t)(p >> 64);
#pragma GCC unroll 8
    for (int j = 1; j < 6; j++) {
        p = (u128)a[j] * bi + t[j] + c1;
        c1 = (uint64_t)(p >> 64);
        p = (u128)k * Q_MOD[j] + (uint64_t)p + c2;
        t[j - 1] = (uint64_t)p;
        c2 = (uint64_t)(p >> 64);
    }
    t[5] = c1 + c2;
}
inline Fq fq_mul(const Fq& a, const Fq& b) {
    uint64_t t[6] = {0, 0, 0, 0, 0, 0};
#pragma GCC unroll 8
    for (int i = 0; i < 6; i++) fq_mul_row(t, a.l, b.l[i]);
    if (ge_mod(t)) sub_mod(t);
    Fq r; memcpy(r.l, t, 48); return r;
}
inline Fq fq_sqr(const Fq& a) { return fq_mul(a, a); }      // (a dedicated 57-product squaring measured SLOWER than the 72-product row loop: 60 vs 50 ns)
inline Fq fq_inverse(const Fq& a) {            // a^{q-2}
    uint64_t e[6]; memcpy(e, Q_MOD, 48); e[0] -= 2;
    Fq acc = fq_one(); bool started = false;
    for (int i = 5; i >= 0; i--)
        for (int b = 63; b >= 0; b--) {
            if (started) acc = fq_sqr(acc);
            if ((e[i] >> b) & 1) { acc = started ? fq_mul(acc, a) : a; started = true; }
        }
    return acc;
}

// Fq2 = Fq[u]/(u² + 5) (curves/src/bls12_377/fq2.rs:29-65), the base field of G2
struct Fq2 {
    Fq c0, c1;
};
inline Fq fq_times5(const Fq& x) { Fq t = fq_dbl(fq_dbl(x)); return fq_add(t, x); }
// one overload set per field so that the group law below is written once
inline Fq f_zero(const Fq*) { return fq_zero(); }
inline Fq f_one(const Fq*) { return fq_one(); }
inline bool f_is_zero(const Fq& a) { return fq_is_zero(a); }
inline Fq f_add(const Fq& a, const Fq& b) { return fq_add(a, b); }
inline Fq f_sub(const Fq& a, const Fq& b) { return fq_sub(a, b); }
inline Fq f_dbl(const Fq& a) { return fq_dbl(a); }
inline Fq f_mul(const Fq& a, const Fq& b) { return fq_mul(a, b); }
inline Fq f_sqr(const Fq& a) { return fq_sqr(a); }
inline Fq f_inverse(const Fq& a) { return fq_inverse(a); }
inline Fq2 f_zero(const Fq2*) { Fq2 r; r.c0 = fq_zero(); r.c1 = fq_zero(); return r; }
inline Fq2 f_one(const Fq2*) { Fq2 r; r.c0 = fq_one(); r.c1 = fq_zero(); return r; }
inline bool f_is_zero(const Fq2& a) { return fq_is_zero(a.c0) && fq_is_zero(a.c1); }
inline Fq2 f_add(const Fq2& a, const Fq2& b) { Fq2 r; r.c0 = fq_add(a.c0, b.c0); r.c1 = fq_add(a.c1, b.c1); return r; }
inline Fq2 f_sub(const Fq2& a, const Fq2& b) { Fq2 r; r.c0 = fq_sub(a.c0, b.c0); r.c1 = fq_sub(a.c1, b.c1); return r; }
inline Fq2 f_dbl(const Fq2& a) { return f_add(a, a); }
inline Fq2 f_mul(const Fq2& a, const Fq2& b) {
    Fq v0 = fq_mul(a.c0, b.c0), v1 = fq_mul(a.c1, b.c1);
    Fq2 r;
    r.c1 = fq_sub(fq_sub(fq_mul(fq_add(a.c0, a.c1), fq_add(b.c0, b.c1)), v0), v1);
    r.c0 = fq_sub(v0, fq_times5(v1));
    return r;
}
inline Fq2 f_sqr(const Fq2& a) { return f_mul(a, a); }
inline Fq2 f_inverse(const Fq2& a) {
    Fq n = fq_inverse(fq_add(fq_sqr(a.c0), fq_times5(fq_sqr(a.c1))));
    Fq2 r; r.c0 = fq_mul(a.c0, n); r.c1 = fq_sub(fq_zero(), fq_mul(a.c1, n));
    return r;
}

template <class F>
struct XyzzT {
    F X, Y, ZZ, ZZZ;
};
typedef XyzzT<Fq> Xyzz;        // 192 bytes: the device's XYZZ image
typedef XyzzT<Fq2> Xyzz2;      // 384 bytes: the device's XYZZ2 image
template <class F> inline XyzzT<F> xyzz_inf_t() { XyzzT<F> r; r.X = r.Y = r.ZZ = r.ZZZ = f_zero((const F*)nullptr); return r; }
inline Xyzz xyzz_inf() { return xyzz_inf_t<Fq>(); }
template <class F> inline bool xyzz_is_inf(const XyzzT<F>& p) { return f_is_zero(p.ZZ); }
template <class F> inline void xyzz_dbl(XyzzT<F>& p) {
    if (xyzz_is_inf(p)) return;
    F U = f_dbl(p.Y), V = f_sqr(U), W = f_mul(U, V), S = f_mul(p.X, V);
    F XX = f_sqr(p.X), M = f_add(f_dbl(XX), XX);
    F X3 = f_sub(f_sqr(M), f_dbl(S));
    F Y3 = f_sub(f_mul(M, f_sub(S, X3)), f_mul(W, p.Y));
    p.X = X3; p.Y = Y3; p.ZZ = f_mul(V, p.ZZ); p.ZZZ = f_mul(W, p.ZZZ);
}
template <class F> inline void xyzz_add(XyzzT<F>& p, const XyzzT<F>& o) {
    if (xyzz_is_inf(o)) return;
    if (xyzz_is_inf(p)) { p = o; return; }
    F U1 = f_mul(p.X, o.ZZ), U2 = f_mul(o.X, p.ZZ), S1 = f_mul(p.Y, o.ZZZ), S2 = f_mul(o.Y, p.ZZZ);
    F P = f_sub(U2, U1), R = f_sub(S2, S1);
    if (f_is_zero(P)) { if (f_is_zero(R)) xyzz_dbl(p); else p = xyzz_inf_t<F>(); return; }
    F PP = f_sqr(P), PPP = f_mul(P, PP), Q = f_mul(U1, PP);
    F X3 = f_sub(f_sub(f_sqr(R), PPP), f_dbl(Q));
    p.Y = f_sub(f_mul(R, f_sub(Q, X3)), f_mul(S1, PPP));
    p.X = X3;
    p.ZZ = f_mul(f_mul(p.ZZ, o.ZZ), PP);
    p.ZZZ = f_mul(f_mul(p.ZZZ, o.ZZZ), PPP);
}
// Writes the image of `result.to_affine().to_projective()`: (x, y, 1) or (0, 1, 0) for infinity —
// projective.rs:51-54, 507-512; affine.rs:331-353.  144 bytes for G1 (out[18]), 288 for G2 (out[36]).
template <class F> inline void xyzz_to_normalised_projective(const XyzzT<F>& p, uint64_t* out) {
    const size_t fb = sizeof(F);
    F one = f_one((const F*)nullptr);
    if (xyzz_is_inf(p)) { memset(out, 0, 3 * fb); memcpy((uint8_t*)out + fb, &one, fb); return; }
    F i = f_inverse(f_mul(p.ZZ, p.ZZZ));
    F x = f_mul(p.X, f_mul(i, p.ZZZ)), y = f_mul(p.Y, f_mul(i, p.ZZ));
    memcpy(out, &x, fb); memcpy((uint8_t*)out + fb, &y, fb); memcpy((uint8_t*)out + 2 * fb, &one, fb);
}
// Jacobian (X, Y, Z) image -> XYZZ (ZZ = Z^2, ZZZ = Z^3)
inline Xyzz xyzz_from_projective(const uint64_t in[18]) {
    Xyzz p; memcpy(p.X.l, in, 48); memcpy(p.Y.l, in + 6, 48);
    Fq Z; memcpy(Z.l, in + 12, 48);
    p.ZZ = fq_sqr(Z); p.ZZZ = fq_mul(p.ZZ, Z);
    if (fq_is_zero(Z)) p = xyzz_inf();
    return p;
}
// (Measured and dropped: a Jacobian doubling chain, 2M + 5S against XYZZ's 5M + 4S, and a dedicated squaring.  On the host the
// 13 additions of the Jacobian doubling and the less regular code cost what the two saved products gain: 620 vs 640 ns per
// doubling; the squaring with 57 word products ran at 60 ns against 50 ns for the row loop.)
// Σ_w 2^{c·w} · window_sum[w]  (Horner from the top window; batched.rs:404-413, standard.rs:107-117).  Every window but the top
// one is c bits wide; the top window's sum comes in `top_sets` parts, sums[nwin − 1 …] (its bucket sets, MsmPlan).
template <class F> inline XyzzT<F> horner_windows(const XyzzT<F>* sums, int nwin, int c, int top_sets = 1) {
    XyzzT<F> total = xyzz_inf_t<F>();
    for (int w = nwin - 1; w >= 0; w--) {
        for (int k = 0; k < c; k++) xyzz_dbl(total);
        xyzz_add(total, sums[w]);
        if (w == nwin - 1) for (int s = 1; s < top_sets; s++) xyzz_add(total, sums[w + s]);
    }
    return total;
}

}}  // namespace b200::host
