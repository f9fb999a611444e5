// Montgomery prime-field arithmetic on 32-bit limbs for sm_90a.
//
// Device restatement of the arithmetic of the reference's
//   Fp256<FrParameters>  (fields/src/fp_256.rs:52, mul :754-817, add/sub :730-750)
//   Fp384<FqParameters>  (fields/src/fp_384.rs:52, mul :771-899)
// Values are the SAME numbers as the reference keeps in memory: little-endian
// limbs of (v · 2^{32N}) mod p, always fully reduced (< p), so a device value
// stored to HBM is byte-identical to the Rust `Fp256.0.0` / `Fp384.0.0` image.
//
// Multiplication is a word-serial interleaved Montgomery product built from
// two carry chains per row ("even" columns and "odd" columns) so that every
// 32x32->64 product lands in an aligned register pair and ptxas can fuse the
// mad.lo.cc / madc.hi.cc pairs into IMAD.WIDE.U32(.X) on the fma pipe
// (see ptx_neg for what keeps the reduction rows fused).
// No tensor cores: this is integer modular arithmetic (BASELINE.json north_star).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace b200 {

// ---------------------------------------------------------------------------
// PTX carry-chain primitives.  Each is one instruction; the CC flag carries
// between consecutive statements (asm volatile keeps their order).
// ---------------------------------------------------------------------------
#define FF_DEV __device__ __forceinline__

FF_DEV uint32_t ptx_add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
FF_DEV uint32_t ptx_addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
FF_DEV uint32_t ptx_addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
FF_DEV uint32_t ptx_sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
FF_DEV uint32_t ptx_subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
FF_DEV uint32_t ptx_subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
FF_DEV uint32_t ptx_mul_lo(uint32_t a, uint32_t b) { uint32_t r; asm volatile("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
FF_DEV uint32_t ptx_mul_hi(uint32_t a, uint32_t b) { uint32_t r; asm volatile("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
FF_DEV uint32_t ptx_mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
FF_DEV uint32_t ptx_madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
FF_DEV uint32_t ptx_madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
FF_DEV uint32_t ptx_madc_hi(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }

// The Montgomery multiplier m = x·INV32 = −x mod 2^32 of a reduction row (INV32 = −1 for both moduli, asserted where it is
// used).  Written as `sub.u32 m, 0, x` on purpose: from the compiler's own `x * INV32` NVVM emits `neg.s32`, and ptxas
// folds that negation into the m·p products, issuing each as IMAD.X + IMAD.HI.U32.X (two fmaheavy instructions and a
// carry chain twice as long) instead of one IMAD.WIDE.U32.X.  tests/test_sass_mix.py checks the instruction mix.
FF_DEV uint32_t ptx_neg(uint32_t x) { uint32_t r; asm volatile("sub.u32 %0, 0, %1;" : "=r"(r) : "r"(x)); return r; }

// ---------------------------------------------------------------------------
// Row helpers.  A running value V is held as two N-limb arrays:
//     V = sum e[k]·2^{32k}  +  sum o[k]·2^{32(k+1)}
// ("o" is offset by one limb).  Products x[j]·y with even j feed e, odd j feed o.
// ---------------------------------------------------------------------------
template <int N>
FF_DEV void row_mul(uint32_t (&acc)[N], const uint32_t* x, uint32_t y) {
    // acc = sum_{j even} x[j]·y·2^{32j}   (x already points at the first column)
#pragma unroll
    for (int j = 0; j < N; j += 2) { acc[j] = ptx_mul_lo(x[j], y); acc[j + 1] = ptx_mul_hi(x[j], y); }
}
template <int N>
FF_DEV void row_mad(uint32_t (&acc)[N], const uint32_t* x, uint32_t y) {
    // acc += sum_{j even} x[j]·y·2^{32j}; leaves the carry-out in CC
    acc[0] = ptx_mad_lo_cc(x[0], y, acc[0]);
    acc[1] = ptx_madc_hi_cc(x[0], y, acc[1]);
#pragma unroll
    for (int j = 2; j < N; j += 2) { acc[j] = ptx_madc_lo_cc(x[j], y, acc[j]); acc[j + 1] = ptx_madc_hi_cc(x[j], y, acc[j + 1]); }
}
template <int N>
FF_DEV void row_mad_shift(uint32_t (&dst)[N], const uint32_t (&src)[N], const uint32_t* x, uint32_t y) {
    // dst[k] = src[k+2] + (sum_{j even} x[j]·y·2^{32j})[k] + carry-in (CC); top two limbs have no src.
#pragma unroll
    for (int j = 0; j < N - 2; j += 2) { dst[j] = ptx_madc_lo_cc(x[j], y, src[j + 2]); dst[j + 1] = ptx_madc_hi_cc(x[j], y, src[j + 3]); }
    dst[N - 2] = ptx_madc_lo_cc(x[N - 2], y, 0u);
    dst[N - 1] = ptx_madc_hi(x[N - 2], y, 0u);
}

// One word-serial step:  V <- (V_prev/2^32 + a·bi + m·p)  with m chosen so the low limb vanishes.
// On entry (ee, oo) hold V_prev BEFORE its pending one-limb right shift (ee[0] == 0).
// On exit  (oo', ee') := (new even array, new odd array) — the roles swap because of the shift,
// so the caller alternates the argument order.
template <int N, class P>
FF_DEV void mont_step(uint32_t (&ev)[N], uint32_t (&od)[N], const uint32_t (&a)[N], uint32_t bi, bool first) {
    // `ev` is the array that is limb-aligned with V after the shift (it was the odd array before);
    // `od` was the even array before the shift: od[1] lands on limb 0, od[2..] become the new odd array.
    if (first) {
        row_mul<N>(od, &a[1], bi);
        row_mul<N>(ev, &a[0], bi);
    } else {
        ev[0] = ptx_add_cc(ev[0], od[1]);
        uint32_t nod[N];
        row_mad_shift<N>(nod, od, &a[1], bi);          // consumes the carry of the add above
#pragma unroll
        for (int k = 0; k < N; k++) od[k] = nod[k];
        row_mad<N>(ev, &a[0], bi);
        od[N - 1] = ptx_addc(od[N - 1], 0u);
    }
    // Montgomery reduction row: m = -ev[0] / p mod 2^32
    static_assert(P::INV32 == 0xffffffffu, "m = ev[0]·INV32 is computed as −ev[0]");
    const uint32_t m = ptx_neg(ev[0]);
    uint32_t pm[N];
#pragma unroll
    for (int k = 0; k < N; k++) pm[k] = P::mod(k);
    row_mad<N>(od, &pm[1], m);                          // odd columns of p (pm[N] is never read: j < N-1)
#ifdef FF_NO_P0_SHORTCUT
    if (false) {
#else
    if (P::MOD0_IS_ONE) {
#endif
        // both BLS12-377 moduli are ≡ 1 mod 2^32: p[0]·m = m, so column 0 is ev[0] + m = 0 with carry
        // (ev[0] != 0) and the high word of that product is 0 — two adds instead of a 32x32->64 multiply.
        ev[0] = ptx_add_cc(ev[0], m);
        ev[1] = ptx_addc_cc(ev[1], 0u);
#pragma unroll
        for (int j = 2; j < N; j += 2) { ev[j] = ptx_madc_lo_cc(pm[j], m, ev[j]); ev[j + 1] = ptx_madc_hi_cc(pm[j], m, ev[j + 1]); }
    } else {
        row_mad<N>(ev, &pm[0], m);
    }
    od[N - 1] = ptx_addc(od[N - 1], 0u);
}

// ---------------------------------------------------------------------------
// Plain H×H-limb product T[2H] = a·b (H even) for the Karatsuba multiplier below.  Products are accumulated by the
// parity of their position i + j: E holds the even positions, O (offset by one limb) the odd ones, so within a row
// the (lo, hi) register pairs of consecutive products tile the accumulator and form ONE carry chain; the carry out of
// a row lands in a limb that holds at most another row's carry.  tests/manual/karatsuba_model.py is a
// statement-level model of this code (and of mul_karatsuba) checked against big integers.
// ---------------------------------------------------------------------------
template <int H>
FF_DEV void mul_wide(const uint32_t* a, const uint32_t* b, uint32_t (&T)[2 * H]) {
    uint32_t E[2 * H], O[2 * H];
#pragma unroll
    for (int k = 0; k < 2 * H; k++) { E[k] = 0u; O[k] = 0u; }
#pragma unroll
    for (int i = 0; i < H; i++) {
        {   // even positions: j ≡ i (mod 2)
#pragma unroll
            for (int j = (i & 1); j < H; j += 2) {
                const int p = i + j;
                if (j == (i & 1)) E[p] = ptx_mad_lo_cc(a[j], b[i], E[p]);
                else E[p] = ptx_madc_lo_cc(a[j], b[i], E[p]);
                E[p + 1] = ptx_madc_hi_cc(a[j], b[i], E[p + 1]);
                if (j + 2 >= H && p + 2 < 2 * H) E[p + 2] = ptx_addc(E[p + 2], 0u);
            }
        }
        {   // odd positions: j ≢ i → O[p − 1], O[p]
#pragma unroll
            for (int j = 1 - (i & 1); j < H; j += 2) {
                const int p = i + j;
                if (j == 1 - (i & 1)) O[p - 1] = ptx_mad_lo_cc(a[j], b[i], O[p - 1]);
                else O[p - 1] = ptx_madc_lo_cc(a[j], b[i], O[p - 1]);
                O[p] = ptx_madc_hi_cc(a[j], b[i], O[p]);
                if (j + 2 >= H && p + 1 < 2 * H - 1) O[p + 1] = ptx_addc(O[p + 1], 0u);
            }
        }
    }
    T[0] = E[0];
    T[1] = ptx_add_cc(E[1], O[0]);
#pragma unroll
    for (int k = 2; k < 2 * H - 1; k++) T[k] = ptx_addc_cc(E[k], O[k - 1]);
    T[2 * H - 1] = ptx_addc(E[2 * H - 1], O[2 * H - 2]);
}
// d = |x − y| over H limbs; returns 1 when x < y
template <int H>
FF_DEV uint32_t abs_diff(const uint32_t* x, const uint32_t* y, uint32_t (&d)[H]) {
    d[0] = ptx_sub_cc(x[0], y[0]);
#pragma unroll
    for (int i = 1; i < H; i++) d[i] = ptx_subc_cc(x[i], y[i]);
    const uint32_t m = ptx_subc(0u, 0u);               // 0xffffffff if x < y
    // conditional two's complement: (d ^ m) + (m & 1)
    d[0] = ptx_add_cc(d[0] ^ m, m & 1u);
#pragma unroll
    for (int i = 1; i < H - 1; i++) d[i] = ptx_addc_cc(d[i] ^ m, 0u);
    d[H - 1] = ptx_addc(d[H - 1] ^ m, 0u);
    return m & 1u;
}

// ---------------------------------------------------------------------------
// Field element
// ---------------------------------------------------------------------------
template <class P>
struct Fp {
    static constexpr int N = P::N;
    static constexpr int WORDS = P::N;
    uint32_t v[N];

    FF_DEV static Fp zero() { Fp r;
#pragma unroll
        for (int i = 0; i < N; i++) r.v[i] = 0u; return r; }
    FF_DEV static Fp one() { Fp r;
#pragma unroll
        for (int i = 0; i < N; i++) r.v[i] = P::r1(i); return r; }
    FF_DEV static Fp r2() { Fp r;
#pragma unroll
        for (int i = 0; i < N; i++) r.v[i] = P::r2(i); return r; }

    FF_DEV bool is_zero() const { uint32_t t = 0;
#pragma unroll
        for (int i = 0; i < N; i++) t |= v[i]; return t == 0; }
    FF_DEV bool operator==(const Fp& o) const { uint32_t t = 0;
#pragma unroll
        for (int i = 0; i < N; i++) t |= v[i] ^ o.v[i]; return t == 0; }
    FF_DEV bool operator!=(const Fp& o) const { return !(*this == o); }

    // r = (x >= p) ? x - p : x      (x < 2p)
    FF_DEV void final_sub() {
        uint32_t t[N];
        t[0] = ptx_sub_cc(v[0], P::mod(0));
#pragma unroll
        for (int i = 1; i < N; i++) t[i] = ptx_subc_cc(v[i], P::mod(i));
        uint32_t borrow = ptx_subc(0u, 0u);            // 0xffffffff if x < p
        if (borrow == 0u) {
#pragma unroll
            for (int i = 0; i < N; i++) v[i] = t[i];
        }
    }

    FF_DEV friend Fp operator+(const Fp& a, const Fp& b) {
        Fp r;
        r.v[0] = ptx_add_cc(a.v[0], b.v[0]);
#pragma unroll
        for (int i = 1; i < N - 1; i++) r.v[i] = ptx_addc_cc(a.v[i], b.v[i]);
        r.v[N - 1] = ptx_addc(a.v[N - 1], b.v[N - 1]);  // moduli leave ≥3 spare bits: no carry out
        r.final_sub();
        return r;
    }
    FF_DEV friend Fp operator-(const Fp& a, const Fp& b) {
        Fp r;
        r.v[0] = ptx_sub_cc(a.v[0], b.v[0]);
#pragma unroll
        for (int i = 1; i < N; i++) r.v[i] = ptx_subc_cc(a.v[i], b.v[i]);
        uint32_t borrow = ptx_subc(0u, 0u);
        if (borrow) {
            r.v[0] = ptx_add_cc(r.v[0], P::mod(0));
#pragma unroll
            for (int i = 1; i < N - 1; i++) r.v[i] = ptx_addc_cc(r.v[i], P::mod(i));
            r.v[N - 1] = ptx_addc(r.v[N - 1], P::mod(N - 1));
        }
        return r;
    }
    FF_DEV Fp neg() const { return is_zero() ? *this : (zero() - *this); }
    FF_DEV Fp dbl() const { return *this + *this; }

    FF_DEV static Fp mul_inline(const Fp& a, const Fp& b) {
        uint32_t e[N], o[N];
#pragma unroll
        for (int i = 0; i < N; i += 2) {
            mont_step<N, P>(e, o, a.v, b.v[i], i == 0);
            mont_step<N, P>(o, e, a.v, b.v[i + 1], false);
        }
        // pending shift + merge: result[k] = e'[k] + o'[k+1]  where (e', o') = (e, o) roles after N steps
        Fp r;
        r.v[0] = ptx_add_cc(e[0], o[1]);
#pragma unroll
        for (int k = 1; k < N - 1; k++) r.v[k] = ptx_addc_cc(e[k], o[k + 1]);
        r.v[N - 1] = ptx_addc(e[N - 1], 0u);
        r.final_sub();
        return r;
    }
    // Out-of-line copy (arguments and result travel in registers — checked in SASS).  Kernels whose hot
    // loop contains many multiplications call this one so the loop stays inside the instruction cache.
    // Karatsuba (below) trades 36 (Fq) / 16 (Fr) of the 32×32→64 multiplications for ≈ 220 / 110 ALU instructions, and
    // measured SLOWER in both fields (tools/ff_microbench.cu): at 4 warps per scheduler the multiplier is bound by issue slots and the carry-chain latency as much as by the
    // fmaheavy pipe, so the word-serial product stays the default; -DFF_KARATSUBA selects the other one.
#ifdef FF_KARATSUBA
    FF_DEV static Fp mul_best(const Fp& a, const Fp& b) { return mul_karatsuba(a, b); }
#else
    FF_DEV static Fp mul_best(const Fp& a, const Fp& b) { return mul_inline(a, b); }
#endif
    static __device__ __noinline__ Fp mul_call(Fp a, Fp b) { return mul_best(a, b); }
    FF_DEV friend Fp operator*(const Fp& a, const Fp& b) {
#ifdef FF_CALL_MUL
        return mul_call(a, b);
#else
        return mul_best(a, b);
#endif
    }
    // T·2^{-32N} mod p for a 2N-limb T < p·2^{32N} (the product of two reduced elements).
    FF_DEV static Fp mont_reduce_wide(const uint32_t (&T)[2 * N]) {
        // Montgomery reduction of the 2N-limb square: V = ev + od·2^32 starts as the low half; every step clears
        // the low limb with m·p, shifts one limb down and lets the next high limb of T in at the top.
        uint32_t ev[N], od[N];
#pragma unroll
        for (int k = 0; k < N; k++) { ev[k] = T[k]; od[k] = 0u; }
        uint32_t pm[N];
#pragma unroll
        for (int k = 0; k < N; k++) pm[k] = P::mod(k);
#pragma unroll
        for (int i = 0; i < N; i++) {
            static_assert(P::INV32 == 0xffffffffu, "m = ev[0]·INV32 is computed as −ev[0]");
            const uint32_t m = ptx_neg(ev[0]);
            row_mad<N>(od, &pm[1], m);
            if (P::MOD0_IS_ONE) {
                ev[0] = ptx_add_cc(ev[0], m);
                ev[1] = ptx_addc_cc(ev[1], 0u);
#pragma unroll
                for (int j = 2; j < N; j += 2) { ev[j] = ptx_madc_lo_cc(pm[j], m, ev[j]); ev[j + 1] = ptx_madc_hi_cc(pm[j], m, ev[j + 1]); }
            } else {
                row_mad<N>(ev, &pm[0], m);
            }
            od[N - 1] = ptx_addc(od[N - 1], 0u);
            // shift one limb: (ev, od) ← (od + ev[1], ev[2..] ‖ T[N+i] ‖ 0) with the carry of the first add rippling up
            uint32_t nev[N], nod[N];
            nev[0] = ptx_add_cc(od[0], ev[1]);
#pragma unroll
            for (int k = 0; k < N - 2; k++) nod[k] = ptx_addc_cc(ev[k + 2], 0u);
            nod[N - 2] = ptx_addc_cc(T[N + i], 0u);
            nod[N - 1] = ptx_addc(0u, 0u);
#pragma unroll
            for (int k = 1; k < N; k++) nev[k] = od[k];
#pragma unroll
            for (int k = 0; k < N; k++) { ev[k] = nev[k]; od[k] = nod[k]; }
        }
        Fp r;
        r.v[0] = ev[0];
        r.v[1] = ptx_add_cc(ev[1], od[0]);
#pragma unroll
        for (int k = 2; k < N; k++) r.v[k] = ptx_addc_cc(ev[k], od[k - 1]);
        r.final_sub();
        return r;
    }
    // Karatsuba (one level, subtractive): a·b = z0 + (z0 + z2 − (a0 − a1)(b0 − b1))·2^{16N} + z2·2^{32N} with three N/2-limb
    // products — 3·(N/2)² = 108 (Fq) / 48 (Fr) 32×32→64 multiplications instead of N² = 144 / 64; the additions run on the
    // ALU pipe, which the multiplier leaves idle.  Then the same N reduction rows as the squaring.
    FF_DEV static Fp mul_karatsuba(const Fp& a, const Fp& b) {
        constexpr int H = N / 2;
        uint32_t T[2 * N];
        uint32_t mid[N + 1];
        {
            uint32_t z0[N], z2[N];
            mul_wide<H>(&a.v[0], &b.v[0], z0);
            mul_wide<H>(&a.v[H], &b.v[H], z2);
            mid[0] = ptx_add_cc(z0[0], z2[0]);
#pragma unroll
            for (int k = 1; k < N; k++) mid[k] = ptx_addc_cc(z0[k], z2[k]);
            mid[N] = ptx_addc(0u, 0u);
#pragma unroll
            for (int k = 0; k < N; k++) { T[k] = z0[k]; T[N + k] = z2[k]; }
        }
        {
            uint32_t da[H], db[H], zm[N];
            const uint32_t sa = abs_diff<H>(&a.v[0], &a.v[H], da), sb = abs_diff<H>(&b.v[0], &b.v[H], db);
            mul_wide<H>(da, db, zm);
            // mid −= zm when the signs agree, += zm otherwise: add (zm ^ mask) and then the two's-complement +1
            const uint32_t mask = (sa == sb) ? 0xffffffffu : 0u;
            mid[0] = ptx_add_cc(mid[0], zm[0] ^ mask);
#pragma unroll
            for (int k = 1; k < N; k++) mid[k] = ptx_addc_cc(mid[k], zm[k] ^ mask);
            mid[N] = ptx_addc(mid[N], mask);
            mid[0] = ptx_add_cc(mid[0], mask & 1u);
#pragma unroll
            for (int k = 1; k < N; k++) mid[k] = ptx_addc_cc(mid[k], 0u);
            mid[N] = ptx_addc(mid[N], 0u);
        }
        T[H] = ptx_add_cc(T[H], mid[0]);
#pragma unroll
        for (int k = 1; k <= N; k++) T[H + k] = ptx_addc_cc(T[H + k], mid[k]);
#pragma unroll
        for (int k = H + N + 1; k < 2 * N - 1; k++) T[k] = ptx_addc_cc(T[k], 0u);
        T[2 * N - 1] = ptx_addc(T[2 * N - 1], 0u);
        return mont_reduce_wide(T);
    }
    // Dedicated squaring: N(N−1)/2 cross products (doubled by a 1-bit shift) + N diagonal products instead of N²,
    // then N Montgomery reduction rows on the 2N-limb square.  Cross products use the same even/odd carry-chain
    // layout as the multiplier: E holds columns of even position, O (offset by one limb) those of odd position.
    FF_DEV static Fp sqr_inline(const Fp& a) {
        uint32_t E[2 * N], O[2 * N];
#pragma unroll
        for (int k = 0; k < 2 * N; k++) { E[k] = 0u; O[k] = 0u; }
#pragma unroll
        for (int i = 0; i < N - 1; i++) {
            // products a_i·a_j, j > i: position i+j.  Same parity as i ⇒ even position ⇒ E; else O (index pos−1).
            {   // j = i+2, i+4, …  (even positions 2i+2, …)
                bool first = true;
#pragma unroll
                for (int j = i + 2; j < N; j += 2) {
                    const int p = i + j;
                    if (first) { E[p] = ptx_mad_lo_cc(a.v[i], a.v[j], E[p]); first = false; }
                    else E[p] = ptx_madc_lo_cc(a.v[i], a.v[j], E[p]);
                    E[p + 1] = ptx_madc_hi_cc(a.v[i], a.v[j], E[p + 1]);
                    if (j + 2 >= N) E[p + 2] = ptx_addc(E[p + 2], 0u);       // untouched so far: receives the carry
                }
            }
            {   // j = i+1, i+3, …  (odd positions 2i+1, …) → O[pos−1]
                bool first = true;
#pragma unroll
                for (int j = i + 1; j < N; j += 2) {
                    const int p = i + j - 1;
                    if (first) { O[p] = ptx_mad_lo_cc(a.v[i], a.v[j], O[p]); first = false; }
                    else O[p] = ptx_madc_lo_cc(a.v[i], a.v[j], O[p]);
                    O[p + 1] = ptx_madc_hi_cc(a.v[i], a.v[j], O[p + 1]);
                    if (j + 2 >= N) O[p + 2] = ptx_addc(O[p + 2], 0u);
                }
            }
        }
        // T = E + (O << 32)
        uint32_t T[2 * N];
        T[0] = E[0];
        T[1] = ptx_add_cc(E[1], O[0]);
#pragma unroll
        for (int k = 2; k < 2 * N - 1; k++) T[k] = ptx_addc_cc(E[k], O[k - 1]);
        T[2 * N - 1] = ptx_addc(E[2 * N - 1], O[2 * N - 2]);
        // T = 2·T (the cross terms appear twice) …
#pragma unroll
        for (int k = 2 * N - 1; k > 0; k--) T[k] = __funnelshift_l(T[k - 1], T[k], 1);
        T[0] <<= 1;
        // … + Σ a_i²·2^{64 i}
        T[0] = ptx_mad_lo_cc(a.v[0], a.v[0], T[0]);
        T[1] = ptx_madc_hi_cc(a.v[0], a.v[0], T[1]);
#pragma unroll
        for (int i = 1; i < N; i++) { T[2 * i] = ptx_madc_lo_cc(a.v[i], a.v[i], T[2 * i]); T[2 * i + 1] = ptx_madc_hi_cc(a.v[i], a.v[i], T[2 * i + 1]); }
        return mont_reduce_wide(T);
    }
    static __device__ __noinline__ Fp sqr_call(Fp a) { return sqr_inline(a); }
    FF_DEV Fp sqr() const {
#if defined(FF_NO_SQR)
        return (*this) * (*this);
#elif defined(FF_CALL_MUL)
        return sqr_call(*this);
#else
        return sqr_inline(*this);
#endif
    }

    // a^e for a fixed public exponent given as 32-bit limbs (MSB-first square-and-multiply)
    template <int L>
    FF_DEV Fp pow_const(const uint32_t (&e)[L]) const {
        Fp acc = one();
        bool started = false;
        for (int i = L - 1; i >= 0; i--) {
            for (int b = 31; b >= 0; b--) {
                if (started) acc = acc.sqr();
                if ((e[i] >> b) & 1u) { acc = started ? acc * (*this) : *this; started = true; }
            }
        }
        return acc;
    }
    // Fermat inverse a^{p-2}; returns zero for zero (callers that need the reference's Option test is_zero first).
    FF_DEV Fp inverse() const {
        uint32_t e[N];
        uint32_t borrow = 2u;                           // e = p - 2
#pragma unroll
        for (int i = 0; i < N; i++) { uint32_t m = P::mod(i); e[i] = m - borrow; borrow = (m < borrow) ? 1u : 0u; }
        return pow_const<N>(e);
    }

    // x/2 mod p (works on Montgomery images too: (x/2)·R = (x·R)/2)
    FF_DEV Fp half() const {
        uint32_t t[N + 1];
        if (v[0] & 1u) {
            t[0] = ptx_add_cc(v[0], P::mod(0));
#pragma unroll
            for (int i = 1; i < N; i++) t[i] = ptx_addc_cc(v[i], P::mod(i));
            t[N] = ptx_addc(0u, 0u);
        } else {
#pragma unroll
            for (int i = 0; i < N; i++) t[i] = v[i];
            t[N] = 0u;
        }
        Fp r;
#pragma unroll
        for (int i = 0; i < N; i++) r.v[i] = __funnelshift_r(t[i], t[i + 1], 1);
        return r;
    }

    FF_DEV Fp to_mont() const { return (*this) * r2(); }
    FF_DEV Fp from_mont() const { Fp o = zero(); o.v[0] = 1u; return (*this) * o; }

    // 128-bit vector global memory access (coalesced across a warp when elements are contiguous)
    FF_DEV static Fp load(const void* p) {
        Fp r; const uint4* q = reinterpret_cast<const uint4*>(p);
#pragma unroll
        for (int i = 0; i < N / 4; i++) { uint4 t = q[i]; r.v[4 * i] = t.x; r.v[4 * i + 1] = t.y; r.v[4 * i + 2] = t.z; r.v[4 * i + 3] = t.w; }
        return r;
    }
    FF_DEV static Fp load_ldg(const void* p) {
        Fp r; const uint4* q = reinterpret_cast<const uint4*>(p);
#pragma unroll
        for (int i = 0; i < N / 4; i++) { uint4 t = __ldg(q + i); r.v[4 * i] = t.x; r.v[4 * i + 1] = t.y; r.v[4 * i + 2] = t.z; r.v[4 * i + 3] = t.w; }
        return r;
    }
    FF_DEV void store(void* p) const {
        uint4* q = reinterpret_cast<uint4*>(p);
#pragma unroll
        for (int i = 0; i < N / 4; i++) q[i] = make_uint4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    }
};

// ---------------------------------------------------------------------------
// Warp-cooperative Montgomery arithmetic: ONE field element spread over a warp, limb j in lane j (lanes ≥ N hold 0).
// A lone warp running the word-serial multiplier above is latency-bound (≈ 700 dependent instructions per product);
// here a product is N iterations of { a·b_i, m·p, shift one limb down } on a carry-save value (lo, hi, ex per lane), with
// three shuffles per iteration, then one ballot-based carry resolution and one ballot-based conditional subtraction:
// ≈ 170 instructions per product for the whole warp.  Used for the single Fermat inversion a CTA shares (msm.cu), where
// 31 lanes would otherwise compute the same 570 products redundantly.  tests/manual/coop_mul_model.py is a statement-by-
// statement model of this code checked against big integers.
// ---------------------------------------------------------------------------
FF_DEV uint32_t coop_carries_in(uint32_t gen, uint32_t prop) {
    // bit j = carry (borrow) into lane j, given the lanes that generate one and the lanes that pass one on
    const uint32_t a = gen | prop;
    return (a + gen) ^ a ^ gen;
}
template <class P>
FF_DEV uint32_t coop_mod_limb(int lane) {
    uint32_t p = 0u;
#pragma unroll
    for (int k = 0; k < P::N; k++) if (lane == k) p = P::mod(k);
    return p;
}
// limbs of a·b·R^{-1} mod p, fully reduced; a, b, p = this lane's limbs; all 32 lanes must call it
template <class P>
FF_DEV uint32_t coop_mul(uint32_t a, uint32_t b, uint32_t p, int lane) {
    constexpr int N = P::N;
    uint32_t lo = 0u, hi = 0u, ex = 0u;
    uint32_t bi = __shfl_sync(0xffffffffu, b, 0);
#pragma unroll
    for (int i = 0; i < N; i++) {
        const uint32_t bnext = __shfl_sync(0xffffffffu, b, (i + 1) % N);      // off the critical path
        asm("mad.lo.cc.u32 %0, %3, %4, %0; madc.hi.cc.u32 %1, %3, %4, %1; addc.u32 %2, %2, 0;" : "+r"(lo), "+r"(hi), "+r"(ex) : "r"(a), "r"(bi));
        const uint32_t m = __shfl_sync(0xffffffffu, lo * P::INV32, 0);       // lane 0 decides the reduction multiple
        asm("mad.lo.cc.u32 %0, %3, %4, %0; madc.hi.cc.u32 %1, %3, %4, %1; addc.u32 %2, %2, 0;" : "+r"(lo), "+r"(hi), "+r"(ex) : "r"(m), "r"(p));
        // lane 0's lo is now 0: divide by 2^32 — V'_j = (V_j >> 32) + lo_{j+1}  (lane 31's own lo is always 0)
        const uint32_t t = __shfl_down_sync(0xffffffffu, lo, 1);
        asm("add.cc.u32 %0, %1, %3; addc.u32 %1, %2, 0;" : "=r"(lo), "+r"(hi), "+r"(ex) : "r"(t));
        ex = 0u;
        bi = bnext;
    }
    // carry-save → canonical limbs: s_j = lo_j + hi_{j-1}, then carries resolved across lanes in one step
    uint32_t up = __shfl_up_sync(0xffffffffu, hi, 1);
    if (lane == 0) up = 0u;
    uint32_t s = lo + up;
    const uint32_t cin = coop_carries_in(__ballot_sync(0xffffffffu, s < up), __ballot_sync(0xffffffffu, s == 0xffffffffu));
    s += (cin >> lane) & 1u;
    // r = s ≥ p ? s − p : s  — the most significant differing limb decides
    const uint32_t gt = __ballot_sync(0xffffffffu, s > p), lt = __ballot_sync(0xffffffffu, s < p);
    if (gt >= lt) {
        const uint32_t bin = coop_carries_in(lt, __ballot_sync(0xffffffffu, s == p));
        s = s - p - ((bin >> lane) & 1u);
    }
    return s;
}
// a^{p-2} for an element every lane of the warp holds (e.g. after a broadcast); every lane returns the inverse.  0 ↦ 0.
template <class P>
FF_DEV Fp<P> coop_inverse(const Fp<P>& v) {
    constexpr int N = P::N;
    const int lane = threadIdx.x & 31;
    const uint32_t p = coop_mod_limb<P>(lane);
    uint32_t x = 0u;
#pragma unroll
    for (int k = 0; k < N; k++) if (lane == k) x = v.v[k];
    uint32_t acc = x;
    bool started = false;
#pragma unroll 1
    for (int i = N - 1; i >= 0; i--) {
        uint32_t e = 0u, borrow_in = 0u;                 // limb i of p − 2 (p ≡ 1 mod 2^32 would borrow; handled generally)
#pragma unroll
        for (int k = 0; k < N; k++) {
            const uint32_t mk = P::mod(k), sub = (k == 0 ? 2u : 0u) + borrow_in;
            const uint32_t ek = mk - sub;
            borrow_in = (mk < sub) ? 1u : 0u;
            if (k == i) e = ek;
        }
#pragma unroll 1
        for (int b = 31; b >= 0; b--) {
            if (started) acc = coop_mul<P>(acc, acc, p, lane);
            if ((e >> b) & 1u) { acc = started ? coop_mul<P>(acc, x, p, lane) : x; started = true; }
        }
    }
    Fp<P> r;
#pragma unroll
    for (int k = 0; k < N; k++) r.v[k] = __shfl_sync(0xffffffffu, acc, k);
    return r;
}

// ---------------------------------------------------------------------------
// BLS12-377 parameters (numbers from curves/src/bls12_377/fr.rs:109-192, fq.rs:85-176,
// re-expressed as 32-bit limbs; cross-checked in tests against oracle/bls12_377.py).
// ---------------------------------------------------------------------------
#define FF_TABLE(name, ...) \
    __host__ __device__ static constexpr uint32_t name(int i) { constexpr uint32_t t[N] = {__VA_ARGS__}; return t[i]; }

struct FrParams {
    static constexpr int N = 8;
    static constexpr uint32_t INV32 = 0xffffffffu;     // -r^{-1} mod 2^32 (low word of INV, fr.rs:137)
    static constexpr bool MOD0_IS_ONE = true;
    FF_TABLE(mod, 0x00000001u, 0x0a118000u, 0xd0000001u, 0x59aa76feu, 0x5c37b001u, 0x60b44d1eu, 0x9a2ca556u, 0x12ab655eu)
    FF_TABLE(r1,  0xfffffff3u, 0x7d1c7fffu, 0x6ffffff2u, 0x7257f50fu, 0x512c0feeu, 0x16d81575u, 0x2bbb9a9du, 0x0d4bda32u)
    FF_TABLE(r2,  0xb861857bu, 0x25d577bau, 0x8860591fu, 0xcc2c27b5u, 0xe5dc8593u, 0xa7cc008fu, 0xeff1c939u, 0x011fdae7u)
};
struct FqParams {
    static constexpr int N = 12;
    static constexpr uint32_t INV32 = 0xffffffffu;     // -q^{-1} mod 2^32 (low word of INV, fq.rs:111)
    static constexpr bool MOD0_IS_ONE = true;
    FF_TABLE(mod, 0x00000001u, 0x8508c000u, 0x30000000u, 0x170b5d44u, 0xba094800u, 0x1ef3622fu, 0x00f5138fu, 0x1a22d9f3u, 0x6ca1493bu, 0xc63b05c0u, 0x17c510eau, 0x01ae3a46u)
    FF_TABLE(r1,  0xffffff68u, 0x02cdffffu, 0x7fffffb1u, 0x51409f83u, 0x8a7d3ff2u, 0x9f7db3a9u, 0x6e7c6305u, 0x7b4e97b7u, 0x803c84e8u, 0x4cf495bfu, 0xe2fdf49au, 0x008d6661u)
    FF_TABLE(r2,  0x9400cd22u, 0xb786686cu, 0xb00431b1u, 0x0329fcaau, 0x62d6b46du, 0x22a5f111u, 0x827dc3acu, 0xbfdf7d03u, 0x41790bf9u, 0x837e92f0u, 0x1e914b88u, 0x006dfccbu)
};
#undef FF_TABLE

using Fr = Fp<FrParams>;
using Fq = Fp<FqParams>;

}  // namespace b200
