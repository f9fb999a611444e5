// Element-wise test kernels for the field arithmetic of ff.cuh / ec.cuh (snarkvm_b200_test_field_op_device).
//
// The machine code of a Montgomery product depends on the translation unit it is compiled in: msm.cu and pairing.cu define
// FF_CALL_MUL, so `a * b` and `a.sqr()` call the out-of-line mul_call / sqr_call there (each its own copy: the library is not
// built with relocatable device code), while ntt.cu inlines them.  ptxas is free to schedule the carry flag differently in each,
// so this header is included by all three and each instance is tested on its own.
// The includer names the entry point with FIELD_TEST_ENTRY before including it; every kernel has internal linkage.
//
// Operands come from the caller (tests/field_corpus.py): n elements of WORDS little-endian 32-bit limbs each, reduced
// Montgomery images unless the op says otherwise.  A result that cannot be correct — a warp-cooperative product whose lanes ≥ N
// are not zero — is reported by writing all-ones limbs, which is never a reduced value.
//
// The copy of the multiplier that runs here is the one inlined into these test kernels, not the one inside the NTT butterflies
// or the MSM kernels: "ntt" tests ff.cuh as compiled without FF_CALL_MUL (inlined into a kernel of ntt.cu), "msm" as compiled
// with it (the out-of-line mul_call / sqr_call of msm.cu, which msm.cu's kernels call too), "pairing" the out-of-line copies of
// pairing.cu, which every Fq6 / Fq12 product of the pairing calls.
#pragma once
#include "ec.cuh"
#include "msm.cuh"   // count_launch
#include "../../include/snarkvm_b200.h"

#ifndef FIELD_TEST_ENTRY
#error "define FIELD_TEST_ENTRY to the name of this translation unit's entry point"
#endif

namespace b200 {
namespace {

template <class F>
FF_DEV F tf_load(const uint32_t* p, size_t i) { F r;
#pragma unroll
    for (int k = 0; k < F::N; k++) r.v[k] = p[i * F::N + k]; return r; }
template <class F>
FF_DEV void tf_store(uint32_t* p, size_t i, const F& x) {
#pragma unroll
    for (int k = 0; k < F::N; k++) p[i * F::N + k] = x.v[k]; }
template <class F>
FF_DEV F tf_poison() { F r;
#pragma unroll
    for (int k = 0; k < F::N; k++) r.v[k] = 0xffffffffu; return r; }

template <class P>
__global__ void __launch_bounds__(128) k_test_field_op(int op, uint32_t* __restrict__ out, const uint32_t* __restrict__ a,
                                                       const uint32_t* __restrict__ b, size_t n) {
    using F = Fp<P>;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const F x = tf_load<F>(a, i), y = tf_load<F>(b, i);
    F r;
    switch (op) {
        case SNARKVM_B200_OP_ADD: r = x + y; break;
        case SNARKVM_B200_OP_SUB: r = x - y; break;
        case SNARKVM_B200_OP_NEG: r = x.neg(); break;
        case SNARKVM_B200_OP_DBL: r = x.dbl(); break;
        case SNARKVM_B200_OP_HALF: r = x.half(); break;
        case SNARKVM_B200_OP_MUL: r = x * y; break;
        case SNARKVM_B200_OP_MUL_INLINE: r = F::mul_inline(x, y); break;
        case SNARKVM_B200_OP_MUL_CALL: r = F::mul_call(x, y); break;
        case SNARKVM_B200_OP_MUL_KARATSUBA: r = F::mul_karatsuba(x, y); break;
        case SNARKVM_B200_OP_SQR: r = x.sqr(); break;
        case SNARKVM_B200_OP_SQR_INLINE: r = F::sqr_inline(x); break;
        case SNARKVM_B200_OP_SQR_CALL: r = F::sqr_call(x); break;
        case SNARKVM_B200_OP_INVERSE: r = x.inverse(); break;
        case SNARKVM_B200_OP_TO_MONT: r = x.to_mont(); break;
        case SNARKVM_B200_OP_FROM_MONT: r = x.from_mont(); break;
        default: r = tf_poison<F>(); break;
    }
    tf_store<F>(out, i, r);
}

// Fq2 elements: c0 then c1, 24 words; TIMES5 reads and writes plain Fq elements (12 words)
__global__ void __launch_bounds__(128) k_test_fq2_op(int op, uint32_t* __restrict__ out, const uint32_t* __restrict__ a,
                                                     const uint32_t* __restrict__ b, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (op == SNARKVM_B200_OP_TIMES5) { tf_store<Fq>(out, i, Fq2::times5(tf_load<Fq>(a, i))); return; }
    Fq2 x, y, r;
    x.c0 = tf_load<Fq>(a, 2 * i); x.c1 = tf_load<Fq>(a, 2 * i + 1);
    y.c0 = tf_load<Fq>(b, 2 * i); y.c1 = tf_load<Fq>(b, 2 * i + 1);
    switch (op) {
        case SNARKVM_B200_OP_ADD: r = x + y; break;
        case SNARKVM_B200_OP_SUB: r = x - y; break;
        case SNARKVM_B200_OP_NEG: r = x.neg(); break;
        case SNARKVM_B200_OP_DBL: r = x.dbl(); break;
        case SNARKVM_B200_OP_MUL: r = x * y; break;
        case SNARKVM_B200_OP_SQR: r = x.sqr(); break;
        case SNARKVM_B200_OP_INVERSE: r = x.inverse(); break;
        default: r.c0 = tf_poison<Fq>(); r.c1 = r.c0; break;
    }
    tf_store<Fq>(out, 2 * i, r.c0); tf_store<Fq>(out, 2 * i + 1, r.c1);
}

// One warp per element; lane 0 writes the result.  COOP_MUL: lane k < N holds limb k of a and b and returns limb k of a·b, and
// lanes ≥ N must return 0; a warp where one of them does not writes all-ones.  That is the only lane check with content: the
// limbs of r are gathered from lanes < N by full-warp shuffles (here for COOP_MUL, inside coop_inverse for COOP_INVERSE), so
// every lane holds the same r by construction and comparing the lanes' copies could never fail.  Every shuffle and vote is
// executed by all 32 lanes.
template <class P>
__global__ void __launch_bounds__(128) k_test_coop_op(int op, uint32_t* __restrict__ out, const uint32_t* __restrict__ a,
                                                      const uint32_t* __restrict__ b, size_t n) {
    using F = Fp<P>;
    constexpr int N = P::N;
    const size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= n) return;                                   // whole warps leave together
    const F x = tf_load<F>(a, w), y = tf_load<F>(b, w);
    F r;
    bool bad = false;
    if (op == SNARKVM_B200_OP_COOP_MUL) {
        uint32_t xl = 0u, yl = 0u;
#pragma unroll
        for (int k = 0; k < N; k++) if (lane == k) { xl = x.v[k]; yl = y.v[k]; }
        const uint32_t s = coop_mul<P>(xl, yl, coop_mod_limb<P>(lane), lane);
        bad = lane >= N && s != 0u;
#pragma unroll
        for (int k = 0; k < N; k++) r.v[k] = __shfl_sync(0xffffffffu, s, k);
    } else {
        r = coop_inverse<P>(x);
    }
    if (__any_sync(0xffffffffu, bad)) r = tf_poison<F>();
    if (lane == 0) tf_store<F>(out, w, r);
}

template <class P>
int tf_launch_field(int op, uint32_t* out, const uint32_t* a, const uint32_t* b, size_t n, cudaStream_t stream) {
    if (op == SNARKVM_B200_OP_COOP_MUL || op == SNARKVM_B200_OP_COOP_INVERSE) {
        k_test_coop_op<P><<<(unsigned)((n * 32 + 127) / 128), 128, 0, stream>>>(op, out, a, b, n);
    } else {
        if (op < SNARKVM_B200_OP_ADD || op > SNARKVM_B200_OP_FROM_MONT) return (int)cudaErrorInvalidValue;
        k_test_field_op<P><<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(op, out, a, b, n);
    }
    return 0;
}

}  // namespace

int FIELD_TEST_ENTRY(int field, int op, void* d_out, const void* d_a, const void* d_b, size_t n, cudaStream_t stream) {
    if (n == 0) return 0;
    if (!d_out || !d_a || !d_b || n > ((size_t)1 << 26)) return (int)cudaErrorInvalidValue;
    uint32_t* out = (uint32_t*)d_out;
    const uint32_t *a = (const uint32_t*)d_a, *b = (const uint32_t*)d_b;
    int rc;
    switch (field) {
        case SNARKVM_B200_FIELD_FR: rc = tf_launch_field<FrParams>(op, out, a, b, n, stream); break;
        case SNARKVM_B200_FIELD_FQ:
            if (op == SNARKVM_B200_OP_TIMES5) { k_test_fq2_op<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(op, out, a, b, n); rc = 0; }
            else rc = tf_launch_field<FqParams>(op, out, a, b, n, stream);
            break;
        case SNARKVM_B200_FIELD_FQ2:
            switch (op) {
                case SNARKVM_B200_OP_ADD: case SNARKVM_B200_OP_SUB: case SNARKVM_B200_OP_NEG: case SNARKVM_B200_OP_DBL:
                case SNARKVM_B200_OP_MUL: case SNARKVM_B200_OP_SQR: case SNARKVM_B200_OP_INVERSE:
                    k_test_fq2_op<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(op, out, a, b, n); rc = 0; break;
                default: rc = (int)cudaErrorInvalidValue;
            }
            break;
        default: rc = (int)cudaErrorInvalidValue;
    }
    if (rc != 0) return rc;
    count_launch();
    return (int)cudaGetLastError();
}

}  // namespace b200
