// Device-resident polynomial helpers around the NTT (SURVEY §8 f2/f3): the pieces of the Varuna prover that sit between
// transforms and would otherwise force a PCIe round trip per polynomial.
//
//   fr_batch_inversion_and_mul_device  — fields/src/lib.rs:78-129 (batch_inversion_and_mul; used by
//                                        snark/varuna/ahp/prover/round_functions/fourth.rs:203-211)
//   poly_divide_by_vanishing_device    — fft/polynomial/dense.rs:162-169 → fft/polynomial/mod.rs:222-256 with the
//                                        divisor x^n − 1
//   poly_evaluate_device               — DensePolynomial::evaluate (fft/polynomial/dense.rs:98-114)
//   csr_serialize_device               — the circuit id's byte stream (snark/varuna/ahp/indexer/circuit.rs:109-121)
//   fr_lincomb_device                  — a LinearCombination of polynomials in one pass (snark/varuna/varuna.rs:256-272)
//   matrix_evals_dot_device            — MatrixEvals::evaluate (snark/varuna/ahp/matrices.rs:114-126)
//
// Every result is a canonical Fr value, so any correct evaluation order is bit-identical to the reference's.
#include "poly.cuh"

#include <algorithm>
#include <cstring>
#include <vector>

#include "ff.cuh"
#include "msm.cuh"   // count_launch, ensure_pool_configured
#include "ntt.cuh"   // NTT_MAX_LG

namespace b200 {

struct FrArg { uint32_t v[8]; };
FF_DEV Fr fr_from_arg(const FrArg& a) { Fr r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = a.v[i]; return r; }

// Segmented launches: thread (or CTA) g of the grid belongs to the last segment whose `first` is ≤ g (segments hold consecutive
// ranges of the grid; empty ones are skipped by the search).
template <class Seg> FF_DEV uint32_t seg_of(const Seg* __restrict__ segs, uint32_t nsegs, uint64_t g) {
    uint32_t lo = 0, hi = nsegs;
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (segs[mid].first <= g) lo = mid; else hi = mid;
    }
    return lo;
}

// ---------------------------------------------------------------------------------------------------------------------
// v_i ← coeff · v_i^{-1}; zeros are skipped and stay zero (lib.rs:107, 121).  Montgomery's trick per thread over K
// elements taken with a grid stride (coalesced), one Fermat inversion per K: ≈ 3 + 380/K multiplications per element.
// ---------------------------------------------------------------------------------------------------------------------
static constexpr int BINV_K = 8;
__global__ void __launch_bounds__(128) k_fr_batch_inverse(uint32_t* __restrict__ v, size_t n, FrArg coeff_arg) {
    const size_t T = (size_t)gridDim.x * blockDim.x, t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    Fr x[BINV_K], pre[BINV_K];
    Fr run = Fr::one();
#pragma unroll
    for (int k = 0; k < BINV_K; k++) {
        size_t i = (size_t)k * T + t;
        x[k] = i < n ? Fr::load(v + i * 8) : Fr::zero();
        pre[k] = run;                                      // product of the non-zero elements before k
        if (!x[k].is_zero()) run = run * x[k];
    }
    Fr inv = run.inverse() * fr_from_arg(coeff_arg);       // run ≠ 0 (one if everything was zero)
#pragma unroll
    for (int k = BINV_K - 1; k >= 0; k--) {
        size_t i = (size_t)k * T + t;
        if (i < n && !x[k].is_zero()) {
            (inv * pre[k]).store(v + i * 8);
            inv = inv * x[k];
        }
    }
}

int fr_batch_inversion_and_mul_device(void* d_v, size_t n, const void* coeff_mont_host, cudaStream_t stream) {
    if (n == 0) return 0;
    if (!d_v || !coeff_mont_host) return (int)cudaErrorInvalidValue;
    FrArg c;
    memcpy(c.v, coeff_mont_host, 32);
    size_t threads = (n + BINV_K - 1) / BINV_K;
    k_fr_batch_inverse<<<(unsigned)((threads + 127) / 128), 128, 0, stream>>>((uint32_t*)d_v, n, c);
    count_launch();
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// p = q·(x^n − 1) + r  ⇒  q_i = Σ_{k ≥ 1} p_{i + k·n},  r_i = p_i + q_i  (q_i = 0 past its end).
// ---------------------------------------------------------------------------------------------------------------------
__global__ void k_divide_by_vanishing(const uint32_t* __restrict__ p, size_t m, size_t n, uint32_t* __restrict__ q,
                                      uint32_t* __restrict__ r) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t qlen = m > n ? m - n : 0, rlen = m < n ? m : n;
    if (i >= qlen && i >= rlen) return;
    Fr acc = Fr::zero();
    for (size_t j = i + n; j < m; j += n) acc = acc + Fr::load_ldg(p + j * 8);
    if (i < qlen) acc.store(q + i * 8);
    if (i < rlen) (acc + Fr::load_ldg(p + i * 8)).store(r + i * 8);
}

// The loop above costs m/n additions per output: fine for the quotient by a large domain (m/n ≤ a few), quadratic for a SMALL
// one — Varuna's first round divides a |C|-coefficient polynomial by the vanishing polynomial of the input domain (n = 4 … 64),
// 2.7·10^11 additions at |C| = 2^20.  View p as rows of n coefficients: q is the exclusive suffix sum DOWN each column.  Blocks of
// RB rows: (1) per-block column sums, (2) a suffix scan over the blocks of each column, (3) every block walks its rows once more
// with its offset — 2m additions, depth RB + #blocks ≈ 2·sqrt(m/n).
__global__ void k_dbv_block_sums(const uint32_t* __restrict__ p, size_t m, size_t n, size_t rb, size_t nblocks, uint32_t* __restrict__ S) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nblocks * n) return;
    const size_t b = t / n, c = t % n;
    Fr acc = Fr::zero();
    for (size_t k = b * rb; k < (b + 1) * rb; k++) { const size_t j = k * n + c; if (j < m) acc = acc + Fr::load_ldg(p + j * 8); }
    acc.store(S + t * 8);
}
__global__ void k_dbv_block_scan(uint32_t* __restrict__ S, size_t n, size_t nblocks) {     // in place: S[b][c] ← Σ_{b' > b} S[b'][c]
    const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n) return;
    Fr run = Fr::zero();
    for (size_t b = nblocks; b-- > 0;) {
        const Fr v = Fr::load(S + (b * n + c) * 8);
        run.store(S + (b * n + c) * 8);
        run = run + v;
    }
}
__global__ void k_dbv_finish(const uint32_t* __restrict__ p, size_t m, size_t n, size_t rb, size_t nblocks, const uint32_t* __restrict__ T,
                             uint32_t* __restrict__ q, uint32_t* __restrict__ r) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nblocks * n) return;
    const size_t b = t / n, c = t % n, qlen = m > n ? m - n : 0, rlen = m < n ? m : n;
    Fr run = Fr::load(T + t * 8);                                                          // Σ of the rows below this block
    for (size_t k = (b + 1) * rb; k-- > b * rb;) {
        const size_t j = k * n + c;
        if (j >= m) continue;
        const Fr v = Fr::load_ldg(p + j * 8);
        if (j < qlen) run.store(q + j * 8);
        if (j < rlen) (run + v).store(r + j * 8);
        run = run + v;
    }
}

int poly_divide_by_vanishing_device(void* d_q, void* d_r, const void* d_p, size_t m, size_t n, cudaStream_t stream) {
    if (n == 0) return (int)cudaErrorInvalidValue;
    if (m == 0) return 0;
    const size_t qlen = m > n ? m - n : 0, rlen = m < n ? m : n, work = qlen > rlen ? qlen : rlen;
    if (!d_p || !d_r || (qlen && !d_q)) return (int)cudaErrorInvalidValue;
    const size_t rows = (m + n - 1) / n;
    if (rows <= 64) {
        k_divide_by_vanishing<<<(unsigned)((work + 255) / 256), 256, 0, stream>>>((const uint32_t*)d_p, m, n, (uint32_t*)d_q, (uint32_t*)d_r);
        count_launch();
        return (int)cudaGetLastError();
    }
    size_t rb = 1;
    while (rb * rb < rows) rb <<= 1;                                                       // ≈ sqrt(rows), a power of two
    const size_t nblocks = (rows + rb - 1) / rb, cells = nblocks * n;
    uint32_t* S = nullptr;
    cudaError_t e = pool_alloc(&S, cells * 32, stream);
    if (e != cudaSuccess) return (int)e;
    k_dbv_block_sums<<<(unsigned)((cells + 127) / 128), 128, 0, stream>>>((const uint32_t*)d_p, m, n, rb, nblocks, S);
    k_dbv_block_scan<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(S, n, nblocks);
    k_dbv_finish<<<(unsigned)((cells + 127) / 128), 128, 0, stream>>>((const uint32_t*)d_p, m, n, rb, nblocks, S, (uint32_t*)d_q, (uint32_t*)d_r);
    count_launch(3);
    int rc = (int)cudaGetLastError();
    cudaFreeAsync(S, stream);
    return rc;
}

// ---------------------------------------------------------------------------------------------------------------------
// Σ c_i z^i for many polynomials at once: a thread runs Horner over EVAL_K consecutive coefficients of its segment and shifts its
// partial by z^{first index}; the CTA adds its 256 partials in shared memory.  Segment j owns the CTAs [first, first + nctas), so
// a long polynomial spreads over many CTAs and a short one takes one; a second launch, one CTA per segment, adds its CTA sums.
// ---------------------------------------------------------------------------------------------------------------------
static constexpr int EVAL_K = 64, EVAL_THREADS = 256;
FF_DEV Fr fr_pow_u64(Fr base, uint64_t e) {
    Fr acc = Fr::one();
    while (e) { if (e & 1) acc = acc * base; base = base.sqr(); e >>= 1; }
    return acc;
}
FF_DEV Fr cta_sum(Fr mine, uint32_t* sh) {
    mine.store(sh + threadIdx.x * 8);
    __syncthreads();
    for (int s = EVAL_THREADS / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) (Fr::load(sh + threadIdx.x * 8) + Fr::load(sh + (threadIdx.x + s) * 8)).store(sh + threadIdx.x * 8);
        __syncthreads();
    }
    return Fr::load(sh);
}
struct EvalSeg {
    const uint32_t* c;
    uint64_t m, first;                                  // first: the segment's first CTA of the partial-sum launch
    uint32_t nctas, reserved;
    FrArg z;
};
__global__ void __launch_bounds__(EVAL_THREADS) k_poly_eval_partial(const EvalSeg* __restrict__ segs, uint32_t nsegs,
                                                                     uint32_t* __restrict__ partial) {
    __shared__ uint4 sh4[EVAL_THREADS * 2];
    const EvalSeg& s = segs[seg_of(segs, nsegs, blockIdx.x)];
    const uint32_t* __restrict__ c = s.c;
    const size_t m = s.m, t = (size_t)(blockIdx.x - s.first) * blockDim.x + threadIdx.x, i0 = t * EVAL_K;
    const Fr z = fr_from_arg(s.z);
    Fr acc = Fr::zero();
    if (i0 < m) {
        const size_t i1 = i0 + EVAL_K < m ? i0 + EVAL_K : m;
        for (size_t i = i1; i-- > i0;) acc = acc * z + Fr::load_ldg(c + i * 8);
        acc = acc * fr_pow_u64(z, (uint64_t)i0);
    }
    Fr sum = cta_sum(acc, reinterpret_cast<uint32_t*>(sh4));
    if (threadIdx.x == 0) sum.store(partial + (size_t)blockIdx.x * 8);
}
// CTA j adds segment j's CTA sums into out[j] (zero for an empty segment)
__global__ void __launch_bounds__(EVAL_THREADS) k_poly_eval_sum(const EvalSeg* __restrict__ segs, const uint32_t* __restrict__ partial,
                                                                 uint32_t* __restrict__ out) {
    __shared__ uint4 sh4[EVAL_THREADS * 2];
    const EvalSeg& s = segs[blockIdx.x];
    const uint32_t* in = partial + s.first * 8;
    Fr acc = Fr::zero();
    for (size_t i = threadIdx.x; i < s.nctas; i += EVAL_THREADS) acc = acc + Fr::load_ldg(in + i * 8);
    Fr sum = cta_sum(acc, reinterpret_cast<uint32_t*>(sh4));
    if (threadIdx.x == 0) sum.store(out + (size_t)blockIdx.x * 8);
}

int poly_evaluate_batch_device(void* out_mont_host, const snarkvm_b200_poly_eval_segment_t* segs, size_t count, cudaStream_t stream) {
    if (count == 0) return 0;
    if (!out_mont_host || !segs || count >= ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    std::vector<EvalSeg> table(count);
    uint64_t ctas = 0;
    for (size_t i = 0; i < count; i++) {
        const snarkvm_b200_poly_eval_segment_t& s = segs[i];
        if (s.m && !s.d_coeffs) return (int)cudaErrorInvalidValue;
        const uint64_t blocks = ((s.m + EVAL_K - 1) / EVAL_K + EVAL_THREADS - 1) / EVAL_THREADS;
        table[i] = EvalSeg{(const uint32_t*)s.d_coeffs, s.m, ctas, (uint32_t)blocks, 0, FrArg{}};
        memcpy(table[i].z.v, s.point_mont, 32);
        ctas += blocks;
    }
    if (ctas >= ((uint64_t)1 << 31)) return (int)cudaErrorInvalidValue;
    if (ctas == 0) { memset(out_mont_host, 0, count * 32); return 0; }
    // scratch: table | partial[ctas] | out[count]
    const size_t off_partial = (count * sizeof(EvalSeg) + 255) & ~(size_t)255, off_out = off_partial + ctas * 32;
    uint8_t* scratch = nullptr;
    cudaError_t e = pool_alloc(&scratch, off_out + count * 32, stream);
    if (e != cudaSuccess) return (int)e;
    const EvalSeg* d_table = (const EvalSeg*)scratch;
    uint32_t *partial = (uint32_t*)(scratch + off_partial), *out = (uint32_t*)(scratch + off_out);
    int rc = (int)cudaMemcpyAsync(scratch, table.data(), count * sizeof(EvalSeg), cudaMemcpyHostToDevice, stream);
    if (rc == 0) {
        k_poly_eval_partial<<<(unsigned)ctas, EVAL_THREADS, 0, stream>>>(d_table, (uint32_t)count, partial);
        k_poly_eval_sum<<<(unsigned)count, EVAL_THREADS, 0, stream>>>(d_table, partial, out);
        count_launch(2);
        rc = (int)cudaGetLastError();
    }
    if (rc == 0) rc = (int)cudaMemcpyAsync(out_mont_host, out, count * 32, cudaMemcpyDeviceToHost, stream);
    cudaFreeAsync(scratch, stream);
    if (rc == 0) rc = (int)cudaStreamSynchronize(stream);
    return rc;
}

int poly_evaluate_device(void* out_mont_host, const void* d_coeffs, size_t m, const void* point_mont_host, cudaStream_t stream) {
    if (!out_mont_host || !point_mont_host) return (int)cudaErrorInvalidValue;
    snarkvm_b200_poly_eval_segment_t s{d_coeffs, m, {}};
    memcpy(s.point_mont, point_mont_host, 32);
    return poly_evaluate_batch_device(out_mont_host, &s, 1, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// Quotient of p / (x − z) — the KZG witness polynomial (polycommit/kzg10/mod.rs:220-241).  q_{L−1} = p_L, q_{i−1} = p_i + z·q_i
// (L = m − 1) is a first-order linear recurrence; it is cut into chunks of LIN_K coefficients:
//   pass 1: each chunk's value at its low end assuming a zero carry-in (A_k),
//   pass 2: one CTA per polynomial chains its chunks, C_k = A_k + z^{len_k}·C_{k+1}, two levels deep, and leaves every chunk's
//           carry-in,
//   pass 3: each chunk reruns its recurrence from the true carry-in and writes q.
// 2 Fr multiplications per coefficient.  Many polynomials share the three launches: segment j owns the chunks [first, first +
// ⌈L/LIN_K⌉) of passes 1 and 3 and CTA j of pass 2.
// ---------------------------------------------------------------------------------------------------------------------
static constexpr int LIN_K = 64, LIN_THREADS = 256;
struct LinSeg {
    const uint32_t* p;
    uint32_t* q;
    uint64_t L, first;                                  // first: the segment's first chunk
    FrArg z;
};
__global__ void k_lin_local(const LinSeg* __restrict__ segs, uint32_t nsegs, uint64_t total, uint32_t* __restrict__ A) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const LinSeg& s = segs[seg_of(segs, nsegs, g)];
    const uint32_t* __restrict__ p = s.p;
    const size_t L = s.L, bot = (g - s.first) * LIN_K, top = bot + LIN_K < L ? bot + LIN_K : L;
    const Fr z = fr_from_arg(s.z);
    Fr acc = Fr::zero();
    for (size_t i = top; i-- > bot;) acc = acc * z + Fr::load_ldg(p + (i + 1) * 8);
    acc.store(A + g * 8);
}
__global__ void __launch_bounds__(LIN_THREADS) k_lin_carry(const LinSeg* __restrict__ segs, const uint32_t* __restrict__ A,
                                                            uint32_t* __restrict__ cin) {
    __shared__ uint4 shB4[LIN_THREADS * 2], shW4[LIN_THREADS * 2];
    uint32_t* shB = reinterpret_cast<uint32_t*>(shB4);
    uint32_t* shW = reinterpret_cast<uint32_t*>(shW4);
    const LinSeg& s = segs[blockIdx.x];
    const size_t L = s.L, nchunks = (L + LIN_K - 1) / LIN_K;
    A += s.first * 8;
    cin += s.first * 8;
    const Fr z = fr_from_arg(s.z);
    const Fr zK = fr_pow_u64(z, LIN_K);
    const Fr zlast = fr_pow_u64(z, (uint64_t)(L - (nchunks - 1) * LIN_K));      // the highest chunk may be short
    const size_t per = (nchunks + LIN_THREADS - 1) / LIN_THREADS;
    const size_t k0 = (size_t)threadIdx.x * per, k1 = k0 + per < nchunks ? k0 + per : nchunks;
    Fr B = Fr::zero(), W = Fr::one();
    for (size_t k = k1; k-- > k0 && k0 < nchunks;) {
        const Fr zl = (k == nchunks - 1) ? zlast : zK;
        B = Fr::load_ldg(A + k * 8) + zl * B;
        W = W * zl;
    }
    B.store(shB + threadIdx.x * 8);
    W.store(shW + threadIdx.x * 8);
    __syncthreads();
    if (threadIdx.x == 0) {                                  // D_t = value entering super-chunk t from above
        Fr D = Fr::zero();
        for (int t = LIN_THREADS - 1; t >= 0; t--) {
            Fr Bt = Fr::load(shB + t * 8), Wt = Fr::load(shW + t * 8);
            D.store(shB + t * 8);                            // carry-in of super-chunk t
            D = Bt + Wt * D;
        }
    }
    __syncthreads();
    Fr C = Fr::load(shB + threadIdx.x * 8);
    for (size_t k = k1; k-- > k0 && k0 < nchunks;) {
        C.store(cin + k * 8);
        const Fr zl = (k == nchunks - 1) ? zlast : zK;
        C = Fr::load_ldg(A + k * 8) + zl * C;
    }
}
__global__ void k_lin_final(const LinSeg* __restrict__ segs, uint32_t nsegs, uint64_t total, const uint32_t* __restrict__ cin) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const LinSeg& s = segs[seg_of(segs, nsegs, g)];
    const uint32_t* __restrict__ p = s.p;
    uint32_t* __restrict__ q = s.q;
    const size_t L = s.L, bot = (g - s.first) * LIN_K, top = bot + LIN_K < L ? bot + LIN_K : L;
    const Fr z = fr_from_arg(s.z);
    Fr acc = Fr::load_ldg(cin + g * 8);
    for (size_t i = top; i-- > bot;) { acc = acc * z + Fr::load_ldg(p + (i + 1) * 8); acc.store(q + i * 8); }
}

int poly_divide_by_linear_batch_device(const snarkvm_b200_poly_divide_segment_t* segs, size_t count, cudaStream_t stream) {
    if (count == 0) return 0;
    if (!segs || count >= ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    std::vector<LinSeg> table;                               // the segments with a non-empty quotient
    uint64_t total = 0;
    for (size_t i = 0; i < count; i++) {
        const snarkvm_b200_poly_divide_segment_t& s = segs[i];
        if (s.m <= 1) continue;
        if (!s.d_q || !s.d_p) return (int)cudaErrorInvalidValue;
        LinSeg t{(const uint32_t*)s.d_p, (uint32_t*)s.d_q, s.m - 1, total, FrArg{}};
        memcpy(t.z.v, s.point_mont, 32);
        table.push_back(t);
        total += (s.m - 1 + LIN_K - 1) / LIN_K;
    }
    if (table.empty()) return 0;
    const size_t n = table.size();
    if (total >= ((uint64_t)1 << 38)) return (int)cudaErrorInvalidValue;      // grid < 2^31 CTAs
    // scratch: table | A[total] | cin[total]
    const size_t off_a = (n * sizeof(LinSeg) + 255) & ~(size_t)255;
    uint8_t* scratch = nullptr;
    cudaError_t e = pool_alloc(&scratch, off_a + total * 64, stream);
    if (e != cudaSuccess) return (int)e;
    const LinSeg* d_table = (const LinSeg*)scratch;
    uint32_t *A = (uint32_t*)(scratch + off_a), *cin = A + total * 8;
    int rc = (int)cudaMemcpyAsync(scratch, table.data(), n * sizeof(LinSeg), cudaMemcpyHostToDevice, stream);
    if (rc == 0) {
        const unsigned grid = (unsigned)((total + 127) / 128);
        k_lin_local<<<grid, 128, 0, stream>>>(d_table, (uint32_t)n, total, A);
        k_lin_carry<<<(unsigned)n, LIN_THREADS, 0, stream>>>(d_table, A, cin);
        k_lin_final<<<grid, 128, 0, stream>>>(d_table, (uint32_t)n, total, cin);
        count_launch(3);
        rc = (int)cudaGetLastError();
    }
    cudaFreeAsync(scratch, stream);
    return rc;
}

int poly_divide_by_linear_device(void* d_q, const void* d_p, size_t m, const void* point_mont_host, cudaStream_t stream) {
    if (m <= 1) return 0;
    if (!point_mont_host) return (int)cudaErrorInvalidValue;
    snarkvm_b200_poly_divide_segment_t s{d_q, d_p, m, {}};
    memcpy(s.point_mont, point_mont_host, 32);
    return poly_divide_by_linear_batch_device(&s, 1, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// z_M = M·z for a sparse R1CS matrix in CSR form — inner_product (snark/varuna/ahp/prover/round_functions/mod.rs:169-189),
// the per-row loop the prover runs for A, B and C (:128-152).  One thread per row (rows hold a handful of entries).
// ---------------------------------------------------------------------------------------------------------------------
// Rows longer than SPMV_LONG entries (a hot variable: the constant one, or — transposed — a variable every constraint uses;
// the reference's TestCircuit puts 2^20 entries of B in ONE column) would serialise a thread: 2.6 s for M(α, ·) of a
// 2^20-constraint circuit.  They leave the thread-per-row kernel through a device-side work list — no host round trip —
// and are cut into segments of SPMV_SEG entries, one CTA per segment, then one CTA per long row adds its segments.
static constexpr uint32_t SPMV_LONG = 256, SPMV_SEG = 2048;
// Many mat-vecs in one pass (every instance of every circuit, or the three transposes of every circuit): thread g takes row
// g − first of its segment; the long rows of all segments share one work list, each entry naming its segment.
struct SpmvSeg {
    const uint32_t *row_ptr, *cols, *vals, *x;
    uint32_t* out;
    uint64_t first, nrows, nnz, nvars;
};
struct SpmvLong { uint32_t seg, row, base, nseg; };
struct SpmvItem { uint32_t seg, row, j; };
__global__ void k_sparse_matvec(const SpmvSeg* __restrict__ segs, uint32_t nsegs, uint64_t total, int* __restrict__ bad_flags,
                                uint32_t* __restrict__ ctr /* [0] long rows, [1] work items */, SpmvLong* __restrict__ long_rows,
                                SpmvItem* __restrict__ items) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const uint32_t s = seg_of(segs, nsegs, g);
    const SpmvSeg& m = segs[s];
    const size_t r = g - m.first;
    const uint32_t e0 = m.row_ptr[r], e1 = m.row_ptr[r + 1];
    if (e1 < e0 || e1 > m.nnz || (r + 1 == m.nrows && e1 != m.nnz)) { bad_flags[s] = 1; return; }   // the work lists are sized by nnz
    if (e1 - e0 > SPMV_LONG) {
        const uint32_t nseg = (e1 - e0 + SPMV_SEG - 1) / SPMV_SEG;
        const uint32_t base = atomicAdd(&ctr[1], nseg), slot = atomicAdd(&ctr[0], 1u);
        long_rows[slot] = SpmvLong{s, (uint32_t)r, base, nseg};
        for (uint32_t j = 0; j < nseg; j++) items[base + j] = SpmvItem{s, (uint32_t)r, j};
        return;
    }
    Fr acc = Fr::zero();
    for (uint32_t e = e0; e < e1; e++) {
        const uint32_t c = m.cols[e];
        if (c >= m.nvars) { bad_flags[s] = 1; continue; }   // out-of-range column: reported, never read
        acc = acc + Fr::load_ldg(m.x + (size_t)c * 8) * Fr::load_ldg(m.vals + (size_t)e * 8);
    }
    acc.store(m.out + r * 8);
}
// Σ over the 256 threads of a CTA (shared memory tree); the result is valid in thread 0
FF_DEV Fr cta_sum_fr(Fr v, uint4* sh) {
    const uint32_t t = threadIdx.x;
    sh[2 * t] = make_uint4(v.v[0], v.v[1], v.v[2], v.v[3]); sh[2 * t + 1] = make_uint4(v.v[4], v.v[5], v.v[6], v.v[7]);
    __syncthreads();
    for (uint32_t d = 128; d >= 1; d >>= 1) {
        if (t < d) {
            Fr a = Fr::load(sh + 2 * t), b = Fr::load(sh + 2 * (t + d));
            a = a + b;
            a.store(sh + 2 * t);
        }
        __syncthreads();
    }
    return Fr::load(sh);
}
__global__ void __launch_bounds__(256) k_spmv_segments(const SpmvSeg* __restrict__ segs, const uint32_t* __restrict__ ctr,
                                                       const SpmvItem* __restrict__ items, uint32_t* __restrict__ partial,
                                                       int* __restrict__ bad_flags) {
    __shared__ uint4 sh[512];
    const uint32_t nitems = ctr[1];
    for (uint32_t it = blockIdx.x; it < nitems; it += gridDim.x) {
        const SpmvItem w = items[it];
        const uint32_t *cols = segs[w.seg].cols, *vals = segs[w.seg].vals, *x = segs[w.seg].x, *row_ptr = segs[w.seg].row_ptr;
        const uint32_t nvars = (uint32_t)segs[w.seg].nvars;
        const uint32_t e0 = row_ptr[w.row] + w.j * SPMV_SEG, rend = row_ptr[w.row + 1], e1 = e0 + SPMV_SEG < rend ? e0 + SPMV_SEG : rend;
        bool bad = false;
        Fr acc = Fr::zero();
        for (uint32_t e = e0 + threadIdx.x; e < e1; e += 256) {
            const uint32_t c = cols[e];
            if (c >= nvars) { bad = true; continue; }
            acc = acc + Fr::load_ldg(x + (size_t)c * 8) * Fr::load_ldg(vals + (size_t)e * 8);
        }
        if (bad) bad_flags[w.seg] = 1;
        const Fr tot = cta_sum_fr(acc, sh);
        if (threadIdx.x == 0) tot.store(partial + (size_t)it * 8);
        __syncthreads();
    }
}
__global__ void __launch_bounds__(256) k_spmv_long_rows(const SpmvSeg* __restrict__ segs, const uint32_t* __restrict__ ctr,
                                                        const SpmvLong* __restrict__ long_rows, const uint32_t* __restrict__ partial) {
    __shared__ uint4 sh[512];
    const uint32_t nlong = ctr[0];
    for (uint32_t k = blockIdx.x; k < nlong; k += gridDim.x) {
        const SpmvLong L = long_rows[k];
        Fr acc = Fr::zero();
        for (uint32_t j = threadIdx.x; j < L.nseg; j += 256) acc = acc + Fr::load(partial + (size_t)(L.base + j) * 8);
        const Fr tot = cta_sum_fr(acc, sh);
        if (threadIdx.x == 0) tot.store(segs[L.seg].out + (size_t)L.row * 8);
        __syncthreads();
    }
}

static int seg_finish(int rc, uint8_t* scratch, const int* bad, size_t count, int64_t* bad_segment, cudaStream_t stream);

int sparse_matvec_batch_device(const snarkvm_b200_spmv_segment_t* segs, size_t count, int64_t* bad_segment, cudaStream_t stream) {
    if (bad_segment) *bad_segment = -1;
    if (count == 0) return 0;
    if (!segs || count >= ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    std::vector<SpmvSeg> table;
    std::vector<size_t> index;                                    // table entry → segment (segments without rows are left out)
    uint64_t total = 0;
    size_t max_long = 0, max_items = 0;
    for (size_t i = 0; i < count; i++) {
        const snarkvm_b200_spmv_segment_t& s = segs[i];
        if (s.nrows == 0) continue;
        if (!s.d_out || !s.d_row_ptr || !s.d_x || (s.nnz && (!s.d_cols || !s.d_vals))) return (int)cudaErrorInvalidValue;
        if (s.nrows >= ((uint64_t)1 << 32) || s.nnz >= ((uint64_t)1 << 32) || s.nvars >= ((uint64_t)1 << 32)) return (int)cudaErrorInvalidValue;
        table.push_back(SpmvSeg{(const uint32_t*)s.d_row_ptr, (const uint32_t*)s.d_cols, (const uint32_t*)s.d_vals, (const uint32_t*)s.d_x,
                                (uint32_t*)s.d_out, total, s.nrows, s.nnz, s.nvars});
        index.push_back(i);
        total += s.nrows;
        const size_t ml = (size_t)s.nnz / SPMV_LONG + 1;
        max_long += ml;
        max_items += (size_t)s.nnz / SPMV_SEG + ml + 1;
    }
    if (table.empty()) return 0;
    // the segment and long-row kernels walk their work lists grid-stride: four CTAs per SM and one CTA per SM
    int dev = 0, sms = 0;
    int rc = (int)cudaGetDevice(&dev);
    if (rc == 0) rc = (int)cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (rc != 0) return rc;
    const size_t n = table.size(), nflags = (n * sizeof(int) + 255) & ~(size_t)255;
    // scratch: bad flags | counters | segment table | long rows | work items | partial sums
    const size_t off_ctr = nflags, off_table = off_ctr + 256, off_long = off_table + ((n * sizeof(SpmvSeg) + 255) & ~(size_t)255),
                 off_items = off_long + ((max_long * sizeof(SpmvLong) + 255) & ~(size_t)255),
                 off_partial = off_items + ((max_items * sizeof(SpmvItem) + 255) & ~(size_t)255), bytes = off_partial + max_items * 32;
    uint8_t* scratch = nullptr;
    cudaError_t e = pool_alloc(&scratch, bytes, stream);
    if (e != cudaSuccess) return (int)e;
    int* bad = (int*)scratch;
    uint32_t* ctr = (uint32_t*)(scratch + off_ctr);
    SpmvSeg* d_table = (SpmvSeg*)(scratch + off_table);
    rc = (int)cudaMemsetAsync(scratch, 0, off_table, stream);     // bad flags and counters
    if (rc == 0) rc = (int)cudaMemcpyAsync(d_table, table.data(), n * sizeof(SpmvSeg), cudaMemcpyHostToDevice, stream);
    if (rc == 0) {
        k_sparse_matvec<<<(unsigned)((total + 127) / 128), 128, 0, stream>>>(d_table, (uint32_t)n, total, bad, ctr, (SpmvLong*)(scratch + off_long),
                                                                           (SpmvItem*)(scratch + off_items));
        k_spmv_segments<<<4 * sms, 256, 0, stream>>>(d_table, ctr, (const SpmvItem*)(scratch + off_items), (uint32_t*)(scratch + off_partial), bad);
        k_spmv_long_rows<<<sms, 256, 0, stream>>>(d_table, ctr, (const SpmvLong*)(scratch + off_long), (const uint32_t*)(scratch + off_partial));
        count_launch(3);
        rc = (int)cudaGetLastError();
    }
    int64_t bad_entry = -1;
    rc = seg_finish(rc, scratch, bad, n, &bad_entry, stream);
    if (bad_segment && bad_entry >= 0) *bad_segment = (int64_t)index[(size_t)bad_entry];
    return rc;
}

int sparse_matvec_device(void* d_out, const void* d_row_ptr, const void* d_cols, const void* d_vals, size_t nrows, const void* d_x,
                         size_t nvars, cudaStream_t stream) {
    if (nrows == 0) return 0;
    if (!d_out || !d_row_ptr || !d_x) return (int)cudaErrorInvalidValue;
    // the number of entries sizes the work lists of the long rows
    uint32_t nnz = 0;
    int rc = (int)cudaMemcpyAsync(&nnz, (const uint32_t*)d_row_ptr + nrows, 4, cudaMemcpyDeviceToHost, stream);
    if (rc == 0) rc = (int)cudaStreamSynchronize(stream);
    if (rc != 0) return rc;
    const snarkvm_b200_spmv_segment_t s{d_row_ptr, d_cols, d_vals, nrows, nnz, d_x, nvars, d_out};
    return sparse_matvec_batch_device(&s, 1, nullptr, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// Elementwise Fr arithmetic on HBM vectors (the `cfg_iter_mut!(..).zip(..)` loops between transforms, e.g.
// polycommit/kzg10/mod.rs:292-297, fft/evaluations.rs:49-74) and the domain's elements (fft/domain.rs:307-309, 980-988).
// op: 0 = a + b, 1 = a − b, 2 = a · b.  out may alias a or b.
// ---------------------------------------------------------------------------------------------------------------------
FF_DEV Fr fr_apply(int op, const Fr& a, const Fr& b) { return op == 0 ? a + b : op == 1 ? a - b : a * b; }
__global__ void k_fr_vec_op(uint32_t* out, const uint32_t* a, const uint32_t* b, size_t n, int op) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) fr_apply(op, Fr::load(a + i * 8), Fr::load(b + i * 8)).store(out + i * 8);
}
__global__ void k_fr_vec_scalar_op(uint32_t* out, const uint32_t* a, FrArg s_arg, size_t n, int op) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) fr_apply(op, Fr::load(a + i * 8), fr_from_arg(s_arg)).store(out + i * 8);
}
// ω_n^i (i < n = 2^lg) from the NTT's table ω_N^j (j < N/2): ω_n^i = ω_N^{i·N/n}, and ω^{i} = −ω^{i − n/2} in the upper half
FF_DEV Fr domain_element(size_t i, int lg, const uint32_t* __restrict__ tw, int lgN) {
    if (lg == 0) return Fr::one();
    const size_t half = (size_t)1 << (lg - 1), j = i < half ? i : i - half;
    const Fr w = Fr::load_ldg(tw + (j << (lgN - lg)) * 8);
    return i < half ? w : w.neg();
}
__global__ void k_domain_elements(uint32_t* __restrict__ out, int lg, const uint32_t* __restrict__ tw, int lgN) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, n = (size_t)1 << lg;
    if (i >= n) return;
    domain_element(i, lg, tw, lgN).store(out + i * 8);
}

int fr_vec_op_device(void* d_out, const void* d_a, const void* d_b, size_t n, int op, cudaStream_t stream) {
    if (n == 0) return 0;
    if (!d_out || !d_a || !d_b || op < 0 || op > 2) return (int)cudaErrorInvalidValue;
    k_fr_vec_op<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((uint32_t*)d_out, (const uint32_t*)d_a, (const uint32_t*)d_b, n, op);
    count_launch();
    return (int)cudaGetLastError();
}
int fr_vec_scalar_op_device(void* d_out, const void* d_a, const void* scalar_mont_host, size_t n, int op, cudaStream_t stream) {
    if (n == 0) return 0;
    if (!d_out || !d_a || !scalar_mont_host || op < 0 || op > 2) return (int)cudaErrorInvalidValue;
    FrArg sc;
    memcpy(sc.v, scalar_mont_host, 32);
    k_fr_vec_scalar_op<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((uint32_t*)d_out, (const uint32_t*)d_a, sc, n, op);
    count_launch();
    return (int)cudaGetLastError();
}
int domain_elements_device(void* d_out, uint32_t lg, cudaStream_t stream) {
    if (!d_out || lg > 30) return (int)cudaErrorInvalidValue;
    const void* tw = nullptr;
    int lgN = 0, rc = 0;
    if (lg > 0 && (rc = ntt_get_twiddles((int)lg, &tw, &lgN)) != 0) return rc;
    const size_t n = (size_t)1 << lg;
    k_domain_elements<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((uint32_t*)d_out, (int)lg, (const uint32_t*)tw, lgN);
    count_launch();
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// The Varuna indexer over a CSR matrix (row_ptr u32 [nrows + 1], cols u32 [nnz], vals Montgomery Fr [nnz]):
//   matrix_evals (snark/varuna/ahp/matrices.rs:138-195) — entry e gets row = ω_R^{row(e)}, col = ω_C^{reindex(col(e))} and
//     row_col_val = val·row·col; entries nnz … |K| − 1 get the padding (1, 1, 0);
//   transpose (matrices.rs:249-270) over the variable domain — a counting sort: histogram of the reindexed columns, exclusive
//     scan, scatter.  Entries land in a transposed row in atomic order; the sums sparse_matvec takes over them are exact.
// row(e) is the last row whose first entry is ≤ e (a binary search of row_ptr, so empty rows are skipped); reindex is
// EvaluationDomain::reindex_by_subdomain (fft/domain.rs:322-344) of the variable domain C by the input domain I, |C| > |I|.
// A column ≥ nvars, or a row_ptr that does not run from 0 to nnz, raises the bad flag; such an entry is never indexed by.
// ---------------------------------------------------------------------------------------------------------------------
struct CsrArgs {
    const uint32_t* row_ptr; const uint32_t* cols; const uint32_t* vals;
    uint32_t nrows, nnz, nvars, input_size, period;    // period = |C| / |I| ≥ 2
};
FF_DEV uint32_t csr_row_of(const uint32_t* __restrict__ row_ptr, uint32_t nrows, uint32_t e) {
    uint32_t lo = 0, hi = nrows;                        // row_ptr[lo] ≤ e < row_ptr[hi]; lo < nrows always
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (__ldg(row_ptr + mid) <= e) lo = mid; else hi = mid;
    }
    return lo;
}
FF_DEV uint32_t reindex_by_subdomain(uint32_t index, uint32_t input_size, uint32_t period) {
    if (index < input_size) return index * period;
    const uint32_t i = index - input_size;
    return i + i / (period - 1) + 1;
}
FF_DEV void csr_check_bounds(const CsrArgs& m, int* bad) {
    if (blockIdx.x == 0 && threadIdx.x == 0 && (m.row_ptr[0] != 0 || m.row_ptr[m.nrows] != m.nnz)) *bad = 1;
}

struct EvalsSeg {
    CsrArgs m;
    uint32_t *row_out, *col_out, *rcv_out;
    uint64_t first, K;
    int lgR, lgC;
};
// one launch over every matrix's K: entry e of segment j; bad[j] is the segment's flag
__global__ void k_matrix_evals(const EvalsSeg* __restrict__ segs, uint32_t nsegs, uint64_t total, const uint32_t* __restrict__ tw, int lgN,
                               int* __restrict__ bad_flags) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const uint32_t j = seg_of(segs, nsegs, g);
    const EvalsSeg& s = segs[j];
    const CsrArgs m = s.m;
    const size_t e = g - s.first;
    int* bad = bad_flags + j;
    uint32_t *row_out = s.row_out, *col_out = s.col_out, *rcv_out = s.rcv_out;
    const int lgR = s.lgR, lgC = s.lgC;
    if (e == 0 && (m.row_ptr[0] != 0 || m.row_ptr[m.nrows] != m.nnz)) *bad = 1;
    if (e >= m.nnz) {                                                       // padding (matrices.rs:174-181)
        Fr::one().store(row_out + e * 8); Fr::one().store(col_out + e * 8); Fr::zero().store(rcv_out + e * 8);
        return;
    }
    const uint32_t c = __ldg(m.cols + e);
    if (c >= m.nvars) {
        *bad = 1;
        Fr::zero().store(row_out + e * 8); Fr::zero().store(col_out + e * 8); Fr::zero().store(rcv_out + e * 8);
        return;
    }
    const Fr r = domain_element(csr_row_of(m.row_ptr, m.nrows, (uint32_t)e), lgR, tw, lgN);
    const Fr cc = domain_element(reindex_by_subdomain(c, m.input_size, m.period), lgC, tw, lgN);
    r.store(row_out + e * 8);
    cc.store(col_out + e * 8);
    (Fr::load_ldg(m.vals + e * 8) * (r * cc)).store(rcv_out + e * 8);
}

__global__ void k_csr_col_histogram(CsrArgs m, uint32_t* __restrict__ counts, int* __restrict__ bad) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    csr_check_bounds(m, bad);
    if (e >= m.nnz) return;
    const uint32_t c = __ldg(m.cols + e);
    if (c >= m.nvars) { *bad = 1; return; }
    atomicAdd(counts + reindex_by_subdomain(c, m.input_size, m.period), 1u);
}

// exclusive scan of n u32 counts into out[0 … n] (out[n] = total): SCAN_TILE per CTA, then one CTA scans the tile sums,
// then every tile adds its offset
static constexpr int SCAN_THREADS = 256, SCAN_PER = 4, SCAN_TILE = SCAN_THREADS * SCAN_PER;
FF_DEV uint32_t cta_exclusive_scan(uint32_t v, uint32_t* sh, uint32_t* total) {
    const uint32_t t = threadIdx.x;
    sh[t] = v;
    __syncthreads();
    for (uint32_t d = 1; d < SCAN_THREADS; d <<= 1) {                      // Hillis–Steele inclusive scan
        const uint32_t add = t >= d ? sh[t - d] : 0;
        __syncthreads();
        sh[t] += add;
        __syncthreads();
    }
    const uint32_t incl = sh[t];
    *total = sh[SCAN_THREADS - 1];
    __syncthreads();
    return incl - v;
}
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_tiles(const uint32_t* __restrict__ in, size_t n, uint32_t* __restrict__ out,
                                                             uint32_t* __restrict__ tile_sums) {
    __shared__ uint32_t sh[SCAN_THREADS];
    const size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_PER;
    uint32_t v[SCAN_PER], run = 0;
#pragma unroll
    for (int k = 0; k < SCAN_PER; k++) { v[k] = base + k < n ? in[base + k] : 0; run += v[k]; }
    uint32_t total;
    uint32_t pre = cta_exclusive_scan(run, sh, &total);
#pragma unroll
    for (int k = 0; k < SCAN_PER; k++) { if (base + k < n) out[base + k] = pre; pre += v[k]; }
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_tile_sums(uint32_t* __restrict__ tile_sums, size_t ntiles, uint32_t* __restrict__ out_total) {
    __shared__ uint32_t sh[SCAN_THREADS];
    uint32_t carry = 0;
    for (size_t b = 0; b < ntiles; b += SCAN_THREADS) {                     // in place, exclusive
        const size_t i = b + threadIdx.x;
        const uint32_t v = i < ntiles ? tile_sums[i] : 0;
        uint32_t total;
        const uint32_t pre = cta_exclusive_scan(v, sh, &total);
        if (i < ntiles) tile_sums[i] = carry + pre;
        carry += total;
    }
    if (threadIdx.x == 0) *out_total = carry;
}
__global__ void k_scan_add(uint32_t* __restrict__ out, size_t n, const uint32_t* __restrict__ tile_sums) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] += tile_sums[i / SCAN_TILE];
}

// cursor[t] starts at the transposed row's first slot; every valid entry takes the next one
__global__ void k_csr_transpose_scatter(CsrArgs m, uint32_t* __restrict__ cursor, uint32_t* __restrict__ t_cols,
                                        uint32_t* __restrict__ t_vals) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m.nnz) return;
    const uint32_t c = __ldg(m.cols + e);
    if (c >= m.nvars) return;
    const uint32_t slot = atomicAdd(cursor + reindex_by_subdomain(c, m.input_size, m.period), 1u);   // < its row's end ≤ nnz
    t_cols[slot] = csr_row_of(m.row_ptr, m.nrows, (uint32_t)e);
    const uint4* src = reinterpret_cast<const uint4*>(m.vals + e * 8);
    uint4* dst = reinterpret_cast<uint4*>(t_vals + (size_t)slot * 8);
    dst[0] = __ldg(src); dst[1] = __ldg(src + 1);
}

// the shared validation of both entry points: everything the kernels index by must fit in u32 and in its domain
static int csr_index_args(CsrArgs* m, const void* d_row_ptr, size_t nrows, const void* d_cols, const void* d_vals, size_t nnz,
                          size_t nvars, size_t input_size, uint32_t lg_variable) {
    if (!d_row_ptr || (nnz && (!d_cols || !d_vals)) || lg_variable > 31) return (int)cudaErrorInvalidValue;
    const size_t V = (size_t)1 << lg_variable;
    if (input_size == 0 || (input_size & (input_size - 1)) || V <= input_size) return (int)cudaErrorInvalidValue;   // domain.rs:327-329
    if (nvars > V || nrows >= ((size_t)1 << 32) || nnz >= ((size_t)1 << 32)) return (int)cudaErrorInvalidValue;
    *m = CsrArgs{(const uint32_t*)d_row_ptr, (const uint32_t*)d_cols, (const uint32_t*)d_vals, (uint32_t)nrows, (uint32_t)nnz,
                 (uint32_t)nvars, (uint32_t)input_size, (uint32_t)(V / input_size)};
    return 0;
}
// reads the bad flag back (synchronising the stream) and frees the scratch
static int csr_finish(int rc, uint8_t* scratch, const int* bad, cudaStream_t stream) {
    int h_bad = 0;
    if (rc == 0) rc = (int)cudaMemcpyAsync(&h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, stream);
    cudaFreeAsync(scratch, stream);
    if (rc == 0) rc = (int)cudaStreamSynchronize(stream);
    if (rc == 0 && h_bad) rc = (int)cudaErrorInvalidValue;
    return rc;
}

// Scratch of a segmented call: [bad flags, one int per segment | the segment table]; the table is copied up and the flags cleared.
template <class Seg> static int seg_scratch(const std::vector<Seg>& table, uint8_t** scratch, int** bad, Seg** d_table, cudaStream_t stream) {
    const size_t nflags = (table.size() * sizeof(int) + 255) & ~(size_t)255;
    cudaError_t e = pool_alloc(scratch, nflags + table.size() * sizeof(Seg), stream);
    if (e != cudaSuccess) return (int)e;
    *bad = (int*)*scratch;
    *d_table = (Seg*)(*scratch + nflags);
    int rc = (int)cudaMemsetAsync(*scratch, 0, nflags, stream);
    if (rc == 0) rc = (int)cudaMemcpyAsync(*d_table, table.data(), table.size() * sizeof(Seg), cudaMemcpyHostToDevice, stream);
    return rc;
}
// reads every segment's bad flag back (one synchronisation), frees the scratch and names the first bad segment
static int seg_finish(int rc, uint8_t* scratch, const int* bad, size_t count, int64_t* bad_segment, cudaStream_t stream) {
    std::vector<int> h_bad(count, 0);
    if (rc == 0) rc = (int)cudaMemcpyAsync(h_bad.data(), bad, count * sizeof(int), cudaMemcpyDeviceToHost, stream);
    cudaFreeAsync(scratch, stream);
    if (rc == 0) rc = (int)cudaStreamSynchronize(stream);
    if (rc != 0) return rc;
    for (size_t i = 0; i < count; i++) {
        if (h_bad[i]) {
            if (bad_segment) *bad_segment = (int64_t)i;
            return (int)cudaErrorInvalidValue;
        }
    }
    return 0;
}

int varuna_matrix_evals_batch_device(const snarkvm_b200_csr_segment_t* segs, size_t count, int64_t* bad_segment, cudaStream_t stream) {
    if (bad_segment) *bad_segment = -1;
    if (count == 0) return 0;
    if (!segs || count >= ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    std::vector<EvalsSeg> table(count);
    uint64_t total = 0;
    uint32_t lg_max = 0;
    for (size_t i = 0; i < count; i++) {
        const snarkvm_b200_csr_segment_t& s = segs[i];
        EvalsSeg& t = table[i];
        int rc = csr_index_args(&t.m, s.d_row_ptr, s.nrows, s.d_cols, s.d_vals, s.nnz, s.nvars, s.input_size, s.lg_variable);
        if (rc != 0) return rc;
        if (!s.d_out[0] || !s.d_out[1] || !s.d_out[2] || s.lg_constraint > 31 || s.lg_non_zero > 31) return (int)cudaErrorInvalidValue;
        if (s.nrows > ((uint64_t)1 << s.lg_constraint) || s.nnz > ((uint64_t)1 << s.lg_non_zero)) return (int)cudaErrorInvalidValue;
        t.row_out = (uint32_t*)s.d_out[0]; t.col_out = (uint32_t*)s.d_out[1]; t.rcv_out = (uint32_t*)s.d_out[2];
        t.first = total;
        t.K = (uint64_t)1 << s.lg_non_zero;
        t.lgR = (int)s.lg_constraint; t.lgC = (int)s.lg_variable;
        total += t.K;
        lg_max = std::max(lg_max, std::max(s.lg_constraint, s.lg_variable));
    }
    const void* tw = nullptr;
    int lgN = 0, rc = ntt_get_twiddles((int)lg_max, &tw, &lgN);
    if (rc != 0) return rc;
    uint8_t* scratch = nullptr;
    int* bad = nullptr;
    EvalsSeg* d_table = nullptr;
    rc = seg_scratch(table, &scratch, &bad, &d_table, stream);
    if (rc != 0 && !scratch) return rc;
    if (rc == 0) {
        k_matrix_evals<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(d_table, (uint32_t)count, total, (const uint32_t*)tw, lgN, bad);
        count_launch();
        rc = (int)cudaGetLastError();
    }
    return seg_finish(rc, scratch, bad, count, bad_segment, stream);
}

int varuna_matrix_evals_device(void* d_row, void* d_col, void* d_row_col_val, const void* d_row_ptr, size_t nrows, const void* d_cols,
                               const void* d_vals, size_t nnz, size_t nvars, size_t input_size, uint32_t lg_constraint,
                               uint32_t lg_variable, uint32_t lg_non_zero, cudaStream_t stream) {
    const snarkvm_b200_csr_segment_t s{d_row_ptr, d_cols, d_vals, nrows, nnz, nvars, input_size, lg_constraint, lg_variable, lg_non_zero, 0,
                                       {d_row, d_col, d_row_col_val}};
    return varuna_matrix_evals_batch_device(&s, 1, nullptr, stream);
}

int csr_transpose_device(void* d_t_row_ptr, void* d_t_cols, void* d_t_vals, const void* d_row_ptr, size_t nrows, const void* d_cols,
                         const void* d_vals, size_t nnz, size_t nvars, size_t input_size, uint32_t lg_variable, cudaStream_t stream) {
    CsrArgs m;
    int rc = csr_index_args(&m, d_row_ptr, nrows, d_cols, d_vals, nnz, nvars, input_size, lg_variable);
    if (rc != 0) return rc;
    if (!d_t_row_ptr || (nnz && (!d_t_cols || !d_t_vals))) return (int)cudaErrorInvalidValue;
    const size_t V = (size_t)1 << lg_variable, ntiles = (V + SCAN_TILE - 1) / SCAN_TILE;
    // scratch: [0] bad flag | counts[V] | cursor[V] | tile sums[ntiles]
    const size_t off_counts = 256, off_cursor = off_counts + ((V * 4 + 255) & ~(size_t)255),
                 off_tiles = off_cursor + ((V * 4 + 255) & ~(size_t)255), total = off_tiles + ntiles * 4;
    uint8_t* scratch = nullptr;
    cudaError_t e = pool_alloc(&scratch, total, stream);
    if (e != cudaSuccess) return (int)e;
    int* bad = (int*)scratch;
    uint32_t *counts = (uint32_t*)(scratch + off_counts), *cursor = (uint32_t*)(scratch + off_cursor), *tiles = (uint32_t*)(scratch + off_tiles);
    uint32_t* t_row_ptr = (uint32_t*)d_t_row_ptr;
    rc = (int)cudaMemsetAsync(scratch, 0, off_cursor, stream);              // bad flag and counts
    if (rc == 0) {
        const unsigned egrid = (unsigned)((nnz + 255) / 256 > 0 ? (nnz + 255) / 256 : 1);
        k_csr_col_histogram<<<egrid, 256, 0, stream>>>(m, counts, bad);
        k_scan_tiles<<<(unsigned)ntiles, SCAN_THREADS, 0, stream>>>(counts, V, t_row_ptr, tiles);
        k_scan_tile_sums<<<1, SCAN_THREADS, 0, stream>>>(tiles, ntiles, t_row_ptr + V);
        k_scan_add<<<(unsigned)((V + 255) / 256), 256, 0, stream>>>(t_row_ptr, V, tiles);
        count_launch(4);
        rc = (int)cudaMemcpyAsync(cursor, t_row_ptr, V * 4, cudaMemcpyDeviceToDevice, stream);
        if (rc == 0 && nnz) {
            k_csr_transpose_scatter<<<egrid, 256, 0, stream>>>(m, cursor, (uint32_t*)d_t_cols, (uint32_t*)d_t_vals);
            count_launch();
        }
        if (rc == 0) rc = (int)cudaGetLastError();
    }
    return csr_finish(rc, scratch, bad, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// The circuit id's byte stream (Circuit::hash, snark/varuna/ahp/indexer/circuit.rs:109-121): a Matrix = Vec<Vec<(Fr, usize)>>
// through serialize_uncompressed (utilities/src/serialize/impls.rs: u64 LE length prefixes, usize as u64 LE; Fr as its 32 LE
// canonical bytes with empty flags, fields/src/macros.rs:190-245):
//     [u64 nrows] then, per row r, [u64 len_r][len_r × (32 B value, u64 column)]
// Row r's header sits at 8 + 8·r + 40·row_ptr[r] and entry e of row r at 16 + 8·r + 40·e, so every thread knows its address: one
// thread per entry (Montgomery → canonical fused in) and one per row header.  A row_ptr that is not non-decreasing from 0 to nnz
// raises the bad flag; its row header is then not written, and no thread writes outside the 8 + 8·nrows + 40·nnz bytes.
// ---------------------------------------------------------------------------------------------------------------------
struct SerializeSeg {
    CsrArgs m;
    uint8_t* out;
    uint64_t first;                                     // nnz + nrows + 1 threads per segment
};
__global__ void k_csr_serialize(const SerializeSeg* __restrict__ segs, uint32_t nsegs, uint64_t total, int* __restrict__ bad_flags) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const uint32_t j = seg_of(segs, nsegs, g);
    const CsrArgs m = segs[j].m;
    uint8_t* __restrict__ out = segs[j].out;
    int* bad = bad_flags + j;
    const size_t t = g - segs[j].first;
    if (t == 0 && (m.row_ptr[0] != 0 || m.row_ptr[m.nrows] != m.nnz)) *bad = 1;
    if (t < m.nnz) {
        const uint32_t e = (uint32_t)t, r = csr_row_of(m.row_ptr, m.nrows, e);
        uint64_t* dst = reinterpret_cast<uint64_t*>(out + 16 + 8 * (size_t)r + 40 * (size_t)e);
        const Fr v = Fr::load_ldg(m.vals + (size_t)e * 8).from_mont();
#pragma unroll
        for (int i = 0; i < 4; i++) dst[i] = (uint64_t)v.v[2 * i] | (uint64_t)v.v[2 * i + 1] << 32;
        dst[4] = __ldg(m.cols + e);
    } else if (t < (size_t)m.nnz + m.nrows) {
        const uint32_t r = (uint32_t)(t - m.nnz), e0 = __ldg(m.row_ptr + r), e1 = __ldg(m.row_ptr + r + 1);
        if (e0 > e1 || e1 > m.nnz) { *bad = 1; return; }
        *reinterpret_cast<uint64_t*>(out + 8 + 8 * (size_t)r + 40 * (size_t)e0) = e1 - e0;
    } else if (t == (size_t)m.nnz + m.nrows) {
        *reinterpret_cast<uint64_t*>(out) = m.nrows;
    }
}

int csr_serialize_batch_device(const snarkvm_b200_csr_segment_t* segs, size_t count, int64_t* bad_segment, cudaStream_t stream) {
    if (bad_segment) *bad_segment = -1;
    if (count == 0) return 0;
    if (!segs || count >= ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    std::vector<SerializeSeg> table(count);
    uint64_t total = 0;
    for (size_t i = 0; i < count; i++) {
        const snarkvm_b200_csr_segment_t& s = segs[i];
        if (!s.d_out[0] || !s.d_row_ptr || (s.nnz && (!s.d_cols || !s.d_vals))) return (int)cudaErrorInvalidValue;
        if (s.nrows >= ((uint64_t)1 << 32) || s.nnz >= ((uint64_t)1 << 32)) return (int)cudaErrorInvalidValue;
        if ((s.nnz && !s.nrows) || ((uintptr_t)s.d_out[0] & 7)) return (int)cudaErrorInvalidValue;
        table[i].m = CsrArgs{(const uint32_t*)s.d_row_ptr, (const uint32_t*)s.d_cols, (const uint32_t*)s.d_vals, (uint32_t)s.nrows,
                             (uint32_t)s.nnz, 0, 0, 0};
        table[i].out = (uint8_t*)s.d_out[0];
        table[i].first = total;
        total += s.nnz + s.nrows + 1;
    }
    uint8_t* scratch = nullptr;
    int* bad = nullptr;
    SerializeSeg* d_table = nullptr;
    int rc = seg_scratch(table, &scratch, &bad, &d_table, stream);
    if (rc != 0 && !scratch) return rc;
    if (rc == 0) {
        k_csr_serialize<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(d_table, (uint32_t)count, total, bad);
        count_launch();
        rc = (int)cudaGetLastError();
    }
    return seg_finish(rc, scratch, bad, count, bad_segment, stream);
}

int csr_serialize_device(void* d_out, size_t out_bytes, const void* d_row_ptr, size_t nrows, const void* d_cols, const void* d_vals, size_t nnz,
                         cudaStream_t stream) {
    if (nrows >= ((size_t)1 << 32) || nnz >= ((size_t)1 << 32) || out_bytes != 8 + 8 * nrows + 40 * nnz) return (int)cudaErrorInvalidValue;
    const snarkvm_b200_csr_segment_t s{d_row_ptr, d_cols, d_vals, nrows, nnz, 0, 0, 0, 0, 0, 0, {d_out, nullptr, nullptr}};
    return csr_serialize_batch_device(&s, 1, nullptr, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// out = Σ_j c_j·p_j over polynomials of different lengths in one pass: each output coefficient is read-modified once instead of
// once per term (the poly_axpy loop).  A term is a view (pointer, length) placed at an offset of its output, optionally repeated
// `reps` times `period` apart: the selector sums of the batched Varuna prover (a quotient by v_n of a degree < 2n product is its
// upper half; a remainder times v_t / v_s is t/s copies of it, s apart) are such terms.  A term whose coefficient is one adds
// p_j without the product; zero coefficients and empty terms are dropped on the host.  Field sums are exact, so the result is the
// sequence of additions' bit for bit.
// Segmented: every output of a call in one launch; thread g writes coefficient g − first of its output, looping over that output's
// terms in the term table.
struct LincombTerm {
    const uint32_t* p;
    uint64_t len, offset, period, reps;
    FrArg c;
};
struct LincombOut {
    uint32_t* out;
    uint64_t n, first, t0, nterms;
};
__global__ void k_fr_lincomb(const LincombOut* __restrict__ outs, uint32_t nouts, uint64_t total, const LincombTerm* __restrict__ terms) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const LincombOut& a = outs[seg_of(outs, nouts, g)];
    const uint64_t i = g - a.first;
    Fr acc = Fr::zero();
    for (uint64_t j = a.t0; j < a.t0 + a.nterms; j++) {
        const LincombTerm& t = terms[j];
        if (i < t.offset) continue;
        uint64_t u = i - t.offset;
        if (t.reps > 1) {
            if (u >= t.period * t.reps) continue;
            u %= t.period;
        }
        if (u >= t.len) continue;
        const Fr x = Fr::load_ldg(t.p + u * 8), c = fr_from_arg(t.c);
        acc = acc + (c == Fr::one() ? x : c * x);
    }
    acc.store(a.out + i * 8);
}

int fr_lincomb_terms_device(const snarkvm_b200_lincomb_output_t* outs, size_t nouts, const snarkvm_b200_lincomb_term_t* terms, size_t nterms,
                            cudaStream_t stream) {
    if (nouts == 0) return 0;
    if (!outs || (nterms && !terms) || nouts >= ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    std::vector<LincombOut> table;
    std::vector<LincombTerm> kept;
    uint64_t total = 0;
    for (size_t i = 0; i < nouts; i++) {
        const snarkvm_b200_lincomb_output_t& o = outs[i];
        if ((o.n && !o.d_out) || o.first_term > nterms || o.nterms > nterms - o.first_term) return (int)cudaErrorInvalidValue;
        LincombOut a{(uint32_t*)o.d_out, o.n, total, kept.size(), 0};
        for (uint64_t j = o.first_term; j < o.first_term + o.nterms; j++) {
            const snarkvm_b200_lincomb_term_t& s = terms[j];
            if (s.len && !s.d_poly) return (int)cudaErrorInvalidValue;
            if (s.reps > 1 && s.period < s.len) return (int)cudaErrorInvalidValue;
            const uint64_t reps = s.reps ? s.reps : 1, step = reps > 1 ? s.period : 0;
            if (s.len && (s.offset > o.n || s.len > o.n || (reps - 1) > (o.n / (step ? step : 1)) ||
                          s.offset + (reps - 1) * step + s.len > o.n)) return (int)cudaErrorInvalidValue;   // every copy ends inside the output
            LincombTerm t{(const uint32_t*)s.d_poly, s.len, s.offset, reps > 1 ? s.period : s.len, reps, FrArg{}};
            memcpy(t.c.v, s.coeff_mont, 32);
            bool zero = true;
            for (int k = 0; k < 8; k++) zero &= t.c.v[k] == 0;
            if (s.len == 0 || s.reps == 0 || zero) continue;                         // zero coefficients and empty terms are dropped
            kept.push_back(t);
            a.nterms++;
        }
        if (o.n == 0) { kept.resize(a.t0); continue; }
        table.push_back(a);
        total += o.n;
    }
    if (total == 0) return 0;
    const size_t off_terms = (table.size() * sizeof(LincombOut) + 255) & ~(size_t)255, bytes = off_terms + kept.size() * sizeof(LincombTerm);
    uint8_t* scratch = nullptr;
    cudaError_t e = pool_alloc(&scratch, bytes, stream);
    if (e != cudaSuccess) return (int)e;
    int rc = (int)cudaMemcpyAsync(scratch, table.data(), table.size() * sizeof(LincombOut), cudaMemcpyHostToDevice, stream);
    if (rc == 0 && !kept.empty())
        rc = (int)cudaMemcpyAsync(scratch + off_terms, kept.data(), kept.size() * sizeof(LincombTerm), cudaMemcpyHostToDevice, stream);
    if (rc == 0) {
        k_fr_lincomb<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>((const LincombOut*)scratch, (uint32_t)table.size(), total,
                                                                          (const LincombTerm*)(scratch + off_terms));
        count_launch();
        rc = (int)cudaGetLastError();
    }
    cudaFreeAsync(scratch, stream);
    return rc;
}

// The capped segment form (at most 12 terms per output, all at offset 0) as a call of the same kernel.
static constexpr int LINCOMB_MAX = 12;
int fr_lincomb_batch_device(const snarkvm_b200_lincomb_segment_t* segs, size_t count, cudaStream_t stream) {
    if (count == 0) return 0;
    if (!segs || count >= ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    std::vector<snarkvm_b200_lincomb_output_t> outs(count);
    std::vector<snarkvm_b200_lincomb_term_t> terms;
    for (size_t i = 0; i < count; i++) {
        const snarkvm_b200_lincomb_segment_t& s = segs[i];
        if (s.nterms > LINCOMB_MAX) return (int)cudaErrorInvalidValue;
        outs[i] = snarkvm_b200_lincomb_output_t{s.d_out, s.n, terms.size(), s.nterms};
        for (uint32_t j = 0; j < s.nterms; j++) {
            snarkvm_b200_lincomb_term_t t{s.d_polys[j], s.lens[j], 0, 0, 1, {}};
            memcpy(t.coeff_mont, s.coeffs_mont[j], 32);
            terms.push_back(t);
        }
    }
    return fr_lincomb_terms_device(outs.data(), count, terms.data(), terms.size(), stream);
}

int fr_lincomb_device(void* d_out, size_t n, const void* const* d_polys, const size_t* lens, const void* coeffs_mont_host, uint32_t nterms,
                      cudaStream_t stream) {
    if (nterms > LINCOMB_MAX || (nterms && (!d_polys || !lens || !coeffs_mont_host))) return (int)cudaErrorInvalidValue;
    snarkvm_b200_lincomb_segment_t s{};
    s.d_out = d_out;
    s.n = n;
    s.nterms = nterms;
    for (uint32_t j = 0; j < nterms; j++) {
        s.d_polys[j] = d_polys[j];
        s.lens[j] = lens[j];
        memcpy(s.coeffs_mont[j], (const uint8_t*)coeffs_mont_host + 32 * (size_t)j, 32);
    }
    return fr_lincomb_batch_device(&s, 1, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// Many independent PolyMultiplier products (fft/polynomial/multiplier.rs:70-134) in one pass: one launch loads every zero-padded
// operand (a into its output, b into scratch), the forward transforms of all 2·count operands go through ntt_batch_device (equal
// sizes share launches), one launch multiplies pointwise, and the inverse transforms of the outputs go through ntt_batch_device.
// ---------------------------------------------------------------------------------------------------------------------
struct PolymulSeg {
    uint32_t* out;
    uint32_t* tmp;
    const uint32_t *a, *b;
    uint64_t first, n, len_a, len_b;
};
__global__ void k_polymul_load(const PolymulSeg* __restrict__ segs, uint32_t nsegs, uint64_t total) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const PolymulSeg& s = segs[seg_of(segs, nsegs, g)];
    const uint64_t i = g - s.first;
    (i < s.len_a ? Fr::load_ldg(s.a + i * 8) : Fr::zero()).store(s.out + i * 8);
    (i < s.len_b ? Fr::load_ldg(s.b + i * 8) : Fr::zero()).store(s.tmp + i * 8);
}
__global__ void k_polymul_pointwise(const PolymulSeg* __restrict__ segs, uint32_t nsegs, uint64_t total) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const PolymulSeg& s = segs[seg_of(segs, nsegs, g)];
    const uint64_t i = g - s.first;
    (Fr::load(s.out + i * 8) * Fr::load(s.tmp + i * 8)).store(s.out + i * 8);
}

int polymul_batch_device(const snarkvm_b200_polymul_job_t* jobs, size_t count, cudaStream_t stream) {
    if (count == 0) return 0;
    if (!jobs || count >= ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    std::vector<PolymulSeg> table(count);
    std::vector<void*> fwd(2 * count), inv(count);
    std::vector<uint32_t> fwd_lg(2 * count), inv_lg(count);
    uint64_t total = 0;
    for (size_t i = 0; i < count; i++) {
        const snarkvm_b200_polymul_job_t& j = jobs[i];
        if (j.lg > NTT_MAX_LG || !j.d_out || !j.d_a || !j.d_b || j.len_a == 0 || j.len_b == 0) return (int)cudaErrorInvalidValue;
        const uint64_t n = (uint64_t)1 << j.lg;
        if (j.len_a > n || j.len_b > n || j.len_a + j.len_b - 1 > n) return (int)cudaErrorInvalidValue;
        table[i] = PolymulSeg{(uint32_t*)j.d_out, nullptr, (const uint32_t*)j.d_a, (const uint32_t*)j.d_b, total, n, j.len_a, j.len_b};
        total += n;
    }
    uint8_t* scratch = nullptr;                                  // segment table | the b operands, concatenated
    const size_t off_tmp = (count * sizeof(PolymulSeg) + 255) & ~(size_t)255;
    cudaError_t e = pool_alloc(&scratch, off_tmp + total * 32, stream);
    if (e != cudaSuccess) return (int)e;
    uint32_t* tmp = (uint32_t*)(scratch + off_tmp);
    for (size_t i = 0; i < count; i++) {
        table[i].tmp = tmp + table[i].first * 8;
        fwd[i] = table[i].out; fwd[count + i] = table[i].tmp; inv[i] = table[i].out;
        fwd_lg[i] = fwd_lg[count + i] = inv_lg[i] = jobs[i].lg;
    }
    const PolymulSeg* d_table = (const PolymulSeg*)scratch;
    const unsigned grid = (unsigned)((total + 255) / 256);
    int rc = (int)cudaMemcpyAsync(scratch, table.data(), count * sizeof(PolymulSeg), cudaMemcpyHostToDevice, stream);
    if (rc == 0) {
        k_polymul_load<<<grid, 256, 0, stream>>>(d_table, (uint32_t)count, total);
        count_launch();
        rc = (int)cudaGetLastError();
    }
    if (rc == 0) rc = ntt_batch_device(fwd.data(), fwd_lg.data(), 2 * count, NTT_FORWARD, NTT_STANDARD, stream);
    if (rc == 0) {
        k_polymul_pointwise<<<grid, 256, 0, stream>>>(d_table, (uint32_t)count, total);
        count_launch();
        rc = (int)cudaGetLastError();
    }
    if (rc == 0) rc = ntt_batch_device(inv.data(), inv_lg.data(), count, NTT_INVERSE, NTT_STANDARD, stream);
    cudaFreeAsync(scratch, stream);
    return rc;
}

// ---------------------------------------------------------------------------------------------------------------------
// Varuna's fourth round (ahp/prover/round_functions/fourth.rs:151-245) on K for every matrix of every circuit: one launch writes
// a = v_rc·row_col_val, b = |R||C|·(r − α)(c − β) and the denominators (r − α)(c − β) (= (α − r)(β − c)) into one concatenated
// buffer; one batch inversion (fields/src/lib.rs:78-129, zeros stay zero) runs over all of them; one launch writes
// f = (v_rc / (|R||C|))·row_col_val / ((r − α)(c − β)).
// ---------------------------------------------------------------------------------------------------------------------
struct Round4Seg {
    const uint32_t *row, *col, *rcv;
    uint32_t *a, *b, *f;
    uint64_t first, n;
    FrArg v_rc, rc, scale, alpha, beta;
};
__global__ void k_round4_evals(const Round4Seg* __restrict__ segs, uint32_t nsegs, uint64_t total, uint32_t* __restrict__ den) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const Round4Seg& s = segs[seg_of(segs, nsegs, g)];
    const uint64_t i = g - s.first;
    const Fr d = (Fr::load_ldg(s.row + i * 8) - fr_from_arg(s.alpha)) * (Fr::load_ldg(s.col + i * 8) - fr_from_arg(s.beta));
    (fr_from_arg(s.v_rc) * Fr::load_ldg(s.rcv + i * 8)).store(s.a + i * 8);
    (fr_from_arg(s.rc) * d).store(s.b + i * 8);
    d.store(den + g * 8);
}
__global__ void k_round4_f(const Round4Seg* __restrict__ segs, uint32_t nsegs, uint64_t total, const uint32_t* __restrict__ inv) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const Round4Seg& s = segs[seg_of(segs, nsegs, g)];
    const uint64_t i = g - s.first;
    (fr_from_arg(s.scale) * Fr::load(inv + g * 8) * Fr::load_ldg(s.rcv + i * 8)).store(s.f + i * 8);
}

// the table's segments (first and n set) in one launch, one batch inversion and one launch for f
static int round4_impl(const std::vector<Round4Seg>& table, uint64_t total, cudaStream_t stream) {
    const size_t count = table.size();
    FrArg one{};
    for (int k = 0; k < 8; k++) one.v[k] = FrParams::r1(k);                   // Montgomery one
    uint8_t* scratch = nullptr;                                                  // segment table | denominators, concatenated
    const size_t off_den = (count * sizeof(Round4Seg) + 255) & ~(size_t)255;
    cudaError_t e = pool_alloc(&scratch, off_den + total * 32, stream);
    if (e != cudaSuccess) return (int)e;
    const Round4Seg* d_table = (const Round4Seg*)scratch;
    uint32_t* den = (uint32_t*)(scratch + off_den);
    int rc = (int)cudaMemcpyAsync(scratch, table.data(), count * sizeof(Round4Seg), cudaMemcpyHostToDevice, stream);
    if (rc == 0) {
        const unsigned grid = (unsigned)((total + 255) / 256);
        const size_t threads = (total + BINV_K - 1) / BINV_K;
        k_round4_evals<<<grid, 256, 0, stream>>>(d_table, (uint32_t)count, total, den);
        k_fr_batch_inverse<<<(unsigned)((threads + 127) / 128), 128, 0, stream>>>(den, total, one);
        k_round4_f<<<grid, 256, 0, stream>>>(d_table, (uint32_t)count, total, den);
        count_launch(3);
        rc = (int)cudaGetLastError();
    }
    cudaFreeAsync(scratch, stream);
    return rc;
}

template <class S> static bool round4_segment(const S& s, uint64_t first, Round4Seg* t) {
    if (s.n == 0 || !s.d_row || !s.d_col || !s.d_row_col_val || !s.d_a || !s.d_b || !s.d_f) return false;
    *t = Round4Seg{(const uint32_t*)s.d_row, (const uint32_t*)s.d_col, (const uint32_t*)s.d_row_col_val, (uint32_t*)s.d_a, (uint32_t*)s.d_b,
                   (uint32_t*)s.d_f, first, s.n, FrArg{}, FrArg{}, FrArg{}, FrArg{}, FrArg{}};
    memcpy(t->v_rc.v, s.v_rc_mont, 32); memcpy(t->rc.v, s.rc_mont, 32); memcpy(t->scale.v, s.f_scale_mont, 32);
    return true;
}

int varuna_round4_evals_batch_device(const snarkvm_b200_round4_batch_segment_t* segs, size_t count, cudaStream_t stream) {
    if (count == 0) return 0;
    if (!segs || count >= ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    std::vector<Round4Seg> table(count);
    uint64_t total = 0;
    for (size_t i = 0; i < count; i++) {
        if (!round4_segment(segs[i], total, &table[i])) return (int)cudaErrorInvalidValue;
        memcpy(table[i].alpha.v, segs[i].alpha_mont, 32); memcpy(table[i].beta.v, segs[i].beta_mont, 32);
        total += segs[i].n;
    }
    return round4_impl(table, total, stream);
}

int varuna_round4_evals_device(const snarkvm_b200_round4_segment_t* segs, size_t count, const void* alpha_mont, const void* beta_mont,
                               cudaStream_t stream) {
    if (count == 0) return 0;
    if (!segs || !alpha_mont || !beta_mont || count >= ((size_t)1 << 31)) return (int)cudaErrorInvalidValue;
    std::vector<Round4Seg> table(count);
    uint64_t total = 0;
    for (size_t i = 0; i < count; i++) {
        if (!round4_segment(segs[i], total, &table[i])) return (int)cudaErrorInvalidValue;
        memcpy(table[i].alpha.v, alpha_mont, 32); memcpy(table[i].beta.v, beta_mont, 32);
        total += segs[i].n;
    }
    return round4_impl(table, total, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// MatrixEvals::evaluate (snark/varuna/ahp/matrices.rs:114-126): with the Lagrange coefficients l of K at a point, the four inner
// products Σ l·row, Σ l·col, Σ l·row·col, Σ l·row_col_val — the matrix's four index polynomials at that point.  row·col is formed
// on the fly (the device index keeps no row_col vector).  Stage 1: one launch over the whole matrix, grid-stride, every CTA
// reduces its four partials in shared memory; stage 2: one CTA per product adds the per-CTA partials.
// ---------------------------------------------------------------------------------------------------------------------
//
// Segmented over many matrices (each with its own K and point): segment j owns CTAs [cta0, cta0 + nctas) of the first launch and
// the four finishing CTAs 4j … 4j + 3 of the second.  Its Lagrange coefficients are either given (`lag`, `computed` = 0) or formed
// on the fly from the inverted denominators 1/(ω^i − τ) that one batch inversion left in `lag` (fft/domain.rs:277-291):
// L_i = c·ω^i/(ω^i − τ) with c = (1 − τ^n)/n.  When τ lies in K, c = 0 and the one zero denominator (left zero by the inversion)
// marks the indicator position (domain.rs:264-275).
static constexpr unsigned DOT_MAX_CTAS = 1024;
struct DotSeg {
    const uint32_t *row, *col, *rcv, *lag;
    uint64_t n, first;                                  // first: the segment's offset in the concatenated denominators
    FrArg tau;
    uint32_t lg, cta0, nctas, computed;
};
FF_DEV uint32_t dot_seg_of_cta(const DotSeg* __restrict__ segs, uint32_t nsegs, uint32_t b) {
    uint32_t lo = 0, hi = nsegs;
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (segs[mid].cta0 <= b) lo = mid; else hi = mid;
    }
    return lo;
}
// den[first + i] = ω_K^i − τ for every segment, and scale[j] = (1 − τ^n)/n
__global__ void k_lagrange_denominators(const DotSeg* __restrict__ segs, uint32_t nsegs, uint64_t total, const uint32_t* __restrict__ tw, int lgN,
                                        uint32_t* __restrict__ den, uint32_t* __restrict__ scale) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const uint32_t j = seg_of(segs, nsegs, g);
    const DotSeg& s = segs[j];
    const size_t i = g - s.first;
    const Fr tau = fr_from_arg(s.tau);
    (domain_element(i, (int)s.lg, tw, lgN) - tau).store(den + g * 8);
    if (i == 0) {
        Fr c = Fr::one() - fr_pow_u64(tau, s.n);
        for (uint32_t k = 0; k < s.lg; k++) c = c.half();
        c.store(scale + (size_t)j * 8);
    }
}
__global__ void __launch_bounds__(EVAL_THREADS) k_matrix_evals_dot(const DotSeg* __restrict__ segs, uint32_t nsegs, uint32_t total_ctas,
                                                                    const uint32_t* __restrict__ tw, int lgN, const uint32_t* __restrict__ scale,
                                                                    uint32_t* __restrict__ partial /* [4][total_ctas] */) {
    __shared__ uint4 sh4[EVAL_THREADS * 2];
    const uint32_t j = dot_seg_of_cta(segs, nsegs, blockIdx.x);
    const DotSeg& sg = segs[j];
    const uint32_t *row = sg.row, *col = sg.col, *rcv = sg.rcv, *lag = sg.lag;
    const size_t n = sg.n, stride = (size_t)sg.nctas * blockDim.x;
    const bool computed = sg.computed != 0;
    const Fr c_j = computed ? Fr::load(scale + (size_t)j * 8) : Fr::zero();
    Fr s[4] = {Fr::zero(), Fr::zero(), Fr::zero(), Fr::zero()};
    for (size_t i = (size_t)(blockIdx.x - sg.cta0) * blockDim.x + threadIdx.x; i < n; i += stride) {
        Fr l = Fr::load_ldg(lag + i * 8);
        if (computed) l = l.is_zero() ? Fr::one() : c_j * l * domain_element(i, (int)sg.lg, tw, lgN);
        const Fr lr = l * Fr::load_ldg(row + i * 8), c = Fr::load_ldg(col + i * 8);
        s[0] = s[0] + lr;
        s[1] = s[1] + l * c;
        s[2] = s[2] + lr * c;
        s[3] = s[3] + l * Fr::load_ldg(rcv + i * 8);
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const Fr t = cta_sum(s[k], reinterpret_cast<uint32_t*>(sh4));
        if (threadIdx.x == 0) t.store(partial + ((size_t)k * total_ctas + blockIdx.x) * 8);
        __syncthreads();
    }
}
// CTA 4j + k adds segment j's partials of product k
__global__ void __launch_bounds__(EVAL_THREADS) k_fr_sum_segments(const DotSeg* __restrict__ segs, const uint32_t* __restrict__ partial,
                                                                   uint32_t total_ctas, uint32_t* __restrict__ out) {
    __shared__ uint4 sh4[EVAL_THREADS * 2];
    const uint32_t j = blockIdx.x / 4, k = blockIdx.x % 4;
    const uint32_t* in = partial + ((size_t)k * total_ctas + segs[j].cta0) * 8;
    Fr acc = Fr::zero();
    for (uint32_t i = threadIdx.x; i < segs[j].nctas; i += EVAL_THREADS) acc = acc + Fr::load_ldg(in + (size_t)i * 8);
    const Fr s = cta_sum(acc, reinterpret_cast<uint32_t*>(sh4));
    if (threadIdx.x == 0) s.store(out + (size_t)blockIdx.x * 8);
}

// table: the segments with row / col / rcv (and lag unless computed) set; runs the Lagrange denominators and their one batch
// inversion when any segment is `computed`, then the dot and finishing launches, one D2H and one synchronisation
static int evals_dot_impl(void* out_mont_host, std::vector<DotSeg>& table, cudaStream_t stream) {
    const size_t count = table.size();
    uint64_t total_den = 0;
    uint32_t total_ctas = 0, lg_max = 0;
    bool any_computed = false;
    for (DotSeg& s : table) {
        const size_t blocks = std::min<size_t>((s.n + EVAL_THREADS - 1) / EVAL_THREADS, DOT_MAX_CTAS);
        s.cta0 = total_ctas;
        s.nctas = (uint32_t)blocks;
        total_ctas += (uint32_t)blocks;
        s.first = total_den;
        if (s.computed) { total_den += s.n; any_computed = true; lg_max = std::max(lg_max, s.lg); }
    }
    if (total_ctas == 0) { memset(out_mont_host, 0, count * 4 * 32); return 0; }
    const void* tw = nullptr;
    int lgN = 0, rc = 0;
    if (any_computed && (rc = ntt_get_twiddles((int)lg_max, &tw, &lgN)) != 0) return rc;
    // scratch: table | scale[count] | den[total_den] | partial[4][total_ctas] | out[count][4]
    const size_t off_scale = (count * sizeof(DotSeg) + 255) & ~(size_t)255, off_den = off_scale + count * 32,
                 off_partial = off_den + total_den * 32, off_out = off_partial + (size_t)4 * total_ctas * 32, bytes = off_out + count * 4 * 32;
    uint8_t* scratch = nullptr;
    cudaError_t e = pool_alloc(&scratch, bytes, stream);
    if (e != cudaSuccess) return (int)e;
    uint32_t *scale = (uint32_t*)(scratch + off_scale), *den = (uint32_t*)(scratch + off_den), *partial = (uint32_t*)(scratch + off_partial),
             *out = (uint32_t*)(scratch + off_out);
    for (DotSeg& s : table) if (s.computed) s.lag = den + s.first * 8;
    DotSeg* d_table = (DotSeg*)scratch;
    rc = (int)cudaMemcpyAsync(d_table, table.data(), count * sizeof(DotSeg), cudaMemcpyHostToDevice, stream);
    if (rc == 0 && total_den) {
        // a table is either all computed (matrix_evals_at_points) or none (matrix_evals_dot), so `first` orders every segment
        k_lagrange_denominators<<<(unsigned)((total_den + 255) / 256), 256, 0, stream>>>(d_table, (uint32_t)count, total_den, (const uint32_t*)tw,
                                                                                         lgN, den, scale);
        const size_t threads = (total_den + BINV_K - 1) / BINV_K;
        FrArg one{};
        for (int k = 0; k < 8; k++) one.v[k] = FrParams::r1(k);                     // Montgomery one
        k_fr_batch_inverse<<<(unsigned)((threads + 127) / 128), 128, 0, stream>>>(den, total_den, one);
        count_launch(2);
    }
    if (rc == 0) {
        k_matrix_evals_dot<<<total_ctas, EVAL_THREADS, 0, stream>>>(d_table, (uint32_t)count, total_ctas, (const uint32_t*)tw, lgN, scale, partial);
        k_fr_sum_segments<<<(unsigned)(4 * count), EVAL_THREADS, 0, stream>>>(d_table, partial, total_ctas, out);
        count_launch(2);
        rc = (int)cudaGetLastError();
    }
    if (rc == 0) rc = (int)cudaMemcpyAsync(out_mont_host, out, count * 4 * 32, cudaMemcpyDeviceToHost, stream);
    cudaFreeAsync(scratch, stream);
    if (rc == 0) rc = (int)cudaStreamSynchronize(stream);
    return rc;
}

int matrix_evals_dot_device(void* out_mont_host, const void* d_row, const void* d_col, const void* d_row_col_val, const void* d_lagrange,
                            size_t n, cudaStream_t stream) {
    if (!out_mont_host) return (int)cudaErrorInvalidValue;
    if (n == 0) { memset(out_mont_host, 0, 4 * 32); return 0; }
    if (!d_row || !d_col || !d_row_col_val || !d_lagrange) return (int)cudaErrorInvalidValue;
    std::vector<DotSeg> table(1);
    table[0] = DotSeg{(const uint32_t*)d_row, (const uint32_t*)d_col, (const uint32_t*)d_row_col_val, (const uint32_t*)d_lagrange, n, 0, FrArg{}, 0, 0, 0, 0};
    return evals_dot_impl(out_mont_host, table, stream);
}

int matrix_evals_at_points_device(void* out_mont_host, const snarkvm_b200_evals_segment_t* segs, size_t count, cudaStream_t stream) {
    if (count == 0) return 0;
    if (!out_mont_host || !segs || count >= ((size_t)1 << 24)) return (int)cudaErrorInvalidValue;
    std::vector<DotSeg> table(count);
    for (size_t i = 0; i < count; i++) {
        const snarkvm_b200_evals_segment_t& s = segs[i];
        if (s.n == 0 || (s.n & (s.n - 1)) || s.n > ((uint64_t)1 << NTT_MAX_LG) || !s.d_row || !s.d_col || !s.d_row_col_val)
            return (int)cudaErrorInvalidValue;
        DotSeg& t = table[i];
        t = DotSeg{(const uint32_t*)s.d_row, (const uint32_t*)s.d_col, (const uint32_t*)s.d_row_col_val, nullptr, s.n, 0, FrArg{}, 0, 0, 0, 1};
        memcpy(t.tau.v, s.point_mont, 32);
        while (((uint64_t)1 << t.lg) < s.n) t.lg++;
    }
    return evals_dot_impl(out_mont_host, table, stream);
}

}  // namespace b200
