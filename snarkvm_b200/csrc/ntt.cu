// See ntt.cuh for semantics and the reference map.
//
// Structure: radix-2 decimation-in-frequency butterflies (the reference's io_helper,
// domain.rs:691-735, butterfly_fn_io :651-656) grouped into passes of S ≤ 8 stages.
// A pass keeps a tile of 2^S rows × 2^Q columns of Fr in shared memory, runs its S
// stages there, and touches HBM once (32 B read + 32 B write per element).  Twiddles
// ω^e come from one precomputed table of ω_N^j (j < N/2) that is strided for smaller
// domains, exactly like precomputation_for_subdomain (domain.rs:895-908); inverse
// transforms use ω^{-e} = −ω^{n/2−e}, so no second table exists.  The last pass writes
// bit-reversed addresses (derange, domain.rs:789-804) so the output is natural-order,
// and fuses the n^{-1} / coset scaling (domain.rs:421, 440-443); the first pass fuses
// the coset pre-scaling g^j (domain.rs:201-206).
#include "ntt.cuh"

#include <map>
#include <mutex>
#include <vector>

#include "ff.cuh"
#include "msm.cuh"   // count_launch
#include "poly.cuh"  // ntt_get_twiddles
#define FIELD_TEST_ENTRY test_field_op_ntt
#include "testops.cuh"   // the field-arithmetic test kernels, compiled here with the multiplier inlined

namespace b200 {

#define CUDA_TRY(x)                                          \
    do {                                                     \
        cudaError_t e_ = (x);                                \
        if (e_ != cudaSuccess) { rc = (int)e_; goto done; }  \
    } while (0)

// TWO_ADIC_ROOT_OF_UNITY (order 2^47), GENERATOR = 22 and its inverse, Montgomery form (fr.rs:115-135)
__constant__ uint32_t FR_ROOT47[8] = {0xda3ad648u, 0xaf80da4du, 0xfc381dacu, 0x5e223adbu, 0xb2f92525u, 0x03ba0666u, 0x3befb0ceu, 0x0f906c5bu};
__constant__ uint32_t FR_GEN[8] = {0xfffffed3u, 0x296c7fffu, 0x6ffffec7u, 0x92921665u, 0x92860e69u, 0x4c01534du, 0xb9819970u, 0x0c79cfc4u};
__constant__ uint32_t FR_GEN_INV[8] = {0xd1745d17u, 0xb76f9745u, 0xafffffffu, 0xfed18274u, 0x5b36a173u, 0xfce61983u, 0x78dc8d16u, 0x068b6ffdu};

FF_DEV Fr fr_from_const(const uint32_t* c) { Fr r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = c[i]; return r; }

// out[k] = ω_N^(2^k), k < lgN   (get_root_of_unity, fields/src/traits/fft_field.rs:38-86)
__global__ void k_root_pow2(Fr* out, int lgN) {
    Fr w = fr_from_const(FR_ROOT47);
    for (int i = lgN; i < 47; i++) w = w.sqr();
    for (int k = 0; k < lgN; k++) { out[k] = w; w = w.sqr(); }
}
// gp[k] = g^(±2^k), k < 40 ; ninv[0] = 2^{-lg} (size_inv, domain.rs:138-139), ninv[1] = 1
__global__ void k_coset_setup(Fr* gp, Fr* ninv, int lg, int inverse) {
    Fr g = fr_from_const(inverse ? FR_GEN_INV : FR_GEN);
    for (int k = 0; k < 40; k++) { gp[k] = g; g = g.sqr(); }
    Fr h = Fr::one();
    for (int k = 0; k < lg; k++) h = h.half();
    ninv[0] = h;
    ninv[1] = Fr::one();
}
// out[j] = scale · Π_{bit k of j} pow2[k + shift]
__global__ void k_pow_table(Fr* out, size_t count, const Fr* __restrict__ pow2, int shift, const Fr* __restrict__ scale) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    Fr acc = scale ? *scale : Fr::one();
    size_t e = j;
    for (int k = shift; e; k++, e >>= 1) if (e & 1) acc = acc * pow2[k];
    out[j] = acc;
}

// ---------------------------------------------------------------------------
// Per-device caches (the FFI is entered concurrently from many threads — SURVEY §8b)
// ---------------------------------------------------------------------------
struct CosetTables { Fr* lo; Fr* hi; Fr* ninv; };   // lo[4096] = g^{±j}, hi[h] = c·g^{±4096h}, ninv[0] = n^{-1}
struct DeviceCache {
    std::mutex mu;
    Fr* tw = nullptr;      // ω_N^j, j < N/2
    int lgN = 0;
    std::map<uint64_t, CosetTables> coset;   // key = lg | dir << 8
};
static DeviceCache g_cache[64];

static int get_twiddles(int lg, const Fr** tw, int* lgN) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    DeviceCache& c = g_cache[dev & 63];
    std::lock_guard<std::mutex> lock(c.mu);
    if (c.lgN < lg) {
        int want = lg < 16 ? 16 : lg;
        Fr *tab = nullptr, *pw = nullptr;
        size_t count = (size_t)1 << (want - 1);
        if ((e = cudaMalloc(&tab, count * sizeof(Fr))) != cudaSuccess) return (int)e;
        if ((e = cudaMalloc(&pw, 64 * sizeof(Fr))) != cudaSuccess) { cudaFree(tab); return (int)e; }
        k_root_pow2<<<1, 1>>>(pw, want);
        k_pow_table<<<(unsigned)((count + 255) / 256), 256>>>(tab, count, pw, 0, nullptr);
        count_launch(2);
        e = cudaDeviceSynchronize();
        cudaFree(pw);
        if (e != cudaSuccess) { cudaFree(tab); return (int)e; }
        // the previous (smaller) table is intentionally kept alive: other threads may still be reading it
        c.tw = tab;
        c.lgN = want;
    }
    *tw = c.tw;
    *lgN = c.lgN;
    return 0;
}

int ntt_get_twiddles(int lg, const void** tw, int* lgN) {
    const Fr* t = nullptr;
    int rc = get_twiddles(lg, &t, lgN);
    *tw = t;
    return rc;
}

static int get_coset_tables(int lg, int inverse, CosetTables* out) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    DeviceCache& c = g_cache[dev & 63];
    std::lock_guard<std::mutex> lock(c.mu);
    uint64_t key = (uint64_t)lg | ((uint64_t)inverse << 8);
    auto it = c.coset.find(key);
    if (it == c.coset.end()) {
        CosetTables t{nullptr, nullptr, nullptr};
        Fr* gp = nullptr;
        size_t nhi = lg > 12 ? ((size_t)1 << (lg - 12)) : 1;
        if ((e = cudaMalloc(&t.lo, 4096 * sizeof(Fr))) != cudaSuccess) return (int)e;
        if ((e = cudaMalloc(&t.hi, nhi * sizeof(Fr))) != cudaSuccess) return (int)e;
        if ((e = cudaMalloc(&t.ninv, 2 * sizeof(Fr))) != cudaSuccess) return (int)e;
        if ((e = cudaMalloc(&gp, 40 * sizeof(Fr))) != cudaSuccess) return (int)e;
        k_coset_setup<<<1, 1>>>(gp, t.ninv, lg, inverse);
        k_pow_table<<<16, 256>>>(t.lo, 4096, gp, 0, nullptr);
        // forward: hi carries no scale; inverse: hi carries n^{-1} so the post-scale is two multiplications
        k_pow_table<<<(unsigned)((nhi + 255) / 256), 256>>>(t.hi, nhi, gp, 12, inverse ? t.ninv : t.ninv + 1);
        count_launch(3);
        e = cudaDeviceSynchronize();
        cudaFree(gp);
        if (e != cudaSuccess) return (int)e;
        it = c.coset.emplace(key, t).first;
    }
    *out = it->second;
    return 0;
}

// ---------------------------------------------------------------------------
// One pass = stages [t0, t0+S) of the DIF network on a 2^S × 2^Q tile in shared memory.
// ---------------------------------------------------------------------------
// Two layout variants measured slower and left OFF (A/B builds, 2^24 forward): the XOR swizzle that removes the last pass's
// transposed-store bank conflicts, and the last pass's ≤ 128 twiddles staged in shared memory — the conflicts and the L1-resident twiddle loads were never on the
// critical path (the butterflies are bound by the multiplier), the extra index arithmetic and shared-memory traffic are.
#ifndef NTT_SMEM_TW
#define NTT_SMEM_TW 0
#endif
#ifndef NTT_SWIZZLE
#define NTT_SWIZZLE 0
#endif
#ifndef NTT_TW_PREFETCH
#define NTT_TW_PREFETCH 0      // measured slower at 2^24: the duplicated index arithmetic costs more issue slots than the hidden twiddle latency returns
#endif
struct PassArgs {
    const Fr* in;
    Fr* out;
    const Fr* tw;        // ω_N^j table
    const Fr* coset_lo;  // may be null
    const Fr* coset_hi;
    const Fr* ninv;      // n^{-1} (used when post == 1)
    int lg, lgN;
    int t0, S, Q;
    int last;            // 1: rows are contiguous sub-arrays, output is bit-reversed scatter
    int inverse;
    uint32_t tile0;      // first tile of this launch (a pass may be launched in column ranges)
    int pre;             // 1: multiply input j by coset_lo/hi (forward coset)
    int post;            // 0 none, 1: × n^{-1}, 2: × coset_lo/hi[k] (hi already carries n^{-1})
    // k_ntt_pass<true>: blockIdx.y is a transform of 2^lg elements at batch[y]; in / out are then the scratch base (transform y's
    // scratch at in/out + y·2^lg) unless in_batch / out_batch select batch[y]
    Fr* const* batch;
    int in_batch, out_batch;
};

FF_DEV Fr coset_factor(const Fr* lo, const Fr* hi, size_t idx) { return lo[idx & 4095] * hi[idx >> 12]; }

// BATCH: the pointer-table form (ntt_batch_device); the one-transform instantiation compiles without it.
template <bool BATCH>
__global__ void __launch_bounds__(256) k_ntt_pass(PassArgs a) {
    // Shared memory holds the tile as two planes of 16-byte halves (low limbs of element i at [i], high limbs at
    // [tile_elems + i]): consecutive threads then touch consecutive 16-byte words — conflict-free LDS/STS.128 — where
    // the 32-byte array-of-structures layout made every access a 2-way bank conflict.
    extern __shared__ uint4 smem_raw[];
    // Column index XOR row index (low Q bits): the last pass fills the tile column by column (consecutive threads →
    // consecutive ROWS, a stride of 2^Q 16-byte words = one bank group), which was an 8-way conflict per store
    // (31.8 M conflicts in round 1's ncu of the last pass, 12× the other passes); with the swizzle consecutive rows land in
    // different bank groups and row-wise accesses stay a permutation of one 128-byte line.
    struct Tile {
        uint4* p; uint32_t n; uint32_t q, cmask;
#if NTT_SWIZZLE
        __device__ __forceinline__ uint32_t sw(uint32_t i) const { return i ^ ((i >> q) & cmask); }
#else
        __device__ __forceinline__ uint32_t sw(uint32_t i) const { return i; }
#endif
        __device__ __forceinline__ Fr get(uint32_t i0) const {
            const uint32_t i = sw(i0);
            uint4 a = p[i], b = p[n + i]; Fr r;
            r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
            return r;
        }
        __device__ __forceinline__ void put(uint32_t i0, const Fr& r) const {
            const uint32_t i = sw(i0);
            p[i] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]); p[n + i] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
        }
    };
    const int S = a.S, Q = a.Q, lg = a.lg, t0 = a.t0;
    const int L = lg - t0 - S;                       // low index bits below the tile's row digit
    const uint32_t rows = 1u << S, cols = 1u << Q, tile_elems = rows << Q;
    const Tile sm{smem_raw, tile_elems, (uint32_t)Q, cols - 1u};
    const size_t tile = (size_t)blockIdx.x + a.tile0;
    const uint32_t tid = threadIdx.x, nthr = blockDim.x;
    const Fr* src = a.in;
    Fr* dst = a.out;
    if (BATCH) {
        Fr* const x = a.batch[blockIdx.y];
        const size_t off = (size_t)blockIdx.y << lg;
        src = a.in_batch ? x : a.in + off;
        dst = a.out_batch ? x : a.out + off;
    }

    size_t H = 0, low_base = 0, hprime_base = 0;
    if (!a.last) { H = tile >> (L - Q); low_base = (tile & (((size_t)1 << (L - Q)) - 1)) << Q; }
    else hprime_base = tile << Q;

    // ---- last pass: its stages use only 2^(S-1) ≤ 128 distinct twiddles ω^{k·2^t0} — staged once per CTA in shared memory ----
    uint4* sm_tw = smem_raw + 2 * tile_elems;
    if (NTT_SMEM_TW && a.last && S > 0) {
        const size_t halfn = (size_t)1 << (lg - 1);
        for (uint32_t k = tid; k < (1u << (S - 1)); k += nthr) {
            Fr w = Fr::one();
            if (k) { const size_t ex = (size_t)k << t0; w = Fr::load(a.tw + ((a.inverse ? halfn - ex : ex) << (a.lgN - lg))); }
            sm_tw[2 * k] = make_uint4(w.v[0], w.v[1], w.v[2], w.v[3]);
            sm_tw[2 * k + 1] = make_uint4(w.v[4], w.v[5], w.v[6], w.v[7]);
        }
    }
    // ---- load (+ optional coset pre-scale) ----
    for (uint32_t e = tid; e < tile_elems; e += nthr) {
        uint32_t d, c;
        size_t idx;
        if (!a.last) { c = e & (cols - 1); d = e >> Q; idx = (H << (S + L)) | ((size_t)d << L) | low_base | c; }
        else {
            d = e & (rows - 1); c = e >> S;
            size_t hp = hprime_base + c;
            size_t Hrow = t0 ? (size_t)(__brevll((unsigned long long)hp) >> (64 - t0)) : 0;
            idx = (Hrow << S) | d;
        }
        Fr x = Fr::load(src + idx);
        if (a.pre) x = x * coset_factor(a.coset_lo, a.coset_hi, idx);
        sm.put((d << Q) | c, x);
    }
    __syncthreads();

    // ---- S butterfly stages ----
    const uint32_t nbf = tile_elems >> 1;
    const int tw_shift = a.lgN - lg;
    for (int u = 0; u < S; u++) {
        const int t = t0 + u;
        const uint32_t hb = S - 1 - u;               // log2 of the local gap (in rows)
#ifndef NTT_UNROLL
#define NTT_UNROLL 1
#endif
        // NTT_UNROLL butterflies per thread per trip with all operands requested up front.  Unroll 2 and 4 measured slower
        // at 2^24 (the extra registers cost more occupancy than the overlapped latency gains), so the default is 1.
#if NTT_TW_PREFETCH
        // (variant, off) The twiddle of the thread's NEXT butterfly is requested before the current one is multiplied: the first two passes read
        // theirs from HBM / L2 (more long-scoreboard stalls per issue than the last pass, whose ≤ 128 twiddles sit in L1), and with shared memory capping the SM at 3 CTAs the 8 extra registers
        // cost no occupancy (≤ 85 registers per thread).
        auto tw_ptr = [&](uint32_t b) -> const Fr* {             // address of butterfly b's twiddle, or null when it is 1
            const uint32_t c = b & (cols - 1), j = b >> Q, r_lo = j & ((1u << hb) - 1u);
            const size_t r = a.last ? (size_t)r_lo : (((size_t)r_lo << L) | low_base | c);
            const size_t ex = r << t;
            return ex ? a.tw + ((a.inverse ? (((size_t)1 << (lg - 1)) - ex) : ex) << tw_shift) : nullptr;
        };
        const Fr* wp = tid < nbf ? tw_ptr(tid) : nullptr;
        Fr wn = Fr::one();
        if (wp) wn = Fr::load(wp);
        for (uint32_t b = tid; b < nbf; b += nthr) {
            const Fr w = wn;
            const bool has = wp != nullptr;
            const uint32_t nb = b + nthr;
            wp = nb < nbf ? tw_ptr(nb) : nullptr;
            if (wp) wn = Fr::load(wp);
            const uint32_t c = b & (cols - 1), j = b >> Q, r_lo = j & ((1u << hb) - 1u);
            const uint32_t d_lo = ((j >> hb) << (hb + 1)) | r_lo;
            const uint32_t il = (d_lo << Q) | c, ih = il + ((1u << hb) << Q);
            const Fr x = sm.get(il), y = sm.get(ih);
            Fr dif = x - y;
            if (has) { dif = dif * w; if (a.inverse) dif = dif.neg(); }
            sm.put(il, x + y); sm.put(ih, dif);
        }
        __syncthreads();
        continue;
#endif
        for (uint32_t b0 = tid; b0 < nbf; b0 += nthr * NTT_UNROLL) {
            Fr x[NTT_UNROLL], y[NTT_UNROLL], w[NTT_UNROLL];
            uint32_t il[NTT_UNROLL], ih[NTT_UNROLL];
            bool live[NTT_UNROLL], tw[NTT_UNROLL];
#pragma unroll
            for (int k = 0; k < NTT_UNROLL; k++) {
                const uint32_t b = b0 + k * nthr;
                live[k] = b < nbf;
                tw[k] = false;
                if (!live[k]) continue;
                uint32_t c = b & (cols - 1), j = b >> Q;
                uint32_t r_lo = j & ((1u << hb) - 1u);
                uint32_t d_lo = ((j >> hb) << (hb + 1)) | r_lo;
                il[k] = (d_lo << Q) | c; ih[k] = il[k] + ((1u << hb) << Q);
                // exponent of ω_n: (index mod gap) · 2^t
                size_t r = a.last ? (size_t)r_lo : (((size_t)r_lo << L) | low_base | c);
                size_t ex = r << t;
                x[k] = sm.get(il[k]); y[k] = sm.get(ih[k]);
                if (ex != 0) {
                    tw[k] = true;
                    if (NTT_SMEM_TW && a.last) {
                        const uint4 w0 = sm_tw[2 * (r_lo << u)], w1 = sm_tw[2 * (r_lo << u) + 1];
                        w[k].v[0] = w0.x; w[k].v[1] = w0.y; w[k].v[2] = w0.z; w[k].v[3] = w0.w;
                        w[k].v[4] = w1.x; w[k].v[5] = w1.y; w[k].v[6] = w1.z; w[k].v[7] = w1.w;
                    } else {
                        w[k] = Fr::load(a.tw + ((a.inverse ? (((size_t)1 << (lg - 1)) - ex) : ex) << tw_shift));
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < NTT_UNROLL; k++) {
                if (!live[k]) continue;
                Fr sum = x[k] + y[k], dif = x[k] - y[k];
                if (tw[k]) { dif = dif * w[k]; if (a.inverse) dif = dif.neg(); }
                sm.put(il[k], sum); sm.put(ih[k], dif);
            }
        }
        __syncthreads();
    }

    // ---- store (+ optional post-scale) ----
    for (uint32_t e = tid; e < tile_elems; e += nthr) {
        uint32_t c = e & (cols - 1), d = e >> Q;
        size_t k;
        if (!a.last) k = (H << (S + L)) | ((size_t)d << L) | low_base | c;
        else {
            size_t drev = S ? (size_t)(__brev(d) >> (32 - S)) : 0;
            k = (drev << t0) | (hprime_base + c);
        }
        Fr x = sm.get((d << Q) | c);
        if (a.post == 1) x = x * (*a.ninv);
        else if (a.post == 2) x = x * coset_factor(a.coset_lo, a.coset_hi, k);
        x.store(dst + k);
    }
}

// derange (domain.rs:789-804) as a stand-alone pass: used only for the NR / RN / RR orders of the FFI, which no
// reference caller requests (they all pass NN, where the permutation is fused into the last NTT pass).
__global__ void k_bitrev_inplace(Fr* x, uint32_t lg) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >> lg) return;
    size_t r = lg ? (size_t)(__brevll((unsigned long long)i) >> (64 - lg)) : 0;
    if (i < r) { Fr a = Fr::load(x + i), b = Fr::load(x + r); b.store(x + i); a.store(x + r); }
}
int fr_bitrev_device(void* d_x, uint32_t lg, cudaStream_t stream) {
    size_t n = (size_t)1 << lg;
    k_bitrev_inplace<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((Fr*)d_x, lg);
    count_launch();
    return (int)cudaGetLastError();
}

__global__ void k_pointwise_mul(Fr* acc, const Fr* __restrict__ x, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) (Fr::load(acc + i) * Fr::load(x + i)).store(acc + i);
}
__global__ void k_fr_convert(Fr* out, const Fr* __restrict__ in, size_t n, int to_mont) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { Fr x = Fr::load(in + i); (to_mont ? x.to_mont() : x.from_mont()).store(out + i); }
}

int fr_pointwise_mul_device(void* d_acc, const void* d_x, size_t n, cudaStream_t stream) {
    if (!n) return 0;
    k_pointwise_mul<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((Fr*)d_acc, (const Fr*)d_x, n);
    count_launch();
    return (int)cudaGetLastError();
}
int fr_from_mont_device(void* d_out, const void* d_in, size_t n, cudaStream_t stream) {
    if (!n) return 0;
    k_fr_convert<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((Fr*)d_out, (const Fr*)d_in, n, 0);
    count_launch();
    return (int)cudaGetLastError();
}
int fr_to_mont_device(void* d_out, const void* d_in, size_t n, cudaStream_t stream) {
    if (!n) return 0;
    k_fr_convert<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((Fr*)d_out, (const Fr*)d_in, n, 1);
    count_launch();
    return (int)cudaGetLastError();
}

static constexpr int MAX_STAGES = 8;    // rows per tile ≤ 256
static constexpr int TILE_LG = 11;      // 2^11 elements × 32 B = 64 KiB of shared memory per CTA
// + the last pass's 2^(S-1) twiddles: ≤ 128 for a multi-pass transform, up to 1024 when a whole transform of ≤ 2^11
// elements is one pass
static inline size_t tw_smem_bytes(int S, bool last) { return NTT_SMEM_TW && last && S > 0 ? ((size_t)32 << (S - 1)) : 0; }

// The passes of one transform: stages [t0, t0 + S) on tiles of 2^S rows × 2^Q columns.
int ntt_make_passes(uint32_t lg, NttPass* out, int* npasses) {
    if (lg > NTT_MAX_LG || !out || !npasses) return (int)cudaErrorInvalidValue;
    const int P = lg <= (uint32_t)TILE_LG ? 1 : (int)((lg + MAX_STAGES - 1) / MAX_STAGES);
    int t0 = 0;
    for (int p = 0; p < P; p++) {
        const int remaining = (int)lg - t0;
        const int S = (remaining + (P - p) - 1) / (P - p);
        const bool last = p == P - 1;
        int Q = TILE_LG - S;
        if (Q > 3) Q = 3;
        if (last) { if (Q > t0) Q = t0; }
        else { const int L = (int)lg - t0 - S; if (Q > L) Q = L; }
        out[p].t0 = t0; out[p].S = S; out[p].Q = Q;
        out[p].tiles = ((size_t)1 << lg) >> (S + Q);
        t0 += S;
    }
    *npasses = P;
    return 0;
}

// Tiles [tile0, tile0 + ntiles) of pass `p`.  Pass 0 reads A; the last pass writes A; everything in between lives in B.
// Tile t of pass 0 holds columns [t·2^Q, (t+1)·2^Q) of the 2^S × 2^(lg−S) row-major view of the input; tile t of the last pass
// produces the same column range of the 2^S × 2^t0 view of the (natural-order) output — which is what lets a host-buffer
// transform upload / download by column ranges underneath those two passes (snarkvm_ntt in api.cu).
// Everything of pass p of a 2^lg transform but its buffers (in, out, batch).
static int pass_args(uint32_t lg, int direction, int type, int p, const NttPass* passes, int P, PassArgs* out) {
    const Fr* tw = nullptr;
    int lgN = 0, rc = 0;
    CosetTables ct{nullptr, nullptr, nullptr};
    const bool inverse = direction == NTT_INVERSE, coset = type == NTT_COSET;
    static std::once_flag smem_once[64];
    if ((rc = get_twiddles((int)lg, &tw, &lgN)) != 0) return rc;
    if (inverse || coset) { if ((rc = get_coset_tables((int)lg, inverse ? 1 : 0, &ct)) != 0) return rc; }
    {
        int dev = 0; cudaGetDevice(&dev);
        std::call_once(smem_once[dev & 63], [] {
            const int smem = (1 << TILE_LG) * (int)sizeof(Fr) + (int)tw_smem_bytes(TILE_LG, true);
            cudaFuncSetAttribute(k_ntt_pass<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
            cudaFuncSetAttribute(k_ntt_pass<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        });
    }
    PassArgs a{};
    a.tw = tw; a.coset_lo = ct.lo; a.coset_hi = ct.hi; a.ninv = ct.ninv;
    a.lg = (int)lg; a.lgN = lgN; a.t0 = passes[p].t0; a.S = passes[p].S; a.Q = passes[p].Q;
    a.last = (p == P - 1) ? 1 : 0;
    a.inverse = inverse ? 1 : 0;
    a.pre = (p == 0 && coset && !inverse) ? 1 : 0;
    a.post = (a.last && inverse) ? (coset ? 2 : 1) : 0;
    *out = a;
    return 0;
}
static inline size_t pass_smem(const PassArgs& a) { return ((size_t)1 << (a.S + a.Q)) * sizeof(Fr) + tw_smem_bytes(a.S, a.last != 0); }

int ntt_launch_pass(void* d_A, void* d_B, uint32_t lg, int direction, int type, int p, size_t tile0, size_t ntiles, cudaStream_t stream) {
    if (lg > NTT_MAX_LG || (direction != NTT_FORWARD && direction != NTT_INVERSE) || (type != NTT_STANDARD && type != NTT_COSET))
        return (int)cudaErrorInvalidValue;
    NttPass passes[8];
    int P = 0, rc = ntt_make_passes(lg, passes, &P);
    if (rc) return rc;
    if (p < 0 || p >= P || tile0 + ntiles > passes[p].tiles || (P > 1 && !d_B)) return (int)cudaErrorInvalidValue;
    if (ntiles == 0) return 0;
    PassArgs a;
    if ((rc = pass_args(lg, direction, type, p, passes, P, &a)) != 0) return rc;
    a.in = (p == 0) ? (const Fr*)d_A : (const Fr*)d_B;
    a.out = (P == 1 || a.last) ? (Fr*)d_A : (Fr*)d_B;
    a.tile0 = (uint32_t)tile0;
    {
        ProfScope pass_scope(PROF_NTT_PASS, stream);
        k_ntt_pass<false><<<(unsigned)ntiles, 256, pass_smem(a), stream>>>(a);
    }
    count_launch();
    return (int)cudaGetLastError();
}

// Transforms of equal size share their launches: blockIdx.y picks the transform from a device-side pointer table, so a size
// of one pass costs one launch for all its transforms and a larger size one launch per pass (each transform has its own
// slice of one scratch buffer).  The twiddle table is built once, for the largest size, before any launch.
static constexpr size_t NTT_BATCH_GRID_Y = 65535;
int ntt_batch_device(void* const* d_data, const uint32_t* lgs, size_t count, int direction, int type, cudaStream_t stream) {
    if (count == 0) return 0;
    if (!d_data || !lgs || (direction != NTT_FORWARD && direction != NTT_INVERSE) || (type != NTT_STANDARD && type != NTT_COSET))
        return (int)cudaErrorInvalidValue;
    std::map<uint32_t, std::vector<Fr*>> by_lg;
    uint32_t lg_max = 0;
    for (size_t i = 0; i < count; i++) {
        if (lgs[i] > NTT_MAX_LG || !d_data[i]) return (int)cudaErrorInvalidValue;
        by_lg[lgs[i]].push_back((Fr*)d_data[i]);
        if (lgs[i] > lg_max) lg_max = lgs[i];
    }
    const Fr* tw = nullptr;
    int lgN = 0, rc = get_twiddles((int)lg_max, &tw, &lgN);
    if (rc) return rc;
    std::vector<Fr*> table;                                   // the pointers of every size, size by size
    table.reserve(count);
    for (auto& g : by_lg) table.insert(table.end(), g.second.begin(), g.second.end());
    Fr** d_table = nullptr;
    if ((rc = (int)pool_alloc(&d_table, count * sizeof(Fr*), stream)) != 0) return rc;
    rc = (int)cudaMemcpyAsync(d_table, table.data(), count * sizeof(Fr*), cudaMemcpyHostToDevice, stream);
    size_t first = 0;
    for (auto it = by_lg.begin(); rc == 0 && it != by_lg.end(); ++it) {
        const uint32_t lg = it->first;
        const size_t n = it->second.size();
        NttPass passes[8];
        int P = 0;
        if ((rc = ntt_make_passes(lg, passes, &P)) != 0) break;
        Fr* scratch = nullptr;
        if (P > 1 && (rc = (int)pool_alloc(&scratch, (n << lg) * sizeof(Fr), stream)) != 0) break;
        for (int p = 0; p < P && rc == 0; p++) {
            PassArgs a;
            if ((rc = pass_args(lg, direction, type, p, passes, P, &a)) != 0) break;
            a.in_batch = p == 0;
            a.out_batch = P == 1 || a.last;
            ProfScope pass_scope(PROF_NTT_PASS, stream);
            for (size_t y0 = 0; y0 < n && rc == 0; y0 += NTT_BATCH_GRID_Y) {
                const size_t ny = n - y0 < NTT_BATCH_GRID_Y ? n - y0 : NTT_BATCH_GRID_Y;
                a.batch = d_table + first + y0;
                a.in = a.out = scratch + (y0 << lg);
                k_ntt_pass<true><<<dim3((unsigned)passes[p].tiles, (unsigned)ny), 256, pass_smem(a), stream>>>(a);
                count_launch();
                rc = (int)cudaGetLastError();
            }
        }
        if (scratch) cudaFreeAsync(scratch, stream);
        first += n;
    }
    cudaFreeAsync(d_table, stream);
    return rc;
}

int ntt_device(void* d_inout, uint32_t lg, int direction, int type, void* d_scratch, cudaStream_t stream) {
    NttPass passes[8];
    int P = 0, rc = ntt_make_passes(lg, passes, &P);
    if (rc) return rc;
    void* B = d_scratch;
    bool own_scratch = false;
    if (P > 1 && !B) {
        if ((rc = (int)pool_alloc(&B, ((size_t)1 << lg) * sizeof(Fr), stream)) != 0) return rc;
        own_scratch = true;
    }
    for (int p = 0; p < P && rc == 0; p++) rc = ntt_launch_pass(d_inout, B, lg, direction, type, p, 0, passes[p].tiles, stream);
    if (own_scratch) cudaFreeAsync(B, stream);
    return rc;
}

}  // namespace b200
