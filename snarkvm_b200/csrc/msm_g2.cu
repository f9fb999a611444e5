// Pippenger MSM over BLS12-377 G2 (points over Fq2) — the device path for the curves the reference sends to
// standard::msm (algorithms/src/msm/variable_base/mod.rs:30-49 → standard.rs:79-118: every curve except BLS12-377 G1).
//
// The curve-independent half is shared with G1 (msm.cu): signed c-bit digits, counting sort by (window, bucket), work items
// of ≤ cap points, 32:1 folding of hot buckets.  The curve-dependent half is the same XYZZ group law instantiated over Fq2
// (ec.cuh: XyzzT<Fq2>, 384-byte accumulators; a mixed addition is 8M + 2S in Fq2 = 28 Fq multiplications):
//   update_buckets      (standard.rs:24-41)  →  k_g2_accumulate      gathers the reference's 200-byte Affine<G2> images
//   running-sum window  (standard.rs:66-74)  →  k_g2_bucket_reduce / k_g2_group_sum
//   window combine      (standard.rs:104-117) →  host Horner (host_ec.hpp, XyzzT<Fq2>)
// The result is a group element, so any window size / digit recoding yields the reference's to_affine() image.  No batched
// affine levels here: G2 MSMs are setup-sized (no Varuna commitment lives in G2) and XYZZ over Fq2 keeps this path small.
#include "msm.cuh"

#define FF_CALL_MUL 1
#include "ec.cuh"

namespace b200 {

static constexpr int X2W = XYZZ2::WORDS;          // 96 words = 384 bytes

// one thread per work item (≤ cap sorted entries of one bucket)
__global__ void __launch_bounds__(128) k_g2_accumulate(const uint8_t* __restrict__ points, size_t stride, const uint32_t* __restrict__ sorted,
                                                       const uint32_t* __restrict__ bucket_start, const uint32_t* __restrict__ item_start,
                                                       uint32_t total_buckets, uint32_t cap, uint32_t* __restrict__ partial) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= item_start[total_buckets]) return;
    uint32_t lo = 0, hi = total_buckets;          // item_start[lo] <= t < item_start[hi]
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (item_start[mid] <= t) lo = mid; else hi = mid; }
    const uint32_t seg = t - item_start[lo], b0 = bucket_start[lo], b1 = bucket_start[lo + 1];
    const uint32_t s0 = b0 + seg * cap, s1 = s0 + cap < b1 ? s0 + cap : b1;
    XYZZ2 acc = XYZZ2::infinity();
#pragma unroll 1
    for (uint32_t k = s0; k < s1; k++) {
        const uint32_t e = sorted[k];
        acc.add_affine(load_affine_g2(points, stride, e & 0x7fffffffu), (e >> 31) != 0u);
    }
    acc.store(partial + (size_t)t * X2W);
}
// hot buckets: fold item partials 32:1
__global__ void __launch_bounds__(128) k_g2_partial_group_sum(const uint32_t* __restrict__ partial_in, const uint32_t* __restrict__ start_in,
                                                              const uint32_t* __restrict__ start_out, uint32_t total_buckets,
                                                              uint32_t* __restrict__ partial_out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= start_out[total_buckets]) return;
    uint32_t lo = 0, hi = total_buckets;
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (start_out[mid] <= t) lo = mid; else hi = mid; }
    const uint32_t g = t - start_out[lo];
    uint32_t i0 = start_in[lo] + g * 32u, i1 = start_in[lo + 1];
    if (i0 + 32u < i1) i1 = i0 + 32u;
    XYZZ2 s = XYZZ2::load(partial_in + (size_t)i0 * X2W);
#pragma unroll 1
    for (uint32_t i = i0 + 1; i < i1; i++) s.add(XYZZ2::load(partial_in + (size_t)i * X2W));
    s.store(partial_out + (size_t)t * X2W);
}
// thread j of window w owns bucket values [j·K + 1, (j+1)·K]: running = Σ S_b, acc = Σ (b − lo + 1)·S_b, out = acc + lo·running
__global__ void __launch_bounds__(128) k_g2_bucket_reduce(const uint32_t* __restrict__ partial, const uint32_t* __restrict__ item_start,
                                                          uint32_t nbuckets, uint32_t chunk, uint32_t chunks_per_window, uint32_t nwin,
                                                          uint32_t* __restrict__ out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= chunks_per_window * nwin) return;
    const uint32_t w = t / chunks_per_window, j = t % chunks_per_window, lo = j * chunk, hi = lo + chunk;
    XYZZ2 running = XYZZ2::infinity(), acc = XYZZ2::infinity();
#pragma unroll 1
    for (uint32_t b = hi; b-- > lo;) {
        const uint32_t wb = w * nbuckets + b, i0 = item_start[wb], i1 = item_start[wb + 1];
#pragma unroll 1
        for (uint32_t i = i0; i < i1; i++) running.add(XYZZ2::load(partial + (size_t)i * X2W));
        acc.add(running);
    }
    if (lo != 0u) acc.add(running.mul_u32(lo));
    acc.store(out + (size_t)t * X2W);
}
__global__ void __launch_bounds__(128) k_g2_group_sum(const uint32_t* __restrict__ in, uint32_t per_row, uint32_t group, uint32_t out_per_row,
                                                      uint32_t rows, uint32_t* __restrict__ out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= out_per_row * rows) return;
    const uint32_t r = t / out_per_row, j = t % out_per_row, i0 = j * group, i1 = i0 + group < per_row ? i0 + group : per_row;
    XYZZ2 s = XYZZ2::infinity();
#pragma unroll 1
    for (uint32_t i = i0; i < i1; i++) s.add(XYZZ2::load(in + ((size_t)r * per_row + i) * X2W));
    s.store(out + (size_t)t * X2W);
}

int msm_g2_window_sums_device(uint32_t* d_window_sums, uint32_t* d_flags, const MsmPlan& plan, const void* d_points, size_t stride,
                              const void* d_scalars, size_t npoints, int mont, cudaStream_t stream) {
    if (!d_window_sums || !d_flags || !d_points || !d_scalars || npoints == 0 || stride < 200 || (stride & 7)) return (int)cudaErrorInvalidValue;
    const uint64_t TB64 = (uint64_t)plan.nwin * plan.nbuckets;
    const size_t entries = npoints * (size_t)plan.nwin;
    if (TB64 >= (1ull << 31) || npoints >= (1ull << 31) || entries >= (1ull << 32)) return (int)cudaErrorInvalidValue;
    const uint32_t TB = (uint32_t)TB64, cap = plan.cap;
    const uint32_t chunk = plan.nbuckets < 16u ? plan.nbuckets : 16u, tree = MSM_TREE_FANIN, chunks_per_set = plan.nbuckets / chunk;
    const size_t max_items = (size_t)TB + entries / cap + 1;
    const size_t cub_bytes = msm_scan_bytes((size_t)TB + 1);
    uint32_t *hist, *bucket_start, *cursors, *items, *item_start, *items2, *cnt_tmp, *sorted, *partial, *partial2, *red_a, *red_b;
    uint8_t* cub_tmp;
    Arena ar;
    auto layout = [&](Arena& a) {
        hist = a.take<uint32_t>((size_t)TB + 1); bucket_start = a.take<uint32_t>((size_t)TB + 1); cursors = a.take<uint32_t>((size_t)TB + 1);
        items = a.take<uint32_t>((size_t)TB + 1); item_start = a.take<uint32_t>((size_t)TB + 1); items2 = a.take<uint32_t>((size_t)TB + 1);
        cnt_tmp = a.take<uint32_t>((size_t)TB + 1);
        sorted = a.take<uint32_t>(entries);
        partial = a.take<uint32_t>(max_items * X2W);
        partial2 = a.take<uint32_t>(((size_t)TB + max_items / 32 + 2) * X2W);
        red_a = a.take<uint32_t>((size_t)plan.nwin * chunks_per_set * X2W);
        red_b = a.take<uint32_t>((size_t)plan.nwin * (chunks_per_set / tree + 1) * X2W);
        cub_tmp = a.take<uint8_t>(cub_bytes);
    };
    layout(ar);
    uint8_t* block = nullptr;
    cudaError_t e = pool_alloc(&block, ar.off, stream);
    if (e != cudaSuccess) return (int)e;
    ar.base = block; ar.off = 0;
    layout(ar);
    int rc = msm_sort_indices(plan, d_scalars, npoints, mont, hist, bucket_start, cursors, sorted, cub_tmp, cub_bytes, d_flags, stream);
    if (rc == 0) rc = msm_items_per_bucket(hist, items, TB, cap, stream);
    if (rc == 0) rc = msm_exclusive_scan(cub_tmp, cub_bytes, items, item_start, (size_t)TB + 1, stream);
    if (rc == 0) {
        k_g2_accumulate<<<(unsigned)((max_items + 127) / 128), 128, 0, stream>>>((const uint8_t*)d_points, stride, sorted, bucket_start, item_start, TB, cap, partial);
        count_launch();
        // worst case: every entry in one bucket
        uint32_t *p = partial, *st = item_start;
        rc = msm_scan_fold(k_g2_partial_group_sum, msm_exclusive_scan, &p, partial2, &st, items2, cnt_tmp, TB, npoints / cap + 1, max_items,
                           cub_tmp, cub_bytes, stream);
        if (rc == 0) {
            const uint32_t nthreads = chunks_per_set * (uint32_t)plan.nwin;
            k_g2_bucket_reduce<<<(nthreads + 127) / 128, 128, 0, stream>>>(p, st, plan.nbuckets, chunk, chunks_per_set, (uint32_t)plan.nwin, red_a);
            count_launch();
            rc = msm_tree_sum(k_g2_group_sum, red_a, red_b, chunks_per_set, (uint32_t)plan.nwin, X2W, d_window_sums, stream);
        }
    }
    cudaFreeAsync(block, stream);
    return rc;
}

// ---------------------------------------------------------------------------
// Synthetic bases: P_i = h(seed, i)·G2 with the G1 generator's multipliers (msm.cu splitmix64 scheme)
// ---------------------------------------------------------------------------
FF_DEV uint64_t splitmix64_g2(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
// G2_GENERATOR_{X,Y}_{C0,C1}, Montgomery limbs (curves/src/bls12_377/g2.rs:228-282)
__constant__ uint32_t G2_GEN[4][12] = {
    {0xb2cfca6du, 0x135aa022u, 0xa0ba2863u, 0x999f96bdu, 0x049d2570u, 0x3b258618u, 0x37f7601du, 0xbac1c559u, 0x160b0ebau, 0x2c17e3ffu, 0x61311156u, 0x01243de0u},
    {0x2bf627a2u, 0xafdc3839u, 0xc2169752u, 0x2fe64cfbu, 0xf1e17646u, 0x83a7358eu, 0xe6d52a7eu, 0x45d36f92u, 0xf6420d6du, 0x88d14c88u, 0x5bd94f8eu, 0x00e0e47cu},
    {0xfe5b5ef8u, 0x19c08814u, 0x43980256u, 0x297c67edu, 0xcfa274a8u, 0x874aef39u, 0x3ca72dfau, 0x2c7a13e8u, 0xb6e40f15u, 0xe54547d6u, 0xa60e9ab3u, 0x00dbfac4u},
    {0x59f2193cu, 0x1543371fu, 0xb505c4ffu, 0xc9c52a35u, 0xbbf1a70fu, 0x96480bceu, 0x6668452bu, 0xcb831ef8u, 0xe4c10a6du, 0x06b4abbeu, 0xf64e4d98u, 0x0105fbcdu}};

__global__ void __launch_bounds__(64) k_generate_bases_g2(uint8_t* points, size_t n, size_t stride, uint64_t seed) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t k = splitmix64_g2(seed ^ splitmix64_g2((uint64_t)i));
    if (k == 0) k = 1;
    AffineT<Fq2> g;
#pragma unroll
    for (int j = 0; j < 12; j++) { g.x.c0.v[j] = G2_GEN[0][j]; g.x.c1.v[j] = G2_GEN[1][j]; g.y.c0.v[j] = G2_GEN[2][j]; g.y.c1.v[j] = G2_GEN[3][j]; }
    g.inf = false;
    XYZZ2 acc = XYZZ2::infinity();
    bool started = false;
#pragma unroll 1
    for (int b = 63; b >= 0; b--) {
        if (started) acc.dbl();
        if ((k >> b) & 1ull) { acc.add_affine(g, false); started = true; }
    }
    store_affine_g2(points, stride, i, acc.to_affine());
}
int msm_generate_bases_g2_device(void* d_points, size_t npoints, size_t stride, uint64_t seed, cudaStream_t stream) {
    if (stride < 200 || (stride & 7)) return (int)cudaErrorInvalidValue;
    if (npoints == 0) return 0;
    k_generate_bases_g2<<<(unsigned)((npoints + 63) / 64), 64, 0, stream>>>((uint8_t*)d_points, npoints, stride, seed);
    count_launch();
    return (int)cudaGetLastError();
}

}  // namespace b200
