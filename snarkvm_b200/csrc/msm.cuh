// Pippenger multi-scalar multiplication over BLS12-377 G1 for sm_90a.
//
// Replaces the hot loops of the reference's VariableBase::msm
// (algorithms/src/msm/variable_base/mod.rs:30-49 → batched.rs:366-415):
//   batched_window  (batched.rs:328-364)  →  k_digits<0/1>                      (signed digits, counting sort by bucket)
//   batch_add       (batched.rs:175-325)  →  k_pair_desc + k_pair_level2 ×(0…5) (Montgomery-trick affine pair levels)
//                                            k_bucket_accumulate(_dense)         (XYZZ sums of what is left, per work item)
//                                            k_partial_group_sum                 (hot buckets: fold item partials 32:1)
//   running sum     (batched.rs:356-361)  →  k_bucket_reduce / k_group_sum
//   window combine  (batched.rs:404-413)  →  host Horner over ≤ 24 window sums (host_ec.hpp)
//
// Design differences (the result is a group element, so any window size / digit
// recoding / coordinate system yields the same to_affine() image):
//   * signed c-bit digits  → 2^(c-1) buckets per window instead of 2^c − 1
//   * counting sort by (window, bucket) with global atomics instead of sort_unstable
//   * batched affine additions only for the first levels (where they fill the GPU), XYZZ mixed additions after
//   * every bucket is cut into work items of ≤ cap points and every pair level is split by OUTPUT elements, so a hot
//     bucket (all scalars equal, repeated bases — benches/msm/variable_base.rs:29-32 — or the carry-only top window)
//     cannot serialise a thread.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace b200 {

// Window layout: windows 0 … nwin−2 have c bits each, the top window (bits (nwin−1)·c …) has c_top bits.  Every window is a
// signed-digit window (digit ∈ [−2^(w−1), 2^(w−1)] for a w-bit window, the carry passed upwards); the top window is wide
// enough that a scalar below 2^253 never makes its digit negative, so no carry leaves it.  A window's buckets are cut into
// bucket SETS of nbuckets = 2^(c−1) buckets: one set per window below the top, top_sets() = 2^(c_top−1) / nbuckets for the top
// window, whose set k holds the digits k·nbuckets + 1 … (k+1)·nbuckets (its window sum carries the k·nbuckets offset).
// The uniform plans are c_top = c, nsets = nwin (nwin = 253 / c + 1).
struct MsmPlan {
    int c;              // bits of every window but the top one
    int nwin;           // number of windows
    uint32_t nbuckets;  // 2^(c-1) buckets per bucket set (bucket value 1 .. 2^(c-1))
    uint32_t cap;       // max points per work item
    int levels;         // batched-affine pair levels run before the XYZZ accumulation (0 = gather + XYZZ only)
    int c_top;          // bits of the top window (= c in the uniform plans)
    int nsets;          // bucket sets per sum: nwin − 1 + top_sets()

    int top_sets() const { return nsets - nwin + 1; }
    int window_bit(int w) const { return w * c; }                                        // first scalar bit of window w
    int window_bits(int w) const { return w == nwin - 1 ? c_top : c; }
    uint32_t window_buckets(int w) const { return 1u << (window_bits(w) - 1); }          // largest digit magnitude
    int window_first_set(int w) const { return w; }                                      // its sets are contiguous from here
    uint32_t set_digit_offset(int s) const { return s >= nwin ? (uint32_t)(s - nwin + 1) * nbuckets : 0u; }
};

// mixed = false: always a uniform plan (the sharded window-sum calls, whose callers fold the sums as Σ 2^{c·w}·S_w, and G2)
MsmPlan msm_make_plan(size_t npoints, bool mixed = true);
MsmPlan msm_make_plan_batch(size_t max_n, size_t total_n);

// One MSM call = `njobs` independent sums over one resident base set.
struct MsmBases {            // base arrays, densified back to back into 128-byte records (their indices follow each other)
    const void* d_points;
    size_t stride, n;
};
struct MsmSegment {          // one scalar vector; segment i of job j adds Σ_k scalars[k]·base[base0 + k] into job j's sum
    const void* d_scalars;   // n × 32 B in HBM
    size_t n;
    uint32_t base0;          // index of its first point in the concatenated base array (0 in table mode)
    uint32_t job;
    int mont;                // 1: Montgomery Fr (polynomial coefficients), converted to canonical integers in the digit kernel
};
// d_window_sums[njobs][flat ? 1 : plan.nwin] XYZZ points (48 words each); *d_flags (device u32, zeroed by the caller) gets bit 0
// set when a scalar has bits 253..255 set.  All pointers are device pointers; scratch comes from the library's private
// stream-ordered pool under the per-device byte budget.  Returns cudaError_t as int.
int msm_core(uint32_t* d_window_sums, uint32_t* d_flags, const MsmPlan& plan, const MsmBases* bases, int nbases,
             const uint32_t* table, size_t table_n, const MsmSegment* segs, int nsegs, int njobs, cudaStream_t stream);

// single sum, canonical scalars: per-window sums Σ_b b·S_{w,b} into d_window_sums[plan.nwin][48]
int msm_window_sums_device(uint32_t* d_window_sums, uint32_t* d_flags, const MsmPlan& plan, const void* d_points, size_t stride,
                           const void* d_scalars, size_t npoints, cudaStream_t stream);

// Resident bases with precomputed tables 2^{c·w}·P_i (w < nwin; 128 B per record): all windows then share ONE bucket set, so
// wide windows are cheap (c = 22, 12 windows at 2^24 instead of 17 / 15).  Table size: npoints · nwin · 128 B.
MsmPlan msm_make_plan_precomputed(size_t npoints);
int msm_precompute_tables_device(uint32_t* d_table, const MsmPlan& plan, const void* d_points, size_t stride, size_t npoints, cudaStream_t stream);
// d_sum: ONE XYZZ point (192 B) = Σ scalars[i]·P_i over the first nscalars (≤ table_n) points
int msm_precomputed_sum_device(uint32_t* d_sum, uint32_t* d_flags, const MsmPlan& plan, const uint32_t* d_table, size_t table_n, const void* d_scalars,
                               size_t nscalars, int mont, cudaStream_t stream);

// Bump allocator over one scratch block: a pass with base = nullptr sizes a layout, a second one over the block hands out the
// same 256-byte-aligned pieces.
struct Arena {
    uint8_t* base = nullptr;
    size_t off = 0;
    template <class T> T* take(size_t count) {
        T* p = base ? (T*)(base + off) : nullptr;
        off += (count * sizeof(T) + 255) & ~(size_t)255;
        return p;
    }
};

// Curve-independent building blocks (signed-digit bucket sort, scans, work-item counts, hot-bucket folds, the 8:1 tree), shared
// with the G2 path:
size_t msm_scan_bytes(size_t count);
// an exclusive scan of `count` u32 that counts its launches (msm_exclusive_scan: two)
using MsmScan = int (*)(void* tmp, size_t tmp_bytes, const uint32_t* in, uint32_t* out, size_t count, cudaStream_t stream);
int msm_exclusive_scan(void* tmp, size_t tmp_bytes, const uint32_t* in, uint32_t* out, size_t count, cudaStream_t stream);
// hist / bucket_start / cursors: nwin·nbuckets + 1 u32 each; sorted: n·nwin u32 (point index | sign << 31, grouped by (window, bucket))
int msm_sort_indices(const MsmPlan& plan, const void* d_scalars, size_t n, int mont, uint32_t* hist, uint32_t* bucket_start, uint32_t* cursors,
                     uint32_t* sorted, void* cub_tmp, size_t cub_bytes, uint32_t* d_flags, cudaStream_t stream);
int msm_items_per_bucket(const uint32_t* hist, uint32_t* items, uint32_t total_buckets, uint32_t cap, cudaStream_t stream);
// Scan-driven 32:1 folds of item partials until every bucket holds one: per round k_group_counts, `scan` and the curve's `fold`
// kernel (k_partial_group_sum, k_g2_partial_group_sum).  *partial / *start (item_start) come in as the accumulation's output and
// go out as the last round's; partial2 / start2 are the other buffers of the ping-pong.
using MsmFoldKernel = void (*)(const uint32_t* partial_in, const uint32_t* start_in, const uint32_t* start_out, uint32_t total_buckets,
                               uint32_t* partial_out);
int msm_scan_fold(MsmFoldKernel fold, MsmScan scan, uint32_t** partial, uint32_t* partial2, uint32_t** start, uint32_t* start2, uint32_t* cnt_tmp,
                  uint32_t total_buckets, size_t worst, size_t total_bound, void* cub_tmp, size_t cub_bytes, cudaStream_t stream);
// the curve's `sum` kernel (k_group_sum, k_g2_group_sum) over groups of MSM_TREE_FANIN; red_a holds the input and is overwritten
static constexpr uint32_t MSM_TREE_FANIN = 8;
using MsmTreeKernel = void (*)(const uint32_t* in, uint32_t per_row, uint32_t group, uint32_t out_per_row, uint32_t rows, uint32_t* out);
int msm_tree_sum(MsmTreeKernel sum, uint32_t* red_a, uint32_t* red_b, uint32_t per_row, uint32_t rows, size_t point_words, uint32_t* out,
                 cudaStream_t stream);

// BLS12-377 G2 (points over Fq2; the curves the reference sends to standard::msm, msm/variable_base/standard.rs:79-118):
// per-window sums Σ_b b·S_{w,b} as XYZZ points over Fq2 (96 words each) into d_window_sums[plan.nwin][96].
// d_points: the reference's Affine<G2> images (x.c0 x.c1 y.c0 y.c1 infinity, stride ≥ 200).
int msm_g2_window_sums_device(uint32_t* d_window_sums, uint32_t* d_flags, const MsmPlan& plan, const void* d_points, size_t stride,
                              const void* d_scalars, size_t npoints, int mont, cudaStream_t stream);
// P_i = h(seed, i)·G2 (same multipliers as the G1 generator)
int msm_generate_bases_g2_device(void* d_points, size_t npoints, size_t stride, uint64_t seed, cudaStream_t stream);

// Deterministic test/bench input: P_i = h(seed, i)·G with a 64-bit multiplier h
// (every point is in the prime-order subgroup because G is).  Writes the reference
// affine layout with the given stride.
int msm_generate_bases_device(void* d_points, size_t npoints, size_t stride, uint64_t seed, cudaStream_t stream);
int msm_generator_mul_device(void* d_points, size_t npoints, size_t stride, const void* d_scalars, cudaStream_t stream);

// `.usrs` uncompressed points (96 B canonical each) → reference Affine images in HBM; *d_invalid counts points that are
// off the curve, out of range or badly flagged.
int srs_decode_device(void* d_out, size_t stride, const void* d_in, size_t npoints, uint32_t* d_invalid, cudaStream_t stream);

// device self-test of ff.cuh's warp-cooperative multiplication / inversion; *d_mismatches (device u32) counts failing warps
int selftest_coop_device(uint32_t nwarps, uint64_t seed, uint32_t* d_mismatches, cudaStream_t stream);
// element-wise arithmetic test kernels (testops.cuh instantiated in msm.cu and in ntt.cu; snarkvm_b200_test_*_device)
int test_field_op_msm(int field, int op, void* d_out, const void* d_a, const void* d_b, size_t n, cudaStream_t stream);
int test_field_op_ntt(int field, int op, void* d_out, const void* d_a, const void* d_b, size_t n, cudaStream_t stream);
int test_field_op_pairing(int field, int op, void* d_out, const void* d_a, const void* d_b, size_t n, cudaStream_t stream);
int test_curve_op_device(int group, int op, void* d_out, const void* d_a, const void* d_b, const uint32_t* d_k, size_t n, cudaStream_t stream);

// out[i] = Σ_r in[r][i]  over `nranks` arrays of `count` XYZZ points (multi-GPU combine).
int xyzz_sum_ranks_device(uint32_t* d_out, const uint32_t* d_in, int nranks, int count, cudaStream_t stream);

// Allocation from the library's private stream-ordered pool of the current device (release threshold = the scratch budget:
// 60 % of the device unless SNARKVM_B200_SCRATCH_LIMIT_GB says otherwise); free with cudaFreeAsync.  The default pool is untouched.
int pool_alloc_raw(void** p, size_t bytes, cudaStream_t stream);
template <class T> inline cudaError_t pool_alloc(T** p, size_t bytes, cudaStream_t stream) { return (cudaError_t)pool_alloc_raw((void**)p, bytes, stream); }
// MSM scratch budget of the current device: bytes allowed in flight, in flight now, and the high-water mark
int msm_scratch_stats(size_t* limit, size_t* in_use, size_t* peak);
int msm_set_scratch_limit(size_t bytes);      // also resets the high-water mark

uint64_t launch_count();
void count_launch(int n = 1);

// Optional per-kernel CUDA-event timing on the launching stream (bench.py's roofline numbers).
enum ProfKind { PROF_MSM_SORT = 0, PROF_MSM_ACCUMULATE = 1, PROF_MSM_REDUCE = 2, PROF_NTT_PASS = 3, PROF_KINDS = 4 };
void prof_enable(bool on);
bool prof_enabled();
// records an event pair around whatever is enqueued on `stream` between begin and end
struct ProfScope {
    cudaEvent_t a = nullptr, b = nullptr;
    cudaStream_t stream;
    int kind;
    ProfScope(int kind, cudaStream_t stream);
    ~ProfScope();
};
// waits for all recorded pairs of `kind`, returns their summed duration and count, and clears them
int prof_collect(int kind, double* total_ms, uint64_t* count);

}  // namespace b200
