// See msm.cuh for the map from reference functions to kernels.
#include "msm.cuh"

#include <atomic>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <utility>
#include <vector>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cub/device/device_scan.cuh>

#define FF_CALL_MUL 1
#include "ec.cuh"
#include "cta_inverse.cuh"
#include "quad.cuh"
#define FIELD_TEST_ENTRY test_field_op_msm
#include "testops.cuh"

namespace b200 {

static std::atomic<uint64_t> g_launches{0};
uint64_t launch_count() { return g_launches.load(); }
void count_launch(int n) { g_launches.fetch_add((uint64_t)n); }

static std::atomic<bool> g_prof{false};
static std::mutex g_prof_mu;
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_recs[PROF_KINDS];
void prof_enable(bool on) { g_prof.store(on); }
bool prof_enabled() { return g_prof.load(); }
ProfScope::ProfScope(int kind_, cudaStream_t stream_) : stream(stream_), kind(kind_) {
    if (!g_prof.load()) return;
    if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) { a = b = nullptr; return; }
    cudaEventRecord(a, stream);
}
ProfScope::~ProfScope() {
    if (!a) return;
    cudaEventRecord(b, stream);
    std::lock_guard<std::mutex> lock(g_prof_mu);
    g_prof_recs[kind].emplace_back(a, b);
}
int prof_collect(int kind, double* total_ms, uint64_t* count) {
    if (kind < 0 || kind >= PROF_KINDS) return (int)cudaErrorInvalidValue;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> recs;
    { std::lock_guard<std::mutex> lock(g_prof_mu); recs.swap(g_prof_recs[kind]); }
    double tot = 0; int rc = 0;
    for (auto& r : recs) {
        float ms = 0;
        cudaError_t e = cudaEventSynchronize(r.second);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, r.first, r.second);
        if (e != cudaSuccess) rc = (int)e; else tot += ms;
        cudaEventDestroy(r.first); cudaEventDestroy(r.second);
    }
    if (total_ms) *total_ms = tot;
    if (count) *count = recs.size();
    return rc;
}

static int ceil_log2(size_t x) { int l = 0; size_t v = x > 1 ? x - 1 : 0; while (v) { l++; v >>= 1; } return l; }
// log2 rounded to the NEAREST integer (in the log domain): the plans below were swept at powers of two, and a size just above one
// — a 2^20-coefficient polynomial plus four blinding terms — belongs to that power's plan, not to the next one's.
static int plan_log2(size_t x) {
    int l = ceil_log2(x < 2 ? 2 : x);
    if (l > 1 && (double)x < 0.70710678118 * (double)((size_t)1 << l)) l--;
    return l;
}

// "w,w,…" or "w*k,…" (k windows of w bits): every width but the last equal, the last one wide enough that the top digit of a
// scalar below 2^253 stays non-negative.  Returns false (and leaves p alone) for anything else.
static bool parse_window_widths(const char* s, MsmPlan& p) {
    std::vector<int> w;
    while (*s) {
        char* end = nullptr;
        long v = strtol(s, &end, 10);
        if (end == s || v < 2 || v > 24) return false;
        long k = 1;
        s = end;
        if (*s == '*') { k = strtol(s + 1, &end, 10); if (end == s + 1 || k < 1 || k > 128) return false; s = end; }
        for (long i = 0; i < k && w.size() <= 128; i++) w.push_back((int)v);
        if (*s == ',') s++;
        else if (*s) return false;
    }
    if (w.size() < 2 || w.size() > 128) return false;
    for (size_t i = 1; i + 1 < w.size(); i++) if (w[i] != w[0]) return false;
    const int c = w[0], nwin = (int)w.size(), c_top = w.back();
    if ((nwin - 1) * c >= 253 || (nwin - 1) * c + c_top < 254) return false;          // top raw ≤ 2^(253 − bit) ≤ 2^(c_top − 1)
    const int top_sets = c_top > c ? 1 << (c_top - c) : 1;
    if (top_sets > 64) return false;
    p.c = c; p.nwin = nwin; p.c_top = c_top; p.nsets = nwin - 1 + top_sets;
    p.nbuckets = 1u << (c - 1);
    return true;
}

MsmPlan msm_make_plan(size_t npoints, bool mixed) {
    MsmPlan p;
    int lg = plan_log2(npoints);
    // Window bits from a sweep (tools/tune_msm.py): wider windows mean fewer
    // bucket additions (n·W) but more buckets to reduce and shorter, more divergent bucket runs.
    int c = lg <= 8 ? 4 : lg <= 12 ? lg - 4 : lg <= 18 ? 11 : lg == 19 ? 13 : lg == 20 ? 15 : lg <= 22 ? 16 : 17;
    const char* ec = getenv("SNARKVM_B200_MSM_C");
    if (ec) { int v = atoi(ec); if (v >= 2 && v <= 24) c = v; }
    p.c = c;
    p.nwin = 253 / c + 1;
    p.nbuckets = 1u << (c - 1);
    p.c_top = c;
    p.nsets = p.nwin;
    // Mixed layouts (tools/sweep_msm_windows.py, DESIGN §4): from 2^24, 13 windows of 18 bits and a 20-bit top window — 14
    // windows instead of 15, every bucket set 2^17 buckets, the top window's digits (≤ 305 881 below r) in four sets.  At 2^22
    // and 2^23 the uniform plans stay ahead (the larger reduction and sort cost more than the 1/15 fewer additions save).
    // SNARKVM_B200_MSM_C asks for a uniform plan; SNARKVM_B200_MSM_WINDOWS names a layout ("18*13,20"), or "0" for the uniform one.
    if (mixed) {
        const char* ew = getenv("SNARKVM_B200_MSM_WINDOWS");
        if (ew && *ew && strcmp(ew, "0") != 0) parse_window_widths(ew, p);
        else if (!ew && !ec && lg >= 24) parse_window_widths("18*13,20", p);
        c = p.c;
    }
    // Aim for ≥ ~300k work items so 132 SMs × (2 × 256-thread CTAs) see several waves, but keep
    // items long enough (≥ 16 points) that the per-item overhead stays in the noise.
    size_t total = npoints * (size_t)p.nwin;
    size_t cap = total / 300000 + 1;
    if (cap < 16) cap = 16;
    p.cap = (uint32_t)cap;
    // Batched-affine pair levels before the XYZZ accumulation pay off only when every level still fills the
    // GPU (tools/ab_pair.py sweep with the record-scatter sort): 5 levels from 2^23, 4 at 2^21–2^22, 3 at 2^20, 2 at 2^19
    // with c = 13, none below.
    int levels = lg >= 23 ? 5 : lg >= 21 ? 4 : lg == 20 ? 3 : lg == 19 ? 2 : 0;
    while (levels > 0 && ((npoints >> (c - 1)) >> levels) < 2) levels--;
    if (const char* e = getenv("SNARKVM_B200_MSM_LEVELS")) { int v = atoi(e); if (v >= 0 && v <= 16) levels = v; }
    p.levels = levels;
    return p;
}

// Plan for `njobs` sums sharing one base set in one pass: the window size follows the LARGEST job (bucket load), the
// number of pair levels follows the TOTAL work (a level is worth it while it fills the machine) as long as the buckets
// of the largest job still hold a few points after the halvings.
MsmPlan msm_make_plan_batch(size_t max_n, size_t total_n) {
    MsmPlan p = msm_make_plan(max_n);
    if (total_n > max_n) {
        int lgt = plan_log2(total_n);
        int levels = lgt >= 23 ? 5 : lgt >= 21 ? 4 : lgt == 20 ? 3 : lgt == 19 ? 2 : 0;
        // (a level the total asks for beyond the largest job's own plan must leave ≥ 4 points per bucket: 8 × 2^20 coefficients with
        // c = 15 hold 64 per bucket, and 4 levels beat 5 there, tools/time_batch.py)
        while (levels > p.levels && ((max_n >> (p.c - 1)) >> levels) < 4) levels--;
        while (levels > 0 && ((max_n >> (p.c - 1)) >> levels) < 2) levels--;
        if (const char* e = getenv("SNARKVM_B200_MSM_LEVELS")) { int v = atoi(e); if (v >= 0 && v <= 16) levels = v; }
        if (levels > p.levels) p.levels = levels;
        size_t cap = total_n * (size_t)p.nwin / 300000 + 1;
        if (cap < 16) cap = 16;
        p.cap = (uint32_t)cap;
    }
    return p;
}

// ---------------------------------------------------------------------------
// Signed-digit recoding of a canonical 253-bit scalar (8 little-endian u32 words).
// digit_w ∈ [-2^(c-1), 2^(c-1)]; returns magnitude and sign for window w given the
// running carry (sequential over w).
// ---------------------------------------------------------------------------
// flat != 0 (precomputed tables 2^{c·w}·P_i): every window feeds the SAME bucket set and the entry names record
// w·flat + i of the table instead of point i.  slot_base: first counter of this job's bucket sets; index_base: position of
// this scalar vector's first point in the call's dense base array.  MONT: the scalars are Montgomery Fr (polynomial
// coefficients) and are converted here (to_bigint, kzg10/mod.rs:469-474).  Scalars with bits 253..255 set are outside
// what nwin windows cover: they raise bit 0 of *flags and the caller returns an error instead of a wrong point.
// Windows below the top one have c_low bits, the top one c_top (MsmPlan); the top window's digits run past nbuckets into the
// sets that follow its first one.
template <bool SCATTER, bool MONT>
__global__ void __launch_bounds__(256) k_digits(const uint32_t* __restrict__ scalars, size_t n, int c_low, int c_top, int nwin,
                                                uint32_t nbuckets, uint32_t* __restrict__ counters /* hist or cursors */,
                                                uint32_t* __restrict__ sorted, size_t flat /* 0, or the table's points per window */,
                                                uint32_t slot_base, uint32_t index_base, uint32_t* __restrict__ flags) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8];
    {
        const uint4* q = reinterpret_cast<const uint4*>(scalars + 8 * i);
        uint4 a = __ldg(q), b = __ldg(q + 1);
        s[0] = a.x; s[1] = a.y; s[2] = a.z; s[3] = a.w; s[4] = b.x; s[5] = b.y; s[6] = b.z; s[7] = b.w;
    }
    if (MONT) {
        Fr x;
#pragma unroll
        for (int k = 0; k < 8; k++) x.v[k] = s[k];
        x = x.from_mont();
#pragma unroll
        for (int k = 0; k < 8; k++) s[k] = x.v[k];
    }
    if (!SCATTER && (s[7] >> 29)) atomicOr(flags, 1u);
    uint32_t carry = 0;
    for (int w = 0; w < nwin; w++) {
        const int c = w == nwin - 1 ? c_top : c_low;
        int bit = w * c_low;
        // dynamic register-array indexing would spill: select the two words with a small switch-free scan
        int wi = bit >> 5, sh = bit & 31;
        uint32_t lo = 0, hi = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) { if (k == wi) lo = s[k]; if (k == wi + 1) hi = s[k]; }
        const uint32_t half = 1u << (c - 1);
        uint32_t raw = (__funnelshift_r(lo, hi, sh) & ((1u << c) - 1u)) + carry;
        uint32_t neg = raw > half ? 1u : 0u;
        uint32_t mag = neg ? (1u << c) - raw : raw;
        carry = neg;
        if (mag != 0u) {
            uint32_t slot = slot_base + (flat ? 0u : (uint32_t)w * nbuckets) + (mag - 1u);
            if (SCATTER) {
                uint32_t pos = atomicAdd(&counters[slot], 1u);
                sorted[pos] = (uint32_t)(flat ? (size_t)w * flat + i : (size_t)index_base + i) | (neg << 31);
            } else {
                atomicAdd(&counters[slot], 1u);
            }
        }
    }
}

__global__ void k_items_per_bucket(const uint32_t* __restrict__ hist, uint32_t* __restrict__ items, uint32_t total_buckets, uint32_t cap,
                                   uint32_t* __restrict__ hot /* may be null; hot[0] = count, hot[1 …] = buckets with more than `keep` items */, uint32_t hot_max,
                                   uint32_t keep) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total_buckets) {
        const uint32_t it = (hist[i] + cap - 1u) / cap;
        items[i] = it;
        if (hot != nullptr && it > keep) { const uint32_t pos = atomicAdd(hot, 1u); if (pos < hot_max) hot[1u + pos] = i; }
    } else if (i == total_buckets) items[i] = 0;
}

// Dense points are 96 B (x, y Montgomery); infinity is encoded as (0, 0), which is not on y² = x³ + 1.
static constexpr int DENSE_WORDS = 24;
static constexpr int BASE_WORDS = 32;       // level-0 copy of the bases: 96 B padded to one 128-byte line per point

struct DensePoint { Fq x, y; bool inf; };
FF_DEV DensePoint load_dense(const uint32_t* p) {
    DensePoint d; d.x = Fq::load_ldg(p); d.y = Fq::load_ldg(p + 12);
    d.inf = d.x.is_zero() && d.y.is_zero();
    return d;
}
FF_DEV void store_dense(uint32_t* p, const DensePoint& d) {
    if (d.inf) { Fq z = Fq::zero(); z.store(p); z.store(p + 12); }
    else { d.x.store(p); d.y.store(p + 12); }
}
// Sort pass of the pair-level path (round 2): instead of an index array that level 0 would have to chase through a
// random gather (ncu: the gathering level ran the multiplier well below the dense levels —
// 32 DRAM lines per LDGSTS instruction, MIO and scoreboard stalls with only 4 warps per scheduler to hide them), the
// scatter writes the RECORDS themselves: point i is read once, and for every window its 96-byte (x, ±y) image goes to the
// slot the bucket cursor hands out.  Level 0 then reads a dense, already signed array exactly like the levels above it.
// The CTA stages its 256 points (x, y, −y) in shared memory and writes each window's records cooperatively, consecutive
// lanes per record, so a store instruction touches 4–6 lines instead of 32.
// rec_words = BASE_WORDS (plain bases, calls of at least REC_LINE_MIN_ENTRIES entries): every record is one whole, aligned
// 128-byte line (x, ±y, 32 B of zeros) written by eight lanes.  At the 96-byte stride (DENSE_WORDS, six lanes) a record covers
// half of a 64-byte unit that the next slot of its bucket fills later from another CTA; in a large call the halves rarely
// meet in L2, and the partial writes cost more than the 33 % extra bytes (H100 SXM at 400 W, 2^24 points, 14 windows: the
// stores alone take 16.6 ms at 96 B and 13.5 ms at 128 B; DESIGN §4).
// FLAT (precomputed tables): window w of point i takes record w·table_n + i of the table (staged per window) and every window
// feeds the job's single bucket set.
// Windows [w_lo, w_hi) of this segment belong to the current group of bucket sets; positions are relative to *pos_base.
static constexpr uint32_t REC_NONE = 0xffffffffu;
// Below this many entries per call, 128-byte records lose to 96-byte ones.  The stores alone per record
// (tools/scatter_probe.py, H100 SXM at 400 W, 14 windows): 96-byte records are 15–23 % faster at 2^14–2^16 points, the two
// tie at 2^18 points (3.7 M entries), and 128-byte records are 16–18 % faster from 2^20 points.  The default plans run pair
// levels from 2^19 points (≥ 10 M entries); smaller calls get here only with forced levels.  The tables' records (FLAT)
// always keep 96 B: one job's table scratch cannot be split into groups and already fills most of the device next to the
// tables.
static constexpr size_t REC_LINE_MIN_ENTRIES = (size_t)1 << 22;
// one window's records of the CTA's 256 points, LANES 16-byte granules per record (6, or 8 with the zero tail).
// The whole lines are stored evict-first (st.global.cs): nothing reads them before level 0, long after they have left L2,
// and with ordinary stores 30 GB of records push the bucket cursors (2.2 M × 4 B at 2^24) out of L2, where every cursor
// atomic needs them (H100 SXM at 700 W, 2^24 points: the scatter 16.4 → 14.2 ms; the stores alone stay at 13.5 ms).  The
// 96-byte records keep ordinary stores: their two halves of a 64-byte unit must meet in L2.
template <uint32_t LANES>
FF_DEV void emit_records(const uint4* sh_rec, const uint32_t* my_pos, uint32_t tid, uint4* __restrict__ dense0) {
    for (uint32_t k = tid; k < 256u * LANES; k += 256u) {
        const uint32_t r = k / LANES, part = k - LANES * r;
        const uint32_t pp = my_pos[r];
        if (pp == REC_NONE) continue;
        const uint32_t src = part < 3u ? part : ((pp >> 31) ? 3u : 0u) + part;       // x0..2 | y0..2 or (−y)0..2
        const uint4 v = part < 6u ? sh_rec[r * 9u + src] : make_uint4(0u, 0u, 0u, 0u);
        uint4* d = dense0 + (size_t)(pp & 0x7fffffffu) * LANES + part;
        if (LANES == 8u) __stcs(d, v);
        else *d = v;
    }
}
template <bool MONT, bool FLAT>
__global__ void __launch_bounds__(256) k_scatter_records(const uint32_t* __restrict__ scalars, size_t n, const uint8_t* __restrict__ points,
                                                         size_t stride, const uint32_t* __restrict__ table, size_t table_n, int c_low, int c_top,
                                                         int nwin, uint32_t nbuckets,
                                                         uint32_t* __restrict__ cursors, uint32_t slot_base, int w_lo, int w_hi,
                                                         const uint32_t* __restrict__ pos_base_ptr, uint4* __restrict__ dense0,
                                                         uint32_t rec_words) {
    __shared__ uint4 sh_rec[256 * 9];                       // per point: x (3 × 16 B), y (3), −y (3)
    __shared__ uint32_t sh_pos[2][256];
    const uint32_t tid = threadIdx.x;
    const size_t i = (size_t)blockIdx.x * 256 + tid;
    const bool live = i < n;
    const uint32_t pos_base = __ldg(pos_base_ptr);
    uint32_t s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = 0u;
    auto stage = [&](Fq x, Fq y, bool inf) {
        Fq yn = y.neg();
        if (inf) { x = Fq::zero(); y = Fq::zero(); yn = Fq::zero(); }      // (0, 0) is the dense encoding of infinity
        uint4* r = sh_rec + tid * 9;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            r[k] = make_uint4(x.v[4 * k], x.v[4 * k + 1], x.v[4 * k + 2], x.v[4 * k + 3]);
            r[3 + k] = make_uint4(y.v[4 * k], y.v[4 * k + 1], y.v[4 * k + 2], y.v[4 * k + 3]);
            r[6 + k] = make_uint4(yn.v[4 * k], yn.v[4 * k + 1], yn.v[4 * k + 2], yn.v[4 * k + 3]);
        }
    };
    if (live) {
        const uint4* q = reinterpret_cast<const uint4*>(scalars + 8 * i);
        uint4 a = __ldg(q), b = __ldg(q + 1);
        s[0] = a.x; s[1] = a.y; s[2] = a.z; s[3] = a.w; s[4] = b.x; s[5] = b.y; s[6] = b.z; s[7] = b.w;
        if (MONT) {
            Fr x;
#pragma unroll
            for (int k = 0; k < 8; k++) x.v[k] = s[k];
            x = x.from_mont();
#pragma unroll
            for (int k = 0; k < 8; k++) s[k] = x.v[k];
        }
        if (!FLAT) {
            AffinePoint pt = load_affine(points, stride, i);
            stage(pt.x, pt.y, pt.inf);
        }
    }
    uint32_t carry = 0;
    // One window at a time (issuing the cursor atomics of 8 windows back to back before one barrier was measured slower at
    // 2^24 — co-resident CTAs in different phases already overlap).
    for (int w = 0; w < w_hi; w++) {
        const int c = w == nwin - 1 ? c_top : c_low;          // (k_digits)
        const int bit = w * c_low, wi = bit >> 5, sh = bit & 31;
        uint32_t lo = 0, hi = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) { if (k == wi) lo = s[k]; if (k == wi + 1) hi = s[k]; }
        const uint32_t half = 1u << (c - 1);
        const uint32_t raw = (__funnelshift_r(lo, hi, sh) & ((1u << c) - 1u)) + carry;
        const uint32_t neg = raw > half ? 1u : 0u;
        const uint32_t mag = neg ? (1u << c) - raw : raw;
        carry = neg;
        if (w < w_lo) continue;
        if (FLAT) {
            if (w > w_lo) __syncthreads();                  // the previous window's records have been written out
            if (live && mag != 0u) {
                const DensePoint d = load_dense(table + ((size_t)w * table_n + i) * BASE_WORDS);
                stage(d.x, d.y, d.inf);
            }
        }
        uint32_t pos = REC_NONE;
        if (live && mag != 0u) pos = (atomicAdd(&cursors[slot_base + (FLAT ? 0u : (uint32_t)w * nbuckets) + (mag - 1u)], 1u) - pos_base) | (neg << 31);
        uint32_t* my_pos = sh_pos[w & 1];
        my_pos[tid] = pos;
        __syncthreads();                                    // also orders the staging of sh_rec before the reads
        if (!FLAT && rec_words == (uint32_t)BASE_WORDS) emit_records<8>(sh_rec, my_pos, tid, dense0);
        else emit_records<6>(sh_rec, my_pos, tid, dense0);
        // the next window writes the other half of sh_pos; its barrier orders this window's reads before the window after
    }
}

// A dense base record: x, y (Montgomery) in one 128-byte line, infinity encoded as (0, 0) — written by k_densify_bases
// (per call) or k_precompute_tables (per SRS).
FF_DEV AffinePoint load_record(const uint32_t* __restrict__ records, uint32_t idx) {
    const uint32_t* p = records + (size_t)idx * 32;
    AffinePoint a;
    a.x = Fq::load_ldg(p); a.y = Fq::load_ldg(p + 12);
    a.inf = a.x.is_zero() && a.y.is_zero();
    return a;
}
// One thread per work item (a run of ≤ cap sorted entries of one bucket): XYZZ mixed additions
// of gathered affine bases.  partial[item] receives the item's sum.
// 128-thread CTAs, 4 per SM (≤ 128 registers/thread, a few hundred bytes of spill): measured faster at 2^24 points
// than 256×1 at 207 registers.  The kernel is bound by
// the IMAD pipe, and 16 warps/SM hide its latency better than 8.
#ifndef MSM_ACC_THREADS
#define MSM_ACC_THREADS 128
#define MSM_ACC_MINBLOCKS 4
#endif
__global__ void __launch_bounds__(MSM_ACC_THREADS, MSM_ACC_MINBLOCKS) k_bucket_accumulate(const uint32_t* __restrict__ records /* 128-byte dense bases or table */,
                                                            const uint32_t* __restrict__ sorted,
                                                            const uint32_t* __restrict__ bucket_start /* [TB+1] */,
                                                            const uint32_t* __restrict__ item_start /* [TB+1] */,
                                                            uint32_t total_buckets, uint32_t cap, uint32_t* __restrict__ partial) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t total_items = item_start[total_buckets];
    if (t >= total_items) return;
    // upper_bound(item_start, t) - 1 : the bucket whose item range contains t
    uint32_t lo = 0, hi = total_buckets;          // invariant: item_start[lo] <= t < item_start[hi]
    while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (item_start[mid] <= t) lo = mid; else hi = mid;
    }
    uint32_t wb = lo;
    uint32_t seg = t - item_start[wb];
    uint32_t b0 = bucket_start[wb], b1 = bucket_start[wb + 1];
    uint32_t s0 = b0 + seg * cap;
    uint32_t s1 = s0 + cap < b1 ? s0 + cap : b1;

    XYZZ acc = XYZZ::infinity();
    // software pipeline: fetch entry k+1 while adding entry k
    uint32_t e = sorted[s0];
    AffinePoint p = load_record(records, e & 0x7fffffffu);
    for (uint32_t k = s0; k < s1; k++) {
        uint32_t e_cur = e;
        AffinePoint p_cur = p;
        if (k + 1 < s1) { e = sorted[k + 1]; p = load_record(records, e & 0x7fffffffu); }
        acc.add_affine(p_cur, (e_cur >> 31) != 0u);
    }
    acc.store(partial + (size_t)t * XYZZ_WORDS);
}

// =================================================================================================
// Batched-affine pair levels (the reference's own idea — batch_add, batched.rs:175-325: pair up the
// points of a bucket, add all pairs with ONE field inversion per batch via Montgomery's trick,
// affine.rs:224-273 — restated for the GPU).  One level halves every bucket: output element i of a
// bucket is in[2i] + in[2i+1] (or a copy of in[2i] when the count is odd).  A lane owns T pairs (across
// bucket boundaries, so hot buckets are spread over many lanes), walks them forward accumulating the
// running product of the denominators (x2 − x1, or 2·y1 for a doubling) into `prefix`, takes one
// inversion shared by its CTA (cta_inverse.cuh), then walks them backward peeling off one inverse per
// pair: 6 Fq mul per addition instead of 10 for an XYZZ mixed add.
// Dense points are 96 B (x, y Montgomery); infinity is encoded as (0, 0), which is not on y² = x³ + 1.
// =================================================================================================
// Without pair levels, the XYZZ accumulation gathers its inputs through `sorted` from a dense, 128-byte-aligned copy of the
// bases made once per call by k_densify_bases: a gathered point then costs one DRAM line instead of the two or three that
// the reference's 104-byte stride straddles.
__global__ void k_densify_bases(const uint8_t* __restrict__ points, size_t stride, size_t n, uint32_t* __restrict__ out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    AffinePoint a = load_affine(points, stride, i);
    DensePoint d; d.x = a.x; d.y = a.y; d.inf = a.inf;
    store_dense(out + i * BASE_WORDS, d);
}
// Precomputed tables for resident bases: record (w, i) = 2^{c·w}·P_i as a dense 128-byte affine record, w < nwin.
// One thread per point walks the doubling chain in XYZZ; every multiple is normalised with ONE field inversion shared by
// the 128 threads of the CTA (cta_inverse.cuh) instead of a Fermat ladder per record: ≈ 9·c + 12 Fq mul per record instead of
// 9·c + 580 (round 1: 6.3 s for the 2^24-point tables).
__global__ void __launch_bounds__(CTA_INV_THREADS) k_precompute_tables(const uint8_t* __restrict__ points, size_t stride, size_t n, int c, int nwin,
                                                            uint32_t* __restrict__ table) {
    __shared__ uint4 sh_inv[CTA_INV_SMEM_BYTES / 16];
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < n;
    AffinePoint a;
    a.x = Fq::zero(); a.y = Fq::zero(); a.inf = true;
    if (live) a = load_affine(points, stride, i);
    DensePoint d; d.x = a.x; d.y = a.y; d.inf = a.inf;
    if (live) store_dense(table + i * BASE_WORDS, d);
    XYZZ q = XYZZ::from_affine(a);
    for (int w = 1; w < nwin; w++) {
        for (int k = 0; k < c; k++) q.dbl();
        const bool inf = q.is_inf();
        Fq z = inf ? Fq::one() : q.ZZ * q.ZZZ;
        Fq iz = cta_shared_inverse_by(z, reinterpret_cast<uint32_t*>(sh_inv), w & 3);
        __syncthreads();                                    // the next round overwrites the shared area
        if (inf) { d.x = Fq::zero(); d.y = Fq::zero(); d.inf = true; }
        else { d.x = q.X * (iz * q.ZZZ); d.y = q.Y * (iz * q.ZZ); d.inf = false; }
        if (live) store_dense(table + ((size_t)w * n + i) * BASE_WORDS, d);
    }
}

static constexpr int PAIR_THREADS = CTA_INV_THREADS;
// Resident CTAs per SM that k_pair_level2 is built for (128 registers per thread) and that the host sizes its waves by when a
// group's pair levels have the GPU to themselves (half as many while another window group is in flight, msm_core).
static constexpr int PAIR_MIN_BLOCKS = 4;
// The pair-level kernels run as k_pair_desc<false> and k_pair_level2<false, PAIR_MIN_BLOCKS>, their only instances.  Their
// template arguments keep the kernel names that profiles and the MSM path tests identify the pair levels by; the bool
// selects nothing.
enum PairKind { PAIR_COPY1 = 0, PAIR_COPY2 = 1, PAIR_INF = 2, PAIR_ADD = 3, PAIR_DBL = 4 };
FF_DEV int classify_pair(const DensePoint& P, const DensePoint& Q, Fq& d) {
    if (Q.inf) return PAIR_COPY1;
    if (P.inf) return PAIR_COPY2;
    if (P.x == Q.x) {
        if (P.y == Q.y && !P.y.is_zero()) { d = P.y.dbl(); return PAIR_DBL; }
        return PAIR_INF;                                   // P + (−P)  (or a 2-torsion point doubled)
    }
    d = Q.x - P.x;
    return PAIR_ADD;
}

// =================================================================================================
// The pair level kernel: warp-interleaved steps and a shared-memory operand ring.
//
// A WARP owns 32·T consecutive pairs and lane l takes pairs W0 + 32·j + l, j < T — any partition works for Montgomery's
// trick.  A lane that owned T consecutive pairs instead would make the 32 lanes of every load touch 32 different DRAM
// pages / L1 lines (ncu: 2.5–4.3 long-scoreboard stall cycles per issued instruction at 65–72 % of the multiplier pipe);
// interleaved, the descriptors, prefix[] and the dense inputs/outputs of a step are contiguous across the warp.  The
// operands of later steps are already on their way into shared memory (cp.async / LDGSTS, 16-byte granules into a
// per-warp [stage][chunk][lane] ring, conflict-free for LDS.128) while the current step multiplies: a descriptor is
// loaded one step before its copies are issued, the copies run three steps ahead in the forward pass and one in the
// backward pass, and the multiplier calls read their operands from shared memory when they need them, so nothing but
// the running inverse is live across a call.  Each record crosses DRAM once per pass (forward: x only; backward: x and
// y); prefix products go to HBM coalesced (48 B per pair) and come back one step late behind the first multiplication
// of the step.
// =================================================================================================
FF_DEV uint32_t smem_addr_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
FF_DEV void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
FF_DEV void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
FF_DEV void cp_async_wait_1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }
FF_DEV void cp_async_wait_0() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
FF_DEV void cp_async_wait_3() { asm volatile("cp.async.wait_group 3;" ::: "memory"); }

static constexpr int RING_CHUNKS = 12;                       // x1 y1 x2 y2, three 16-byte chunks each
static constexpr int RING_STAGE_U4 = RING_CHUNKS * 32;       // uint4 per warp per stage (6 KiB)
static constexpr int PAIR2_SMEM = PAIR_THREADS * 48 + 4 * 2 * RING_STAGE_U4 * 16;   // shared inversion + 4 warps × 2 stages

FF_DEV Fq ring_fq(const uint4* slot) {                       // slot = &ring[(stage·12 + first chunk)·32 + lane]
    Fq r;
#pragma unroll
    for (int i = 0; i < 3; i++) { uint4 t = slot[i * 32]; r.v[4 * i] = t.x; r.v[4 * i + 1] = t.y; r.v[4 * i + 2] = t.z; r.v[4 * i + 3] = t.w; }
    return r;
}

// Bucket search for a warp of consecutive indices.  `off` is an exclusive scan over nb buckets (off[nb] = total) and every
// lane holds an index x < off[nb], nondecreasing across the lanes; the lane's bucket is the largest b with off[b] <= x.
// warp_bucket_first: one binary search for a warp-uniform x (every lane walks the same path, so each step is one broadcast
// load).  warp_bucket_walk: from a warp-uniform bucket b with off[b] <= x on every lane, lane l loads off[b + 1 + l] and
// counts the boundaries at or below its x with a five-step shuffle search over the warp — one load per 32 buckets, so buckets
// smaller than a warp and buckets of millions of entries cost the same.  Lanes still past the 32 loaded boundaries after two
// rounds (long runs of empty buckets) finish with their own binary search.
FF_DEV uint32_t warp_bucket_first(const uint32_t* __restrict__ off, uint32_t nb, uint32_t x) {
    uint32_t lo = 0, hi = nb;                             // off[lo] <= x < off[hi]
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(off + mid) <= x) lo = mid; else hi = mid; }
    return lo;
}
FF_DEV uint32_t warp_bucket_walk(const uint32_t* __restrict__ off, uint32_t nb, uint32_t b, uint32_t x) {
    const int lane = threadIdx.x & 31;
    uint32_t res = b;
    bool done = false;
    for (int round = 0;; round++) {
        const uint32_t k = b + 1u + (uint32_t)lane;
        const uint32_t e = k <= nb ? __ldg(off + k) : 0xffffffffu;
        uint32_t c = 0;                                   // boundaries off[b + 1 … b + c] <= x  (c ≤ 31 here)
#pragma unroll
        for (uint32_t s = 16; s >= 1; s >>= 1)
            if (__shfl_sync(0xffffffffu, e, (int)(c + s - 1u)) <= x) c += s;
        const uint32_t e31 = __shfl_sync(0xffffffffu, e, 31);
        if (!done && e31 > x) { res = b + c; done = true; }
        if (__all_sync(0xffffffffu, done)) return res;
        b += 32u;                                         // off[b] = e31 <= x on every lane not done
        if (round == 1) break;
    }
    if (!done) { uint32_t lo = b, hi = nb; while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(off + mid) <= x) lo = mid; else hi = mid; } res = lo; }
    return res;
}

// Pair descriptors, written once per level by k_pair_desc so that the pair kernel never chases off_out → off_in → sorted in
// its instruction stream: it reads 8 bytes per pair, coalesced, two steps ahead.  Only real pairs (both inputs present) get a
// descriptor and a lane step: pair j of the level is the i-th pair of its bucket b, i = j − pair_off[b] (pair_off = scan of
// ⌊cnt/2⌋), its inputs are off_in[b] + 2i and the one after, and it writes output off_out[b] + i (off_out = scan of ⌈cnt/2⌉,
// so the output layout is that of all outputs, the pairs of a bucket first).  desc[j] = (index of the first input in the
// level's dense input, output position).
// The single input of a bucket with an odd count is not a step: the same kernel copies it to the bucket's last output.
static constexpr int DESC_CHUNKS = 8;                    // 32-pair chunks per warp: one binary search per 256 pairs
template <bool>
__global__ void __launch_bounds__(256) k_pair_desc(const uint32_t* __restrict__ off_in,
                                                   const uint32_t* __restrict__ off_out, const uint32_t* __restrict__ pair_off,
                                                   uint32_t total_buckets, uint2* __restrict__ desc,
                                                   const uint32_t* __restrict__ in_base_ptr /* *in_base_ptr = position of element 0, or null */,
                                                   const uint32_t* __restrict__ records, uint32_t in_words, uint32_t* __restrict__ dense_out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t in_base = in_base_ptr ? __ldg(in_base_ptr) : 0u;
    // ---- single inputs: one thread per bucket ----
    if (t < total_buckets) {
        const uint32_t end = __ldg(off_in + t + 1);
        if ((end - __ldg(off_in + t)) & 1u) {
            const uint32_t idx = end - 1u;
            const DensePoint P = load_dense(records + (size_t)(idx - in_base) * in_words);
            store_dense(dense_out + (size_t)(__ldg(off_out + t + 1) - 1u) * DENSE_WORDS, P);
        }
    }
    // ---- pairs: 32 · DESC_CHUNKS consecutive ones per warp ----
    const uint32_t total = __ldg(pair_off + total_buckets);
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t j0_64 = (uint64_t)(t >> 5) * (32u * DESC_CHUNKS);
    if (j0_64 >= total) return;                           // warp-uniform
    uint32_t j0 = (uint32_t)j0_64;
    uint32_t b = warp_bucket_first(pair_off, total_buckets, j0);
    for (int c = 0; c < DESC_CHUNKS && j0 < total; c++, j0 += 32u) {
        const uint32_t j = j0 + lane < total ? j0 + lane : total - 1u;
        const uint32_t bj = warp_bucket_walk(pair_off, total_buckets, b, j);
        b = __shfl_sync(0xffffffffu, bj, 31);             // the next chunk starts at or after the last lane's bucket
        if (j0 + lane < total) {
            const uint32_t i = j - __ldg(pair_off + bj);
            const uint32_t idx = __ldg(off_in + bj) + 2u * i, o = __ldg(off_out + bj) + i;
            desc[j] = make_uint2(idx - in_base, o);
        }
    }
}

struct PairDesc {            // one lane's pair of one step
    uint32_t p, o;           // first input (the second is p + 1) and output position as written by k_pair_desc — possibly
                             // still in flight: only touch them when the step is issued / computed
    bool valid;              // the pair exists (known from the indices alone, never from loaded data)
};
// descriptor of step j for this lane (dlane = desc + W0 + lane); steps outside [0, nv) do not exist
FF_DEV PairDesc pair_load_desc(int64_t j, uint32_t nv, const uint2* __restrict__ dlane) {
    PairDesc d; d.p = 0; d.o = 0; d.valid = false;
    if (j < 0 || j >= (int64_t)nv) return d;
    const uint2 v = __ldg(dlane + 32 * j);
    d.p = v.x; d.o = v.y; d.valid = true;
    return d;
}
// in_words: stride of the dense inputs — the call's record stride at level 0 (BASE_WORDS or DENSE_WORDS, see
// REC_LINE_MIN_ENTRIES), DENSE_WORDS above
FF_DEV const uint32_t* pair_src(const PairDesc& d, int which, const uint32_t* __restrict__ records, uint32_t in_words) {
    return records + (size_t)(d.p + (uint32_t)which) * in_words;
}
// copies of step operands into ring stage `st` of `chunks` 16-byte chunks per lane: backward (FULL) x1 y1 x2 y2 in 12 chunks,
// forward x1 x2 in 6 chunks
template <bool FULL>
FF_DEV void pair_issue(const PairDesc& d, uint4* ring, int st, int lane, const uint32_t* __restrict__ records, uint32_t in_words, int chunks) {
    if (d.valid) {
        const uint32_t dst = smem_addr_u32(ring + (size_t)st * (size_t)(chunks * 32) + lane);
        const uint32_t* p = pair_src(d, 0, records, in_words);
#pragma unroll
        for (int k = 0; k < (FULL ? 6 : 3); k++) cp_async16(dst + (uint32_t)k * 512u, p + 4 * k);
        const uint32_t* q = pair_src(d, 1, records, in_words);
#pragma unroll
        for (int k = 0; k < (FULL ? 6 : 3); k++) cp_async16(dst + (uint32_t)((FULL ? 6 : 3) + k) * 512u, q + 4 * k);
    }
    cp_async_commit();
}
// full classification of one pair from global memory (rare path of the forward pass: equal x, or an x that is 0)
FF_DEV int pair_classify_global(const PairDesc& d, const uint32_t* __restrict__ records, uint32_t in_words, Fq& den) {
    const DensePoint P = load_dense(pair_src(d, 0, records, in_words));
    const DensePoint Q = load_dense(pair_src(d, 1, records, in_words));
    return classify_pair(P, Q, den);
}

// The shared inversion is a bubble — one warp works while the CTA's other warps wait at the barrier, and CTAs that start
// together reach it together — so (i) the inverting warp computes ONE inverse limb-per-lane (coop_inverse, ff.cuh) instead
// of 32 redundant copies, and (ii) every CTA takes a slot number from a per-SM counter: slot & 3 names the inverting warp, so
// the CTAs resident on an SM invert on different sub-partitions whatever the block → SM mapping is.
template <bool, int MINB>
__global__ void __launch_bounds__(PAIR_THREADS, MINB) k_pair_level2(const uint32_t* __restrict__ records /* the level's dense input */,
                                                         uint32_t in_words, const uint2* __restrict__ desc,
                                                         const uint32_t* __restrict__ total_ptr,
                                                         uint32_t T_bound, uint32_t* __restrict__ prefix, uint32_t* __restrict__ dense_out,
                                                         uint32_t* __restrict__ sm_slots) {
    (void)T_bound;
    extern __shared__ uint4 pair2_smem[];
    __shared__ uint32_t sh_slot;
    uint32_t* sh_inv = reinterpret_cast<uint32_t*>(pair2_smem);                       // 128 × 48 B
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint4* ring = pair2_smem + PAIR_THREADS * 3 + (size_t)warp * 2 * RING_STAGE_U4;    // this warp's two stages
    if (threadIdx.x == 0) {
        uint32_t smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        sh_slot = atomicAdd(sm_slots + (smid & 255u), 1u);
    }
    __syncthreads();
    const int inv_warp = (int)(sh_slot & 3u);
    const uint32_t total = __ldg(total_ptr);
    // Steps per lane from the level's ACTUAL pair count: the host sizes the grid (whole waves) from an upper bound, Σ cnt/2,
    // and every lane walks all T steps, so T from the bound would make the whole grid that much slower.  Any partition works
    // for Montgomery's trick and the outputs do not depend on it.
    const uint64_t lanes = (uint64_t)gridDim.x * PAIR_THREADS;
    const uint32_t T = total > lanes ? (uint32_t)((total + lanes - 1) / lanes) : 1u;      // ≤ T_bound
    const uint64_t w0_64 = ((uint64_t)blockIdx.x * (PAIR_THREADS / 32) + (uint32_t)warp) * 32ull * T + (uint32_t)lane;   // this lane's first pair
    uint32_t nv = 0;                                                                   // steps that exist for this lane
    if (w0_64 < total) { const uint64_t left = (total - w0_64 + 31) / 32; nv = left < T ? (uint32_t)left : T; }
    const uint2* dlane = desc + w0_64;
    uint32_t* plane = prefix + w0_64 * 12;                                             // prefix of step j at plane + j·32·12

    // ---------------- forward: running product of the denominators ----------------
    // A forward step is ONE multiplication, far shorter than a DRAM access: the x-only operands (96 B per lane) fit
    // FOUR ring stages where the backward pass has two, so the copies run three steps ahead of the multiplier
    // (ncu, round 2: with one step of lead the forward loop held 21 % of the kernel's stall samples for 4 % of its instructions).
    Fq run = Fq::one();
    {
        constexpr int PF = 3;                                                   // steps of lead; PF + 1 stages of 6 chunks
        PairDesc q0 = pair_load_desc(0, nv, dlane), q1 = pair_load_desc(1, nv, dlane), q2 = pair_load_desc(2, nv, dlane);
        pair_issue<false>(q0, ring, 0, lane, records, in_words, 6);
        pair_issue<false>(q1, ring, 1, lane, records, in_words, 6);
        pair_issue<false>(q2, ring, 2, lane, records, in_words, 6);
        PairDesc ahead = pair_load_desc(PF, nv, dlane);
        for (uint32_t j = 0; j < T; j++) {
            pair_issue<false>(ahead, ring, (int)((j + PF) & 3u), lane, records, in_words, 6);       // step j+3 (descriptor loaded a step ago)
            const PairDesc cur = q0;
            q0 = q1; q1 = q2; q2 = ahead;
            ahead = pair_load_desc((int64_t)j + PF + 1, nv, dlane);                             // not touched until the next iteration
            cp_async_wait_3();
            Fq d = Fq::one();
            if (cur.valid) {
                const uint4* slot_p = ring + (size_t)(j & 3u) * (6 * 32) + lane;
                Fq x1 = ring_fq(slot_p), x2 = ring_fq(slot_p + 3 * 32);
                if (x1 == x2 || x1.is_zero() || x2.is_zero()) {
                    Fq den;
                    if (pair_classify_global(cur, records, in_words, den) >= PAIR_ADD) d = den;
                } else {
                    d = x2 - x1;
                }
            }
            run = run * d;
            if (cur.valid) run.store(plane + (size_t)j * (32 * 12));
        }
        cp_async_wait_0();
    }
    Fq inv = cta_shared_inverse_by(run, sh_inv, inv_warp);
    // ---------------- backward: one inverse per pair, then the affine addition ----------------
    {
        PairDesc cur = pair_load_desc((int64_t)T - 1, nv, dlane);
        pair_issue<true>(cur, ring, 0, lane, records, in_words, 12);
        PairDesc nxt = pair_load_desc((int64_t)T - 2, nv, dlane);
        for (uint32_t k = 0; k < T; k++) {
            const uint32_t j = T - 1 - k;
            pair_issue<true>(nxt, ring, (int)((k + 1) & 1u), lane, records, in_words, 12);
            PairDesc nn = pair_load_desc((int64_t)j - 2, nv, dlane);
            Fq pf = Fq::one();
            if (cur.valid && j != 0) pf = Fq::load(plane + (size_t)(j - 1) * (32 * 12));     // behind the first multiplication
            cp_async_wait_1();
            const uint4* slot_p = ring + (size_t)(k & 1u) * RING_STAGE_U4 + lane;
            // classify (same decisions as the forward pass); a step that does not exist multiplies by one and stores nothing
            int kind = PAIR_COPY1;
            Fq d = Fq::one(), num = Fq::zero();
            if (cur.valid) {
                Fq x1 = ring_fq(slot_p), x2 = ring_fq(slot_p + 6 * 32);
                if (x1 == x2 || x1.is_zero() || x2.is_zero()) {
                    DensePoint P, Q;
                    P.x = x1; P.y = ring_fq(slot_p + 3 * 32); P.inf = P.x.is_zero() && P.y.is_zero();
                    Q.x = x2; Q.y = ring_fq(slot_p + 9 * 32); Q.inf = Q.x.is_zero() && Q.y.is_zero();
                    Fq den;
                    kind = classify_pair(P, Q, den);
                    if (kind >= PAIR_ADD) d = den;
                    if (kind == PAIR_ADD) num = Q.y - P.y;
                    else if (kind == PAIR_DBL) { Fq xx = P.x.sqr(); num = xx.dbl() + xx; }
                } else {
                    kind = PAIR_ADD;
                    d = x2 - x1;
                    const Fq y1 = ring_fq(slot_p + 3 * 32), y2 = ring_fq(slot_p + 9 * 32);
                    num = y2 - y1;
                }
            }
            Fq inv_next = inv * d;
            Fq inv_d = (j != 0) ? inv * pf : inv;
            inv = inv_next;
            Fq lambda = num * inv_d;
            Fq x3 = lambda.sqr();
            {
                Fq x1 = ring_fq(slot_p), x2 = ring_fq(slot_p + 6 * 32);
                x3 = x3 - x1 - x2;
                Fq t = x1 - x3;
                Fq y3 = lambda * t;
                if (cur.valid) {
                    DensePoint R;
                    if (kind >= PAIR_ADD) {
                        Fq y1 = ring_fq(slot_p + 3 * 32);
                        R.x = x3; R.y = y3 - y1; R.inf = false;
                    } else if (kind == PAIR_INF) {
                        R.inf = true; R.x = Fq::zero(); R.y = Fq::zero();
                    } else {
                        const int c0 = (kind == PAIR_COPY2) ? 6 : 0;
                        R.x = ring_fq(slot_p + c0 * 32); R.y = ring_fq(slot_p + (c0 + 3) * 32);
                        R.inf = R.x.is_zero() && R.y.is_zero();
                    }
                    store_dense(dense_out + (size_t)cur.o * DENSE_WORDS, R);      // consecutive pairs: consecutive outputs, but for singles between
                }
            }
            cur = nxt; nxt = nn;
        }
        cp_async_wait_0();
    }
}

// a pair level's counts per bucket: outputs ⌈cnt/2⌉ and pairs ⌊cnt/2⌋
__global__ void k_halve_counts(const uint32_t* __restrict__ off_in, uint32_t* __restrict__ cnt_out, uint32_t* __restrict__ pairs_out,
                               uint32_t total_buckets) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total_buckets) { const uint32_t c = off_in[i + 1] - off_in[i]; cnt_out[i] = (c + 1u) >> 1; pairs_out[i] = c >> 1; }
    else if (i == total_buckets) { cnt_out[i] = 0; pairs_out[i] = 0; }
}
__global__ void k_items_from_offsets(const uint32_t* __restrict__ off, uint32_t* __restrict__ items, uint32_t total_buckets, uint32_t cap,
                                     uint32_t* __restrict__ hot, uint32_t hot_max, uint32_t keep) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total_buckets) {
        const uint32_t it = (off[i + 1] - off[i] + cap - 1u) / cap;
        items[i] = it;
        if (hot != nullptr && it > keep) { const uint32_t pos = atomicAdd(hot, 1u); if (pos < hot_max) hot[1u + pos] = i; }
    } else if (i == total_buckets) items[i] = 0;
}

// XYZZ accumulation of what the pair levels left: contiguous dense points, no gather, no signs.
__global__ void __launch_bounds__(MSM_ACC_THREADS, MSM_ACC_MINBLOCKS) k_bucket_accumulate_dense(
    const uint32_t* __restrict__ dense, const uint32_t* __restrict__ bucket_start, const uint32_t* __restrict__ item_start,
    uint32_t total_buckets, uint32_t cap, uint32_t* __restrict__ partial) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t total_items = item_start[total_buckets];
    const uint32_t t0 = t & ~31u;                         // the warp's first item (blockDim is a multiple of 32)
    if (t0 >= total_items) return;                        // warp-uniform: the search below needs the whole warp
    const uint32_t wb = warp_bucket_walk(item_start, total_buckets, warp_bucket_first(item_start, total_buckets, t0),
                                         t < total_items ? t : total_items - 1u);
    if (t >= total_items) return;
    uint32_t seg = t - item_start[wb];
    uint32_t b0 = bucket_start[wb], b1 = bucket_start[wb + 1];
    uint32_t s0 = b0 + seg * cap, s1 = s0 + cap < b1 ? s0 + cap : b1;
    XYZZ acc = XYZZ::infinity();
    DensePoint p = load_dense(dense + (size_t)s0 * DENSE_WORDS);
    for (uint32_t k = s0; k < s1; k++) {
        AffinePoint cur; cur.x = p.x; cur.y = p.y; cur.inf = p.inf;
        if (k + 1 < s1) p = load_dense(dense + (size_t)(k + 1) * DENSE_WORDS);
        acc.add_affine(cur, false);
    }
    acc.store(partial + (size_t)t * XYZZ_WORDS);
}

// Hot buckets (all scalars equal; or the top signed-digit window, which holds only the carry and therefore
// puts ~n/2 points into ONE bucket) produce thousands of item partials for one bucket.  They are folded
// 32 at a time by as many threads as there are groups, pass after pass, until every bucket has one partial.
__global__ void k_group_counts(const uint32_t* __restrict__ start_in, uint32_t* __restrict__ cnt_out, uint32_t total_buckets) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total_buckets) cnt_out[i] = (start_in[i + 1] - start_in[i] + 31u) >> 5;
    else if (i == total_buckets) cnt_out[i] = 0;
}
__global__ void __launch_bounds__(128) k_partial_group_sum(const uint32_t* __restrict__ partial_in, const uint32_t* __restrict__ start_in,
                                                            const uint32_t* __restrict__ start_out, uint32_t total_buckets,
                                                            uint32_t* __restrict__ partial_out) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= start_out[total_buckets]) return;
    uint32_t lo = 0, hi = total_buckets;
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (start_out[mid] <= t) lo = mid; else hi = mid; }
    uint32_t g = t - start_out[lo];
    uint32_t i0 = start_in[lo] + g * 32u, i1 = start_in[lo + 1];
    if (i0 + 32u < i1) i1 = i0 + 32u;
    XYZZ s = XYZZ::load(partial_in + (size_t)i0 * XYZZ_WORDS);
    for (uint32_t i = i0 + 1; i < i1; i++) s.add(XYZZ::load(partial_in + (size_t)i * XYZZ_WORDS));
    s.store(partial_out + (size_t)t * XYZZ_WORDS);
}

// rounds of 32:1 folds a bucket with `cnt` item partials takes until at most `keep` are left
FF_DEV uint32_t fold_rounds_of(uint32_t cnt, uint32_t& final_cnt, uint32_t keep = 32u) {
    uint32_t r = 0;
    while (cnt > keep) { cnt = (cnt + 31u) >> 5; r++; }
    final_cnt = cnt;
    return r;
}

// Σ of a bucket's item partials
FF_DEV XYZZ bucket_sum(const uint32_t* __restrict__ partial, const uint32_t* __restrict__ item_start, uint32_t wb) {
    uint32_t i0 = item_start[wb], i1 = item_start[wb + 1];
    XYZZ s = XYZZ::infinity();
    for (uint32_t i = i0; i < i1; i++) {
        if (i == i0) s = XYZZ::load(partial + (size_t)i * XYZZ_WORDS);
        else s.add(XYZZ::load(partial + (size_t)i * XYZZ_WORDS));
    }
    return s;
}

// Digit offset of the buckets of set `set` of a launch (MsmPlan::set_digit_offset): the sets of the launch are sets set0, set0 + 1, …
// of the call, per_job of them per sum, and set k ≥ 1 above the top window's first set `top_first` holds the digits k·nbuckets + b + 1.
// Its window sum is Σ_b (k·nbuckets + b + 1)·S_b = (the usual Σ_b (b + 1)·S_b) + k·nbuckets·Σ_b S_b.  Uniform plans: all zero.
struct SetOffsets {
    uint32_t set0, per_job, top_first, nbuckets;
    FF_DEV uint32_t of(uint32_t set) const {
        const uint32_t s = (set0 + set) % per_job;
        return s > top_first ? (s - top_first) * nbuckets : 0u;
    }
};
static SetOffsets set_offsets(const MsmPlan& plan, bool flat, uint32_t set0) {
    if (flat) return SetOffsets{0u, 1u, 0u, 0u};
    return SetOffsets{set0, (uint32_t)plan.nsets, (uint32_t)plan.nwin - 1u, plan.nbuckets};
}

// Thread j of window w owns bucket values [lo, hi] = [j·K + 1, (j+1)·K]:
//   running = Σ S_b ; acc = Σ (b − lo + 1)·S_b   (top-down running sum, batched.rs:356-361)
//   out = acc + (lo − 1)·running = Σ b·S_b over the chunk.
// PAIRS: the chunk's entry for the quad-lane combine levels instead — out[2t] = Σ (b − lo + 1)·S_b, out[2t + 1] = Σ S_b — which
// apply the chunk's offset as 8:1 weighted folds (k_combine_level_quad).  The (lo − 1)·running product costs this thread ≈ 24
// more dependent point operations (16 doublings + the additions of lo's bits) on top of its 32: 43 % of the kernel at 2^24 points.
// folds > 0 (PAIRS only): hot buckets were folded down to ONE partial by k_fold_hot_quad (keep = 1); that partial sits at the bucket's
// offset in `partial` or, after an odd number of rounds, in `partial_b`.
template <bool PAIRS>
__global__ void __launch_bounds__(128) k_bucket_reduce(const uint32_t* __restrict__ partial, const uint32_t* __restrict__ item_start,
                                                        uint32_t nbuckets, uint32_t chunk, uint32_t chunks_per_window,
                                                        uint32_t nwin, uint32_t* __restrict__ out,
                                                        const uint32_t* __restrict__ partial_b = nullptr, int folds = 0,
                                                        SetOffsets so = SetOffsets{0u, 1u, 0u, 0u}) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= chunks_per_window * nwin) return;
    uint32_t w = t / chunks_per_window, j = t % chunks_per_window;
    uint32_t lo = j * chunk, hi = lo + chunk;                 // 0-based bucket indices [lo, hi)
    XYZZ running = XYZZ::infinity(), acc = XYZZ::infinity();
    for (uint32_t b = hi; b-- > lo;) {
        XYZZ s;
        if (PAIRS && folds > 0) {
            const uint32_t wb = w * nbuckets + b, i0 = item_start[wb];
            uint32_t cnt = item_start[wb + 1] - i0;
            const uint32_t r = fold_rounds_of(cnt, cnt, 1u);
            s = cnt ? XYZZ::load(((r & 1u) ? partial_b : partial) + (size_t)i0 * XYZZ_WORDS) : XYZZ::infinity();
        } else
            s = bucket_sum(partial, item_start, w * nbuckets + b);
        running.add(s);
        acc.add(running);
    }
    if (PAIRS) {
        acc.store(out + (size_t)t * 2 * XYZZ_WORDS);
        running.store(out + ((size_t)t * 2 + 1) * XYZZ_WORDS);
        return;
    }
    const uint32_t lo_off = lo + so.of(w);                   // bucket value of index lo is lo+1 (+ the set's digit offset)
    if (lo_off != 0u) acc.add(running.mul_u32(lo_off));
    acc.store(out + (size_t)t * XYZZ_WORDS);
}

// out[j] = Σ in[j·group .. min((j+1)·group, per_row)) for each of `rows` independent rows.
__global__ void __launch_bounds__(128) k_group_sum(const uint32_t* __restrict__ in, uint32_t per_row, uint32_t group,
                                                    uint32_t out_per_row, uint32_t rows, uint32_t* __restrict__ out) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= out_per_row * rows) return;
    uint32_t r = t / out_per_row, j = t % out_per_row;
    uint32_t i0 = j * group, i1 = i0 + group < per_row ? i0 + group : per_row;
    XYZZ s = XYZZ::infinity();
    for (uint32_t i = i0; i < i1; i++) s.add(XYZZ::load(in + ((size_t)r * per_row + i) * XYZZ_WORDS));
    s.store(out + (size_t)t * XYZZ_WORDS);
}

// =================================================================================================
// Latency path for small MSMs (≤ 2^18 points: a few thousand buckets, every kernel a handful of CTAs).  A lone thread's Fq
// multiplications are latency-bound, so a chain of 16 mixed additions per work item, 32 + 24 per reduction chunk and 8 per tree
// level dominated the call at 2^12–2^16 points.  Here the chains are cut across lanes:
//   * k_bucket_accumulate_g8 — EIGHT lanes per work item: each lane adds every 8th entry, then a 3-step shuffle butterfly;
//   * the reduction tail below — four lanes per point operation.
// =================================================================================================
FF_DEV XYZZ shfl_xor_xyzz(const XYZZ& a, int m) {
    XYZZ r;
#pragma unroll
    for (int j = 0; j < 12; j++) {
        r.X.v[j] = __shfl_xor_sync(0xffffffffu, a.X.v[j], m); r.Y.v[j] = __shfl_xor_sync(0xffffffffu, a.Y.v[j], m);
        r.ZZ.v[j] = __shfl_xor_sync(0xffffffffu, a.ZZ.v[j], m); r.ZZZ.v[j] = __shfl_xor_sync(0xffffffffu, a.ZZZ.v[j], m);
    }
    return r;
}

static constexpr int ACC_G = 8;
__global__ void __launch_bounds__(128, 4) k_bucket_accumulate_g8(const uint32_t* __restrict__ records, const uint32_t* __restrict__ sorted,
                                                                 const uint32_t* __restrict__ bucket_start, const uint32_t* __restrict__ item_start,
                                                                 uint32_t total_buckets, uint32_t cap, uint32_t* __restrict__ partial) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x, item = t / ACC_G, sub = t % ACC_G;
    const bool valid = item < item_start[total_buckets];
    XYZZ acc = XYZZ::infinity();
    if (valid) {
        uint32_t lo = 0, hi = total_buckets;          // item_start[lo] <= item < item_start[hi]
        while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (item_start[mid] <= item) lo = mid; else hi = mid; }
        const uint32_t seg = item - item_start[lo];
        const uint32_t b0 = bucket_start[lo], b1 = bucket_start[lo + 1];
        const uint32_t s0 = b0 + seg * cap, s1 = s0 + cap < b1 ? s0 + cap : b1;
        uint32_t k = s0 + sub;
        if (k < s1) {
            uint32_t e = sorted[k];
            AffinePoint p = load_record(records, e & 0x7fffffffu);
            for (; k < s1; k += ACC_G) {
                const uint32_t e_cur = e;
                const AffinePoint p_cur = p;
                if (k + ACC_G < s1) { e = sorted[k + ACC_G]; p = load_record(records, e & 0x7fffffffu); }
                acc.add_affine(p_cur, (e_cur >> 31) != 0u);
            }
        }
    }
#pragma unroll 1
    for (int m = ACC_G / 2; m >= 1; m >>= 1) { XYZZ o = shfl_xor_xyzz(acc, m); acc.add(o); }
    if (valid && sub == 0) acc.store(partial + (size_t)item * XYZZ_WORDS);
}

// =================================================================================================
// The reduction tail with FOUR LANES PER POINT (quad.cuh): an XYZZ addition costs 4 dependent multiplications instead of 14.
//   * k_bucket_accumulate_q8 — one WARP per work item: quad s adds every 8th entry (mixed additions), 3-step butterfly
//                              over the eight quads (sizes where the whole problem is a few thousand items);
//   * k_bucket_reduce_quad   — one warp per 8 buckets: 3-step suffix scan + 3-step sum give (Σ (l+1)·S_l, Σ S_l);
//   * k_window_combine_quad  — one CTA per bucket set folds the (acc, run) entries 8 at a time, level after level in
//                              shared memory: acc' = Σ acc_s + w·Σ s·run_s, run' = Σ run_s for entries spanning w buckets.
// =================================================================================================
FF_DEV XYZZ load_xyzz_plain(const uint32_t* p) {              // global or shared memory, 16-byte aligned
    XYZZ r; const uint4* q = reinterpret_cast<const uint4*>(p);
    uint32_t w[XYZZ_WORDS];
#pragma unroll
    for (int i = 0; i < XYZZ_WORDS / 4; i++) { const uint4 t = q[i]; w[4 * i] = t.x; w[4 * i + 1] = t.y; w[4 * i + 2] = t.z; w[4 * i + 3] = t.w; }
#pragma unroll
    for (int j = 0; j < 12; j++) { r.X.v[j] = w[j]; r.Y.v[j] = w[12 + j]; r.ZZ.v[j] = w[24 + j]; r.ZZZ.v[j] = w[36 + j]; }
    return r;
}
FF_DEV void store_xyzz_plain(uint32_t* p, const XYZZ& a) {
    uint4* q = reinterpret_cast<uint4*>(p);
    uint32_t w[XYZZ_WORDS];
#pragma unroll
    for (int j = 0; j < 12; j++) { w[j] = a.X.v[j]; w[12 + j] = a.Y.v[j]; w[24 + j] = a.ZZ.v[j]; w[36 + j] = a.ZZZ.v[j]; }
#pragma unroll
    for (int i = 0; i < XYZZ_WORDS / 4; i++) q[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
}

__global__ void __launch_bounds__(128, 2) k_bucket_accumulate_q8(const uint32_t* __restrict__ records, const uint32_t* __restrict__ sorted,
                                                                 const uint32_t* __restrict__ bucket_start, const uint32_t* __restrict__ item_start,
                                                                 uint32_t total_buckets, uint32_t cap, uint32_t* __restrict__ partial) {
    const uint32_t item = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (item >= item_start[total_buckets]) return;               // whole warps
    const Quad Q = Quad::here();
    uint32_t lo = 0, hi = total_buckets;                         // item_start[lo] <= item < item_start[hi]
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (item_start[mid] <= item) lo = mid; else hi = mid; }
    const uint32_t seg = item - item_start[lo];
    const uint32_t b0 = bucket_start[lo], b1 = bucket_start[lo + 1];
    const uint32_t s0 = b0 + seg * cap, s1 = s0 + cap < b1 ? s0 + cap : b1;
    XYZZ acc = XYZZ::infinity();
    {
        // lockstep over the item (see k_bucket_reduce_quad): every quad makes every trip, ∞ beyond the item's end
        AffinePoint p; p.x = Fq::zero(); p.y = Fq::zero(); p.inf = true;
        uint32_t e = 0;
        uint32_t k = s0 + (uint32_t)Q.slot;
        if (k < s1) { e = sorted[k]; p = load_record(records, e & 0x7fffffffu); }
#pragma unroll 1
        for (uint32_t base = s0; base < s1; base += 8, k += 8) {
            __syncwarp();
            const uint32_t e_cur = e;
            const AffinePoint p_cur = p;
            p.inf = true;
            if (k + 8 < s1) { e = sorted[k + 8]; p = load_record(records, e & 0x7fffffffu); }
            acc = quad_add_affine(acc, p_cur, (e_cur >> 31) != 0u, Q);
        }
    }
    acc = slot_sum(acc, Q);
    if ((threadIdx.x & 31u) == 0u) acc.store(partial + (size_t)item * XYZZ_WORDS);
}

// Hot buckets without scans.  Some buckets are hot by construction: the top window of a 253-bit scalar has a handful of digit
// values (c = 8: 16 buckets share all n points) or is the carry alone (c = 11: one bucket with ≈ 0.14·n points), equal scalars
// add more.  A bucket's item partials stay at partial[item_start[b] …]; a round replaces every 32 consecutive ones by their sum at
// the SAME base offset of the other buffer (count → ⌈count / 32⌉) while the count exceeds 32, so no offsets are recomputed and
// each bucket knows from its own count how many rounds it took part in and which buffer holds its partials.  k_items_per_bucket
// lists the buckets with more than 32 items; warp w works on hot bucket w / 32 and takes every 32nd group of it, quad s of the
// warp adds entries s, s + 8, … of the group.  Rounds launched for the worst case find nothing to do and return.
__global__ void __launch_bounds__(128) k_fold_hot_quad(const uint32_t* __restrict__ in, const uint32_t* __restrict__ item_start,
                                                       const uint32_t* __restrict__ hot, uint32_t hot_max, uint32_t round, uint32_t keep,
                                                       uint32_t* __restrict__ out) {
    uint32_t nhot = hot[0];
    if (nhot > hot_max) nhot = hot_max;
    const Quad Q = Quad::here();
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5, w0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    for (uint32_t h = w0 >> 5; h < nhot; h += nwarps >> 5) {             // whole warps; nwarps is a multiple of 32
        const uint32_t b = hot[1u + h];
        const uint32_t i0 = item_start[b];
        uint32_t cnt = item_start[b + 1] - i0;
        bool live = true;
        for (uint32_t r = 0; r < round; r++) { if (cnt <= keep) live = false; cnt = (cnt + 31u) >> 5; }
        if (!live || cnt <= keep) continue;                             // this bucket finished in an earlier round
        const uint32_t groups = (cnt + 31u) >> 5;
        for (uint32_t g = w0 & 31u; g < groups; g += 32u) {
            const uint32_t k = g << 5, end = k + 32u < cnt ? k + 32u : cnt;
            XYZZ s = XYZZ::infinity();
#pragma unroll 1
            for (uint32_t i = k; i < end; i += 8u) {                    // lockstep: every quad makes every trip
                __syncwarp();
                XYZZ v = XYZZ::infinity();
                if (i + (uint32_t)Q.slot < end) v = XYZZ::load(in + (size_t)(i0 + i + (uint32_t)Q.slot) * XYZZ_WORDS);
                s = quad_add(s, v, Q);
            }
            s = slot_sum(s, Q);
            if ((threadIdx.x & 31u) == 0u) s.store(out + (size_t)(i0 + g) * XYZZ_WORDS);
        }
    }
}

// out[(set·chunks + chunk)·2] = Σ_l (l + 1)·S_{8·chunk + l},  out[… + 1] = Σ_l S_{8·chunk + l}
// The item partials of bucket b start at item_start[b] in partial_a, or, after an odd number of folds (fold_rounds_of its
// item count), in partial_b.  `folds` = 0: no fold kernel ran (every bucket has one partial or the caller folded already).
__global__ void __launch_bounds__(128) k_bucket_reduce_quad(const uint32_t* __restrict__ partial_a, const uint32_t* __restrict__ partial_b,
                                                            const uint32_t* __restrict__ item_start, int folds,
                                                            uint32_t nbuckets, uint32_t chunks, uint32_t nsets, uint32_t* __restrict__ out) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (warp >= nsets * chunks) return;                                 // whole warps only
    const Quad Q = Quad::here();
    const uint32_t set = warp / chunks, ch = warp % chunks, b = ch * 8u + (uint32_t)Q.slot;
    XYZZ s = XYZZ::infinity();
    {
        // The eight quads walk their buckets in LOCKSTEP (trip count = the largest item count of the warp, ∞ operands beyond a
        // quad's own count, a __syncwarp per trip): quads that leave a loop at different trips are scheduled one after the other
        // from then on, which made each addition cost 8×.
        uint32_t i0 = 0, cnt = 0;
        const uint32_t* partial = partial_a;
        if (b < nbuckets) {
            const uint32_t wb = set * nbuckets + b;
            i0 = item_start[wb];
            cnt = item_start[wb + 1] - i0;
            if (folds) { if (fold_rounds_of(cnt, cnt) & 1u) partial = partial_b; }
        }
        const uint32_t trips = __reduce_max_sync(0xffffffffu, cnt);
#pragma unroll 1
        for (uint32_t i = 0; i < trips; i++) {
            __syncwarp();
            XYZZ t = XYZZ::infinity();
            if (i < cnt) t = XYZZ::load(partial + (size_t)(i0 + i) * XYZZ_WORDS);
            s = quad_add(s, t, Q);
        }
    }
    const XYZZ run = slot_suffix_scan(s, Q);
    const XYZZ acc = slot_sum(run, Q);
    if ((threadIdx.x & 31u) == 0u) {
        acc.store(out + (size_t)warp * 2 * XYZZ_WORDS);
        run.store(out + ((size_t)warp * 2 + 1) * XYZZ_WORDS);
    }
}

// One 8:1 fold of (acc, run) entries that span 2^lgw buckets each: acc' = Σ_s acc_s + 2^lgw·Σ_s s·run_s, run' = Σ_s run_s.
// Called by one warp with slot s holding entry 8·group + s (∞ beyond the end); every lane returns acc', `run_out` = run'.
FF_DEV XYZZ combine_fold_quad(const XYZZ& a, const XYZZ& r, int lgw, const Quad& Q, XYZZ& run_out) {
    XYZZ A = slot_sum(a, Q);
    const XYZZ suf = slot_suffix_scan(r, Q);                            // Σ_{s' ≥ s} run_s'
    XYZZ W = slot_sum(Q.slot == 0 ? XYZZ::infinity() : suf, Q);         // Σ_{s ≥ 1} suffix_s = Σ_s s·run_s
#pragma unroll 1
    for (int k = 0; k < lgw; k++) W = quad_dbl(W, Q);
    run_out = suf;                                                      // slot 0 holds the total
    return quad_add(A, W, Q);
}
// one level for sets with more than 64 entries: m entries per set → ceil(m / 8), one warp per output entry
__global__ void __launch_bounds__(128) k_combine_level_quad(const uint32_t* __restrict__ in, uint32_t m, uint32_t nsets, int lgw, uint32_t* __restrict__ out) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, groups = (m + 7u) / 8u;
    if (warp >= nsets * groups) return;
    const Quad Q = Quad::here();
    const uint32_t set = warp / groups, g = warp % groups, j = g * 8u + (uint32_t)Q.slot;
    XYZZ a = XYZZ::infinity(), r = XYZZ::infinity();
    if (j < m) { a = load_xyzz_plain(in + ((size_t)set * m + j) * 2 * XYZZ_WORDS); r = load_xyzz_plain(in + (((size_t)set * m + j) * 2 + 1) * XYZZ_WORDS); }
    XYZZ run;
    const XYZZ A = combine_fold_quad(a, r, lgw, Q, run);
    if ((threadIdx.x & 31u) == 0u) {
        store_xyzz_plain(out + (size_t)warp * 2 * XYZZ_WORDS, A);
        store_xyzz_plain(out + ((size_t)warp * 2 + 1) * XYZZ_WORDS, run);
    }
}
// The same fold with ONE QUAD per group, its 8 entries walked from the top with running sums (Σ s·run_s = Σ_{s ≥ 1} running after
// entry s): 23 additions per group instead of 9 scan / sum steps that all eight quads of a warp execute — 4× fewer warp
// instructions.  For levels with thousands of groups (4096 → 512 entries per window at 2^24 points), where the
// multiplier's throughput matters more than the depth of one group's chain.
__global__ void __launch_bounds__(128) k_combine_level_quadseq(const uint32_t* __restrict__ in, uint32_t m, uint32_t nsets, int lgw, uint32_t* __restrict__ out) {
    const uint32_t quad = (blockIdx.x * blockDim.x + threadIdx.x) >> 2, groups = (m + 7u) / 8u;
    if (quad >= nsets * groups) return;                                 // whole quads; no warp-wide exchange below
    const Quad Q = Quad::here();
    const uint32_t set = quad / groups, g = quad % groups, first = g * 8u;
    const uint32_t cnt = m - first < 8u ? m - first : 8u;
    XYZZ A = XYZZ::infinity(), running = XYZZ::infinity(), W = XYZZ::infinity();
#pragma unroll 1
    for (uint32_t s = cnt; s-- > 0u;) {
        const size_t e = ((size_t)set * m + first + s) * 2;
        A = quad_add(A, load_xyzz_plain(in + e * XYZZ_WORDS), Q);
        running = quad_add(running, load_xyzz_plain(in + (e + 1) * XYZZ_WORDS), Q);
        if (s >= 1u) W = quad_add(W, running, Q);
    }
#pragma unroll 1
    for (int k = 0; k < lgw; k++) W = quad_dbl(W, Q);
    A = quad_add(A, W, Q);
    if (Q.q == 0) {
        store_xyzz_plain(out + (size_t)quad * 2 * XYZZ_WORDS, A);
        store_xyzz_plain(out + ((size_t)quad * 2 + 1) * XYZZ_WORDS, running);
    }
}
// window sum of a set from its m0 ≤ 64 entries (each spanning 2^lgw0 buckets): one CTA per set, 8:1 per level through
// shared memory
// k·a (double-and-add from the top bit) by one quad
FF_DEV XYZZ quad_mul_u32(const XYZZ& a, uint32_t k, const Quad& Q) {
    XYZZ r = XYZZ::infinity();
#pragma unroll 1
    for (int b = 31 - __clz(k); b >= 0; b--) {
        r = quad_dbl(r, Q);
        if ((k >> b) & 1u) r = quad_add(r, a, Q);
    }
    return r;
}
static constexpr int COMBINE_QUAD_MAX_WARPS = 8;
__global__ void __launch_bounds__(32 * COMBINE_QUAD_MAX_WARPS) k_window_combine_quad(const uint32_t* __restrict__ in, uint32_t m0, int lgw0, uint32_t* __restrict__ out,
                                                                                      SetOffsets so) {
    __shared__ __align__(16) uint32_t sm[COMBINE_QUAD_MAX_WARPS][2][XYZZ_WORDS];
    const uint32_t set = blockIdx.x, warp = threadIdx.x >> 5;
    const Quad Q = Quad::here();
    const uint32_t* src = in + (size_t)set * m0 * 2 * XYZZ_WORDS;
    uint32_t m = m0;
    int lgw = lgw0;
    for (;;) {                                                          // m ≤ 64 → ≤ 8 → 1
        const uint32_t groups = (m + 7u) / 8u;
        XYZZ A, run;
        if (warp < groups) {
            const uint32_t j = warp * 8u + (uint32_t)Q.slot;
            XYZZ a = XYZZ::infinity(), r = XYZZ::infinity();
            if (j < m) { a = load_xyzz_plain(src + (size_t)j * 2 * XYZZ_WORDS); r = load_xyzz_plain(src + ((size_t)j * 2 + 1) * XYZZ_WORDS); }
            A = combine_fold_quad(a, r, lgw, Q, run);
            if (groups == 1u) {
                // slot 0 holds the set's Σ S_b in `run`: add the digit offset's multiple of it (the top window's upper sets)
                const uint32_t off = so.of(set);
                if (off != 0u && Q.slot == 0) A = quad_add(A, quad_mul_u32(run, off, Q), Q);
                if ((threadIdx.x & 31u) == 0u) A.store(out + (size_t)set * XYZZ_WORDS);
            }
        }
        if (groups == 1u) break;
        __syncthreads();                                                // the previous level's entries have been read
        if (warp < groups && (threadIdx.x & 31u) == 0u) { store_xyzz_plain(&sm[warp][0][0], A); store_xyzz_plain(&sm[warp][1][0], run); }
        __syncthreads();
        src = &sm[0][0][0];
        m = groups; lgw += 3;
    }
}

__global__ void k_xyzz_sum_ranks(const uint32_t* __restrict__ in, int nranks, int count, uint32_t* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    XYZZ s = XYZZ::load(in + (size_t)i * XYZZ_WORDS);
    for (int r = 1; r < nranks; r++) s.add(XYZZ::load(in + ((size_t)r * count + i) * XYZZ_WORDS));
    s.store(out + (size_t)i * XYZZ_WORDS);
}

int xyzz_sum_ranks_device(uint32_t* d_out, const uint32_t* d_in, int nranks, int count, cudaStream_t stream) {
    k_xyzz_sum_ranks<<<(count + 31) / 32, 32, 0, stream>>>(d_in, nranks, count, d_out);
    count_launch();
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------
// Scratch: one private stream-ordered pool per device (the default pool is left alone) and a byte budget that
// bounds how much MSM scratch is in flight per device.  The FFI is entered concurrently from many rayon workers
// (sonic_pc/mod.rs:186-245): without the gate, a burst of large commitments would each take tens of GB and the
// losers would fail with cudaErrorMemoryAllocation (⇒ silent CPU fallback on the Rust side); with it they queue.
// ---------------------------------------------------------------------------
// The second stream of a pipelined call (msm_core) and the events that order its window groups against the caller's stream.
// One per lease that asks for it, created once and reused: a lease hands its MsmAux back when its call has enqueued its work,
// so there are as many as there were concurrent pipelined calls, never one per call.
struct MsmAux {
    cudaStream_t stream = nullptr;
    cudaEvent_t sorted = nullptr, joined = nullptr, handoff[2] = {nullptr, nullptr};
};
struct DeviceScratch {
    std::mutex mu;
    std::condition_variable cv;
    cudaMemPool_t pool = nullptr;
    size_t limit = 0, in_use = 0, peak = 0, total = 0;
    bool ready = false;
    std::vector<MsmAux*> aux_free;
};
static DeviceScratch g_scratch[64];

// Default scratch budget and pool release threshold: 60 % of the device.  On an 80 GB H100 that keeps the 48 GB of a
// one-group 2^24-point MSM with 128-byte level-0 records cached between calls; a call whose scratch exceeds the threshold
// has its memory unmapped and mapped again on every call (one 49 GB group: 348 ms per call against 116 ms of kernels, H100
// SXM at 700 W).
static size_t default_scratch_bytes(size_t total) { return total / 5 * 3; }

static int scratch_init(DeviceScratch& ds, int dev) {
    if (ds.ready) return 0;
    size_t free_b = 0, total_b = 0;
    cudaError_t e = cudaMemGetInfo(&free_b, &total_b);
    if (e != cudaSuccess) return (int)e;
    size_t limit = default_scratch_bytes(total_b);
    if (const char* v = getenv("SNARKVM_B200_SCRATCH_LIMIT_GB")) { long g = atol(v); if (g >= 1) limit = (size_t)g << 30; }
    cudaMemPoolProps props = {};
    props.allocType = cudaMemAllocationTypePinned;
    props.handleTypes = cudaMemHandleTypeNone;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    if ((e = cudaMemPoolCreate(&ds.pool, &props)) != cudaSuccess) return (int)e;
    uint64_t thr = limit;                                             // keep up to `limit` cached between calls, not more
    cudaMemPoolSetAttribute(ds.pool, cudaMemPoolAttrReleaseThreshold, &thr);
    ds.limit = limit;
    ds.total = total_b;
    ds.ready = true;
    return 0;
}
// bytes of pair-level scratch one call splits its bucket sets into groups for: the default budget, whatever limit msm_set_scratch_limit sets
static int scratch_group_budget(size_t* out) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    DeviceScratch& ds = g_scratch[dev & 63];
    std::lock_guard<std::mutex> lock(ds.mu);
    int rc = scratch_init(ds, dev);
    if (rc) return rc;
    *out = default_scratch_bytes(ds.total);
    return 0;
}
// small, ungated allocations (window sums, NTT scratch, polynomial temporaries) from the same private pool
int pool_alloc_raw(void** p, size_t bytes, cudaStream_t stream) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    DeviceScratch& ds = g_scratch[dev & 63];
    {
        std::lock_guard<std::mutex> lock(ds.mu);
        int rc = scratch_init(ds, dev);
        if (rc) return rc;
    }
    return (int)cudaMallocFromPoolAsync(p, bytes ? bytes : 16, ds.pool, stream);
}
struct ScratchLease { DeviceScratch* ds; size_t bytes; };
static void CUDART_CB scratch_release_cb(void* p) {
    ScratchLease* l = (ScratchLease*)p;
    { std::lock_guard<std::mutex> lock(l->ds->mu); l->ds->in_use -= l->bytes; }
    l->ds->cv.notify_all();
    delete l;
}
static int aux_create(MsmAux** out) {
    MsmAux* a = new MsmAux;
    cudaError_t e = cudaStreamCreateWithFlags(&a->stream, cudaStreamNonBlocking);
    for (cudaEvent_t* ev : {&a->sorted, &a->joined, &a->handoff[0], &a->handoff[1]})
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(ev, cudaEventDisableTiming);
    if (e != cudaSuccess) {
        for (cudaEvent_t ev : {a->sorted, a->joined, a->handoff[0], a->handoff[1]}) if (ev) cudaEventDestroy(ev);
        if (a->stream) cudaStreamDestroy(a->stream);
        delete a;
        return (int)e;
    }
    *out = a;
    return 0;
}
// blocks until `bytes` fit in the device's budget (a request larger than the whole budget runs alone), then allocates; with
// `aux`, the lease also carries an auxiliary stream and its events
static int scratch_acquire(void** out, size_t bytes, cudaStream_t stream, DeviceScratch** ds_out, MsmAux** aux = nullptr) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    DeviceScratch& ds = g_scratch[dev & 63];
    MsmAux* a = nullptr;
    {
        std::unique_lock<std::mutex> lock(ds.mu);
        int rc = scratch_init(ds, dev);
        if (rc) return rc;
        ds.cv.wait(lock, [&] { return ds.in_use == 0 || ds.in_use + bytes <= ds.limit; });
        ds.in_use += bytes;
        if (ds.in_use > ds.peak) ds.peak = ds.in_use;
        if (aux && !ds.aux_free.empty()) { a = ds.aux_free.back(); ds.aux_free.pop_back(); }
    }
    e = aux && !a ? (cudaError_t)aux_create(&a) : cudaSuccess;
    if (e == cudaSuccess) e = cudaMallocFromPoolAsync(out, bytes, ds.pool, stream);
    if (e != cudaSuccess) {
        {
            std::lock_guard<std::mutex> lock(ds.mu);
            ds.in_use -= bytes;
            if (a) ds.aux_free.push_back(a);
        }
        ds.cv.notify_all();
        return (int)e;
    }
    *ds_out = &ds;
    if (aux) *aux = a;
    return 0;
}
// frees in stream order and returns the bytes to the budget when the stream gets there.  The auxiliary stream goes back to the
// free list at once: whatever the call left on it is already ordered before the caller's stream reaches the free, and a later
// call that takes it queues behind that work (its own event waits are captured when it enqueues them).
static void scratch_release(void* p, size_t bytes, cudaStream_t stream, DeviceScratch* ds, MsmAux* aux = nullptr) {
    if (aux) { std::lock_guard<std::mutex> lock(ds->mu); ds->aux_free.push_back(aux); }
    cudaFreeAsync(p, stream);
    ScratchLease* l = new ScratchLease{ds, bytes};
    if (cudaLaunchHostFunc(stream, scratch_release_cb, l) != cudaSuccess) scratch_release_cb(l);
}
int msm_scratch_stats(size_t* limit, size_t* in_use, size_t* peak) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    DeviceScratch& ds = g_scratch[dev & 63];
    std::lock_guard<std::mutex> lock(ds.mu);
    if (limit) *limit = ds.limit;
    if (in_use) *in_use = ds.in_use;
    if (peak) *peak = ds.peak;
    return 0;
}

int msm_set_scratch_limit(size_t bytes) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    if (bytes == 0) return (int)cudaErrorInvalidValue;
    DeviceScratch& ds = g_scratch[dev & 63];
    {
        std::lock_guard<std::mutex> lock(ds.mu);
        int rc = scratch_init(ds, dev);
        if (rc) return rc;
        ds.limit = bytes;
        ds.peak = ds.in_use;
        uint64_t thr = bytes;
        cudaMemPoolSetAttribute(ds.pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    ds.cv.notify_all();
    return 0;
}

// How msm_core runs a call after its bucket sort.  msm_path() is the one place that decides it; every later phase switches on one
// of these fields.
struct MsmPath {
    enum Acc { ACC_DENSE, ACC_THREAD, ACC_G8, ACC_Q8 } acc;         // XYZZ sums of the records the pair levels leave, or of
                                                                    // gathered points: one thread, 8 lanes or a warp per item
    uint32_t item_cap;                                              // points per work item of the XYZZ accumulation
    enum Fold { FOLD_SCAN, FOLD_HOT32, FOLD_HOT1 } fold;            // scan 32:1, or the hot list keeping 32 or 1 partials
    enum Tail { TAIL_QUAD_SMALL, TAIL_QUAD_LARGE, TAIL_CLASSIC } tail;
    uint32_t hot_keep() const { return fold == FOLD_HOT1 ? 1u : 32u; }
};

static MsmPath msm_path(const MsmPlan& plan, uint32_t total_buckets, size_t max_entries, size_t set_cap) {
    MsmPath p;
    const bool gather = plan.levels == 0;
    // Small problems take the quad-lane latency path (k_bucket_reduce_quad, k_window_combine_quad).  Large bucket sets: quad-lane
    // combine levels after the per-chunk reduction (measured with tools/phase_sizes.py: faster at 2^20, 2^22 and 2^24; at 2^19 —
    // 4096 buckets per window, 256 chunks — the shorter classic chain wins).
    p.tail = plan.nbuckets <= 1024u ? MsmPath::TAIL_QUAD_SMALL : plan.nbuckets >= 16384u ? MsmPath::TAIL_QUAD_LARGE : MsmPath::TAIL_CLASSIC;
    // The small-set quad reduction adds up to 32 partials per bucket itself; without pair levels the buckets with more are folded
    // 32:1 per round, scan-free, from a device-side list of them.  The large-set tail folds its hot buckets the same way down to
    // ONE partial per bucket (a lone thread adds what is left of a bucket in k_bucket_reduce, so nothing may be left), instead of
    // two scan + copy passes over every bucket.  Everything else takes the scan folds: the classic tail, and pair levels with
    // ≤ 1024 buckets per set, whose folds are followed by the small-set quad tail.
    p.fold = p.tail == MsmPath::TAIL_QUAD_SMALL && gather ? MsmPath::FOLD_HOT32
           : p.tail == MsmPath::TAIL_QUAD_LARGE         ? MsmPath::FOLD_HOT1
                                                        : MsmPath::FOLD_SCAN;
    p.item_cap = plan.cap;
    if (!gather) {
        p.acc = MsmPath::ACC_DENSE;
    } else if (p.tail == MsmPath::TAIL_QUAD_SMALL && (size_t)total_buckets + max_entries / 32 <= 1100) {
        // round 2 (quad.cuh): four lanes per point operation.  One warp per work item (k_bucket_accumulate_q8) while the whole
        // problem is a few thousand buckets — every lane of the warp executes every multiplication, so it costs 3× the
        // multiplier time of the one-thread kernel and only pays while the GPU is mostly idle; the item holds up to 1/16 of a
        // bucket set, so a bucket has ≤ 17 item partials, k_bucket_reduce_quad adds them itself and the 32:1 folds are skipped.
        // (measured with tools/phase_sizes.py: the warp-per-item kernel wins at 2^8 points and loses from 2^10, where the 1400
        // items no longer fit one wave of 255-register warps)
        p.acc = MsmPath::ACC_Q8;
        const size_t cap16 = ((set_cap + 15) / 16 + 7) & ~(size_t)7;
        p.item_cap = (uint32_t)(cap16 < 32 ? 32 : cap16);
    } else if (max_entries <= 100000) {
        // (measured: eight lanes per item win only while the whole problem is a few CTAs — up to 2^10 points, equal at 2^12, and
        // from 2^14 they lose to the butterfly's extra additions)
        p.acc = MsmPath::ACC_G8;
        p.item_cap = 8 * 4;                                       // eight lanes per item, four points each
    } else {
        p.acc = MsmPath::ACC_THREAD;
        // latency-bound sizes (2^12 … 2^15 points): 4 … 8 dependent mixed additions per thread instead of 16; the extra item
        // partials of a bucket cost the quad reduction 4 multiplication steps each (swept with tools/phase_sizes.py: 4 wins at
        // 2^12, 8 at 2^13 … 2^15)
        if (p.fold == MsmPath::FOLD_HOT32 && max_entries <= 900000) p.item_cap = max_entries <= 150000 ? 4 : 8;
    }
    return p;
}

// One msm_core call: what its phases read, and its scratch as msm_core lays it out.  A pipelined call has one MsmCall per
// scratch set: the same shared arrays (hist, bucket_start, cursors, sm_slots), its own stream and everything else its own.
struct MsmCall {
    MsmPlan plan;
    MsmPath path;
    bool flat;
    const uint32_t* table;
    size_t flat_n;                        // table mode: the table's points per window, else 0
    uint32_t sets_per_job, wins_per_job, rec_words;
    uint32_t chunk, chunks_per_set;       // buckets per thread of the per-chunk reduction, and such chunks per bucket set
    size_t set_cap, hot_max;
    int sm_count;
    cudaStream_t stream;
    cudaEvent_t handoff;                  // pipelined: recorded on `stream` after a group's record scatter
    uint8_t* cub_tmp;
    size_t cub_bytes;
    uint32_t *hist, *bucket_start, *cursors, *items, *item_start, *items2, *sorted, *cnt_tmp, *partial, *partial2, *hot_dev, *red_a, *red_b;
    uint32_t *dense_bases, *dense0, *off_a, *off_b, *dense_a, *dense_b, *prefix, *pair_cnt, *pair_off, *sm_slots;
    uint2* desc;
};
struct MsmGroup {                         // windows [u0, u0 + un) of the call, i.e. its bucket sets [w0, w0 + wn)
    uint32_t u0, un, w0, wn, tb;
    const uint32_t* bs;                   // tb + 1 absolute offsets into `sorted` (gather) or the level-0 records
    size_t entries;                       // bound on the group's entries
    size_t items_bound, items_launched;   // from the accumulation: ≥ the item count of any single bucket, of the whole group
    const uint32_t *partial, *start;      // from the folds: the item partials and their per-bucket offsets the tail reads
    int quad_rounds;
    int pair_ctas;                        // pair levels: resident CTAs per SM their waves are sized for
};

// the pair levels' dynamic shared memory limit (set once per device), and the current device's SM count
static int msm_device_setup(int* sm_count) {
    static std::once_flag smem_once[64];
    int dev = 0; cudaGetDevice(&dev);
    std::call_once(smem_once[dev & 63], [] {
        cudaFuncSetAttribute(k_pair_level2<false, PAIR_MIN_BLOCKS>, cudaFuncAttributeMaxDynamicSharedMemorySize, PAIR2_SMEM);
    });
    return (int)cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev);
}
// msm_core's scans: one launch each, over a `uint32_t*` input (CUB instantiates its scan kernels per input type, and these are
// the ones msm_core runs; msm_exclusive_scan's take `const uint32_t*` and count two)
static int scan_counted_once(void* tmp, size_t tmp_bytes, const uint32_t* in, uint32_t* out, size_t count, cudaStream_t stream) {
    count_launch();
    return (int)cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, const_cast<uint32_t*>(in), out, (int)count, stream);
}
static void launch_digits(bool scatter, const MsmPlan& plan, const MsmSegment& sg, size_t flat_n, uint32_t slot_base, uint32_t* counters,
                          uint32_t* sorted, uint32_t* d_flags, cudaStream_t stream) {
    const auto k = !scatter ? (sg.mont ? k_digits<false, true> : k_digits<false, false>) : (sg.mont ? k_digits<true, true> : k_digits<true, false>);
    k<<<(unsigned)((sg.n + 255) / 256), 256, 0, stream>>>((const uint32_t*)sg.d_scalars, sg.n, plan.c, plan.c_top, plan.nwin, plan.nbuckets,
                                                          counters, sorted, flat_n, slot_base, sg.base0, d_flags);
    count_launch();
}
// Bucket sort of all jobs and windows: histogram of every segment's digits into `hist` (TB + 1 counters, keyed by (job, bucket
// set, bucket)), its exclusive scan into `bucket_start` and `cursors`, and, given `sorted`, the scatter of the entries into it.
// Without `sorted` only the histogram runs (the pair levels' record scatter follows per window group).
static int msm_bucket_sort(const MsmPlan& plan, const MsmSegment* segs, int nsegs, uint32_t sets_per_job, size_t flat_n, uint32_t TB,
                           uint32_t* hist, uint32_t* bucket_start, uint32_t* cursors, uint32_t* sorted, void* cub_tmp, size_t cub_bytes,
                           MsmScan scan, uint32_t* d_flags, cudaStream_t stream) {
    for (int pass = 0; pass < (sorted ? 2 : 1); pass++) {
        for (int i = 0; i < nsegs; i++)
            if (segs[i].n) launch_digits(pass == 1, plan, segs[i], flat_n, segs[i].job * sets_per_job * plan.nbuckets, pass ? cursors : hist,
                                         pass ? sorted : nullptr, d_flags, stream);
        if (pass == 0) {
            int rc = scan(cub_tmp, cub_bytes, hist, bucket_start, (size_t)TB + 1, stream);
            if (rc == 0) rc = (int)cudaMemcpyAsync(cursors, bucket_start, (size_t)(TB + 1) * 4, cudaMemcpyDeviceToDevice, stream);
            if (rc) return rc;
            count_launch();                                       // the cursor copy
        }
    }
    return (int)cudaGetLastError();
}

// the gather path's points: every base array, back to back as 128-byte records
static int msm_densify(const MsmBases* bases, int nbases, uint32_t* dense_bases, cudaStream_t stream) {
    size_t at = 0;
    for (int i = 0; i < nbases; i++) {
        if (bases[i].n == 0) continue;
        k_densify_bases<<<(unsigned)((bases[i].n + 255) / 256), 256, 0, stream>>>((const uint8_t*)bases[i].d_points, bases[i].stride, bases[i].n,
                                                                                dense_bases + at * BASE_WORDS);
        count_launch();
        at += bases[i].n;
    }
    return (int)cudaGetLastError();
}

// Gather path: work items of ≤ item_cap sorted entries per bucket, each summed in XYZZ from the densified bases or the tables.
// The item count and its scan run outside every profiling scope.
static int msm_gather_accumulate(const MsmCall& mc, MsmGroup& g) {
    const uint32_t cap = mc.path.item_cap;
    k_items_per_bucket<<<(g.tb + 256) / 256, 256, 0, mc.stream>>>(mc.hist + (size_t)g.w0 * mc.plan.nbuckets, mc.items, g.tb, cap,
                                                                  mc.path.fold != MsmPath::FOLD_SCAN ? mc.hot_dev : nullptr,
                                                                  (uint32_t)mc.hot_max, mc.path.hot_keep());
    count_launch();
    const int rc = scan_counted_once(mc.cub_tmp, mc.cub_bytes, mc.items, mc.item_start, (size_t)g.tb + 1, mc.stream);
    if (rc) return rc;
    const size_t group_items = (size_t)g.tb + g.entries / cap + 1;
    g.items_launched = group_items;
    // q8: ≤ 17 partials per bucket, summed by k_bucket_reduce_quad without folds
    g.items_bound = mc.path.acc == MsmPath::ACC_Q8 ? 1 : mc.set_cap / cap + 1;
    const uint32_t* src = mc.flat ? mc.table : mc.dense_bases;
    ProfScope acc_scope(PROF_MSM_ACCUMULATE, mc.stream);
    if (mc.path.acc == MsmPath::ACC_Q8)
        k_bucket_accumulate_q8<<<(unsigned)((group_items * 32 + 127) / 128), 128, 0, mc.stream>>>(src, mc.sorted, g.bs, mc.item_start, g.tb, cap, mc.partial);
    else if (mc.path.acc == MsmPath::ACC_G8)
        k_bucket_accumulate_g8<<<(unsigned)((group_items * ACC_G + 127) / 128), 128, 0, mc.stream>>>(src, mc.sorted, g.bs, mc.item_start, g.tb, cap, mc.partial);
    else
        k_bucket_accumulate<<<(unsigned)((group_items + MSM_ACC_THREADS - 1) / MSM_ACC_THREADS), MSM_ACC_THREADS, 0, mc.stream>>>(
            src, mc.sorted, g.bs, mc.item_start, g.tb, cap, mc.partial);
    count_launch();
    return (int)cudaGetLastError();
}

static void launch_scatter_records(const MsmCall& mc, const MsmSegment& sg, const uint8_t* points, size_t stride, int w_lo, int w_hi, const uint32_t* bs) {
    const auto k = mc.flat ? (sg.mont ? k_scatter_records<true, true> : k_scatter_records<false, true>)
                           : (sg.mont ? k_scatter_records<true, false> : k_scatter_records<false, false>);
    k<<<(unsigned)((sg.n + 255) / 256), 256, 0, mc.stream>>>((const uint32_t*)sg.d_scalars, sg.n, points, stride, mc.table, mc.flat_n, mc.plan.c,
                                                             mc.plan.c_top, mc.plan.nwin, mc.plan.nbuckets, mc.cursors,
                                                             sg.job * mc.sets_per_job * mc.plan.nbuckets, w_lo, w_hi, bs, (uint4*)mc.dense0, mc.rec_words);
    count_launch();
}
// Pair-level path: the group's level-0 records, the batched-affine pair levels over them, and the XYZZ sums of what is left.
// seg_points / seg_stride: where each segment's points start in its base array (nullptr / 0 in table mode).
static int msm_pair_accumulate(const MsmCall& mc, MsmGroup& g, const MsmSegment* segs, int nsegs, const uint8_t* const* seg_points,
                               const size_t* seg_stride) {
    const cudaStream_t stream = mc.stream;
    const uint32_t tb = g.tb;
    {
        // this group's records: every segment re-derives its digits and emits the windows that fall into the group
        ProfScope sort_scope(PROF_MSM_SORT, stream);
        for (int i = 0; i < nsegs; i++) {
            const MsmSegment& sg = segs[i];
            if (sg.n == 0) continue;
            // windows of this segment inside the group: its job's windows are [job·wins, (job+1)·wins)
            const int64_t first = (int64_t)sg.job * mc.wins_per_job;
            int w_lo, w_hi;
            if (mc.flat) {                                                                // one set per job: all windows or none
                if (first < (int64_t)g.u0 || first >= (int64_t)g.u0 + g.un) continue;
                w_lo = 0; w_hi = mc.plan.nwin;
            } else {
                const int64_t lo_w = (int64_t)g.u0 - first, hi_w = (int64_t)g.u0 + g.un - first;
                w_lo = lo_w < 0 ? 0 : (int)lo_w; w_hi = hi_w > mc.plan.nwin ? mc.plan.nwin : (int)hi_w;
                if (w_lo >= w_hi) continue;
            }
            launch_scatter_records(mc, sg, seg_points[i], seg_stride[i], w_lo, w_hi, g.bs);
        }
    }
    // the next group (other stream) scatters from here on.  Handing over later, once this group's first level is ready, ran
    // that scatter beside this group's pair levels but slowed both (2^24 points, H100 80GB HBM3, 700 W: 92.2 against 90.1 ms).
    if (mc.handoff) {
        const cudaError_t e = cudaEventRecord(mc.handoff, stream);
        if (e != cudaSuccess) return (int)e;
    }
    ProfScope acc_scope(PROF_MSM_ACCUMULATE, stream);
    const uint32_t* off_in = g.bs;
    uint32_t* off_bufs[2] = {mc.off_a, mc.off_b};
    uint32_t* dense_bufs[2] = {mc.dense_a, mc.dense_b};
    const uint32_t* dense_in = mc.dense0;
    size_t bound = g.entries;                                // upper bound on the level's input count
    int rc = 0;
    for (int l = 0; l < mc.plan.levels; l++) {
        uint32_t* off_out = off_bufs[l & 1];
        uint32_t* dense_out = dense_bufs[l & 1];
        k_halve_counts<<<(tb + 256) / 256, 256, 0, stream>>>(off_in, mc.cnt_tmp, mc.pair_cnt, tb);
        count_launch();
        if ((rc = scan_counted_once(mc.cub_tmp, mc.cub_bytes, mc.cnt_tmp, off_out, (size_t)tb + 1, stream)) != 0) return rc;
        if ((rc = scan_counted_once(mc.cub_tmp, mc.cub_bytes, mc.pair_cnt, mc.pair_off, (size_t)tb + 1, stream)) != 0) return rc;
        // pairs: Σ ⌊cnt/2⌋ ≤ Σ cnt/2; all outputs (pairs and single inputs): Σ ⌈cnt/2⌉ ≤ Σ cnt/2 + #buckets
        const size_t pair_bound = bound / 2;
        bound = bound / 2 + tb;
        // Whole waves: 132 SMs × 4 resident CTAs × 128 threads = 67584 lanes run at once on an H100; give every lane
        // the same number T of pairs and launch an integer number of such waves, so no partial last wave
        // idles most of the machine (a level is one long-running CTA per slot, not many short ones).  While another
        // group is in flight a wave is 2 CTAs per SM (g.pair_ctas), half the register file, so the other stream's
        // launches find room beside it.
        const size_t wave = (size_t)mc.sm_count * g.pair_ctas * PAIR_THREADS;
        size_t waves = (pair_bound + 1024 * wave - 1) / (1024 * wave);
        if (waves == 0) waves = 1;
        size_t T = (pair_bound + waves * wave - 1) / (waves * wave);
        if (T == 0) T = 1;
        const size_t nthreads = pair_bound > T ? (pair_bound + T - 1) / T : 1;
        const unsigned lgrid = (unsigned)((nthreads + 127) / 128);
        // one thread per bucket (single inputs) and one warp per 32·DESC_CHUNKS pairs
        const size_t desc_warps = (pair_bound + 32 * DESC_CHUNKS - 1) / (32 * DESC_CHUNKS);
        const size_t desc_threads = desc_warps * 32 > (size_t)tb ? desc_warps * 32 : (size_t)tb;
        const unsigned dgrid = (unsigned)((desc_threads + 255) / 256);
        // level 0 reads the group's records, whose first one sits at the absolute position *bs (off_in = bs); its
        // outputs and all later levels are group-relative (the scans start at 0)
        const uint32_t in_words = l == 0 ? mc.rec_words : (uint32_t)DENSE_WORDS;
        k_pair_desc<false><<<dgrid, 256, 0, stream>>>(off_in, off_out, mc.pair_off, tb, mc.desc, l == 0 ? g.bs : nullptr, dense_in, in_words, dense_out);
        k_pair_level2<false, PAIR_MIN_BLOCKS><<<lgrid, 128, PAIR2_SMEM, stream>>>(dense_in, in_words, mc.desc, mc.pair_off + tb, (uint32_t)T, mc.prefix,
                                                                                 dense_out, mc.sm_slots);
        count_launch(2);
        off_in = off_out;
        dense_in = dense_out;
    }
    k_items_from_offsets<<<(tb + 256) / 256, 256, 0, stream>>>(off_in, mc.items, tb, mc.plan.cap,
                                                               mc.path.fold != MsmPath::FOLD_SCAN ? mc.hot_dev : nullptr, (uint32_t)mc.hot_max,
                                                               mc.path.hot_keep());
    count_launch();
    if ((rc = scan_counted_once(mc.cub_tmp, mc.cub_bytes, mc.items, mc.item_start, (size_t)tb + 1, stream)) != 0) return rc;
    const size_t group_items = (size_t)tb + bound / mc.plan.cap + 1;
    g.items_bound = ((mc.set_cap >> mc.plan.levels) + 1) / mc.plan.cap + 1;
    g.items_launched = group_items;
    k_bucket_accumulate_dense<<<(unsigned)((group_items + MSM_ACC_THREADS - 1) / MSM_ACC_THREADS), MSM_ACC_THREADS, 0, stream>>>(
        dense_in, off_in, mc.item_start, tb, mc.plan.cap, mc.partial);
    count_launch();
    return (int)cudaGetLastError();
}

// List-driven quad folds of the hot buckets, 32:1 per round, as many rounds as the worst case needs for no bucket to hold more
// than `keep` item partials.  The partials stay at their bucket's offset, alternating between partial and partial2 by the round's
// parity.  Returns the number of rounds.
static int msm_fold_hot(const MsmCall& mc, size_t worst, uint32_t keep) {
    int rounds = 0;
    const uint32_t* p_in = mc.partial;
    uint32_t* p_out = mc.partial2;
    while (worst > keep) {
        k_fold_hot_quad<<<(unsigned)mc.sm_count * 8, 128, 0, mc.stream>>>(p_in, mc.item_start, mc.hot_dev, (uint32_t)mc.hot_max, (uint32_t)rounds, keep, p_out);
        count_launch();
        worst = (worst + 31) / 32;
        rounds++;
        const uint32_t* t = p_in; p_in = p_out; p_out = (uint32_t*)t;
    }
    return rounds;
}
static int msm_fold(const MsmCall& mc, MsmGroup& g) {
    uint32_t *partial = mc.partial, *start = mc.item_start;
    g.quad_rounds = 0;
    int rc = 0;
    if (mc.path.fold != MsmPath::FOLD_SCAN) g.quad_rounds = msm_fold_hot(mc, g.items_bound, mc.path.hot_keep());
    else rc = msm_scan_fold(k_partial_group_sum, scan_counted_once, &partial, mc.partial2, &start, mc.items2, mc.cnt_tmp, g.tb, g.items_bound,
                            g.items_launched, mc.cub_tmp, mc.cub_bytes, mc.stream);
    g.partial = partial;
    g.start = start;
    return rc ? rc : (int)cudaGetLastError();
}
// bucket reduction and window combine of the group's bucket sets into its window sums
static int msm_tail(const MsmCall& mc, const MsmGroup& g, uint32_t* group_sums) {
    const cudaStream_t stream = mc.stream;
    const uint32_t nbuckets = mc.plan.nbuckets, wn = g.wn, chunks_per_set = mc.chunks_per_set;
    const SetOffsets so = set_offsets(mc.plan, mc.flat, g.w0);
    if (mc.path.tail == MsmPath::TAIL_QUAD_SMALL) {
        const uint32_t qchunks = (nbuckets + 7u) / 8u;                          // ≤ 128
        k_bucket_reduce_quad<<<(wn * qchunks * 32u + 127u) / 128u, 128, 0, stream>>>(
            g.partial, mc.path.fold == MsmPath::FOLD_HOT32 ? mc.partial2 : g.partial, g.start, g.quad_rounds, nbuckets, qchunks, wn, mc.red_a);
        const uint32_t* ent = mc.red_a;
        uint32_t m = qchunks;
        int lgw = 3;
        if (m > 64u) {                                                          // c = 11: 128 entries → 16
            const uint32_t groups = (m + 7u) / 8u;
            k_combine_level_quad<<<(wn * groups * 32u + 127u) / 128u, 128, 0, stream>>>(ent, m, wn, lgw, mc.red_b);
            count_launch();
            ent = mc.red_b; m = groups; lgw += 3;
        }
        k_window_combine_quad<<<wn, 32u * ((m + 7u) / 8u), 0, stream>>>(ent, m, lgw, group_sums, so);
        count_launch(2);
        return (int)cudaGetLastError();
    }
    const uint32_t nthreads = chunks_per_set * wn;
    if (mc.path.tail == MsmPath::TAIL_QUAD_LARGE) {
        // one thread per 16-bucket chunk leaves its (weighted sum, sum) pair; the chunk offsets are applied by 8:1 quad-lane
        // folds (span 16 → 128 → 1024 → …), the last ≤ 64 entries of a set inside one CTA
        k_bucket_reduce<true><<<(nthreads + 127) / 128, 128, 0, stream>>>(g.partial, g.start, nbuckets, mc.chunk, chunks_per_set, wn, mc.red_a,
                                                                            mc.partial2, g.quad_rounds);
        count_launch(1);
        const uint32_t* ent = mc.red_a;
        uint32_t* other = mc.red_b;
        uint32_t m = chunks_per_set;
        int lgw = 0;
        while ((1u << lgw) < mc.chunk) lgw++;
        while (m > 64u) {
            const uint32_t groups = (m + 7u) / 8u;
            if ((size_t)wn * groups >= 2048)                    // many groups: one quad each, sequential
                k_combine_level_quadseq<<<(unsigned)(((size_t)wn * groups * 4 + 127) / 128), 128, 0, stream>>>(ent, m, wn, lgw, other);
            else
                k_combine_level_quad<<<(wn * groups * 32u + 127u) / 128u, 128, 0, stream>>>(ent, m, wn, lgw, other);
            count_launch();
            uint32_t* done = other; other = (uint32_t*)ent; ent = done;
            m = groups; lgw += 3;
        }
        k_window_combine_quad<<<wn, 32u * ((m + 7u) / 8u), 0, stream>>>(ent, m, lgw, group_sums, so);
        count_launch();
        return (int)cudaGetLastError();
    }
    k_bucket_reduce<false><<<(nthreads + 127) / 128, 128, 0, stream>>>(g.partial, g.start, nbuckets, mc.chunk, chunks_per_set, wn, mc.red_a,
                                                                         nullptr, 0, so);
    count_launch(1);
    return msm_tree_sum(k_group_sum, mc.red_a, mc.red_b, chunks_per_set, wn, XYZZ_WORDS, group_sums, stream);
}

// The general form: `njobs` independent sums (one per committed polynomial), each fed by one or more scalar segments,
// over ONE set of resident bases.  All jobs go through one digit/sort pass keyed by (job, window, bucket), one set of pair
// levels and one reduction; d_window_sums receives njobs × (flat ? 1 : nwin) XYZZ points, job-major.
// table != nullptr: "flat" mode over precomputed tables (record w·table_n + i = 2^{c·w}·P_i): all windows of a job share
// one bucket set, so the pipeline sees ONE set of n·nwin entries per job and writes a single sum per job.
int msm_core(uint32_t* d_window_sums, uint32_t* d_flags, const MsmPlan& plan, const MsmBases* bases, int nbases,
             const uint32_t* table, size_t table_n, const MsmSegment* segs, int nsegs, int njobs, cudaStream_t stream) {
    const bool flat = table != nullptr;
    const uint32_t sets_per_job = flat ? 1u : (uint32_t)plan.nsets;  // bucket sets to reduce per job
    const uint32_t wins_per_job = flat ? 1u : (uint32_t)plan.nwin;   // windows per job, each ≤ one scalar's worth of entries
    if (njobs < 1 || nsegs < 1 || (!flat && nbases < 1)) return (int)cudaErrorInvalidValue;
    if (plan.nsets < plan.nwin || plan.nwin < 1 || (flat && plan.nsets != plan.nwin)) return (int)cudaErrorInvalidValue;
    const uint64_t TB64 = (uint64_t)njobs * sets_per_job * plan.nbuckets;
    if (TB64 >= (1ull << 31)) return (int)cudaErrorInvalidValue;
    const uint32_t TB = (uint32_t)TB64;
    size_t total_scalars = 0, total_bases = 0;
    std::vector<size_t> job_n((size_t)njobs, 0);
    for (int i = 0; i < nbases; i++) {
        if (bases[i].stride < 104 || (bases[i].stride & 7)) return (int)cudaErrorInvalidValue;
        total_bases += bases[i].n;
    }
    for (int i = 0; i < nsegs; i++) {
        if (segs[i].job >= (uint32_t)njobs) return (int)cudaErrorInvalidValue;
        if (flat ? (segs[i].base0 != 0 || segs[i].n > table_n) : ((size_t)segs[i].base0 + segs[i].n > total_bases)) return (int)cudaErrorInvalidValue;
        total_scalars += segs[i].n;
        job_n[segs[i].job] += segs[i].n;
    }
    size_t max_job_n = 0;
    for (size_t v : job_n) if (v > max_job_n) max_job_n = v;
    const size_t max_entries = total_scalars * (size_t)plan.nwin;
    if (total_scalars == 0 || total_bases >= (1ull << 31) || max_entries >= (1ull << 32)) return (int)cudaErrorInvalidValue;
    if (flat && table_n * (size_t)plan.nwin >= (1ull << 31)) return (int)cudaErrorInvalidValue;
    const int levels = plan.levels;
    const size_t set_cap = flat ? max_job_n * (size_t)plan.nwin : max_job_n;   // most entries one bucket set (or one bucket) can hold
    // pair levels: the sort scatters level-0 records (k_scatter_records) and every level is dense; the XYZZ-only path keeps
    // the index sort + gather
    const uint32_t rec_words = !flat && max_entries >= REC_LINE_MIN_ENTRIES ? BASE_WORDS : DENSE_WORDS;   // level-0 record stride
    // a scalar segment must lie inside one base array (the record scatter reads its points through one pointer)
    std::vector<const uint8_t*> seg_points((size_t)nsegs, nullptr);
    std::vector<size_t> seg_stride((size_t)nsegs, 0);
    if (levels > 0 && !flat) {
        for (int i = 0; i < nsegs; i++) {
            size_t off = 0; bool found = segs[i].n == 0;
            for (int k = 0; k < nbases && !found; k++) {
                if (segs[i].base0 >= off && (size_t)segs[i].base0 + segs[i].n <= off + bases[k].n) {
                    seg_points[i] = (const uint8_t*)bases[k].d_points + ((size_t)segs[i].base0 - off) * bases[k].stride;
                    seg_stride[i] = bases[k].stride;
                    found = true;
                }
                off += bases[k].n;
            }
            if (!found) return (int)cudaErrorInvalidValue;
        }
    }

    // Everything after the bucket sort runs per GROUP of whole windows (all bucket sets of a window together), so the dense
    // scratch of the pair levels (≈ 212 B per entry with 128-byte level-0 records) stays inside the budget of the device's
    // cached scratch.  A window holds at most one entry per scalar whatever the number of its sets.
    size_t budget = 0;
    int rc = scratch_group_budget(&budget);
    if (rc) return rc;
    if (const char* e = getenv("SNARKVM_B200_MSM_SCRATCH_GB")) { long v = atol(e); if (v >= 1) budget = (size_t)v << 30; }
    if (const char* e = getenv("SNARKVM_B200_MSM_SCRATCH_MB")) { long v = atol(e); if (v >= 1) budget = (size_t)v << 20; }      // tests: force many groups
    const uint32_t nwins = (uint32_t)njobs * wins_per_job;
    uint32_t gu = nwins;                                          // windows per group
    // per entry: dense_a 48 + prefix 24 + descriptors 4, plus the level-0 records (dense_b reuses them: level 0 is their last
    // reader), 96 or 128 B (rec_words), with 8 B for the item partials and per-bucket arrays
    const size_t per_win = set_cap * (size_t)(84 + 4 * rec_words) + 1;
    // Pipelined: at least two groups, alternating between the caller's stream and an auxiliary one, so that one group's pair
    // levels run beside the other's (the two streams' CTAs share the SMs, 2 + 2 per SM) and one group's tail beside the other's
    // levels.  Two groups are in flight, each with its own scratch set and sized for half the budget: on an 80 GB H100, 2^24
    // points run 7 + 7 windows in about the scratch one 14-window group took (DESIGN §3).  Only while half the budget still
    // holds two windows: each group re-reads every scalar and point for its scatter, and a 2^26-point shard in 14 one-window
    // groups was slower than in five serial groups of three (H100 80GB HBM3, 700 W: 452.5 against 409.7 ms).  And only from
    // 2^22 entries per window: below that a group's levels are a few milliseconds in all (2^20 points: 10.66 → 10.35 ms, within
    // run-to-run spread), and one group keeps half the launches.
    const bool pipelined = levels > 0 && !flat && nwins >= 2 && set_cap >= ((size_t)1 << 22) && budget / 2 / per_win >= 2;
    if (levels > 0) {
        size_t fit = (pipelined ? budget / 2 : budget) / per_win;
        if (fit < 1) fit = 1;
        if (pipelined && fit > (nwins + 1) / 2) fit = (nwins + 1) / 2;
        if (fit < gu) {
            const uint32_t ngroups = (uint32_t)((nwins + fit - 1) / fit);          // equal groups (15 windows in 3 groups: 5 + 5 + 5, not 7 + 7 + 1)
            gu = (nwins + ngroups - 1) / ngroups;
        }
    }
    // first bucket set of window u of the call (job-major; a window's sets are contiguous, the top window's come last in its job)
    auto set_of = [&](uint32_t u) { return (u / wins_per_job) * sets_per_job + u % wins_per_job; };
    uint32_t gw = 0;                                              // bucket sets of the largest group
    for (uint32_t u0 = 0; u0 < nwins; u0 += gu) {
        const uint32_t s = set_of(u0 + (nwins - u0 < gu ? nwins - u0 : gu)) - set_of(u0);
        if (s > gw) gw = s;
    }
    const uint32_t TBg = gw * plan.nbuckets;                      // buckets of the largest group
    size_t entries_g = set_cap * (size_t)gu;                      // most entries a group can hold
    if (entries_g > max_entries) entries_g = max_entries;
    if (levels > 0 && entries_g >= 0x7fffffffull) return (int)cudaErrorInvalidValue;      // record positions carry the sign in bit 31

    MsmCall mc = {};
    mc.plan = plan;
    mc.path = msm_path(plan, TB, max_entries, set_cap);
    mc.flat = flat;
    mc.table = table;
    mc.flat_n = flat ? table_n : 0;
    mc.sets_per_job = sets_per_job;
    mc.wins_per_job = wins_per_job;
    mc.rec_words = rec_words;
    mc.set_cap = set_cap;
    mc.stream = stream;
    const size_t max_items = (size_t)TBg + entries_g / (mc.path.item_cap < plan.cap ? mc.path.item_cap : plan.cap) + 1;
    mc.hot_max = max_items / 2 + 1;                               // buckets with more than hot_keep() (1 or 32) item partials
    const size_t dense_cap_a = entries_g / 2 + TBg + 1, dense_cap_b = entries_g / 4 + 2 * (size_t)TBg + 1;
    if ((rc = msm_device_setup(&mc.sm_count)) != 0) return rc;
    // The reduction tail is a chain of dependent point additions per thread (latency-bound for a lone warp): short chunks
    // and a narrow (8:1) tree keep that chain short — what matters at 2^16–2^20 points, where the tail is 20–50 % of the call.
    mc.chunk = plan.nbuckets < 16u ? plan.nbuckets : 16u;
    mc.chunks_per_set = plan.nbuckets / mc.chunk;
    const uint32_t tree = MSM_TREE_FANIN, chunks_per_set = mc.chunks_per_set;

    if (cub::DeviceScan::ExclusiveSum(nullptr, mc.cub_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)(TB + 1), stream) != cudaSuccess) return (int)cudaErrorUnknown;
    if (mc.cub_bytes < 16) mc.cub_bytes = 16;

    // ---- one scratch block, carved up: the arrays every group shares, then one set of the rest per group in flight ----
    const int nsets = pipelined ? 2 : 1;
    MsmCall mcs[2];
    auto layout = [&](Arena& a) {
        mc.hist = a.take<uint32_t>((size_t)TB + 1);
        mc.bucket_start = a.take<uint32_t>((size_t)TB + 1);
        mc.cursors = a.take<uint32_t>((size_t)TB + 1);
        mc.sorted = levels > 0 ? nullptr : a.take<uint32_t>(max_entries);
        if (!flat && levels == 0) mc.dense_bases = a.take<uint32_t>(total_bases * (size_t)BASE_WORDS);
        if (levels > 0) mc.sm_slots = a.take<uint32_t>(256);   // one counter for both streams' CTAs on an SM
        for (int k = 0; k < nsets; k++) {
            MsmCall& m = mcs[k];
            m = mc;
            m.items = a.take<uint32_t>((size_t)TBg + 1);
            m.item_start = a.take<uint32_t>((size_t)TBg + 1);
            m.items2 = a.take<uint32_t>((size_t)TBg + 1);
            m.cnt_tmp = a.take<uint32_t>((size_t)TBg + 1);
            m.partial = a.take<uint32_t>(max_items * XYZZ_WORDS);
            m.partial2 = a.take<uint32_t>((mc.path.fold != MsmPath::FOLD_SCAN ? max_items : (size_t)TBg + max_items / 32 + 2) * XYZZ_WORDS);      // quad folds keep the item layout
            m.hot_dev = a.take<uint32_t>(mc.hot_max + 2);
            m.red_a = a.take<uint32_t>((size_t)gw * (2 * chunks_per_set > 2 * ((plan.nbuckets + 7u) / 8u) ? 2 * chunks_per_set : 2 * ((plan.nbuckets + 7u) / 8u)) * XYZZ_WORDS);
            m.red_b = a.take<uint32_t>((size_t)gw * (chunks_per_set / tree + 1 > 2 * ((plan.nbuckets + 63u) / 64u) + 2 ? chunks_per_set / tree + 1 : 2 * ((plan.nbuckets + 63u) / 64u) + 2) * XYZZ_WORDS);
            m.cub_tmp = a.take<uint8_t>(mc.cub_bytes);           // CUB temp storage is never shared across streams
            if (levels > 0) {
                m.dense0 = a.take<uint32_t>(entries_g * (size_t)rec_words);
                m.off_a = a.take<uint32_t>((size_t)TBg + 1);
                m.off_b = a.take<uint32_t>((size_t)TBg + 1);
                m.dense_a = a.take<uint32_t>(dense_cap_a * DENSE_WORDS);
                // level 1 writes its outputs (96-byte points) over the level-0 records: only level 0 reads them, and the next
                // group on this set scatters after this group's accumulation in stream order
                if (levels > 1) m.dense_b = dense_cap_b * DENSE_WORDS <= entries_g * (size_t)rec_words ? m.dense0 : a.take<uint32_t>(dense_cap_b * DENSE_WORDS);
                m.prefix = a.take<uint32_t>(dense_cap_a * 12);
                m.desc = a.take<uint2>(dense_cap_a);
                m.pair_cnt = a.take<uint32_t>((size_t)TBg + 1);
                m.pair_off = a.take<uint32_t>((size_t)TBg + 1);
            }
        }
    };
    Arena ar;
    layout(ar);
    const size_t scratch_bytes = ar.off;
    void* block = nullptr;
    DeviceScratch* ds = nullptr;
    MsmAux* aux = nullptr;
    if ((rc = scratch_acquire(&block, scratch_bytes, stream, &ds, pipelined ? &aux : nullptr)) != 0) return rc;
    ar.base = (uint8_t*)block; ar.off = 0;
    layout(ar);
    mc = mcs[0];
    if (pipelined) {
        mcs[0].handoff = aux->handoff[0];
        mcs[1].stream = aux->stream;
        mcs[1].handoff = aux->handoff[1];
    }

    rc = (int)cudaMemsetAsync(mc.hist, 0, (size_t)(TB + 1) * 4, stream);
    if (rc == 0 && mc.sm_slots) rc = (int)cudaMemsetAsync(mc.sm_slots, 0, 256 * 4, stream);
    // the hot list: one window group here, reset per group below with folds to one partial
    if (rc == 0 && mc.path.fold == MsmPath::FOLD_HOT32) rc = (int)cudaMemsetAsync(mc.hot_dev, 0, 4, stream);
    if (rc == 0) {
        ProfScope sort_scope(PROF_MSM_SORT, stream);
        rc = msm_bucket_sort(plan, segs, nsegs, sets_per_job, mc.flat_n, TB, mc.hist, mc.bucket_start, mc.cursors, mc.sorted, mc.cub_tmp,
                             mc.cub_bytes, scan_counted_once, d_flags, stream);
    }
    if (rc == 0 && !flat && levels == 0) {
        ProfScope acc_scope(PROF_MSM_ACCUMULATE, stream);
        rc = msm_densify(bases, nbases, mc.dense_bases, stream);
    }
    // Pipelined: group i runs on stream i & 1 with scratch set i & 1, so a set is reused only by the group two later on the
    // same stream, after this one in stream order.  The auxiliary stream starts after the bucket sort, and every group starts
    // its record scatter after the previous group's (on the other stream), so the two scatters never compete for HBM.
    if (rc == 0 && pipelined) {
        rc = (int)cudaEventRecord(aux->sorted, stream);
        if (rc == 0) rc = (int)cudaStreamWaitEvent(aux->stream, aux->sorted, 0);
    }
    const uint32_t ngroups = (nwins + gu - 1) / gu;
    for (uint32_t i = 0, u0 = 0; rc == 0 && u0 < nwins; i++, u0 += gu) {
        const MsmCall& m = mcs[pipelined ? i & 1 : 0];
        if (i > 0 && pipelined && (rc = (int)cudaStreamWaitEvent(m.stream, mcs[(i - 1) & 1].handoff, 0)) != 0) break;
        MsmGroup g = {};
        g.u0 = u0;
        g.un = nwins - u0 < gu ? nwins - u0 : gu;
        g.w0 = set_of(u0);
        g.wn = set_of(u0 + g.un) - g.w0;
        g.tb = g.wn * plan.nbuckets;
        g.bs = mc.bucket_start + (size_t)g.w0 * plan.nbuckets;
        g.entries = set_cap * (size_t)g.un;
        if (g.entries > max_entries) g.entries = max_entries;
        // the last group runs alone once the one before it ends: full waves
        g.pair_ctas = pipelined && i + 1 < ngroups ? PAIR_MIN_BLOCKS / 2 : PAIR_MIN_BLOCKS;
        if (m.path.fold == MsmPath::FOLD_HOT1 && (rc = (int)cudaMemsetAsync(m.hot_dev, 0, 4, m.stream)) != 0) break;
        rc = levels == 0 ? msm_gather_accumulate(m, g) : msm_pair_accumulate(m, g, segs, nsegs, seg_points.data(), seg_stride.data());
        if (rc) break;
        ProfScope red_scope(PROF_MSM_REDUCE, m.stream);
        rc = msm_fold(m, g);
        if (rc == 0) rc = msm_tail(m, g, d_window_sums + (size_t)g.w0 * XYZZ_WORDS);
    }
    // the result (and the free below) is in stream order on the caller's stream, whatever ran on the auxiliary one
    if (pipelined) {
        cudaError_t e = cudaEventRecord(aux->joined, aux->stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(stream, aux->joined, 0);
        if (e != cudaSuccess) cudaStreamSynchronize(aux->stream);          // free nothing the auxiliary stream may still use
        if (rc == 0) rc = (int)e;
    }
    scratch_release(block, scratch_bytes, stream, ds, aux);
    return rc;
}

// ---- building blocks shared with the G2 path (msm_g2.cu): the curve-independent half of Pippenger ----
size_t msm_scan_bytes(size_t count) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)count);
    return bytes < 16 ? 16 : bytes;
}
int msm_exclusive_scan(void* tmp, size_t tmp_bytes, const uint32_t* in, uint32_t* out, size_t count, cudaStream_t stream) {
    count_launch(2);
    return (int)cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, in, out, (int)count, stream);
}
int msm_sort_indices(const MsmPlan& plan, const void* d_scalars, size_t n, int mont, uint32_t* hist, uint32_t* bucket_start, uint32_t* cursors,
                     uint32_t* sorted, void* cub_tmp, size_t cub_bytes, uint32_t* d_flags, cudaStream_t stream) {
    if (plan.nsets != plan.nwin || plan.c_top != plan.c) return (int)cudaErrorInvalidValue;        // G2 takes the uniform plans
    const uint32_t TB = (uint32_t)plan.nwin * plan.nbuckets;
    const int rc = (int)cudaMemsetAsync(hist, 0, (size_t)(TB + 1) * 4, stream);
    if (rc) return rc;
    const MsmSegment sg{d_scalars, n, 0u, 0u, mont};
    return msm_bucket_sort(plan, &sg, 1, (uint32_t)plan.nwin, 0, TB, hist, bucket_start, cursors, sorted, cub_tmp, cub_bytes, msm_exclusive_scan,
                           d_flags, stream);
}
int msm_items_per_bucket(const uint32_t* hist, uint32_t* items, uint32_t total_buckets, uint32_t cap, cudaStream_t stream) {
    k_items_per_bucket<<<(total_buckets + 256) / 256, 256, 0, stream>>>(hist, items, total_buckets, cap, nullptr, 0u, 32u);
    count_launch();
    return (int)cudaGetLastError();
}
// fold item partials 32:1 until no bucket can hold more than one (worst case: all entries in one bucket).  `worst` (≥ the item
// count of any single bucket) only decides when to stop; a round's launch covers Σ_b ceil(items_b / 32) ≤ #buckets + total/32
// outputs, where `total_bound` bounds the items of ALL buckets (a few hot buckets over a full background need far more outputs
// than total_buckets + worst/32).
int msm_scan_fold(MsmFoldKernel fold, MsmScan scan, uint32_t** partial, uint32_t* partial2, uint32_t** start, uint32_t* start2, uint32_t* cnt_tmp,
                  uint32_t total_buckets, size_t worst, size_t total_bound, void* cub_tmp, size_t cub_bytes, cudaStream_t stream) {
    uint32_t *p_in = *partial, *p_out = partial2, *st_in = *start, *st_out = start2;
    int rc = 0;
    while (worst > 1) {
        k_group_counts<<<(total_buckets + 256) / 256, 256, 0, stream>>>(st_in, cnt_tmp, total_buckets);
        count_launch();
        if ((rc = scan(cub_tmp, cub_bytes, cnt_tmp, st_out, (size_t)total_buckets + 1, stream)) != 0) break;
        const size_t out_bound = (size_t)total_buckets + total_bound / 32 + 1;
        total_bound = out_bound;
        fold<<<(unsigned)((out_bound + 127) / 128), 128, 0, stream>>>(p_in, st_in, st_out, total_buckets, p_out);
        count_launch();
        worst = (worst + 31) / 32;
        std::swap(p_in, p_out);
        std::swap(st_in, st_out);
    }
    *partial = p_in;
    *start = st_in;
    return rc ? rc : (int)cudaGetLastError();
}
// tree over `rows` rows of `per_row` partial sums (red_a): groups of MSM_TREE_FANIN until one point per row remains in `out`
int msm_tree_sum(MsmTreeKernel sum, uint32_t* red_a, uint32_t* red_b, uint32_t per_row, uint32_t rows, size_t point_words, uint32_t* out,
                 cudaStream_t stream) {
    if (per_row == 1) return (int)cudaMemcpyAsync(out, red_a, (size_t)rows * point_words * 4, cudaMemcpyDeviceToDevice, stream);
    const uint32_t* src = red_a;
    uint32_t* bufs[2] = {red_b, red_a};
    int which = 0;
    while (per_row > 1) {
        const uint32_t out_per_row = (per_row + MSM_TREE_FANIN - 1) / MSM_TREE_FANIN;
        uint32_t* target = out_per_row == 1 ? out : bufs[which];
        sum<<<(out_per_row * rows + 127) / 128, 128, 0, stream>>>(src, per_row, MSM_TREE_FANIN, out_per_row, rows, target);
        count_launch();
        src = target; which ^= 1; per_row = out_per_row;
    }
    return (int)cudaGetLastError();
}

int msm_window_sums_device(uint32_t* d_window_sums, uint32_t* d_flags, const MsmPlan& plan, const void* d_points, size_t stride,
                           const void* d_scalars, size_t npoints, cudaStream_t stream) {
    MsmBases b{d_points, stride, npoints};
    MsmSegment sg{d_scalars, npoints, 0u, 0u, 0};
    return msm_core(d_window_sums, d_flags, plan, &b, 1, nullptr, 0, &sg, 1, 1, stream);
}

MsmPlan msm_make_plan_precomputed(size_t npoints) {
    MsmPlan p;
    int lg = ceil_log2(npoints < 2 ? 2 : npoints);
    // one bucket set for all windows ⇒ the bucket reduction is paid once and wide windows are cheap.  Swept with the record
    // scatter feeding dense pair levels (tools/tune_precomputed.py): c = 20 from 2^22 (13 windows), c = 17 at 2^20–2^21.
    int c = lg >= 22 ? 20 : lg >= 20 ? 17 : lg >= 8 ? lg - 2 : 6;
    if (const char* e = getenv("SNARKVM_B200_MSM_PRE_C")) { int v = atoi(e); if (v >= 2 && v <= 24) c = v; }
    p.c = c;
    p.nwin = 253 / c + 1;
    p.nbuckets = 1u << (c - 1);
    p.c_top = c;
    p.nsets = p.nwin;
    size_t total = npoints * (size_t)p.nwin;
    size_t cap = total / 300000 + 1;
    if (cap < 16) cap = 16;
    p.cap = (uint32_t)cap;
    int levels = lg >= 24 ? 5 : lg >= 22 ? 4 : lg >= 20 ? 3 : 1;
    if (const char* e = getenv("SNARKVM_B200_MSM_PRE_LEVELS")) { int v = atoi(e); if (v >= 1 && v <= 16) levels = v; }
    p.levels = levels;
    return p;
}

int msm_precompute_tables_device(uint32_t* d_table, const MsmPlan& plan, const void* d_points, size_t stride, size_t npoints,
                                 cudaStream_t stream) {
    if (stride < 104 || (stride & 7) || npoints == 0) return (int)cudaErrorInvalidValue;
    k_precompute_tables<<<(unsigned)((npoints + 127) / 128), 128, 0, stream>>>((const uint8_t*)d_points, stride, npoints, plan.c, plan.nwin, d_table);
    count_launch();
    return (int)cudaGetLastError();
}

int msm_precomputed_sum_device(uint32_t* d_sum, uint32_t* d_flags, const MsmPlan& plan, const uint32_t* d_table, size_t table_n, const void* d_scalars,
                               size_t nscalars, int mont, cudaStream_t stream) {
    MsmSegment sg{d_scalars, nscalars, 0u, 0u, mont};
    return msm_core(d_sum, d_flags, plan, nullptr, 0, d_table, table_n, &sg, 1, 1, stream);
}

// ---------------------------------------------------------------------------
// Synthetic bases: P_i = h(seed, i)·G
// ---------------------------------------------------------------------------
FF_DEV uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
__constant__ uint32_t G1_GEN_X[12] = {0xec301b95u, 0x1042a645u, 0xc1060f28u, 0x5a990780u, 0xa9007a5bu, 0x684a8ab3u,
                                      0x257ba63fu, 0x1c35a184u, 0xfea8e32eu, 0xb2b2abd2u, 0x23fb2017u, 0x017df3a2u};   // g1.rs:225-236 (Montgomery)
__constant__ uint32_t G1_GEN_Y[12] = {0xe2801ab9u, 0xbc5a1ae8u, 0xcbfe13b0u, 0xd4f3c861u, 0x4e949f13u, 0xecdd5ffcu,
                                      0x7503667du, 0x8f87199bu, 0x7dc4fe1cu, 0x0f0b1b83u, 0x053eaabeu, 0x004bcc7eu};   // g1.rs:242-253

__global__ void __launch_bounds__(128) k_generate_bases(uint8_t* points, size_t n, size_t stride, uint64_t seed) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t k = splitmix64(seed ^ splitmix64((uint64_t)i));
    if (k == 0) k = 1;
    AffinePoint g;
#pragma unroll
    for (int j = 0; j < 12; j++) { g.x.v[j] = G1_GEN_X[j]; g.y.v[j] = G1_GEN_Y[j]; }
    g.inf = false;
    XYZZ acc = XYZZ::infinity();
    bool started = false;
    for (int b = 63; b >= 0; b--) {
        if (started) acc.dbl();
        if ((k >> b) & 1ull) { acc.add_affine(g, false); started = true; }
    }
    store_affine(points, stride, i, acc.to_affine());
}

// ---------------------------------------------------------------------------
// SRS ingest (SURVEY §8 f4, first half): uncompressed canonical points of a `.usrs` file
// (x LE 48 B, y LE 48 B, flags in the top two bits of the last byte: bit 6 = infinity —
// utilities/src/serialize/flags.rs:72-98, curves/src/templates/macros.rs:86-96,136) → the reference's
// in-memory Affine image (Montgomery x, y, infinity flag) straight in HBM, with the on-curve check
// y² = x³ + 1 (affine.rs:205-215) and the canonical-range check (< q) counted into *invalid.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_srs_decode(const uint8_t* __restrict__ in, size_t n, uint8_t* __restrict__ out, size_t stride,
                                                     uint32_t* __restrict__ invalid) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(in + i * 96);     // 96-byte records are 4-byte aligned after the 8-byte header
    Fq x, y;
#pragma unroll
    for (int k = 0; k < 12; k++) { x.v[k] = __ldg(w + k); y.v[k] = __ldg(w + 12 + k); }
    const uint32_t flags = y.v[11] >> 30;                                   // bit 31 = y sign (unused when uncompressed), bit 30 = infinity
    y.v[11] &= 0x3fffffffu;
    AffinePoint a;
    bool bad = false;
    if (flags & 1u) {
        a.x = Fq::zero(); a.y = Fq::one(); a.inf = true;                    // Affine::zero(), affine.rs:57-59
        bad = (flags & 2u) != 0u;                                           // (sign, infinity) both set is not a valid encoding
    } else {
        // canonical range: x, y < q  ⇔  (v − q) borrows
        Fq tx = x, ty = y;
        tx.final_sub(); ty.final_sub();
        bad = (tx != x) || (ty != y);
        a.x = x.to_mont(); a.y = y.to_mont(); a.inf = false;
        Fq lhs = a.y.sqr(), rhs = a.x.sqr() * a.x + Fq::one();
        bad = bad || (lhs != rhs);
    }
    if (bad) atomicAdd(invalid, 1u);
    store_affine(out, stride, i, a);
}
int srs_decode_device(void* d_out, size_t stride, const void* d_in, size_t npoints, uint32_t* d_invalid, cudaStream_t stream) {
    if (stride < 104 || (stride & 7) || ((uintptr_t)d_in & 3)) return (int)cudaErrorInvalidValue;
    cudaError_t e = cudaMemsetAsync(d_invalid, 0, 4, stream);
    if (e != cudaSuccess) return (int)e;
    if (npoints == 0) return 0;
    k_srs_decode<<<(unsigned)((npoints + 127) / 128), 128, 0, stream>>>((const uint8_t*)d_in, npoints, (uint8_t*)d_out, stride, d_invalid);
    count_launch();
    return (int)cudaGetLastError();
}

// Self-test of the warp-cooperative field arithmetic (ff.cuh coop_mul / coop_inverse) against the per-thread multiplier:
// warp w takes pseudo-random elements a, b (and the edge values 0, 1, p − 1), checks coop_mul(a, b) == a·b limb by limb and
// coop_inverse(a)·a == 1.  *mismatches counts failures.
__global__ void __launch_bounds__(128) k_selftest_coop(uint32_t nwarps, uint64_t seed, uint32_t* __restrict__ mismatches) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= nwarps) return;
    Fq a, b;
#pragma unroll
    for (int k = 0; k < 12; k += 2) {
        uint64_t ra = splitmix64(seed + 0x100ull * w + (uint64_t)k), rb = splitmix64(~seed + 0x100ull * w + (uint64_t)k);
        a.v[k] = (uint32_t)ra; a.v[k + 1] = (uint32_t)(ra >> 32); b.v[k] = (uint32_t)rb; b.v[k + 1] = (uint32_t)(rb >> 32);
    }
    a.v[11] &= 0x00ffffffu; b.v[11] &= 0x00ffffffu;             // < 2^376 < q: already reduced
    if (w == 0) a = Fq::zero();
    if (w == 1) a = Fq::one();
    if (w == 2) a = Fq::zero() - Fq::one();
    if (w == 3) { a = Fq::zero() - Fq::one(); b = a; }
    if (w == 4) {                                              // long carry chains: 2^352 − 1 times R
#pragma unroll
        for (int k = 0; k < 12; k++) a.v[k] = k < 11 ? 0xffffffffu : 0u;
        b = Fq::one();
    }
    const uint32_t p = coop_mod_limb<FqParams>(lane);
    uint32_t al = 0u, bl = 0u;
#pragma unroll
    for (int k = 0; k < 12; k++) { if (lane == k) { al = a.v[k]; bl = b.v[k]; } }
    const uint32_t prod = coop_mul<FqParams>(al, bl, p, lane);
    const Fq want = a * b;
    uint32_t wl = 0u;
#pragma unroll
    for (int k = 0; k < 12; k++) if (lane == k) wl = want.v[k];
    bool bad = prod != wl;
    const Fq inv = coop_inverse<FqParams>(a);
    const Fq one = inv * a;
    if (a.is_zero()) bad = bad || !inv.is_zero();
    else bad = bad || (one != Fq::one()) || (inv != a.inverse());
    // the Karatsuba multiplier against the word-serial schoolbook one, per lane, Fq and Fr: random operands, operands whose
    // halves are equal / swapped (every sign combination of the middle term), 0, 1, p − 1
    {
        const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
        Fq x, y;
        Fr u, v;
#pragma unroll
        for (int k = 0; k < 12; k += 2) {
            uint64_t rx = splitmix64(seed * 3 + 0x1000ull * t + (uint64_t)k), ry = splitmix64(~seed * 5 + 0x1000ull * t + (uint64_t)k);
            x.v[k] = (uint32_t)rx; x.v[k + 1] = (uint32_t)(rx >> 32); y.v[k] = (uint32_t)ry; y.v[k + 1] = (uint32_t)(ry >> 32);
        }
        x.v[11] &= 0x00ffffffu; y.v[11] &= 0x00ffffffu;
        if ((t & 7u) == 1u) { for (int k = 0; k < 6; k++) { y.v[k] = x.v[k + 6]; y.v[k + 6] = x.v[k]; } y.v[11] &= 0x00ffffffu; y.v[5] = x.v[11]; }
        if ((t & 7u) == 2u) { for (int k = 0; k < 6; k++) x.v[k + 6] = x.v[k]; x.v[11] &= 0x00ffffffu; }
        if (t == 8u) x = Fq::zero();
        if (t == 9u) y = Fq::one();
        if (t == 10u) { x = Fq::zero() - Fq::one(); y = x; }
        if (t == 11u) { x = Fq::zero() - Fq::one(); }
#pragma unroll
        for (int k = 0; k < 8; k++) { u.v[k] = x.v[k] ^ y.v[11 - k]; v.v[k] = y.v[k] + x.v[11 - k]; }
        u.v[7] &= 0x0fffffffu; v.v[7] &= 0x0fffffffu;
        if ((t & 7u) == 3u) { for (int k = 0; k < 4; k++) v.v[k + 4] = v.v[k]; v.v[7] &= 0x0fffffffu; }
        if (t == 12u) { u = Fr::zero() - Fr::one(); v = u; }
        bool bad2 = Fq::mul_karatsuba(x, y) != Fq::mul_inline(x, y) || Fq::mul_karatsuba(x, x) != Fq::sqr_inline(x);
        bad2 = bad2 || Fr::mul_karatsuba(u, v) != Fr::mul_inline(u, v) || Fr::mul_karatsuba(v, v) != Fr::sqr_inline(v);
        bad = bad || bad2;
    }
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicAdd(mismatches, 1u);
}
int selftest_coop_device(uint32_t nwarps, uint64_t seed, uint32_t* d_mismatches, cudaStream_t stream) {
    cudaError_t e = cudaMemsetAsync(d_mismatches, 0, 4, stream);
    if (e != cudaSuccess) return (int)e;
    k_selftest_coop<<<(nwarps * 32 + 127) / 128, 128, 0, stream>>>(nwarps, seed, d_mismatches);
    count_launch();
    return (int)cudaGetLastError();
}

// Element-wise group operations for snarkvm_b200_test_curve_op_device (operands from the caller, see the header).
template <class F>
__global__ void __launch_bounds__(128) k_test_curve_op(int op, uint32_t* __restrict__ out, const uint32_t* __restrict__ a,
                                                       const uint32_t* __restrict__ b, const uint32_t* __restrict__ k, size_t n) {
    using Pt = XyzzT<F>;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Pt x = Pt::load(a + i * Pt::WORDS);
    const Pt y = Pt::load(b + i * Pt::WORDS);
    switch (op) {
        case SNARKVM_B200_OP_XYZZ_ADD: x.add(y); break;
        case SNARKVM_B200_OP_XYZZ_ADD_AFFINE: {
            AffineT<F> q; q.x = y.X; q.y = y.Y; q.inf = y.is_inf();
            x.add_affine(q, k[i] != 0u);
            break;
        }
        case SNARKVM_B200_OP_XYZZ_DBL: x.dbl(); break;
        case SNARKVM_B200_OP_XYZZ_MUL_U32: x = x.mul_u32(k[i]); break;
        default: {                                          // XYZZ_TO_AFFINE
            const AffineT<F> q = x.to_affine();
            x.X = q.x; x.Y = q.y; x.ZZ = F::zero(); x.ZZZ = F::zero();
            x.store(out + i * Pt::WORDS);
            out[i * Pt::WORDS + 2 * F::WORDS] = q.inf ? 1u : 0u;
            return;
        }
    }
    x.store(out + i * Pt::WORDS);
}
// the quad.cuh operations: four lanes per element, lane 0 of the quad writes the result (all-ones when the lanes disagree)
__global__ void __launch_bounds__(128) k_test_quad_op(int op, uint32_t* __restrict__ out, const uint32_t* __restrict__ a,
                                                      const uint32_t* __restrict__ b, const uint32_t* __restrict__ k, size_t n) {
    const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
    if (i >= n) return;                                     // the four lanes of a quad leave together
    const Quad Q = Quad::here();
    const XYZZ x = XYZZ::load(a + i * XYZZ_WORDS), y = XYZZ::load(b + i * XYZZ_WORDS);
    XYZZ r;
    if (op == SNARKVM_B200_OP_QUAD_ADD) r = quad_add(x, y, Q);
    else if (op == SNARKVM_B200_OP_QUAD_DBL) r = quad_dbl(x, Q);
    else {
        AffinePoint q; q.x = y.X; q.y = y.Y; q.inf = y.is_inf();
        r = quad_add_affine(x, q, k[i] != 0u, Q);
    }
    uint32_t w[XYZZ_WORDS];
    r.store(w);
    bool bad = false;
#pragma unroll
    for (int j = 0; j < XYZZ_WORDS; j++) {                  // unconditional: all four lanes of Q.mask take part in every shuffle
        const uint32_t w0 = __shfl_sync(Q.mask, w[j], 0, 4);
        bad = bad | (w0 != w[j]);
    }
    bad = __any_sync(Q.mask, bad);
    if (Q.q == 0) {
#pragma unroll
        for (int j = 0; j < XYZZ_WORDS; j++) out[i * XYZZ_WORDS + j] = bad ? 0xffffffffu : w[j];
    }
}
int test_curve_op_device(int group, int op, void* d_out, const void* d_a, const void* d_b, const uint32_t* d_k, size_t n, cudaStream_t stream) {
    if (n == 0) return 0;
    if (!d_out || !d_a || !d_b || !d_k || n > ((size_t)1 << 24)) return (int)cudaErrorInvalidValue;
    uint32_t* out = (uint32_t*)d_out;
    const uint32_t *a = (const uint32_t*)d_a, *b = (const uint32_t*)d_b;
    const unsigned blocks = (unsigned)((n + 127) / 128);
    if (op >= SNARKVM_B200_OP_XYZZ_ADD && op <= SNARKVM_B200_OP_XYZZ_TO_AFFINE) {
        if (group == SNARKVM_B200_GROUP_G1) k_test_curve_op<Fq><<<blocks, 128, 0, stream>>>(op, out, a, b, d_k, n);
        else if (group == SNARKVM_B200_GROUP_G2) k_test_curve_op<Fq2><<<blocks, 128, 0, stream>>>(op, out, a, b, d_k, n);
        else return (int)cudaErrorInvalidValue;
    } else if (op >= SNARKVM_B200_OP_QUAD_ADD && op <= SNARKVM_B200_OP_QUAD_ADD_AFFINE && group == SNARKVM_B200_GROUP_G1) {
        k_test_quad_op<<<(unsigned)((4 * n + 127) / 128), 128, 0, stream>>>(op, out, a, b, d_k, n);
    } else {
        return (int)cudaErrorInvalidValue;
    }
    count_launch();
    return (int)cudaGetLastError();
}

// P_i = s_i·G for canonical 253-bit scalars s_i in HBM (a universal setup with a KNOWN trapdoor for tests and benches:
// s_i = β^i gives powers_of_beta_g, s_i = γβ^i powers_of_beta_times_gamma_g; kzg10/data_structures.rs UniversalParams)
__global__ void __launch_bounds__(128) k_generator_mul(uint8_t* points, size_t n, size_t stride, const uint32_t* __restrict__ scalars) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t k[8];
#pragma unroll
    for (int j = 0; j < 8; j++) k[j] = scalars[8 * i + j];
    AffinePoint g;
#pragma unroll
    for (int j = 0; j < 12; j++) { g.x.v[j] = G1_GEN_X[j]; g.y.v[j] = G1_GEN_Y[j]; }
    g.inf = false;
    XYZZ acc = XYZZ::infinity();
    bool started = false;
#pragma unroll 1
    for (int w = 7; w >= 0; w--) {
        uint32_t kw = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) if (j == w) kw = k[j];
#pragma unroll 1
        for (int b = 31; b >= 0; b--) {
            if (started) acc.dbl();
            if ((kw >> b) & 1u) { acc.add_affine(g, false); started = true; }
        }
    }
    store_affine(points, stride, i, acc.to_affine());
}
int msm_generator_mul_device(void* d_points, size_t npoints, size_t stride, const void* d_scalars, cudaStream_t stream) {
    if (stride < 104 || (stride & 7)) return (int)cudaErrorInvalidValue;
    if (npoints == 0) return 0;
    k_generator_mul<<<(unsigned)((npoints + 127) / 128), 128, 0, stream>>>((uint8_t*)d_points, npoints, stride, (const uint32_t*)d_scalars);
    count_launch();
    return (int)cudaGetLastError();
}

int msm_generate_bases_device(void* d_points, size_t npoints, size_t stride, uint64_t seed, cudaStream_t stream) {
    if (stride < 104 || (stride & 7)) return (int)cudaErrorInvalidValue;
    if (npoints == 0) return 0;
    k_generate_bases<<<(unsigned)((npoints + 127) / 128), 128, 0, stream>>>((uint8_t*)d_points, npoints, stride, seed);
    count_launch();
    return (int)cudaGetLastError();
}

}  // namespace b200
