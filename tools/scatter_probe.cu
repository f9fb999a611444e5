// Kernels of tools/scatter_probe.py: the level-0 record scatter of the resident G1 MSM (k_scatter_records, msm.cu) taken
// apart, to see where its time goes.  Built at run time by the probe into a temporary directory:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -shared -Xcompiler -fPIC -o scatter_probe.so scatter_probe.cu
// Variants (template MODE):
//   AS_BUILT    the shipped kernel's work: point reads, digits, cursor atomics, barriers, 96-byte records by six lanes each
//   NO_STORE    AS_BUILT without the record stores
//   STORES      positions from an earlier AS_BUILT run (pos[w·n + i]) instead of the cursor atomics: reads + stores
//   LINES       STORES, each record one whole 128-byte line (x, ±y, 32 B of zeros) by eight lanes at a 128-byte stride
//   PAIRED      STORES at the 96-byte stride, two records written by the same 12 lanes to slots 2k, 2k+1 (a synthetic
//               pairing: the slot pair is taken from the first record's position, so the stores cover three whole 64-byte
//               units; the data is meaningless, the addresses are those of STORES)
//   LINES_ATOMIC    AS_BUILT with LINES' 128-byte records (cursor atomics and stores)
//   LINES_ATOMIC_CS LINES_ATOMIC with evict-first stores (st.global.cs), so the records do not push the cursors out of L2
#include "../snarkvm_b200/csrc/ec.cuh"

using namespace b200;

enum { AS_BUILT = 0, NO_STORE = 1, STORES = 2, LINES = 3, PAIRED = 4, RECORD_POS = 5, LINES_ATOMIC = 6, LINES_ATOMIC_CS = 7 };
static constexpr uint32_t NONE = 0xffffffffu;

__device__ __forceinline__ uint32_t digit_of(const uint32_t* s, int w, int nwin, int c_low, int c_top, uint32_t& carry, uint32_t& neg) {
    const int c = w == nwin - 1 ? c_top : c_low;
    const int bit = w * c_low, wi = bit >> 5, sh = bit & 31;
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) { if (k == wi) lo = s[k]; if (k == wi + 1) hi = s[k]; }
    const uint32_t half = 1u << (c - 1);
    const uint32_t raw = (__funnelshift_r(lo, hi, sh) & ((1u << c) - 1u)) + carry;
    neg = raw > half ? 1u : 0u;
    const uint32_t mag = neg ? (1u << c) - raw : raw;
    carry = neg;
    return mag;
}

__global__ void k_probe_hist(const uint32_t* __restrict__ scalars, size_t n, int c_low, int c_top, int nwin, uint32_t nbuckets,
                             uint32_t* __restrict__ hist) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8];
    const uint4* q = reinterpret_cast<const uint4*>(scalars + 8 * i);
    uint4 a = __ldg(q), b = __ldg(q + 1);
    s[0] = a.x; s[1] = a.y; s[2] = a.z; s[3] = a.w; s[4] = b.x; s[5] = b.y; s[6] = b.z; s[7] = b.w;
    uint32_t carry = 0, neg = 0;
    for (int w = 0; w < nwin; w++) {
        const uint32_t mag = digit_of(s, w, nwin, c_low, c_top, carry, neg);
        if (mag != 0u) atomicAdd(&hist[(uint32_t)w * nbuckets + mag - 1u], 1u);
    }
}

template <int MODE>
__global__ void __launch_bounds__(256) k_probe_scatter(const uint32_t* __restrict__ scalars, size_t n, const uint8_t* __restrict__ points,
                                                       size_t stride, int c_low, int c_top, int nwin, uint32_t nbuckets,
                                                       uint32_t* __restrict__ cursors, uint32_t* __restrict__ pos_io, uint4* __restrict__ dense) {
    __shared__ uint4 sh_rec[256 * 9];
    __shared__ uint32_t sh_pos[2][256];
    const uint32_t tid = threadIdx.x;
    const size_t i = (size_t)blockIdx.x * 256 + tid;
    const bool live = i < n;
    uint32_t s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = 0u;
    if (live) {
        const uint4* q = reinterpret_cast<const uint4*>(scalars + 8 * i);
        uint4 a = __ldg(q), b = __ldg(q + 1);
        s[0] = a.x; s[1] = a.y; s[2] = a.z; s[3] = a.w; s[4] = b.x; s[5] = b.y; s[6] = b.z; s[7] = b.w;
        AffinePoint pt = load_affine(points, stride, i);
        Fq x = pt.x, y = pt.y, yn = pt.y.neg();
        if (pt.inf) { x = Fq::zero(); y = Fq::zero(); yn = Fq::zero(); }
        uint4* r = sh_rec + tid * 9;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            r[k] = make_uint4(x.v[4 * k], x.v[4 * k + 1], x.v[4 * k + 2], x.v[4 * k + 3]);
            r[3 + k] = make_uint4(y.v[4 * k], y.v[4 * k + 1], y.v[4 * k + 2], y.v[4 * k + 3]);
            r[6 + k] = make_uint4(yn.v[4 * k], yn.v[4 * k + 1], yn.v[4 * k + 2], yn.v[4 * k + 3]);
        }
    }
    uint32_t carry = 0;
    for (int w = 0; w < nwin; w++) {
        uint32_t neg = 0;
        const uint32_t mag = digit_of(s, w, nwin, c_low, c_top, carry, neg);
        uint32_t pos = NONE;
        if (MODE == STORES || MODE == LINES || MODE == PAIRED) {
            if (live) pos = pos_io[(size_t)w * n + i];
        } else if (live && mag != 0u) {
            pos = atomicAdd(&cursors[(uint32_t)w * nbuckets + (mag - 1u)], 1u) | (neg << 31);
        }
        if (MODE == RECORD_POS && live) pos_io[(size_t)w * n + i] = pos;
        uint32_t* my_pos = sh_pos[w & 1];
        my_pos[tid] = pos;
        __syncthreads();
        if (MODE == NO_STORE) {
            // a store no position ever reaches (positions stay below 2^31 records) keeps the point reads and the staging alive
            if (pos == 0xfffffffeu) dense[tid] = sh_rec[tid * 9u];
        } else if (MODE == AS_BUILT || MODE == STORES || MODE == RECORD_POS) {
            for (uint32_t k = tid; k < 256u * 6u; k += 256u) {
                const uint32_t r = k / 6u, part = k - 6u * r;
                const uint32_t pp = my_pos[r];
                if (pp == NONE) continue;
                const uint32_t src = part < 3u ? part : ((pp >> 31) ? 3u : 0u) + part;
                dense[(size_t)(pp & 0x7fffffffu) * 6u + part] = sh_rec[r * 9u + src];
            }
        } else if (MODE == LINES || MODE == LINES_ATOMIC || MODE == LINES_ATOMIC_CS) {
            for (uint32_t k = tid; k < 256u * 8u; k += 256u) {
                const uint32_t r = k >> 3, part = k & 7u;
                const uint32_t pp = my_pos[r];
                if (pp == NONE) continue;
                const uint32_t src = part < 3u ? part : ((pp >> 31) ? 3u : 0u) + part;
                const uint4 v = part < 6u ? sh_rec[r * 9u + src] : make_uint4(0u, 0u, 0u, 0u);
                uint4* d = dense + (size_t)(pp & 0x7fffffffu) * 8u + part;
                if (MODE == LINES_ATOMIC_CS) __stcs(d, v); else *d = v;
            }
        } else if (MODE == PAIRED) {
            for (uint32_t k = tid; k < 128u * 12u; k += 256u) {
                const uint32_t p = k / 12u, sub = k - 12u * p, r = 2u * p + (sub >= 6u ? 1u : 0u), part = sub >= 6u ? sub - 6u : sub;
                const uint32_t p0 = my_pos[2u * p], pp = my_pos[r];
                if (p0 == NONE || pp == NONE) continue;
                const uint32_t slot = ((p0 & 0x7fffffffu) & ~1u) + (sub >= 6u ? 1u : 0u);
                const uint32_t src = part < 3u ? part : ((pp >> 31) ? 3u : 0u) + part;
                dense[(size_t)slot * 6u + part] = sh_rec[r * 9u + src];
            }
        }
    }
}

extern "C" int probe_hist(const void* scalars, size_t n, int c_low, int c_top, int nwin, uint32_t nbuckets, void* hist, void* stream) {
    k_probe_hist<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint32_t*)scalars, n, c_low, c_top, nwin, nbuckets,
                                                                                 (uint32_t*)hist);
    return (int)cudaGetLastError();
}

extern "C" int probe_scatter(int mode, const void* scalars, size_t n, const void* points, size_t stride, int c_low, int c_top, int nwin,
                             uint32_t nbuckets, void* cursors, void* pos, void* dense, void* stream) {
    const unsigned grid = (unsigned)((n + 255) / 256);
    cudaStream_t st = (cudaStream_t)stream;
#define PROBE_LAUNCH(M)                                                                                                         \
    k_probe_scatter<M><<<grid, 256, 0, st>>>((const uint32_t*)scalars, n, (const uint8_t*)points, stride, c_low, c_top, nwin, \
                                             nbuckets, (uint32_t*)cursors, (uint32_t*)pos, (uint4*)dense)
    switch (mode) {
        case AS_BUILT: PROBE_LAUNCH(AS_BUILT); break;
        case NO_STORE: PROBE_LAUNCH(NO_STORE); break;
        case STORES: PROBE_LAUNCH(STORES); break;
        case LINES: PROBE_LAUNCH(LINES); break;
        case PAIRED: PROBE_LAUNCH(PAIRED); break;
        case RECORD_POS: PROBE_LAUNCH(RECORD_POS); break;
        case LINES_ATOMIC: PROBE_LAUNCH(LINES_ATOMIC); break;
        case LINES_ATOMIC_CS: PROBE_LAUNCH(LINES_ATOMIC_CS); break;
        default: return (int)cudaErrorInvalidValue;
    }
#undef PROBE_LAUNCH
    return (int)cudaGetLastError();
}
