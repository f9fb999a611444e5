// Poseidon duplex sponge on the device: PoseidonSponge<F, 2, 1> (algorithms/src/crypto_hash/poseidon.rs), one thread per transcript.
//
//   k_poseidon_check<P>        one thread per transcript: its operation list against the array sizes, its absorbed elements < p
//   k_poseidon_transcripts<P>  one thread per transcript: its operations in order on its own sponge state (3 F in registers)
//
// A transcript is a straight line of operations (SNARKVM_B200_POSEIDON_*): absorb n native elements from the input array, squeeze n
// native elements, or squeeze n nonnative Fr elements, full (252 bits) or short (168 bits).  Each operation is the reference's
// AlgebraicSponge call of the same name, including its mode handling: the permutation runs lazily, before the first element an
// operation adds or reads in a full rate, so the sequence of permutations is exactly the reference's (absorb_internal /
// squeeze_internal never permute after their last chunk; absorbing after a squeeze, or squeezing after an absorb, permutes first).
// A zero-length operation changes nothing, as in the reference.
//
// The permutation: 39 rounds of (ark, S-box x^17, MDS), the four first and four last full.  x^17 is four squarings and a product;
// the MDS is nine products.  8·(15 + 9) + 31·(5 + 9) = 626 products per permutation, every one through the out-of-line multiplier
// (FF_CALL_MUL), so the loop body stays small.  The round keys and the MDS come from HBM once per block into shared memory.
//
// get_bits / get_fe (poseidon.rs:436-492): a squeezed element goes out of Montgomery form, its low size_in_bits − 1 bits are taken
// most significant first, and consecutive groups of 252 (or 168) bits are read as big-endian integers — below 2^252 < r, so each is
// already a reduced Fr, written in Montgomery form.  Bits beyond the last group are dropped (get_bits' truncate).
//
// A resumable transcript keeps its sponge between calls in a state record (d_state, one per transcript): the three state elements
// (Montgomery F), then one word for DuplexSpongeMode (0 absorbing, 1 squeezing) and one for next_absorb_index / next_squeeze_index
// (0 … RATE), then two zero words, so that every record is a whole number of 16-byte lines.  The sponge kernel loads the record
// before the first operation and stores it after the last; without records a transcript starts fresh (zeros, absorbing at 0) and
// nothing is stored.  Both entry points are this one path.
//
// The check kernel runs first; the sponge kernel reads its verdict and writes nothing when any transcript or record is malformed.
#include "msm.cuh"

#define FF_CALL_MUL 1
#include "ff.cuh"
#include "poseidon.cuh"
#include "../../include/snarkvm_b200.h"

namespace b200 {
namespace {

constexpr int P_RATE = 2, P_WIDTH = 3, P_FULL = 8, P_PARTIAL = 31, P_ROUNDS = P_FULL + P_PARTIAL;
constexpr int P_PARAMS = P_ROUNDS * P_WIDTH + P_WIDTH * P_WIDTH;           // ark then mds, in elements
constexpr uint32_t NO_BAD = 0xffffffffu;
constexpr int FULL_NONNATIVE_BITS = 252, SHORT_NONNATIVE_BITS = 168;
constexpr int THREADS = 128;
constexpr uint32_t MODE_ABSORBING = 0, MODE_SQUEEZING = 1;

template <class P> struct StateWords { static constexpr int value = P_WIDTH * P::N + 4; };   // a state record, in 32-bit words

template <class P> struct FieldBits;                                         // MODULUS_BITS (F::size_in_bits())
template <> struct FieldBits<FrParams> { static constexpr int value = 253; };
template <> struct FieldBits<FqParams> { static constexpr int value = 377; };

// a < p on the raw limbs: an image ≥ p is no field element
template <class P>
FF_DEV bool is_canonical(const Fp<P>& a) {
    (void)ptx_sub_cc(a.v[0], P::mod(0));
#pragma unroll
    for (int i = 1; i < P::N; i++) (void)ptx_subc_cc(a.v[i], P::mod(i));
    return ptx_subc(0u, 0u) != 0u;
}

// x^17 = ((x²)²)²)² · x
template <class P>
FF_DEV Fp<P> sbox(const Fp<P>& x) {
    const Fp<P> x16 = x.sqr().sqr().sqr().sqr();
    return x16 * x;
}

template <class P>
FF_DEV void permute(Fp<P> (&s)[P_WIDTH], const Fp<P>* ark, const Fp<P>* mds) {
#pragma unroll 1
    for (int r = 0; r < P_ROUNDS; r++) {
        const bool full = r < P_FULL / 2 || r >= P_FULL / 2 + P_PARTIAL;
#pragma unroll
        for (int i = 0; i < P_WIDTH; i++) s[i] = s[i] + ark[r * P_WIDTH + i];
        s[0] = sbox(s[0]);
        if (full) { s[1] = sbox(s[1]); s[2] = sbox(s[2]); }
        Fp<P> t[P_WIDTH];
#pragma unroll
        for (int i = 0; i < P_WIDTH; i++) t[i] = s[0] * mds[i * P_WIDTH] + s[1] * mds[i * P_WIDTH + 1] + s[2] * mds[i * P_WIDTH + 2];
#pragma unroll
        for (int i = 0; i < P_WIDTH; i++) s[i] = t[i];
    }
}

// one thread per transcript: its state record (when there are records) holds elements below p, a known mode and an index ≤ RATE,
// every operation of [op_start[t], op_start[t + 1]) has a known kind and a range inside its array, and every element it absorbs is
// below p; otherwise *bad_min receives t
template <class P>
__global__ void __launch_bounds__(THREADS) k_poseidon_check(const uint32_t* __restrict__ ops, const uint32_t* __restrict__ op_start,
                                                            uint32_t ntranscripts, uint32_t nops, const uint32_t* __restrict__ in,
                                                            uint64_t nin, uint64_t nout, uint64_t nout_fr, const uint32_t* __restrict__ state,
                                                            uint32_t* __restrict__ bad_min) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntranscripts) return;
    const uint32_t s = op_start[t], e = op_start[t + 1];
    bool ok = s <= e && e <= nops;
    if (state) {
        const uint32_t* rec = state + (size_t)t * StateWords<P>::value;
#pragma unroll 1
        for (int i = 0; ok && i < P_WIDTH; i++) ok = is_canonical(Fp<P>::load(rec + i * P::N));
        const uint32_t mode = rec[P_WIDTH * P::N], idx = rec[P_WIDTH * P::N + 1];
        ok = ok && (mode == MODE_ABSORBING || mode == MODE_SQUEEZING) && idx <= (uint32_t)P_RATE;
    }
#pragma unroll 1
    for (uint32_t k = s; ok && k < e; k++) {
        const uint32_t kind = ops[3 * k], n = ops[3 * k + 1], off = ops[3 * k + 2];
        const uint64_t end = (uint64_t)off + n;
        if (kind == SNARKVM_B200_POSEIDON_ABSORB) {
            ok = end <= nin;
#pragma unroll 1
            for (uint32_t i = 0; ok && i < n; i++) ok = is_canonical(Fp<P>::load(in + ((size_t)off + i) * P::N));
        } else if (kind == SNARKVM_B200_POSEIDON_SQUEEZE) {
            ok = end <= nout;
        } else if (kind == SNARKVM_B200_POSEIDON_SQUEEZE_NONNATIVE || kind == SNARKVM_B200_POSEIDON_SQUEEZE_SHORT_NONNATIVE) {
            ok = end <= nout_fr;
        } else {
            ok = false;
        }
    }
    if (!ok) atomicMin(bad_min, t);
}

// get_fe's bit stream: `acc` collects up to 252 bits, most significant first; every `width` bits make one Fr
struct BitsToFr {
    uint32_t acc[8];
    int have;
    uint32_t done;
    FF_DEV void reset() {
#pragma unroll
        for (int i = 0; i < 8; i++) acc[i] = 0u;
        have = 0;
    }
    // appends the `nbits` low bits of `w`, most significant first; writes each completed element to out[done++] while done < count
    FF_DEV void push(uint32_t w, int nbits, int width, uint32_t count, uint32_t* __restrict__ out) {
#pragma unroll 1
        for (int b = nbits - 1; b >= 0 && done < count; b--) {
#pragma unroll
            for (int i = 7; i > 0; i--) acc[i] = __funnelshift_l(acc[i - 1], acc[i], 1);
            acc[0] = (acc[0] << 1) | ((w >> b) & 1u);
            if (++have == width) {
                Fr x;
#pragma unroll
                for (int i = 0; i < 8; i++) x.v[i] = acc[i];
                (x * Fr::r2()).store(out + (size_t)done * 8);                // < 2^252 < r: reduced; to Montgomery form
                done++;
                reset();
            }
        }
    }
};

template <class P>
__global__ void __launch_bounds__(THREADS) k_poseidon_transcripts(const uint32_t* __restrict__ params, const uint32_t* __restrict__ ops,
                                                                  const uint32_t* __restrict__ op_start, uint32_t ntranscripts,
                                                                  const uint32_t* __restrict__ in, uint32_t* __restrict__ out,
                                                                  uint32_t* __restrict__ out_fr, uint32_t* __restrict__ state,
                                                                  const uint32_t* __restrict__ bad_min) {
    using F = Fp<P>;
    __shared__ __align__(16) uint32_t sh[P_PARAMS * P::N];
    if (*bad_min != NO_BAD) return;                                          // a malformed transcript: no output at all
    for (int i = threadIdx.x; i < P_PARAMS * P::N; i += blockDim.x) sh[i] = params[i];
    __syncthreads();
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntranscripts) return;
    const F* ark = reinterpret_cast<const F*>(sh);
    const F* mds = ark + P_ROUNDS * P_WIDTH;
    constexpr int ELEMENT_BITS = FieldBits<P>::value - 1;                    // get_bits' bits per squeezed element
    constexpr int TOP_BITS = ELEMENT_BITS - 32 * (P::N - 1);                 // of them, in the top limb
    static_assert(TOP_BITS > 0 && TOP_BITS <= 32, "the low size_in_bits − 1 bits reach into the top limb");

    F s[P_WIDTH] = {F::zero(), F::zero(), F::zero()};
    bool squeezing = false;                                                  // DuplexSpongeMode
    int idx = 0;                                                             // next_absorb_index / next_squeeze_index
    uint32_t* rec = state ? state + (size_t)t * StateWords<P>::value : nullptr;
    if (rec) {
#pragma unroll
        for (int i = 0; i < P_WIDTH; i++) s[i] = F::load(rec + i * P::N);
        squeezing = rec[P_WIDTH * P::N] == MODE_SQUEEZING;
        idx = (int)rec[P_WIDTH * P::N + 1];
    }
    const uint32_t e = op_start[t + 1];
#pragma unroll 1
    for (uint32_t k = op_start[t]; k < e; k++) {
        const uint32_t kind = ops[3 * k], n = ops[3 * k + 1], off = ops[3 * k + 2];
        if (n == 0) continue;
        const bool absorb = kind == SNARKVM_B200_POSEIDON_ABSORB;
        const bool nonnative = kind >= SNARKVM_B200_POSEIDON_SQUEEZE_NONNATIVE;
        const int width = kind == SNARKVM_B200_POSEIDON_SQUEEZE_SHORT_NONNATIVE ? SHORT_NONNATIVE_BITS : FULL_NONNATIVE_BITS;
        // elements this operation adds or reads: get_fe(n) squeezes ⌈n·width / ELEMENT_BITS⌉
        const uint32_t count = nonnative ? (uint32_t)(((uint64_t)n * width + ELEMENT_BITS - 1) / ELEMENT_BITS) : n;
        // a change of direction permutes before the first element; so does a full rate (the idx == RATE test below)
        if (absorb == squeezing) { idx = P_RATE; squeezing = !absorb; }
        BitsToFr bits;
        bits.reset();
        bits.done = 0;
#pragma unroll 1
        for (uint32_t i = 0; i < count; i++) {
            if (idx == P_RATE) { permute<P>(s, ark, mds); idx = 0; }
            if (absorb) {
                const F x = F::load(in + ((size_t)off + i) * P::N);
                if (idx == 0) s[1] = s[1] + x; else s[2] = s[2] + x;
            } else {
                const F x = idx == 0 ? s[1] : s[2];
                if (!nonnative) {
                    x.store(out + ((size_t)off + i) * P::N);
                } else {
                    const F c = x.from_mont();
                    uint32_t* dst = out_fr + (size_t)off * 8;
                    bits.push(c.v[P::N - 1], TOP_BITS, width, n, dst);
#pragma unroll
                    for (int l = P::N - 2; l >= 0; l--) bits.push(c.v[l], 32, width, n, dst);
                }
            }
            idx++;
        }
    }
    if (rec) {
#pragma unroll
        for (int i = 0; i < P_WIDTH; i++) s[i].store(rec + i * P::N);
        reinterpret_cast<uint4*>(rec + P_WIDTH * P::N)[0] = make_uint4(squeezing ? MODE_SQUEEZING : MODE_ABSORBING, (uint32_t)idx, 0u, 0u);
    }
}

template <class P>
int run(const void* d_params, const uint32_t* d_ops, const uint32_t* d_op_start, size_t ntranscripts, size_t nops, const void* d_in,
        size_t nin, void* d_out, size_t nout, void* d_out_fr, size_t nout_fr, void* d_state, uint32_t* d_bad, cudaStream_t stream) {
    const unsigned blocks = (unsigned)((ntranscripts + THREADS - 1) / THREADS);
    k_poseidon_check<P><<<blocks, THREADS, 0, stream>>>(d_ops, d_op_start, (uint32_t)ntranscripts, (uint32_t)nops, (const uint32_t*)d_in,
                                                        nin, nout, nout_fr, (const uint32_t*)d_state, d_bad);
    count_launch();
    int rc = (int)cudaGetLastError();
    if (rc != 0) return rc;
    k_poseidon_transcripts<P><<<blocks, THREADS, 0, stream>>>((const uint32_t*)d_params, d_ops, d_op_start, (uint32_t)ntranscripts,
                                                              (const uint32_t*)d_in, (uint32_t*)d_out, (uint32_t*)d_out_fr, (uint32_t*)d_state,
                                                              d_bad);
    count_launch();
    return (int)cudaGetLastError();
}

}  // namespace

int poseidon_transcripts_device(int field, const void* d_params, const uint32_t* d_ops, const uint32_t* d_op_start, size_t ntranscripts,
                                size_t nops, const void* d_in, size_t nin, void* d_out, size_t nout, void* d_out_fr, size_t nout_fr,
                                void* d_state, int64_t* bad_transcript, cudaStream_t stream) {
    if (bad_transcript) *bad_transcript = -1;
    if (field != SNARKVM_B200_FIELD_FR && field != SNARKVM_B200_FIELD_FQ) return (int)cudaErrorInvalidValue;
    if (ntranscripts == 0) return 0;
    if (!d_params || !d_op_start || ntranscripts >= NO_BAD || nops >= NO_BAD) return (int)cudaErrorInvalidValue;
    if ((nops && !d_ops) || (nin && !d_in) || (nout && !d_out) || (nout_fr && !d_out_fr)) return (int)cudaErrorInvalidValue;
    if (((uintptr_t)d_params | (uintptr_t)d_in | (uintptr_t)d_out | (uintptr_t)d_out_fr | (uintptr_t)d_state) & 15)
        return (int)cudaErrorInvalidValue;
    if (((uintptr_t)d_ops | (uintptr_t)d_op_start) & 3) return (int)cudaErrorInvalidValue;
    uint32_t* d_bad = nullptr;
    cudaError_t e = pool_alloc(&d_bad, 256, stream);
    if (e != cudaSuccess) return (int)e;
    int rc = (int)cudaMemsetAsync(d_bad, 0xff, 4, stream);
    if (rc == 0) {
        rc = field == SNARKVM_B200_FIELD_FQ
                 ? run<FqParams>(d_params, d_ops, d_op_start, ntranscripts, nops, d_in, nin, d_out, nout, d_out_fr, nout_fr, d_state, d_bad,
                                              stream)
                 : run<FrParams>(d_params, d_ops, d_op_start, ntranscripts, nops, d_in, nin, d_out, nout, d_out_fr, nout_fr, d_state, d_bad,
                                              stream);
    }
    uint32_t h_bad = NO_BAD;
    if (rc == 0) rc = (int)cudaMemcpyAsync(&h_bad, d_bad, 4, cudaMemcpyDeviceToHost, stream);
    cudaFreeAsync(d_bad, stream);
    if (rc == 0) rc = (int)cudaStreamSynchronize(stream);
    if (rc != 0) return rc;
    if (h_bad != NO_BAD) {
        if (bad_transcript) *bad_transcript = (int64_t)h_bad;
        return (int)cudaErrorInvalidValue;
    }
    return 0;
}

}  // namespace b200
