// Radix-2 NTT over the BLS12-377 scalar field Fr for sm_90a.
//
// Replaces EvaluationDomain::{fft,ifft,coset_fft,coset_ifft}_in_place
// (algorithms/src/fft/domain.rs:169-221; cores :374-444; butterflies :651-773;
// bit reversal :789-804; coset scaling :239-254) and PolyMultiplier::multiply
// (algorithms/src/fft/polynomial/multiplier.rs:70-134).
//
// Semantics (bit-exact: every Fr value is canonical, so any correct algorithm
// yields identical limbs):
//   Forward/Standard : y_k = Σ_j x_j ω^{jk}, natural order in and out
//   Inverse/Standard : x_j = n^{-1} Σ_k y_k ω^{-jk}
//   Forward/Coset    : x_j ← x_j·g^j (g = 22) then Forward/Standard
//   Inverse/Coset    : Inverse/Standard then x_j ← x_j·g^{-j}
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace b200 {

enum NttDirection { NTT_FORWARD = 0, NTT_INVERSE = 1 };
enum NttType { NTT_STANDARD = 0, NTT_COSET = 1 };

// In-place (natural → natural) transform of 2^lg Fr elements at d_inout.  d_scratch must hold
// 2^lg elements when lg > NTT_SINGLE_PASS_MAX_LG (may be null otherwise; if null the scratch
// is taken from the stream-ordered pool).  Returns cudaError_t as int.
int ntt_device(void* d_inout, uint32_t lg, int direction, int type, void* d_scratch, cudaStream_t stream);

// `count` in-place transforms, transform i of 2^lgs[i] elements at d_data[i] (HOST array of device pointers), all with the same
// direction and type and each with ntt_device's result.  Transforms of equal size share their launches; sizes may be mixed.
int ntt_batch_device(void* const* d_data, const uint32_t* lgs, size_t count, int direction, int type, cudaStream_t stream);

// One transform = ntt_make_passes(lg) passes; pass p may be launched in tile ranges (see ntt.cu for the tile ↔ column-range map).
struct NttPass { int t0, S, Q; size_t tiles; };
int ntt_make_passes(uint32_t lg, NttPass* out /* ≥ 8 entries */, int* npasses);
int ntt_launch_pass(void* d_A, void* d_B, uint32_t lg, int direction, int type, int pass, size_t tile0, size_t ntiles, cudaStream_t stream);

// in-place bit-reversal permutation of 2^lg Fr elements (NR / RN / RR orders)
int fr_bitrev_device(void* d_x, uint32_t lg, cudaStream_t stream);

// d_acc[i] *= d_x[i]
int fr_pointwise_mul_device(void* d_acc, const void* d_x, size_t n, cudaStream_t stream);

// Montgomery <-> canonical conversion of n Fr elements (to_bigint / from_bigint, fp_256.rs:362-413)
int fr_from_mont_device(void* d_out, const void* d_in, size_t n, cudaStream_t stream);
int fr_to_mont_device(void* d_out, const void* d_in, size_t n, cudaStream_t stream);

static constexpr uint32_t NTT_MAX_LG = 30;

}  // namespace b200
