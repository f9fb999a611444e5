// Poseidon duplex sponge on the device (poseidon.cu): many independent PoseidonSponge<F, 2, 1> transcripts per launch.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace b200 {

// the header documents the operation list, the layouts and the error contract (snarkvm_b200_poseidon_transcripts_device and
// _resume_device); d_state = nullptr is a fresh sponge per transcript with nothing stored
int poseidon_transcripts_device(int field, const void* d_params, const uint32_t* d_ops, const uint32_t* d_op_start, size_t ntranscripts,
                                size_t nops, const void* d_in, size_t nin, void* d_out, size_t nout, void* d_out_fr, size_t nout_fr,
                                void* d_state, int64_t* bad_transcript, cudaStream_t stream);

}  // namespace b200
