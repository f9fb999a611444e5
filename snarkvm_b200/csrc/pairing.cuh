// BLS12-377 pairing on the device (pairing.cu): G2 preparation and products of pairings over a table of checks.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace b200 {

int g2_prepare_device(void* d_prepared, const void* d_points, size_t npoints, size_t stride, int64_t* bad_point, cudaStream_t stream);
int pairing_products_device(void* d_gt, uint32_t* d_is_one, void* d_miller, const void* d_g1, size_t g1_stride, const uint32_t* d_g2_index,
                            size_t npairs, const void* d_prepared, size_t nprepared, const uint32_t* d_check_start, size_t nchecks,
                            int64_t* bad_check, cudaStream_t stream);
// element-wise tower and line-step operations for snarkvm_b200_test_tower_op_device (the header documents op, k and the layouts)
int test_tower_op_device(int op, int k, void* d_out, const void* d_a, const void* d_b, const void* d_c, size_t n, cudaStream_t stream);

}  // namespace b200
