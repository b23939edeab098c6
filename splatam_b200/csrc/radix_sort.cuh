// radix_sort.cuh -- hand-written stable LSD radix sort of (u32 key, u32 value) pairs for the two orderings of the
// rasterizer (Gaussians by depth bits; tile instances by tile id), replacing the reference's
// cub::DeviceRadixSort::SortPairs (X/cuda_rasterizer/rasterizer_impl.cu:304-309).  See radix_sort.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

namespace sb {

// Scratch for one sort of up to `capacity` pairs over `bits` key bits (8-bit digits): the per-tile digit counts that
// every pass re-uses, the digit totals, and one ping-pong pair buffer.  Never decreases as the capacity grows, so a
// temp sized for one capacity serves every smaller one.
size_t radix_temp_bytes(int capacity, int bits);

// Stable ascending sort of the n pairs (keys_in[i], vals_in ? vals_in[i] : i) by key bits [begin_bit, end_bit).
//   n = n_dev ? min(*n_dev, capacity) : capacity   (n_dev: device-side count, read by the kernels -- no host sync)
// The result is written to (keys_out, vals_out); keys_in / vals_in are not modified.  All launches go to `st`.
int radix_sort_pairs(const uint32_t* keys_in, const uint32_t* vals_in, uint32_t* keys_out, uint32_t* vals_out,
                     int capacity, const int32_t* n_dev, int begin_bit, int end_bit, void* temp, size_t temp_bytes,
                     cudaStream_t st);

}  // namespace sb
