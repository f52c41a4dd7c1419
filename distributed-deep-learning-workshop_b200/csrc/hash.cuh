// Counter-based 32-bit hash shared by the kernels that draw random numbers on the device: dropout (gap_fwd / gap_bwd in
// elementwise.cu) and data augmentation (augment.cu).  Stateless, so a draw is a pure function of its three words and
// any kernel, any launch shape and the host-side Python references reproduce it bit for bit.
#pragma once
#include <stdint.h>

namespace b200 {

__host__ __device__ __forceinline__ uint32_t hash_u32(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t h = a * 0x9E3779B1u ^ (b + 0x7F4A7C15u) * 0x85EBCA77u ^ (c + 0x165667B1u) * 0xC2B2AE3Du;
  h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12; h *= 0x297A2D39u; h ^= h >> 15;
  return h;
}

}  // namespace b200
