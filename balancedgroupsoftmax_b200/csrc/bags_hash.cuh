// Counter-based sampling keys, shared by the head's "others" sampler (bags_kernels.cuh) and the RPN's anchor sampler
// (bags_anchor_target.cu).  A header of its own, with no kernel, so that a translation unit can use it without
// instantiating another's kernels.  tests/sampler_oracle.py restates both functions in numpy.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bags {

__device__ __forceinline__ uint32_t mix32(uint32_t x) {  // murmur3 finaliser
  x ^= x >> 16; x *= 0x85ebca6bu; x ^= x >> 13; x *= 0xc2b2ae35u; x ^= x >> 16;
  return x;
}
// for a fixed (seed, g), a bijection of n: the last step, mix32(h ^ n), is one
__device__ __forceinline__ uint32_t sample_key(unsigned long long seed, int g, int n) {
  uint32_t h = mix32(static_cast<uint32_t>(seed) ^ 0x9e3779b9u);
  h = mix32(h ^ static_cast<uint32_t>(seed >> 32));
  h = mix32(h ^ (static_cast<uint32_t>(g) * 0x632be5abu + 0x7f4a7c15u));
  h = mix32(h ^ static_cast<uint32_t>(n));
  return h;
}

}  // namespace bags
