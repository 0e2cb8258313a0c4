// THCCeilDiv of the THC runtime, for the reference's NMS extension (see THC.h beside it).
#pragma once

template <typename T>
__host__ __device__ __forceinline__ T THCCeilDiv(T a, T b) {
  return (a + b - 1) / b;
}
