// Block-wide radix-select step shared by the sampling and beam-search kernels (sampling.cu, beam.cu): one 8-bit digit of an
// order-preserving key.  Needs blockDim.x >= 256.
#pragma once

// hist[256] (by bin) -> the largest bin b whose count summed with every bin above it reaches k, and the count above b
__device__ __forceinline__ void radix_bucket(const int* hist, int k, int* wsum, int* out_bin, int* out_above) {
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  int h = 0, s = 0;
  if (t < 256) {
    h = hist[255 - t];                                   // thread t holds bins in descending order
    s = h;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane == 31) wsum[w] = s;
  }
  __syncthreads();
  if (t < 256) {
    for (int i = 0; i < w; ++i) s += wsum[i];
    if (s >= k && s - h < k) {
      *out_bin = 255 - t;
      *out_above = s - h;
    }
  }
  __syncthreads();
}
