// Warp and block reductions with one fixed summation order (lane- or thread-strided partials, xor butterfly 16 -> 1 inside the warp,
// warp partials through shared memory, butterfly again), and the two row routines built on them: the LayerNorm statistics of an fp32
// row and the tied-embedding logits + log-sum-exp of the LM heads.
#pragma once
#include <cuda_runtime.h>

namespace pg {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum for blockDim.x <= 1024 (result broadcast to all threads). sh: 33 floats of shared memory.
__device__ __forceinline__ float block_sum(float v, float* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sh[w] = v;
  __syncthreads();
  float t = (threadIdx.x < nw) ? sh[threadIdx.x] : 0.f;
  if (w == 0) {
    t = warp_sum(t);
    if (lane == 0) sh[32] = t;
  }
  __syncthreads();
  return sh[32];
}

// Two-pass LayerNorm statistics (mean, then centred variance; eps = 1e-5 like torch.nn.LayerNorm) of row[0..d), one block per row.
__device__ __forceinline__ void block_ln_stats(const float* row, int d, float* sh, float& mean, float& rstd) {
  float s = 0.f;
  for (int j = threadIdx.x; j < d; j += blockDim.x) s += row[j];
  mean = block_sum(s, sh) / d;
  float ss = 0.f;
  for (int j = threadIdx.x; j < d; j += blockDim.x) {
    const float c = row[j] - mean;
    ss += c * c;
  }
  rstd = rsqrtf(block_sum(ss, sh) / d + 1e-5f);
}

// logits[v] = y . w[v, :] (+ bias[v]) for v < vocab, one warp per vocabulary row; returns lse = log sum_v exp(logits[v]), valid in
// warp 0 only (the other warps get 0). y (shared memory, d floats) must be complete: the caller synchronises before the call.
__device__ __forceinline__ float block_logits_lse(const float* y, int d, const float* w, const float* bias, int vocab, float* logits) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int v = warp; v < vocab; v += nw) {
    const float* wr = w + static_cast<long long>(v) * d;
    float acc = 0.f;
    for (int j = lane; j < d; j += 32) acc = fmaf(y[j], wr[j], acc);
    acc = warp_sum(acc);
    if (lane == 0) logits[v] = bias ? acc + bias[v] : acc;
  }
  __syncthreads();
  if (warp != 0) return 0.f;
  float m = -INFINITY;
  for (int v = lane; v < vocab; v += 32) m = fmaxf(m, logits[v]);
  m = warp_max(m);
  float se = 0.f;
  for (int v = lane; v < vocab; v += 32) se += expf(logits[v] - m);
  se = warp_sum(se);
  return m + logf(se);
}

}  // namespace pg
