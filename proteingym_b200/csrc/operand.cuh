// The operand row formats of common.h, device side: the only place that spells out the plane order, the 2^11 gain of the lo8 plane
// and the fp32 -> fp16 / e4m3 conversions. A row is addressed as (row pointer, lo_off, pw, fmt, scale):
//   fmt 0  [hi fp16]
//   fmt 1  [hi fp16 | lo fp16]         lo plane at element lo_off
//   fmt 2  [hi fp16 | lo8 | hi8]       e4m3 planes of pw bytes each from byte 2 * lo_off: lo8 = e4m3(lo * 2^11 * s), hi8 = e4m3(hi * s)
//   weights (fmt 2 of the W side)      [hi fp16 (K) | hi8 (K bytes) | lo8 (K bytes)] with the matrix scale t
// hi = fp16(v), lo = v - hi. The stores differ only in how many columns one thread holds; each keeps the rounding of the kernels it
// serves (packed cvt for column pairs, saturating hi + RN lo for one and four columns).
#pragma once
#include "ptx.cuh"

namespace pg {

constexpr float LO8_GAIN = 2048.f;  // 2^11: brings the fp16 residual into the range of hi before the shared e4m3 scale

// fp32 -> fp16 hi (+ residual lo), saturating so an outlier cannot become inf
__device__ __forceinline__ __half f2h_sat(float v) {
  unsigned short u;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(u) : "f"(v));
  return __ushort_as_half(u);
}
__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
  return static_cast<uint32_t>(__half_as_ushort(a)) | (static_cast<uint32_t>(__half_as_ushort(b)) << 16);
}
__device__ __forceinline__ float2 unpack_h2(uint32_t h) { return __half22float2(*reinterpret_cast<const __half2*>(&h)); }
__device__ __forceinline__ void split_hi_lo(float v, __half& hi, __half& lo) {
  hi = f2h_sat(v);
  lo = __float2half_rn(v - __half2float(hi));
}
__device__ __forceinline__ uint8_t e4m3_byte(float v) { return static_cast<uint8_t>(cvt_e4m3x2(v, 0.f) & 0xff); }

// Columns col, col + 1 (col even), packed saturating converts. The GEMM and wgmma attention epilogues write the same thing out by
// hand to keep a row's plane addresses in registers across their column blocks (gemm_tc.cu).
__device__ __forceinline__ void store_operand_pair(__half* row, long long lo_off, int pw, int fmt, float scale, long long col, float x0, float x1) {
  const uint32_t hi = cvt_f16x2_rn(x0, x1);
  const float2 hf = unpack_h2(hi);
  // plane addresses ahead of the format branches: with an unrolled column loop they become one base per plane plus constants
  __half* p = row + col;
  __half* plo = row + lo_off + col;
  uint8_t* f8 = reinterpret_cast<uint8_t*>(row + lo_off) + col;
  *reinterpret_cast<uint32_t*>(p) = hi;
  if (fmt == 1) {
    *reinterpret_cast<uint32_t*>(plo) = cvt_f16x2_rn(x0 - hf.x, x1 - hf.y);
  } else if (fmt == 2) {
    const float sl = scale * LO8_GAIN;
    *reinterpret_cast<uint16_t*>(f8) = static_cast<uint16_t>(cvt_e4m3x2((x0 - hf.x) * sl, (x1 - hf.y) * sl));
    *reinterpret_cast<uint16_t*>(f8 + pw) = static_cast<uint16_t>(cvt_e4m3x2(hf.x * scale, hf.y * scale));
  }
}

// Columns col .. col + 3 (col a multiple of 4).
__device__ __forceinline__ void store_operand_quad(__half* row, long long lo_off, int pw, int fmt, float scale, long long col, const float (&y)[4]) {
  __half h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) split_hi_lo(y[j], h[j], l[j]);
  *reinterpret_cast<uint2*>(row + col) = make_uint2(pack_h2(h[0], h[1]), pack_h2(h[2], h[3]));
  if (fmt == 1) {
    *reinterpret_cast<uint2*>(row + lo_off + col) = make_uint2(pack_h2(l[0], l[1]), pack_h2(l[2], l[3]));
  } else if (fmt == 2) {
    uint8_t* f8 = reinterpret_cast<uint8_t*>(row + lo_off);
    const float sl = scale * LO8_GAIN;
    *reinterpret_cast<uint32_t*>(f8 + col) =
        pack4_e4m3((y[0] - __half2float(h[0])) * sl, (y[1] - __half2float(h[1])) * sl, (y[2] - __half2float(h[2])) * sl,
                   (y[3] - __half2float(h[3])) * sl);
    *reinterpret_cast<uint32_t*>(f8 + pw + col) =
        pack4_e4m3(__half2float(h[0]) * scale, __half2float(h[1]) * scale, __half2float(h[2]) * scale, __half2float(h[3]) * scale);
  }
}
// Zeros in columns col .. col + 3 of every plane (the padding columns [d, pw) of a row).
__device__ __forceinline__ void zero_operand_quad(__half* row, long long lo_off, int pw, int fmt, long long col) {
  *reinterpret_cast<uint2*>(row + col) = make_uint2(0u, 0u);
  if (fmt == 1) {
    *reinterpret_cast<uint2*>(row + lo_off + col) = make_uint2(0u, 0u);
  } else if (fmt == 2) {
    uint8_t* f8 = reinterpret_cast<uint8_t*>(row + lo_off);
    *reinterpret_cast<uint32_t*>(f8 + col) = 0u;
    *reinterpret_cast<uint32_t*>(f8 + pw + col) = 0u;
  }
}

// One column.
__device__ __forceinline__ void store_operand_one(__half* row, long long lo_off, int pw, int fmt, float scale, long long col, float v) {
  __half hi, lo;
  split_hi_lo(v, hi, lo);
  row[col] = hi;
  if (fmt == 1) {
    row[lo_off + col] = lo;
  } else if (fmt == 2) {
    uint8_t* f8 = reinterpret_cast<uint8_t*>(row + lo_off);
    const float hf = __half2float(hi);
    f8[col] = e4m3_byte((v - hf) * scale * LO8_GAIN);
    f8[pw + col] = e4m3_byte(hf * scale);
  }
}
// One column of a weight row in the fp16 + e4m3 format: [hi fp16 (K) | hi8 | lo8], t = the matrix scale.
__device__ __forceinline__ void store_weight_f8_one(__half* row, int K, float t, int k, float v) {
  __half hi, lo;
  split_hi_lo(v, hi, lo);
  uint8_t* f8 = reinterpret_cast<uint8_t*>(row + K);
  const float hf = __half2float(hi);
  row[k] = hi;
  f8[k] = e4m3_byte(hf * t);
  f8[K + k] = e4m3_byte((v - hf) * t * LO8_GAIN);
}

// v[0..N) = hi (+ lo when lo_off > 0) of N = 2, 4 or 8 consecutive columns at p: one 4-, 8- or 16-byte load per plane.
template <int N>
struct alignas(2 * N) HalfVec { uint32_t w[N / 2]; };
template <int N>
__device__ __forceinline__ void load_operand(const __half* p, long long lo_off, float* v) {
  const HalfVec<N> hv = *reinterpret_cast<const HalfVec<N>*>(p);
#pragma unroll
  for (int i = 0; i < N / 2; ++i) {
    const float2 f = unpack_h2(hv.w[i]);
    v[2 * i] = f.x; v[2 * i + 1] = f.y;
  }
  if (lo_off > 0) {
    const HalfVec<N> lv = *reinterpret_cast<const HalfVec<N>*>(p + lo_off);
#pragma unroll
    for (int i = 0; i < N / 2; ++i) {
      const float2 f = unpack_h2(lv.w[i]);
      v[2 * i] += f.x; v[2 * i + 1] += f.y;
    }
  }
}

}  // namespace pg
