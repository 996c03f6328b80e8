// K4 (v1) — fused multi-head self-attention, head_dim 64, equal-length sequences, flash-style online softmax.
// Reference arithmetic: esm/multihead_attention.py:357 (QK^T), :379 (fp32 softmax), :387 (PV); q arrives pre-scaled
// (the hd^-1/2 of :261 is folded into the packed q weights) and, for ESM2, already rotated (GEMM epilogue).
//
// This version uses warp-level mma.sync (m16n8k16, fp16 in / fp32 accumulate) with cp.async double-buffered K/V tiles.
// It is the correctness baseline for the attention path; the wgmma version (attention_wgmma.cu) is the hot kernel.
// With NSEG == 3 every operand is an fp16 hi+lo pair and each product runs three passes (hi*hi + lo*hi + hi*lo).
#include "common.h"
#include "operand.cuh"

namespace pg {

namespace {

constexpr int AQ = 64;  // queries per CTA (4 warps x 16 rows)
constexpr int AK = 64;  // keys per pipeline step
constexpr int TILE_BYTES = 64 * 128;  // 64 rows x 64 fp16

__device__ __forceinline__ uint32_t tile_addr(uint32_t tile, int row, int chunk) {
  return tile + row * 128 + ((chunk ^ (row & 7)) << 4);
}

// cp.async a 64x64 fp16 tile (rows r0.. of sequence base pointer `src`, pitch ld elements); rows >= nrows are zero-filled.
__device__ __forceinline__ void load_tile(uint32_t tile, const __half* src, long long ld, int r0, int nrows) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int id = threadIdx.x + i * 128;
    const int row = id >> 3, ch = id & 7;
    const bool ok = (r0 + row) < nrows;
    const __half* g = src + (ok ? (static_cast<long long>(r0 + row) * ld + ch * 8) : 0);
    cp_async_16(tile_addr(tile, row, ch), g, ok ? 16u : 0u);
  }
}

template <int NSEG>
__global__ void __launch_bounds__(128) attn_mma_kernel(AttnLaunch a) {
  extern __shared__ __align__(128) uint8_t smem_attn[];
  constexpr int NP = (NSEG == 3) ? 2 : 1;  // hi (+ lo) planes
  const uint32_t sQ = smem_u32(smem_attn);                 // [NP] tiles
  const uint32_t sK = sQ + NP * TILE_BYTES;                // [2 stages][NP]
  const uint32_t sV = sK + 2 * NP * TILE_BYTES;            // [2 stages][NP]

  const int q0 = a.q_begin + blockIdx.x * AQ, head = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int d = a.heads * 64;
  const __half* base = a.qkv + static_cast<long long>(b) * a.T * a.ld;
  const __half* qp = base + head * 64;
  const __half* kp = base + d + head * 64;
  const __half* vp = base + 2 * d + head * 64;
  const int nkb = a.causal ? ((min(q0 + AQ, a.T) + AK - 1) / AK) : ((a.T + AK - 1) / AK);
  const float slope = a.alibi_slopes ? a.alibi_slopes[head] : 0.f;
  constexpr float LOG2E = 1.4426950408889634f;

#pragma unroll
  for (int pl = 0; pl < NP; ++pl) load_tile(sQ + pl * TILE_BYTES, qp + pl * a.lo_off, a.ld, q0, a.T);
#pragma unroll
  for (int pl = 0; pl < NP; ++pl) {
    load_tile(sK + pl * TILE_BYTES, kp + pl * a.lo_off, a.ld, 0, a.T);
    load_tile(sV + pl * TILE_BYTES, vp + pl * a.lo_off, a.ld, 0, a.T);
  }
  cp_async_commit();

  uint32_t qf[NP][4][4];
  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const int qrow0 = q0 + warp * 16 + g, qrow1 = qrow0 + 8;

  for (int kb = 0; kb < nkb; ++kb) {
    const int st = kb & 1;
    if (kb + 1 < nkb) {
#pragma unroll
      for (int pl = 0; pl < NP; ++pl) {
        load_tile(sK + ((st ^ 1) * NP + pl) * TILE_BYTES, kp + pl * a.lo_off, a.ld, (kb + 1) * AK, a.T);
        load_tile(sV + ((st ^ 1) * NP + pl) * TILE_BYTES, vp + pl * a.lo_off, a.ld, (kb + 1) * AK, a.T);
      }
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (kb == 0) {
#pragma unroll
      for (int pl = 0; pl < NP; ++pl)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          ldmatrix_x4(qf[pl][ks], tile_addr(sQ + pl * TILE_BYTES, warp * 16 + (lane & 15), ks * 2 + (lane >> 4)));
    }
    const uint32_t kt = sK + st * NP * TILE_BYTES, vt = sV + st * NP * TILE_BYTES;

    // ---- S = Q K^T (16 x 64 per warp) ----
    float s[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        uint32_t kf[4];
        ldmatrix_x4(kf, tile_addr(kt, n * 8 + (lane & 7), j * 4 + (lane >> 3)));
        mma_16816(s[n], qf[0][2 * j], kf[0], kf[1]);
        mma_16816(s[n], qf[0][2 * j + 1], kf[2], kf[3]);
        if (NSEG == 3) {
          mma_16816(s[n], qf[NP - 1][2 * j], kf[0], kf[1]);      // q_lo * k_hi
          mma_16816(s[n], qf[NP - 1][2 * j + 1], kf[2], kf[3]);
          uint32_t kl[4];
          ldmatrix_x4(kl, tile_addr(kt + TILE_BYTES, n * 8 + (lane & 7), j * 4 + (lane >> 3)));
          mma_16816(s[n], qf[0][2 * j], kl[0], kl[1]);           // q_hi * k_lo
          mma_16816(s[n], qf[0][2 * j + 1], kl[2], kl[3]);
        }
      }
    }
    // ---- bias / masks, online softmax in the log2 domain ----
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int kidx = kb * AK + n * 8 + 2 * t + (c & 1);
        const int qidx = (c < 2) ? qrow0 : qrow1;
        float v = s[n][c] + slope * static_cast<float>(kidx);
        if (kidx >= a.T || (a.causal && kidx > qidx)) v = -INFINITY;
        s[n][c] = v * LOG2E;
      }
      mx0 = fmaxf(mx0, fmaxf(s[n][0], s[n][1]));
      mx1 = fmaxf(mx1, fmaxf(s[n][2], s[n][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    // rows beyond T (padding rows of the last query tile) may see only masked keys when causal: keep them finite
    const float ms0 = (mn0 == -INFINITY) ? 0.f : mn0, ms1 = (mn1 == -INFINITY) ? 0.f : mn1;
    const float al0 = exp2f(m0 - ms0), al1 = exp2f(m1 - ms1);
    m0 = mn0; m1 = mn1;
    l0 *= al0; l1 *= al1;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      o[n][0] *= al0; o[n][1] *= al0; o[n][2] *= al1; o[n][3] *= al1;
      s[n][0] = exp2f(s[n][0] - ms0); s[n][1] = exp2f(s[n][1] - ms0);
      s[n][2] = exp2f(s[n][2] - ms1); s[n][3] = exp2f(s[n][3] - ms1);
      l0 += s[n][0] + s[n][1];
      l1 += s[n][2] + s[n][3];
    }
    // ---- O += P V ----
#pragma unroll
    for (int j = 0; j < 4; ++j) {  // 16 keys per step
      uint32_t ph[4], pl4[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float x0 = s[2 * j + (u >> 1)][(u & 1) * 2], x1 = s[2 * j + (u >> 1)][(u & 1) * 2 + 1];
        const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
        ph[u] = pack_h2(h0, h1);
        if (NSEG == 3) pl4[u] = pack_h2(__float2half_rn(x0 - __half2float(h0)), __float2half_rn(x1 - __half2float(h1)));
      }
#pragma unroll
      for (int np = 0; np < 4; ++np) {  // pairs of 8-wide head-dim tiles
        uint32_t vf[4];
        const int row = j * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
        const int chunk = np * 2 + (lane >> 4);
        ldmatrix_x4_trans(vf, tile_addr(vt, row, chunk));
        mma_16816(o[2 * np], ph, vf[0], vf[1]);
        mma_16816(o[2 * np + 1], ph, vf[2], vf[3]);
        if (NSEG == 3) {
          mma_16816(o[2 * np], pl4, vf[0], vf[1]);
          mma_16816(o[2 * np + 1], pl4, vf[2], vf[3]);
          uint32_t vl[4];
          ldmatrix_x4_trans(vl, tile_addr(vt + TILE_BYTES, row, chunk));
          mma_16816(o[2 * np], ph, vl[0], vl[1]);
          mma_16816(o[2 * np + 1], ph, vl[2], vl[3]);
        }
      }
    }
    __syncthreads();  // everyone done with stage `st` before it is refilled
  }

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float r0 = 1.f / l0, r1 = 1.f / l1;
  __half* orow0 = a.out + (static_cast<long long>(b) * a.T + qrow0) * a.ldo;
  __half* orow1 = a.out + (static_cast<long long>(b) * a.T + qrow1) * a.ldo;
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    const int col = head * 64 + n * 8 + 2 * t;
    if (qrow0 < a.T) store_operand_pair(orow0, a.out_lo_off, 0, a.out_fmt, 0.f, col, o[n][0] * r0, o[n][1] * r0);
    if (qrow1 < a.T) store_operand_pair(orow1, a.out_lo_off, 0, a.out_fmt, 0.f, col, o[n][2] * r1, o[n][3] * r1);
  }
}

}  // namespace

int launch_attention(const AttnLaunch& al, cudaStream_t s) {
  if (al.B <= 0 || al.T <= 0) return PG_OK;
  AttnLaunch a = al;
  if (int rc = resolve_out_fmt(a.out_fmt, a.out_lo_off, a.out_scale, "attention")) return rc;
  if (a.out_fmt == 2) return set_error(PG_ERR_UNSUPPORTED, "attention: the mma.sync kernel writes fp16 planes only");
  if (a.perm_C) return set_error(PG_ERR_UNSUPPORTED, "attention: the column-attention row order is only in the wgmma kernel (attention_wgmma.cu)");
  if (a.ld % 8 || a.lo_off % 8 || a.ldo % 2 || a.out_lo_off % 2) return set_error(PG_ERR_ARG, "attention: misaligned pitches");
  if (a.nseg != 1 && a.nseg != 3) return set_error(PG_ERR_ARG, "attention: nseg must be 1 or 3");
  if (a.heads > 65535 || a.B > 65535) return set_error(PG_ERR_ARG, "attention: grid too large");
  if (a.q_begin < 0 || a.q_begin >= a.T) return set_error(PG_ERR_ARG, "attention: bad q_begin");
  dim3 grid((a.T - a.q_begin + AQ - 1) / AQ, a.heads, a.B);
  if (a.nseg == 1) {
    const int smem = 5 * TILE_BYTES;
    attn_mma_kernel<1><<<grid, 128, smem, s>>>(a);
  } else {
    const int smem = 10 * TILE_BYTES;
    int dev = 0;
    PG_CUDA_OK(cudaGetDevice(&dev));
    static bool set[64] = {};  // the attribute is per device
    if (dev < 64 && !set[dev]) {
      PG_CUDA_OK(cudaFuncSetAttribute(attn_mma_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      set[dev] = true;
    }
    attn_mma_kernel<3><<<grid, 128, smem, s>>>(a);
  }
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

}  // namespace pg
