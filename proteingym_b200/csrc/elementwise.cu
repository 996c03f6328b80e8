// K1 (embedding), K2 (LayerNorm -> fp16 hi/lo), K5 (masked-row LM head + log-softmax), K6 (mutant scoring gather).
// These are the HBM-bound helpers of the path (SURVEY.md §2.3); all arithmetic is fp32.
#include "common.h"
#include "operand.cuh"
#include "reduce.cuh"

namespace pg {

namespace {

// ---------------------------------------------------------------------------------------------------------------
// K2: one warp per row. Two-pass (mean, then centred variance) like torch.nn.LayerNorm; eps = 1e-5
// (esm/modules.py:68-81). Reads 4*d bytes, writes 2*d (hi) [+ 2*d (lo)] bytes per row.
// Each output plane is dp >= d wide: columns [d, dp) of every plane written are zeros (the K padding of the next GEMM when d is
// not a multiple of 64; statistics are over d only).
template <int MAXV, bool PAD>  // float4 vectors per lane, d <= MAXV*128; PAD: dp > d (a separate instance keeps the unpadded one lean)
__global__ void layernorm_f16_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, int rows, int d, int dp_, __half* __restrict__ out,
                                     long long ldo, long long lo_off, int fmt, float scale, int perm_R, int perm_C,
                                     const __half* __restrict__ base, int base_T) {
  const int warps_per_block = blockDim.x >> 5;
  const int dp = PAD ? dp_ : d;
  const long long row = static_cast<long long>(blockIdx.x) * warps_per_block + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + row * ldx);
  const int nv = d >> 2;
  float4 v[MAXV];
  // delta-operand mode: the shared base row is read after the two reductions (holding it in registers from here on would halve the
  // occupancy of this latency-bound kernel: measured 74 vs 47 ms/step); an L1 prefetch now hides most of that later latency
  const uint2* qr = base ? reinterpret_cast<const uint2*>(base + (row % base_T) * static_cast<long long>(d)) : nullptr;  // 4 halves per entry
  if (qr) {
    for (int o = lane * 16; o < nv; o += 512) asm volatile("prefetch.global.L1 [%0];" ::"l"(qr + o));  // one 128-byte line per lane
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + i * 32;
    if (idx < nv) {
      v[i] = xr[idx];
      s += v[i].x + v[i].y + v[i].z + v[i].w;
    }
  }
  const float mean = warp_sum(s) / d;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + i * 32;
    if (idx < nv) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
      ss += a * a + b * b + c * c + e * e;
    }
  }
  const float rstd = rsqrtf(warp_sum(ss) / d + 1e-5f);
  // perm_C > 0: input rows are (b, r, c) with c fastest; the output row is (b, c, r) — the column-attention layout of an alignment
  long long orow_idx = row;
  if (perm_C > 0) {
    const long long rc = static_cast<long long>(perm_R) * perm_C;
    const long long b = row / rc, rem = row % rc;
    orow_idx = (b * perm_C + rem % perm_C) * perm_R + rem / perm_C;
  }
  __half* orow = out + orow_idx * ldo;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + i * 32;
    if (idx < nv) {
      const float4 g = reinterpret_cast<const float4*>(gamma)[idx];
      const float4 b = reinterpret_cast<const float4*>(beta)[idx];
      float y[4] = {(v[i].x - mean) * rstd * g.x + b.x, (v[i].y - mean) * rstd * g.y + b.y,
                    (v[i].z - mean) * rstd * g.z + b.z, (v[i].w - mean) * rstd * g.w + b.w};
      if (qr) {  // delta-operand mode: the difference to the shared base row, formed in fp32 before the fp16 rounding
        const uint2 q = __ldg(qr + idx);
        const float2 q01 = __half22float2(*reinterpret_cast<const __half2*>(&q.x)), q23 = __half22float2(*reinterpret_cast<const __half2*>(&q.y));
        y[0] -= q01.x; y[1] -= q01.y; y[2] -= q23.x; y[3] -= q23.y;
      }
      store_operand_quad(orow, lo_off, dp, fmt, scale, idx * 4, y);
    }
  }
  if (!PAD) return;
  for (int c = d + lane * 4; c < dp; c += 128) zero_operand_quad(orow, lo_off, dp, fmt, c);  // 4 per lane (d and dp are multiples of 4)
}

// ---------------------------------------------------------------------------------------------------------------
// K1: one block per token row. x = E[tok] (zero for the masked token) * dropout_scale + Pos[t + 2]; optional LN-before.
// (esm1.py:123-139, esm2.py:83-94, modules.py:254-271.)  No padding exists on this path.
__global__ void embed_kernel(EmbedLaunch e) {
  __shared__ float sh[33];
  const long long r = blockIdx.x;  // row within this chunk
  const int p = static_cast<int>(r / e.T), t = static_cast<int>(r % e.T);
  const int gp = e.p_offset + p;
  const int ws = e.win_start ? e.win_start[gp] : 0;
  const int mpos = e.positions ? e.positions[gp] : -1;
  const int gi = ws + t;
  const bool masked = (gi == mpos);
  const int tok = masked ? e.mask_idx : e.tokens[gi < e.n_tokens ? gi : e.n_tokens - 1];
  // mask_ratio_observed = (#mask tokens)/T ; WT sequences never contain <mask> themselves
  const bool has_mask = (mpos >= ws && mpos < ws + e.T) || e.force_mask_scale;
  float scale = 1.f;
  if (e.token_dropout) {
    const float ratio = has_mask ? 1.0f / static_cast<float>(e.T) : 0.f;
    scale = (1.f - 0.15f * 0.8f) / (1.f - ratio);
  }
  const float* er = e.embed + static_cast<long long>(tok) * e.d;
  const float* pr = e.pos_table ? e.pos_table + static_cast<long long>(t + 2) * e.d : nullptr;
  float* xr = e.x + r * e.d;
  for (int j = threadIdx.x; j < e.d; j += blockDim.x) {
    float v = er[j];
    if (e.token_dropout) v = (masked ? 0.f : v) * scale;
    if (pr) v += pr[j];
    xr[j] = v;
  }
  if (e.lnb_gamma) {  // every thread reads back the columns it wrote itself
    float mean, rstd;
    block_ln_stats(xr, e.d, sh, mean, rstd);
    for (int j = threadIdx.x; j < e.d; j += blockDim.x) xr[j] = (xr[j] - mean) * rstd * e.lnb_gamma[j] + e.lnb_beta[j];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// K5a: gather the rows to emit and apply emb_layer_norm_after -> scratch_a [P, d]
__global__ void head_gather_ln_kernel(HeadLaunch h) {
  __shared__ float sh[33];
  const int p = blockIdx.x;
  const long long src = h.all_rows ? p : static_cast<long long>(p) * h.T + h.row_in_seq[p];
  const float* xr = h.x + src * h.d;
  float mean, rstd;
  block_ln_stats(xr, h.d, sh, mean, rstd);
  float* o = h.scratch_a + static_cast<long long>(p) * h.d;
  for (int j = threadIdx.x; j < h.d; j += blockDim.x) o[j] = (xr[j] - mean) * rstd * h.lna_g[j] + h.lna_b[j];
}

// K5b: scratch_b[P, d] = gelu(scratch_a[P, d] * dense_w[d, d]^T + dense_b)   (fp32 SIMT, 64x64 tiles, 4x4 per thread)
__global__ void __launch_bounds__(256) head_dense_kernel(const float* __restrict__ A, const float* __restrict__ W,
                                                         const float* __restrict__ bias, float* __restrict__ C, int M, int N,
                                                         int K) {
  __shared__ float As[16][65];
  __shared__ float Ws[16][65];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int r = i >> 4, c = i & 15;
      As[c][r] = (m0 + r < M && k0 + c < K) ? A[static_cast<long long>(m0 + r) * K + k0 + c] : 0.f;
      Ws[c][r] = (n0 + r < N && k0 + c < K) ? W[static_cast<long long>(n0 + r) * K + k0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      float a[4], w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        a[i] = As[k][ty * 4 + i];
        w[i] = Ws[k][tx * 4 + i];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
    }
    __syncthreads();
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
      if (m < M && n < N) {
        const float v = acc[i][j] + bias[n];
        C[static_cast<long long>(m) * N + n] = 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
      }
    }
}

// K5c: per row: LayerNorm -> logits over vocab (tied embedding + bias) -> log_softmax.  One block (128 thr) per row.
__global__ void head_logits_kernel(HeadLaunch h) {
  __shared__ float sh[33];
  extern __shared__ float dyn[];  // d floats: normalised row; then vocab logits
  float* y = dyn;
  float* logits = dyn + h.d;
  const int p = blockIdx.x;
  const float* xr = h.scratch_b + static_cast<long long>(p) * h.d;
  float mean, rstd;
  block_ln_stats(xr, h.d, sh, mean, rstd);
  for (int j = threadIdx.x; j < h.d; j += blockDim.x) y[j] = (xr[j] - mean) * rstd * h.ln_g[j] + h.ln_b[j];
  __syncthreads();
  const float lse = block_logits_lse(y, h.d, h.out_w, h.out_b, h.vocab, logits);
  if (threadIdx.x < 32)
    for (int v = threadIdx.x; v < h.vocab; v += 32) h.out[static_cast<long long>(p) * h.vocab + v] = logits[v] - lse;
}

// ---------------------------------------------------------------------------------------------------------------
// K6: score[m] = sum over sites (table[row, mt] - table[row, wt]); sequential per mutant => fixed summation order.
__global__ void score_kernel(const float* __restrict__ table, int n_rows, int vocab, const int32_t* __restrict__ site_row,
                             const int32_t* __restrict__ site_wt, const int32_t* __restrict__ site_mt,
                             const int32_t* __restrict__ row_offsets, int M, float* __restrict__ out) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float s = 0.f;
  for (int i = row_offsets[m]; i < row_offsets[m + 1]; ++i) {
    const int r = site_row[i];
    const float* tr = table + static_cast<long long>(r) * vocab;
    s += tr[site_mt[i]] - tr[site_wt[i]];
  }
  out[m] = s;
}

// ---------------------------------------------------------------------------------------------------------------
// Last-layer pruning (exact): only the masked row of each copy feeds the LM head, so in the final layer the attention
// output, out_proj, LayerNorm and MLP are needed for ONE query row per sequence (SURVEY.md §0.3c). K and V still come
// from all rows. One warp per (sequence, head); fp32 SIMT arithmetic on the fp16 hi(+lo) q/k/v.
__global__ void __launch_bounds__(128) attn_single_query_kernel(const __half* __restrict__ qkv, long long ld, long long lo_off,
                                                                const int32_t* __restrict__ row_sel, int B, int T, int heads,
                                                                __half* __restrict__ out, long long ldo, long long out_lo_off,
                                                                int out_fmt, float out_scale) {
  const int wid = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wid >= B * heads) return;
  const int b = wid / heads, h = wid % heads, lane = threadIdx.x & 31;
  const int d = heads * 64;
  const __half* base = qkv + static_cast<long long>(b) * T * ld;
  auto load64 = [&](const __half* p, float (&v)[64]) {
#pragma unroll
    for (int c = 0; c < 8; ++c) load_operand<8>(p + c * 8, lo_off, v + c * 8);
  };
  float q[64];
  load64(base + static_cast<long long>(row_sel[b]) * ld + h * 64, q);
  float m = -INFINITY, l = 0.f, acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  for (int j = lane; j < T; j += 32) {
    float kv[64];
    load64(base + static_cast<long long>(j) * ld + d + h * 64, kv);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) s = fmaf(q[i], kv[i], s);
    const float mn = fmaxf(m, s);
    const float corr = __expf(m - mn), pj = __expf(s - mn);
    m = mn;
    l = l * corr + pj;
    load64(base + static_cast<long long>(j) * ld + 2 * d + h * 64, kv);
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = fmaf(acc[i], corr, pj * kv[i]);
  }
  const float mw = warp_max(m);
  const float sc = (m == -INFINITY) ? 0.f : __expf(m - mw);  // lanes that saw no key (T < 32) contribute nothing
  l = warp_sum(l * sc);
  const float rl = 1.f / l;
  __half* orow = out + static_cast<long long>(b) * ldo;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const float v = warp_sum(acc[i] * sc) * rl;
    if (lane == (i & 31)) store_operand_one(orow, out_lo_off, d, out_fmt, out_scale, h * 64 + i, v);
  }
}

// ESM C attention (esm/layers/attention.py:50-60, rotary.py:36-65): q = q_ln(q) and k = k_ln(k) — LayerNorm over the full width d,
// weight only, eps 1e-5 — then rotate-half rotary on every 64-wide head (token index t = row % T, tables [T, 32]) and q *= 64^-1/2
// (exact). In place on the fp16 hi [+ lo] q/k rows (fmt 0 / 1) the QKV GEMM wrote: the statistics span the whole row, 7.5-9 of the
// GEMM's 128-column tiles, so they cannot live in its epilogue. One warp per (row, q or k); lane l holds columns 64h + l and
// 64h + 32 + l of every head h, which is exactly a rotary pair.
template <int MAXH>
__global__ void __launch_bounds__(256) qk_ln_rotary_kernel(__half* __restrict__ qkv, long long ld, long long lo_off, int rows, int heads,
                                                           const float* __restrict__ q_gamma, const float* __restrict__ k_gamma,
                                                           const float* __restrict__ rot_cos, const float* __restrict__ rot_sin, int T) {
  const long long w = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= 2LL * rows) return;
  const long long row = w >> 1;
  const int is_k = static_cast<int>(w & 1), lane = threadIdx.x & 31, d = heads * 64;
  __half* p = qkv + row * ld + is_k * d;
  const float* g = is_k ? k_gamma : q_gamma;
  float a[MAXH], b[MAXH];
  float s = 0.f;
#pragma unroll
  for (int h = 0; h < MAXH; ++h) {
    if (h < heads) {
      a[h] = __half2float(p[64 * h + lane]);
      b[h] = __half2float(p[64 * h + 32 + lane]);
      if (lo_off > 0) {
        a[h] += __half2float(p[lo_off + 64 * h + lane]);
        b[h] += __half2float(p[lo_off + 64 * h + 32 + lane]);
      }
      s += a[h] + b[h];
    }
  }
  const float mean = warp_sum(s) / d;
  float ss = 0.f;
#pragma unroll
  for (int h = 0; h < MAXH; ++h) {
    if (h < heads) {
      const float x = a[h] - mean, y = b[h] - mean;
      ss += x * x + y * y;
    }
  }
  const float rstd = rsqrtf(warp_sum(ss) / d + 1e-5f);
  const int t = static_cast<int>(row % T);
  const float co = __ldg(rot_cos + t * 32 + lane), si = __ldg(rot_sin + t * 32 + lane);
  const float sc = is_k ? 1.f : 0.125f;
  const int fmt = lo_off > 0 ? 1 : 0;
#pragma unroll
  for (int h = 0; h < MAXH; ++h) {
    if (h < heads) {
      const float x = (a[h] - mean) * rstd * __ldg(g + 64 * h + lane), y = (b[h] - mean) * rstd * __ldg(g + 64 * h + 32 + lane);
      store_operand_one(p, lo_off, d, fmt, 0.f, 64 * h + lane, (x * co - y * si) * sc);
      store_operand_one(p, lo_off, d, fmt, 0.f, 64 * h + 32 + lane, (y * co + x * si) * sc);
    }
  }
}

__global__ void gather_rows_kernel(const float* __restrict__ x, const int32_t* __restrict__ row_sel, int T, int d,
                                   float* __restrict__ xc) {
  const int b = blockIdx.x;
  const float4* src = reinterpret_cast<const float4*>(x + (static_cast<long long>(b) * T + row_sel[b]) * d);
  float4* dst = reinterpret_cast<float4*>(xc + static_cast<long long>(b) * d);
  for (int j = threadIdx.x; j < d / 4; j += blockDim.x) dst[j] = src[j];
}

}  // namespace

int launch_attn_single_query(const __half* qkv, int64_t ld, int64_t lo_off, const int32_t* row_sel, int B, int T, int heads,
                             __half* out, int64_t ldo, int64_t out_lo_off, cudaStream_t s, int out_fmt, float out_scale) {
  if (B <= 0) return PG_OK;
  if (int rc = resolve_out_fmt(out_fmt, out_lo_off, out_scale, "attn_single_query")) return rc;
  attn_single_query_kernel<<<(B * heads + 3) / 4, 128, 0, s>>>(qkv, ld, lo_off, row_sel, B, T, heads, out, ldo, out_lo_off, out_fmt,
                                                              out_scale);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_qk_ln_rotary(__half* qkv, int64_t ld, int64_t lo_off, int rows, int heads, const float* q_gamma, const float* k_gamma,
                        const float* rot_cos, const float* rot_sin, int T, cudaStream_t s) {
  if (rows <= 0) return PG_OK;
  if (heads <= 0 || heads > 24 || T <= 0 || !q_gamma || !k_gamma || !rot_cos || !rot_sin)
    return set_error(PG_ERR_ARG, "qk_ln_rotary: needs 1..24 heads of 64, T > 0, q/k weights and rotary tables");
  const long long warps = 2LL * rows;
  qk_ln_rotary_kernel<24><<<static_cast<unsigned>((warps + 7) / 8), 256, 0, s>>>(qkv, ld, lo_off, rows, heads, q_gamma, k_gamma, rot_cos,
                                                                               rot_sin, T);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_gather_rows(const float* x, const int32_t* row_sel, int B, int T, int d, float* xc, cudaStream_t s) {
  if (B <= 0) return PG_OK;
  gather_rows_kernel<<<B, 128, 0, s>>>(x, row_sel, T, d, xc);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

static __global__ void scatter_rows_kernel(const uint8_t* __restrict__ src, long long src_pitch, uint8_t* __restrict__ dst, long long dst_pitch,
                                    const int32_t* __restrict__ row_sel, int T, int row_bytes) {
  const int b = blockIdx.x;
  const uint4* s = reinterpret_cast<const uint4*>(src + b * src_pitch);
  uint4* d = reinterpret_cast<uint4*>(dst + (static_cast<long long>(b) * T + row_sel[b]) * dst_pitch);
  for (int i = threadIdx.x; i < row_bytes / 16; i += blockDim.x) d[i] = s[i];
}

int launch_scatter_rows(const void* src, int64_t src_pitch_bytes, void* dst, int64_t dst_pitch_bytes, const int32_t* row_sel, int B, int T,
                        int row_bytes, cudaStream_t s) {
  if (B <= 0) return PG_OK;
  if (row_bytes % 16 || src_pitch_bytes % 16 || dst_pitch_bytes % 16 || (reinterpret_cast<uintptr_t>(src) & 15) ||
      (reinterpret_cast<uintptr_t>(dst) & 15))
    return set_error(PG_ERR_ARG, "scatter_rows: rows must be 16-byte aligned multiples of 16 bytes");
  scatter_rows_kernel<<<B, 256, 0, s>>>(static_cast<const uint8_t*>(src), src_pitch_bytes, static_cast<uint8_t*>(dst), dst_pitch_bytes,
                                        row_sel, T, row_bytes);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_layernorm_f16(const float* x, int64_t ldx, const float* gamma, const float* beta, int rows, int d, __half* out,
                         int64_t ldo, int64_t lo_off, cudaStream_t s, int fmt, float scale, int perm_R, int perm_C, const __half* base,
                         int base_T, int dp) {
  if (rows <= 0) return PG_OK;
  if (base && (base_T <= 0 || perm_C > 0)) return set_error(PG_ERR_ARG, "layernorm: a base needs base_T > 0 and no row permutation");
  if (perm_C > 0 && (perm_R <= 0 || rows % (perm_R * perm_C))) return set_error(PG_ERR_ARG, "layernorm: rows must be whole [R, C] alignments");
  if (dp <= 0) dp = d;
  if (d % 4 || dp % 4 || dp < d || ldx % 4 || ldo % 4 || lo_off % 4) return set_error(PG_ERR_ARG, "layernorm: d, the plane width and pitches must be multiples of 4");
  if (base && dp != d) return set_error(PG_ERR_ARG, "layernorm: a base needs unpadded rows");
  if (int rc = resolve_out_fmt(fmt, lo_off, scale, "layernorm")) return rc;
  const int wpb = 8;
  const int grid = (rows + wpb - 1) / wpb;
#define PG_LN(MAXV)                                                                                                               \
  (dp > d ? layernorm_f16_kernel<MAXV, true><<<grid, wpb * 32, 0, s>>>(x, ldx, gamma, beta, rows, d, dp, out, ldo, lo_off, fmt, scale, \
                                                                       perm_R, perm_C, base, base_T)                                 \
          : layernorm_f16_kernel<MAXV, false><<<grid, wpb * 32, 0, s>>>(x, ldx, gamma, beta, rows, d, dp, out, ldo, lo_off, fmt, scale, \
                                                                        perm_R, perm_C, base, base_T))
  if (d <= 128 * 4) PG_LN(4);
  else if (d <= 128 * 10) PG_LN(10);
  else if (d <= 128 * 20) PG_LN(20);
  else if (d <= 128 * 40) PG_LN(40);
#undef PG_LN
  else return set_error(PG_ERR_UNSUPPORTED, "layernorm: d > 5120");
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_embed(const EmbedLaunch& e, cudaStream_t s) {
  const long long rows = static_cast<long long>(e.P) * e.T;
  if (rows <= 0) return PG_OK;
  embed_kernel<<<static_cast<unsigned>(rows), 256, 0, s>>>(e);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_head(const HeadLaunch& h, cudaStream_t s) {
  if (h.P <= 0) return PG_OK;
  head_gather_ln_kernel<<<h.P, 256, 0, s>>>(h);
  dim3 grid((h.d + 63) / 64, (h.P + 63) / 64);
  head_dense_kernel<<<grid, 256, 0, s>>>(h.scratch_a, h.dense_w, h.dense_b, h.scratch_b, h.P, h.d, h.d);
  head_logits_kernel<<<h.P, 128, (h.d + h.vocab) * sizeof(float), s>>>(h);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_score(const float* table, int n_rows, int vocab, const int32_t* site_row, const int32_t* site_wt,
                 const int32_t* site_mt, const int32_t* row_offsets, int M, float* out, cudaStream_t s) {
  if (M <= 0) return PG_OK;
  score_kernel<<<(M + 255) / 256, 256, 0, s>>>(table, n_rows, vocab, site_row, site_wt, site_mt, row_offsets, M, out);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

}  // namespace pg
