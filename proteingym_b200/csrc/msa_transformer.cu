// Alignment-specific kernels of the MSA Transformer forward (esm/model/msa_transformer.py:150-222, esm/axial_attention.py):
// the embedding of a [B, R, C] block of masked alignments, and the data movement + softmax around the two tensor-core GEMMs of the
// TIED row attention (axial_attention.py:115-181):
//     S[b,h][i,j] = sum_r sum_d q[b,r,i,h,d] k[b,r,j,h,d]          one [C, C] map per head, K = R * 64   (grouped GEMM, gemm_tc.cu)
//     P           = softmax_j(S / sqrt(R))                          (q carries head_dim^-1/2 already)
//     ctx[b,r,i,h,:] = sum_j P[b,h][i,j] v[b,r,j,h,:]               N = R * 64, K = C                     (grouped GEMM)
// Both products are plain "A x W^T" GEMMs once q / k are regrouped as [(b,h,i), (r,d)], v as [(b,h,r,d), j] and the result is
// scattered back to token rows; those regroupings are the 128-byte-chunk permutations and the 64x64 transpose below (HBM-bound
// copies, ~5 % of a layer). The column attention needs nothing here: LayerNorm writes its rows in (b, c, r) order and the
// attention kernel writes its output back in (b, r, c) order (attention_tc4.cu perm_C).
#include "common.h"
#include "operand.cuh"
#include "reduce.cuh"

namespace pg {
namespace {

// One block per token row (b, r, c): x = LayerNorm_before(E[tok] + Pos[c + 2] + RowPos[r]); the token at (row 0, column positions[p])
// is <mask>. msa_transformer.py:157-172; LearnedPositionalEmbedding positions = column + 2 (modules.py:254-271), no padding here.
constexpr int EMB_MAXV = 8;  // d <= 256 * 8
__global__ void msa_embed_kernel(MsaEmbedLaunch e) {
  __shared__ float sh[33];
  const long long row = blockIdx.x;
  const int c = static_cast<int>(row % e.Cw);
  const int r = static_cast<int>((row / e.Cw) % e.R);
  const int b = static_cast<int>(row / (static_cast<long long>(e.Cw) * e.R));
  const int p = e.p_offset + b;
  const int col = (e.win_start ? e.win_start[p] : 0) + c;
  int tok = e.tokens[static_cast<long long>(r) * e.Cfull + col];
  if (r == 0 && col == e.positions[p]) tok = e.mask_idx;
  const float* et = e.embed + static_cast<long long>(tok) * e.d;
  const float* pt = e.pos_table + static_cast<long long>(c + 2) * e.d;
  const float* rt = e.row_pos ? e.row_pos + static_cast<long long>(r) * e.d : nullptr;
  float v[EMB_MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < EMB_MAXV; ++i) {
    const int k = threadIdx.x + i * blockDim.x;
    v[i] = 0.f;
    if (k < e.d) {
      v[i] = et[k] + pt[k];
      if (rt) v[i] += rt[k];
      s += v[i];
    }
  }
  const float mean = block_sum(s, sh) / e.d;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < EMB_MAXV; ++i) {
    const int k = threadIdx.x + i * blockDim.x;
    if (k < e.d) ss += (v[i] - mean) * (v[i] - mean);
  }
  const float rstd = rsqrtf(block_sum(ss, sh) / e.d + 1e-5f);
  float* xr = e.x + row * e.d;
#pragma unroll
  for (int i = 0; i < EMB_MAXV; ++i) {
    const int k = threadIdx.x + i * blockDim.x;
    if (k < e.d) xr[k] = (v[i] - mean) * rstd * e.gamma[k] + e.beta[k];
  }
}

// q and k of the fused projection, token rows (b, r, i) x [plane][which][h][64] -> tied rows (b, h, i) x [plane][r][64].
// One block per (b, i, which): thread = (plane, head, 16-byte unit) walks the R alignment rows with pointer increments only (a
// per-chunk index decomposition made the first version of this copy instruction-bound: five integer divisions per 16 bytes).
// Per step a block reads np x H x 128 contiguous bytes of one token row and appends one 128-byte chunk to each of its np x H tied rows.
__global__ void tied_gather_qk_kernel(const __half* __restrict__ qkv, long long ldq, long long lo_off, int R, int C, int H, int np,
                                      int Cp, __half* __restrict__ tq, __half* __restrict__ tk, long long ldt) {
  const int i = blockIdx.x, which = blockIdx.y, b = blockIdx.z;
  const int t = threadIdx.x;
  if (t >= np * H * 8) return;
  const int u = t & 7, h = (t >> 3) % H, pl = (t >> 3) / H;
  const int d = H * 64;
  const uint4* src = reinterpret_cast<const uint4*>(qkv + (static_cast<long long>(b) * R * C + i) * ldq + pl * lo_off + which * d + h * 64) + u;
  uint4* dst = reinterpret_cast<uint4*>((which ? tk : tq) + ((static_cast<long long>(b) * H + h) * Cp + i) * ldt +
                                        static_cast<long long>(pl) * R * 64) + u;
  const long long sstep = static_cast<long long>(C) * ldq / 8;  // one alignment row further, in 16-byte units
#pragma unroll 4
  for (int r = 0; r < R; ++r) dst[r * 8] = src[r * sstep];
}

// v, token rows (b, r, j) x [plane][2d + h*64 + dd] -> tied rows (b, h, r, dd) x [plane][j] (j padded with zeros to Kp): 64x64 tiles
// through shared memory.
__global__ void tied_transpose_v_kernel(const __half* __restrict__ qkv, long long ldq, long long lo_off, int R, int C, int H, int Kp,
                                        __half* __restrict__ tv, long long ldv) {
  __shared__ __half tile[64][72];
  const int jt = blockIdx.x, r = blockIdx.y;
  const int h = blockIdx.z % H;
  const int bp = blockIdx.z / H;  // b * np + plane
  const int np = (lo_off > 0) ? 2 : 1;
  const int b = bp / np, pl = bp % np;
  const int d = H * 64;
  const int t = threadIdx.x;
  {
    const int j = jt * 64 + (t >> 2), d0 = (t & 3) * 16;
    uint4 a = make_uint4(0, 0, 0, 0), c = a;
    if (j < C) {
      const __half* src = qkv + ((static_cast<long long>(b) * R + r) * C + j) * ldq + pl * lo_off + 2 * d + h * 64 + d0;
      a = reinterpret_cast<const uint4*>(src)[0];
      c = reinterpret_cast<const uint4*>(src)[1];
    }
    *reinterpret_cast<uint4*>(&tile[t >> 2][d0]) = a;
    *reinterpret_cast<uint4*>(&tile[t >> 2][d0 + 8]) = c;
  }
  __syncthreads();
  {
    const int dd = t & 63, j0 = (t >> 6) * 16;  // consecutive lanes read consecutive head-dim columns of the tile: no bank conflicts
    __align__(16) __half out[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) out[k] = tile[j0 + k][dd];
    __half* dst = tv + (((static_cast<long long>(b) * H + h) * R + r) * 64 + dd) * ldv + static_cast<long long>(pl) * Kp + jt * 64 + j0;
    reinterpret_cast<uint4*>(dst)[0] = *reinterpret_cast<const uint4*>(&out[0]);
    reinterpret_cast<uint4*>(dst)[1] = *reinterpret_cast<const uint4*>(&out[8]);
  }
}

// One warp per attention row (b, h, i): P = softmax_j(scale * S[., j]), j < C, as fp16 hi [+ lo] planes of Kp columns (zero padded).
__global__ void tied_softmax_kernel(const float* __restrict__ S, long long lds, int G, int C, int Cp, int Kp, float scale,
                                    __half* __restrict__ P, long long ldp, int np) {
  const long long w = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= static_cast<long long>(G) * C) return;
  const long long row = (w / C) * Cp + (w % C);
  const float* s = S + row * lds;
  float m = -INFINITY;
  for (int j = lane; j < C; j += 32) m = fmaxf(m, s[j] * scale);
  m = warp_max(m);
  float l = 0.f;
  for (int j = lane; j < C; j += 32) l += expf(s[j] * scale - m);
  l = warp_sum(l);
  __half* p = P + row * ldp;
  for (int j = lane; j < Kp; j += 32) {
    const float v = (j < C) ? expf(s[j] * scale - m) / l : 0.f;
    store_operand_one(p, Kp, 0, np == 2 ? 1 : 0, 0.f, j, v);
  }
}

// Context rows back to token order: for every (b, h, i, r) the 64-column chunk r of tied row (b, h, i) goes to columns h*64.. of token
// row (b, r, i), plane by plane (fp16 planes: 128-byte chunks; e4m3 planes: 64-byte chunks). One block per (b, i); thread = (plane,
// head, 16-byte unit) walks r with pointer increments, so a block writes whole planes of one token row per step.
struct ScatterPlanes {
  int n;                       // planes
  long long src_off[3], dst_off[3];  // byte offset of the plane in a tied row / in a token row
  int cb[3];                   // chunk bytes: 128 or 64
  int first[4];                // first thread of each plane (first[n] = threads in use)
};
__global__ void tied_scatter_out_kernel(const uint8_t* __restrict__ src, long long src_pitch, uint8_t* __restrict__ dst, long long dst_pitch,
                                        ScatterPlanes P, int R, int C, int H, int Cp) {
  const int i = blockIdx.x, b = blockIdx.y;
  const int t = threadIdx.x;
  if (t >= P.first[P.n]) return;
  int pl = 0;
  while (pl + 1 < P.n && t >= P.first[pl + 1]) ++pl;
  const int upc = P.cb[pl] >> 4;  // 16-byte units per chunk
  const int k = t - P.first[pl];
  const int u = k % upc, h = k / upc;
  const uint4* s = reinterpret_cast<const uint4*>(src + ((static_cast<long long>(b) * H + h) * Cp + i) * src_pitch + P.src_off[pl]) + u;
  uint4* d = reinterpret_cast<uint4*>(dst + (static_cast<long long>(b) * R * C + i) * dst_pitch + P.dst_off[pl] + static_cast<long long>(h) * P.cb[pl]) + u;
  const long long dstep = static_cast<long long>(C) * dst_pitch / 16;
#pragma unroll 4
  for (int r = 0; r < R; ++r) d[r * dstep] = s[r * upc];
}

// ---- exact pruning of the last layer: only (row 0, column sel[b]) of each alignment feeds the LM head ------------------------------
// Its column attention needs the row-attention output at column sel[b] for every alignment row, and that needs ONE row of each head's
// tied attention map: S1[b,h,j] = scale * sum_r q[b,r,sel_b,h,:] . k[b,r,j,h,:]. fp32 SIMT arithmetic on the fp16 hi(+lo) planes; K and
// V are read once (HBM-bound), everything downstream runs on B*R (then B) rows.
// grid (C, B), block H * 16: thread = (head, 4 of the 64 head dims)
__global__ void tied_col_scores_kernel(const __half* __restrict__ qkv, long long ldq, long long lo_off, const int32_t* __restrict__ sel,
                                       int R, int C, int H, float scale, float* __restrict__ S1) {
  const int j = blockIdx.x, b = blockIdx.y;
  const int h = threadIdx.x >> 4, l = threadIdx.x & 15;
  const bool live = h < H;  // the block is padded to whole warps (the shuffles below need them)
  const int hh = live ? h : 0;
  const int d = H * 64;
  const __half* q = qkv + (static_cast<long long>(b) * R * C + sel[b]) * ldq + hh * 64 + l * 4;
  const __half* k = qkv + (static_cast<long long>(b) * R * C + j) * ldq + d + hh * 64 + l * 4;
  const long long step = static_cast<long long>(C) * ldq;
  float acc = 0.f;
  for (int r = 0; r < (live ? R : 0); ++r) {
    float a[4], c[4];
    load_operand<4>(q + r * step, lo_off, a);
    load_operand<4>(k + r * step, lo_off, c);
    acc = fmaf(a[0], c[0], fmaf(a[1], c[1], fmaf(a[2], c[2], fmaf(a[3], c[3], acc))));
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o, 16);
  if (live && l == 0) S1[(static_cast<long long>(b) * H + h) * C + j] = acc * scale;
}
// one warp per (b, h): in-place softmax over the C keys
__global__ void tied_col_softmax_kernel(float* __restrict__ S1, int G, int C) {
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= G) return;
  float* s = S1 + static_cast<long long>(w) * C;
  float m = -INFINITY;
  for (int j = lane; j < C; j += 32) m = fmaxf(m, s[j]);
  m = warp_max(m);
  float l = 0.f;
  for (int j = lane; j < C; j += 32) l += expf(s[j] - m);
  l = warp_sum(l);
  for (int j = lane; j < C; j += 32) s[j] = expf(s[j] - m) / l;
}
// grid (R, B), block H * 16: ctx[(b, r)][h, :] = sum_j P1[b,h,j] v[b,r,j,h,:], written as an operand row (common.h formats)
__global__ void tied_col_context_kernel(const __half* __restrict__ qkv, long long ldq, long long lo_off, const float* __restrict__ P1, int R,
                                        int C, int H, __half* __restrict__ out, long long ldo, long long out_lo_off, int out_fmt,
                                        float out_scale) {
  const int r = blockIdx.x, b = blockIdx.y;
  const int h = threadIdx.x >> 4, l = threadIdx.x & 15;
  if (h >= H) return;
  const int d = H * 64;
  const __half* v = qkv + (static_cast<long long>(b) * R + r) * C * ldq + 2 * d + h * 64 + l * 4;
  const float* p = P1 + (static_cast<long long>(b) * H + h) * C;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j = 0; j < C; ++j) {
    const float pj = __ldg(p + j);
    float x[4];
    load_operand<4>(v + j * ldq, lo_off, x);
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i] = fmaf(pj, x[i], acc[i]);
  }
  store_operand_quad(out + (static_cast<long long>(b) * R + r) * ldo, out_lo_off, d, out_fmt, out_scale, h * 64 + l * 4, acc);
}
// xr[(b, r)] = x[(b, r, sel[b])]: the residual rows of column sel[b]. grid (R, B)
__global__ void msa_gather_col_kernel(const float* __restrict__ x, const int32_t* __restrict__ sel, int R, int C, int d, float* __restrict__ xr) {
  const int r = blockIdx.x, b = blockIdx.y;
  const float4* src = reinterpret_cast<const float4*>(x + ((static_cast<long long>(b) * R + r) * C + sel[b]) * d);
  float4* dst = reinterpret_cast<float4*>(xr + (static_cast<long long>(b) * R + r) * d);
  for (int k = threadIdx.x; k < d / 4; k += blockDim.x) dst[k] = src[k];
}

}  // namespace

int launch_msa_embed(const MsaEmbedLaunch& e, cudaStream_t s) {
  const long long rows = static_cast<long long>(e.B) * e.R * e.Cw;
  if (rows <= 0) return PG_OK;
  if (e.d > 256 * EMB_MAXV) return set_error(PG_ERR_UNSUPPORTED, "msa embed: embed_dim > 2048");
  msa_embed_kernel<<<static_cast<unsigned>(rows), 256, 0, s>>>(e);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_tied_gather_qk(const __half* qkv, int64_t ldq, int64_t lo_off, int B, int R, int C, int H, int Cp, __half* tq, __half* tk,
                          int64_t ldt, cudaStream_t s) {
  const int np = lo_off > 0 ? 2 : 1;
  if (np * H * 8 > 1024 || B > 65535) return set_error(PG_ERR_UNSUPPORTED, "tied attention: more than 64 heads or 65535 alignments per pass");
  dim3 grid(C, 2, B);
  tied_gather_qk_kernel<<<grid, (np * H * 8 + 31) / 32 * 32, 0, s>>>(qkv, ldq, lo_off, R, C, H, np, Cp, tq, tk, ldt);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_tied_transpose_v(const __half* qkv, int64_t ldq, int64_t lo_off, int B, int R, int C, int H, int Kp, __half* tv, int64_t ldv,
                            cudaStream_t s) {
  const int np = lo_off > 0 ? 2 : 1;
  if (R > 65535 || static_cast<long long>(B) * np * H > 65535) return set_error(PG_ERR_ARG, "tied attention: grid too large");
  dim3 grid(Kp / 64, R, B * np * H);
  tied_transpose_v_kernel<<<grid, 256, 0, s>>>(qkv, ldq, lo_off, R, C, H, Kp, tv, ldv);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_tied_softmax(const float* S, int64_t lds, int G, int C, int Cp, int Kp, float scale, __half* P, int64_t ldp, int np, cudaStream_t s) {
  const long long rows = static_cast<long long>(G) * C;
  tied_softmax_kernel<<<static_cast<unsigned>((rows + 7) / 8), 256, 0, s>>>(S, lds, G, C, Cp, Kp, scale, P, ldp, np);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

// fmt: operand format of both buffers (common.h); tied rows hold N = R * 64 columns per plane, token rows d = H * 64.
int launch_tied_scatter_out(const __half* ot, int64_t ldo_t, __half* out, int64_t ldo, int fmt, int B, int R, int C, int H, int Cp,
                            cudaStream_t s) {
  const long long Nt = static_cast<long long>(R) * 64, d = static_cast<long long>(H) * 64;
  ScatterPlanes P{};
  auto add = [&](long long so, long long dof, int cb) {
    P.src_off[P.n] = so; P.dst_off[P.n] = dof; P.cb[P.n] = cb;
    P.first[P.n + 1] = P.first[P.n] + H * (cb >> 4);
    ++P.n;
  };
  add(0, 0, 128);
  if (fmt == 1) add(2 * Nt, 2 * d, 128);
  if (fmt == 2) { add(2 * Nt, 2 * d, 64); add(3 * Nt, 3 * d, 64); }
  if (P.first[P.n] > 1024 || B > 65535) return set_error(PG_ERR_UNSUPPORTED, "tied attention: more than 64 heads or 65535 alignments per pass");
  dim3 grid(C, B);
  tied_scatter_out_kernel<<<grid, (P.first[P.n] + 31) / 32 * 32, 0, s>>>(reinterpret_cast<const uint8_t*>(ot), ldo_t * 2,
                                                                         reinterpret_cast<uint8_t*>(out), ldo * 2, P, R, C, H, Cp);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_tied_col_attention(const __half* qkv, int64_t ldq, int64_t lo_off, const int32_t* sel, int B, int R, int C, int H, float scale,
                              float* S1, __half* out, int64_t ldo, int64_t out_lo_off, int out_fmt, float out_scale, cudaStream_t s) {
  if (H * 16 > 1024 || B > 65535 || R > 2147483647 / 2) return set_error(PG_ERR_UNSUPPORTED, "tied attention: more than 64 heads or 65535 alignments per pass");
  if (int rc = resolve_out_fmt(out_fmt, out_lo_off, out_scale, "tied attention")) return rc;
  tied_col_scores_kernel<<<dim3(C, B), (H * 16 + 31) / 32 * 32, 0, s>>>(qkv, ldq, lo_off, sel, R, C, H, scale, S1);
  tied_col_softmax_kernel<<<(B * H + 7) / 8, 256, 0, s>>>(S1, B * H, C);
  tied_col_context_kernel<<<dim3(R, B), (H * 16 + 31) / 32 * 32, 0, s>>>(qkv, ldq, lo_off, S1, R, C, H, out, ldo, out_lo_off, out_fmt, out_scale);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_msa_gather_col(const float* x, const int32_t* sel, int B, int R, int C, int d, float* xr, cudaStream_t s) {
  if (B > 65535) return set_error(PG_ERR_UNSUPPORTED, "msa: more than 65535 alignments per pass");
  msa_gather_col_kernel<<<dim3(R, B), 128, 0, s>>>(x, sel, R, C, d, xr);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

}  // namespace pg
