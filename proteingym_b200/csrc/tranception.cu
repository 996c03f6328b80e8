// Tranception-specific helper kernels (HBM-bound, fp32 arithmetic):
//   gather_embed_kernel   x[row] = wte[ids[row]] (+ wpe[pos])                      (model_pytorch.py:526-532, no position table;
//                         GPT-2 modeling_gpt2.py GPT2Model.forward: inputs_embeds + position_embeds)
//   qkv_conv_kernel       depthwise causal conv (k = 1,3,5,7 by head group) on q, k and v + the 1/sqrt(hd) query scale
//                         (model_pytorch.py:73-88, :240-251, :158-159)
//   ar_head_kernel        ln_f -> lm_head (optional bias) -> log_softmax -> optional retrieval-prior fusion -> log p(next token)
//                         (model_pytorch.py:612, :783, :806-830; utils/scoring_utils.py:121-128)
//   lm_combine_kernel     the per-tile (max, sum exp) partials of the fused LM head (GEMM epi 7) -> log p(next token)
//   seq_sum_kernel        per-sequence sum over the real (non-pad) predicted tokens, fixed order
#include "common.h"
#include "operand.cuh"
#include "reduce.cuh"

namespace pg {

namespace {

// wpe (optional): learned positions, row r at position r % T + pos_off (a suffix after a shared prefix starts at pos_off).
__global__ void gather_embed_kernel(const int32_t* __restrict__ ids, const float* __restrict__ wte, int d, int vocab,
                                    float* __restrict__ x, const float* __restrict__ wpe, int T, int pos_off) {
  const long long r = blockIdx.x;
  int tok = ids[r];
  tok = tok < 0 ? 0 : (tok >= vocab ? vocab - 1 : tok);
  const float4* src = reinterpret_cast<const float4*>(wte + static_cast<long long>(tok) * d);
  float4* dst = reinterpret_cast<float4*>(x + r * d);
  if (wpe == nullptr) {
    for (int j = threadIdx.x; j < d / 4; j += blockDim.x) dst[j] = src[j];
    return;
  }
  const float4* pe = reinterpret_cast<const float4*>(wpe + (r % T + pos_off) * d);
  for (int j = threadIdx.x; j < d / 4; j += blockDim.x) {
    const float4 a = src[j], b = pe[j];
    dst[j] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
}

// Depthwise conv: the block stages a [CV_T + 6 rows] x [CV_C channels] tile (hi and lo planes) in shared memory with cp.async —
// every byte of the tile is in flight at once, independent of the arithmetic — then each thread walks down time for ONE channel pair
// with a 7-deep register window (16 tap registers, so several blocks fit per SM). One warp = the 64 channels of one head, hence
// uniform in its conv group.
// taps: [3 (q,k,v)][4 groups][64 channels][8] = 7 look-back taps + bias.
// in/out: [B*T, ld] fp16 with columns [q | k | v] (+ lo plane at lo_off). out[t] = bias + sum_o tap[o] * in[t - o].
// Blocks are numbered channel tile fastest, then time tile, then sequence.
constexpr int CV_T = 64;
constexpr int CV_C = 256;
// `prefix` (optional): the 6 raw q/k/v rows that precede row 0 of every sequence (same pitch and planes) — the look-back of a
// suffix whose earlier rows were computed elsewhere (exact wild-type-prefix reuse); null = start of sequence (zeros).
template <int NP>
__global__ void __launch_bounds__(128) qkv_conv_kernel(const __half* __restrict__ in, __half* __restrict__ out, long long ld,
                                                       long long lo_off, int T, int heads, const float* __restrict__ taps, float qscale,
                                                       const __half* __restrict__ prefix) {
  extern __shared__ __align__(16) uint8_t cv_smem[];
  constexpr int ROWS = CV_T + 6;
  constexpr int ROWB = CV_C * 2;                      // bytes per staged row and plane
  const int ctiles = 3 * heads * 64 / CV_C, ttiles = (T + CV_T - 1) / CV_T;
  const int c0 = (blockIdx.x % ctiles) * CV_C, t0 = (blockIdx.x / ctiles % ttiles) * CV_T, b = blockIdx.x / (ctiles * ttiles);
  const long long row0 = static_cast<long long>(b) * T;
  const uint32_t sbase = smem_u32(cv_smem);
  // ---- stage: rows t0-6 .. t0+CV_T-1 (zero-filled outside [0, T)), 32 16-byte chunks per row and plane ----
  for (int id = threadIdx.x; id < NP * ROWS * (ROWB / 16); id += blockDim.x) {
    const int ch = id % (ROWB / 16);
    const int r = (id / (ROWB / 16)) % ROWS;
    const int pl = id / ((ROWB / 16) * ROWS);
    const int t = t0 - 6 + r;
    bool ok = t >= 0 && t < T;
    const __half* g = in + (ok ? (row0 + t) * ld + c0 + ch * 8 + pl * lo_off : 0);
    if (t < 0 && prefix != nullptr) {
      ok = true;
      g = prefix + static_cast<long long>(6 + t) * ld + c0 + ch * 8 + pl * lo_off;
    }
    cp_async_16(sbase + (pl * ROWS + r) * ROWB + ch * 16, g, ok ? 16u : 0u);
  }
  cp_async_commit();
  // ---- this thread's channel pair: taps while the tile is in flight ----
  const int c = c0 + 2 * threadIdx.x;
  const int d = heads * 64;
  const int which = c / d, head = (c % d) / 64, chn = c % 64;
  const int group = head / (heads / 4);
  float tap[2][8];
  {
    const float4* tp4 = reinterpret_cast<const float4*>(taps + ((static_cast<long long>(which) * 4 + group) * 64 + chn) * 8);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float4 a = __ldg(tp4 + 2 * i), bq = __ldg(tp4 + 2 * i + 1);
      tap[i][0] = a.x; tap[i][1] = a.y; tap[i][2] = a.z; tap[i][3] = a.w;
      tap[i][4] = bq.x; tap[i][5] = bq.y; tap[i][6] = bq.z; tap[i][7] = bq.w;
    }
  }
  const float sc = which == 0 ? qscale : 1.f;
  cp_async_wait<0>();
  __syncthreads();
  auto rd = [&](int r, float (&v)[2]) {  // staged row r of this thread's channel pair; the lo plane lies ROWS staged rows further
    load_operand<2>(reinterpret_cast<const __half*>(cv_smem + r * ROWB) + 2 * threadIdx.x, NP == 2 ? ROWS * CV_C : 0, v);
  };
  float win[7][2];  // win[o] = input row t - o
#pragma unroll
  for (int o = 1; o < 7; ++o) rd(6 - o, win[o]);     // staged row index of time t0 - o is 6 - o
  const int nt = (T - t0) < CV_T ? (T - t0) : CV_T;
#pragma unroll 4
  for (int tt = 0; tt < nt; ++tt) {
    rd(6 + tt, win[0]);
    float acc[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float a = tap[i][7];
#pragma unroll
      for (int o = 0; o < 7; ++o) a = fmaf(tap[i][o], win[o][i], a);  // taps beyond the group's kernel length are zero
      acc[i] = a * sc;
    }
    store_operand_pair(out + (row0 + t0 + tt) * ld, lo_off, 0, NP == 2 ? 1 : 0, 0.f, c, acc[0], acc[1]);
#pragma unroll
    for (int o = 6; o > 0; --o) {
      win[o][0] = win[o - 1][0];
      win[o][1] = win[o - 1][1];
    }
  }
}

struct ArHeadParams {
  const float* x; int d; int T; int vocab;
  const int32_t* ids; const int32_t* lens;
  const float* lnf_g; const float* lnf_b; const float* wte;
  const float* bias;  // [vocab] or null
  int label_off;      // head column of token id v is v - label_off (ProGen2: the head holds vocabulary rows 5..29)
  ArFusion f;
  float* tok_logp;  // [B*T]
};

// Retrieval fusion of one log-probability (Tranception model_pytorch.py:806-830; TranceptEVE model_pytorch.py:1100-1116, and the
// non-focus-column fallbacks of :1118-1133 which the host encodes in the row indices): v = vocabulary column, r = token row.
__device__ __forceinline__ float fuse_logp(const ArFusion& f, int vocab, long long r, int v, float lp) {
  if (!f.prior_row || v < f.first_col) return lp;
  const int pr = f.prior_row[r];
  if (pr >= 0) {
    float m = (1.f - f.alpha) * lp + f.alpha * f.log_prior[static_cast<long long>(pr) * vocab + v];
    if (f.prior_row2) {
      const int pr2 = f.prior_row2[r];
      if (pr2 >= 0) m = (1.f - f.beta) * m + f.beta * f.log_prior2[static_cast<long long>(pr2) * vocab + v];
    }
    return m;
  }
  if (pr == -2) return (1.f - f.alpha) * lp;
  return lp;
}

// One block (128 threads) per token row r = (b, t): log p(ids[b, t+1] | ids[b, <=t]); 0 for t >= len-1, NaN for a next token outside
// the head's columns.
__global__ void ar_head_kernel(ArHeadParams p) {
  __shared__ float sh[33];
  extern __shared__ float dyn[];
  float* y = dyn;
  float* logits = dyn + p.d;
  const long long r = blockIdx.x;
  const int b = static_cast<int>(r / p.T), t = static_cast<int>(r % p.T);
  const int len = p.lens[b];
  if (t + 1 >= len) {  // block-uniform
    if (threadIdx.x == 0) p.tok_logp[r] = 0.f;
    return;
  }
  const float* xr = p.x + r * p.d;
  float mean, rstd;
  block_ln_stats(xr, p.d, sh, mean, rstd);
  for (int j = threadIdx.x; j < p.d; j += blockDim.x) y[j] = (xr[j] - mean) * rstd * p.lnf_g[j] + p.lnf_b[j];
  __syncthreads();
  const float lse = block_logits_lse(y, p.d, p.wte, p.bias, p.vocab, logits);
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    if (p.f.out_logprobs)
      for (int v = lane; v < p.vocab; v += 32) p.f.out_logprobs[r * p.vocab + v] = fuse_logp(p.f, p.vocab, r, v, logits[v] - lse);
    if (lane == 0) {
      const int label = p.ids[r + 1] - p.label_off;
      p.tok_logp[r] = (label < 0 || label >= p.vocab) ? NAN : fuse_logp(p.f, p.vocab, r, label, logits[label] - lse);
    }
  }
}

// One warp per token row r = (b, t) of the fused LM head: the row's (max, sum exp) partials of `tiles` N tiles merged in fixed order
// (lane k takes tiles k, k + 32, ..., then a fixed shuffle tree), lse = max + log(sum), log p = target logit - lse. out_logprobs rows
// hold the row's logits (epi 7's lm_logits) and are turned into log-probabilities in place.
__global__ void lm_combine_kernel(const float2* __restrict__ part, int tiles, const float* __restrict__ tgt, const int32_t* __restrict__ ids,
                                  const int32_t* __restrict__ lens, long long rows, int T, int vocab, float* __restrict__ out_logprobs,
                                  float* __restrict__ tok_logp) {
  const long long r = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const int t = static_cast<int>(r % T);
  if (t + 1 >= lens[r / T]) {
    if (lane == 0) tok_logp[r] = 0.f;
    return;
  }
  float m = -INFINITY, s = 0.f;
  for (int k = lane; k < tiles; k += 32) {
    const float2 q = part[r * tiles + k];
    const float mn = fmaxf(m, q.x);
    s = s * expf(m - mn) + q.y * expf(q.x - mn);
    m = mn;
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float mo = __shfl_xor_sync(0xffffffffu, m, o), so = __shfl_xor_sync(0xffffffffu, s, o);
    const float mn = fmaxf(m, mo);
    // lanes with no tile (tiles < 32) carry m = -inf, s = 0: exp(-inf - mn) = 0, and mn is finite as soon as one lane has a tile
    s = (m == -INFINITY ? 0.f : s * expf(m - mn)) + (mo == -INFINITY ? 0.f : so * expf(mo - mn));
    m = mn;
  }
  const float lse = m + logf(s);
  if (out_logprobs)
    for (int v = lane; v < vocab; v += 32) out_logprobs[r * vocab + v] -= lse;
  if (lane == 0) {
    const int label = ids[r + 1];
    tok_logp[r] = (label < 0 || label >= vocab) ? NAN : tgt[r] - lse;
  }
}

// One warp per sequence: sum tok_logp[b, 0 .. len-2] (lane-strided partials, then a fixed shuffle tree).
__global__ void seq_sum_kernel(const float* __restrict__ tok_logp, const int32_t* __restrict__ lens, int B, int T,
                               float* __restrict__ out) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int lane = threadIdx.x & 31;
  const int n = lens[b] - 1;
  float s = 0.f;
  for (int t = lane; t < n; t += 32) s += tok_logp[static_cast<long long>(b) * T + t];
  s = warp_sum(s);
  if (lane == 0) out[b] = s;
}

}  // namespace

int launch_gather_embed(const int32_t* ids, const float* wte, long long rows, int d, int vocab, float* x, cudaStream_t s, const float* wpe,
                        int T, int pos_off) {
  if (rows <= 0) return PG_OK;
  if (T <= 0) return set_error(PG_ERR_ARG, "gather_embed: T must be positive");
  gather_embed_kernel<<<static_cast<unsigned>(rows), 128, 0, s>>>(ids, wte, d, vocab, x, wpe, T, pos_off);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_qkv_conv(const __half* in, __half* out, int64_t ld, int64_t lo_off, int B, int T, int heads, const float* taps,
                    float qscale, cudaStream_t s, const __half* prefix) {
  const long long ctiles = 3 * heads * 64 / CV_C, ttiles = (T + CV_T - 1) / CV_T;
  const long long n = B * ttiles * ctiles;
  if (n <= 0) return PG_OK;
  if (heads % 4) return set_error(PG_ERR_ARG, "qkv_conv: heads must be a multiple of 4");
  if (n > 0x7FFFFFFFll) return set_error(PG_ERR_ARG, "qkv_conv: grid too large");
  const unsigned grid = static_cast<unsigned>(n);
  const int np = lo_off > 0 ? 2 : 1;
  const int smem = np * (CV_T + 6) * CV_C * 2;
  int dev = 0;
  PG_CUDA_OK(cudaGetDevice(&dev));
  static bool attr[64] = {};  // the attribute is per device
  if (dev < 64 && !attr[dev]) {
    PG_CUDA_OK(cudaFuncSetAttribute(qkv_conv_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * (CV_T + 6) * CV_C * 2));
    attr[dev] = true;
  }
  if (np == 2) qkv_conv_kernel<2><<<grid, 128, smem, s>>>(in, out, ld, lo_off, T, heads, taps, qscale, prefix);
  else qkv_conv_kernel<1><<<grid, 128, smem, s>>>(in, out, ld, lo_off, T, heads, taps, qscale, prefix);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_ar_head(const float* x, int d, int B, int T, int vocab, const int32_t* ids, const int32_t* lens, const float* lnf_g,
                   const float* lnf_b, const float* wte, const float* bias, int label_off, const ArFusion& fusion, float* tok_logp,
                   float* out_sum, cudaStream_t s) {
  if (B <= 0 || T <= 0) return PG_OK;
  ArHeadParams p{x, d, T, vocab, ids, lens, lnf_g, lnf_b, wte, bias, label_off, fusion, tok_logp};
  ar_head_kernel<<<static_cast<unsigned>(static_cast<long long>(B) * T), 128, (d + vocab) * sizeof(float), s>>>(p);
  seq_sum_kernel<<<(B + 3) / 4, 128, 0, s>>>(tok_logp, lens, B, T, out_sum);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_lm_head_combine(const float2* part, int tiles, const float* tgt, const int32_t* ids, const int32_t* lens, int B, int T, int vocab,
                           float* out_logprobs, float* tok_logp, float* out_sum, cudaStream_t s) {
  if (B <= 0 || T <= 0) return PG_OK;
  const long long rows = static_cast<long long>(B) * T;
  lm_combine_kernel<<<static_cast<unsigned>((rows + 3) / 4), 128, 0, s>>>(part, tiles, tgt, ids, lens, rows, T, vocab, out_logprobs, tok_logp);
  seq_sum_kernel<<<(B + 3) / 4, 128, 0, s>>>(tok_logp, lens, B, T, out_sum);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

}  // namespace pg
