// K3 — wgmma/TMA GEMM with fused epilogues for the linear layers of the ESM / Tranception forward
// (reference ops: esm/multihead_attention.py:243-261,395; esm/modules.py:138-140; SURVEY.md §2.3).
//
//   C[M,N] = epilogue( A[M,K] * W[N,K]^T + bias )        A, W K-major (row-major), fp32 accumulate in registers.
//
// Precision (the reference is fp32). Every operand x is an fp16 pair hi = rn(x), lo = rn(x - hi). Three operand modes:
//   nseg 1  single pass            hi*hi                                                     (fast mode, ~1e-2 on scores)
//   nseg 3  fp16 x3                hi*hi + lo*hi + hi*lo, all f16 wgmma                      (3 tensor-pipe units)
//   nseg 2  fp16 + fp8 cross terms hi*hi (f16) + [lo8 | hi8] * [hi8 | lo8]^T (e4m3 wgmma, K-concatenated, 2x rate)
//           with lo8 = e4m3(lo * 2^11 * s), hi8 = e4m3(hi * s): s = a fixed power of two on the A side (applied by the producing
//           kernel), a per-row power of two t_n on the W side (chosen at load time); the epilogue rescales by 1/(2^11 s t_n).
//           2 tensor-pipe units; emulated on CPU at true ESM-1v size: 3.0e-4 max score error (scripts/precision_f8.py).
//
// Accumulation: the K loop is cut into CHUNKS. Each chunk accumulates into a register tile from zero (the tensor core's own
// accumulation), and the chunk is then added to a second register tile in round-to-nearest fp32 (fixed order, so results stay
// deterministic). The small-magnitude cross terms come first, the hi*hi product is split into pieces of <= kchunk (default 1280)
// along K. The e4m3 wgmma of sm_90 keeps only ~14 bits while it accumulates, so its chunks are single k-blocks (128 products);
// tiny ESM2 golden table in f16f8 on an H100: max |log-prob error| 1.9e-4 this way, 2.1e-4 with the cross terms as one chunk.
//
// Structure (one persistent CTA per SM, 384 threads = 3 warpgroups, 128 x 128 output tiles; by default the CTAs run as clusters of
// two that share the W tile: each CTA loads 64 of its 128 rows and multicasts them to both, so a k-block costs 24 KB of L2 -> SM
// traffic per CTA instead of 32 KB — the 128 x 128 tile is bound by that traffic, not by the tensor cores):
//   warpgroup 0   TMA producer (one elected thread of warp 0): cp.async.bulk.tensor 2D tiles (128 rows x 128 B of A, 128 rows
//                 x 128 B of W, 128B swizzle; a row of 128 B is 64 fp16 or 128 e4m3 along K) into a 6-stage ring; 40 registers
//   warpgroups 1-2 consumers, rows [0, 64) and [64, 128) of the tile: wgmma m64n128 (K = 16 fp16 / 32 e4m3: 32 B of each row) x4
//                 per stage, then bias / erf-GELU / relu^2 / rotary / SwiGLU / tanh-GELU and fp16 hi [+ fp16 lo | + e4m3 planes for the next GEMM]
//                 stored straight from the accumulator fragments, or added into the fp32 residual stream (one owner per element), or
//                 (epi 7, K16) reduced to per-tile log-softmax partials of an LM head without storing the logits
// Roofline: tensor bound. Algorithmic FLOPs = 2*M*N*K; issued tensor-pipe work = x1 / x2 / x3 by mode.
#include <cstdlib>
#include <cstring>
#include <unordered_map>

#include "common.h"
#include "operand.cuh"

namespace pg {

namespace {

constexpr int BM = 128, BN = 128, BK = 64, STAGES = 6;
static_assert(BN == GEMM_BN, "common.h GEMM_BN sizes the LM-head partial buffers");
constexpr int GEMM_THREADS = 384;
constexpr uint32_t A_BYTES = BM * BK * 2;  // 16 KiB
constexpr uint32_t B_BYTES = BN * BK * 2;  // 16 KiB
constexpr uint32_t OFF_B = STAGES * A_BYTES;
constexpr uint32_t OFF_BAR = OFF_B + STAGES * B_BYTES;
constexpr uint32_t GEMM_SMEM = OFF_BAR + 256 + 1024;  // + barriers + 1 KiB alignment slack
constexpr int MAX_SEGS = 24;
constexpr int CONSUMER_WARPS = 8;

// One run of k-blocks with fixed operand planes. kind: 0 = fp16 (columns in elements), 1 = e4m3 (columns in bytes).
// commit: 1 = the chunk ends after this segment (fold the chunk into the accumulator).
struct GemmSeg {
  int a_col, b_col, nkb;
  short kind, commit;
};

struct GemmKParams {
  int M, N, K;
  int nsegs;
  float a_inv;            // 1 / (2^11 * s_A)
  const float* w_inv;     // [N] 1 / t_n
  int w_uniform;          // every w_inv[n] is the same value (weights packed by the library: one scale per matrix)
  GemmSeg seg[MAX_SEGS];
  const float* bias;
  __half* out; long long ldo; long long out_lo_off;
  float* resid; long long ldr;
  int out_fmt;            // 0 fp16 hi; 1 fp16 hi + fp16 lo; 2 fp16 hi + e4m3 [lo8 | hi8] byte planes
  float out_scale;        // out_fmt 2: s of the consuming GEMM (hi8 = e4m3(hi*s), lo8 = e4m3(lo*2^11*s))
  const float* rot_cos; const float* rot_sin; int rot_T; int rot_dim;
  int rot_half;           // 32: 64-wide head slots, tables [T, 32]; 64: 128-wide slots (one per N tile), tables [T, 64]
  int tiles_m, tiles_n;
  int prefetch;           // k-blocks of L2 look-ahead for the A operand (0 = off)
  // delta-operand mode (common.h GemmLaunch): shared base rows added before / subtracted after the activation, masked rows skipped
  const float* base_pre; const __half* base_post; int base_T; const int* mask_pos;
  int grp_rows_a, grp_rows_b;  // grouped (block-diagonal) mode: A rows [g*grp_rows_a, (g+1)*grp_rows_a) pair with W rows g*grp_rows_b + n
  // LM-head log-softmax partials (epi 7; common.h GemmLaunch)
  float2* lm_part; float* lm_tgt; float* lm_logits; const int32_t* lm_ids; const int32_t* lm_lens; int lm_T;
};

// Exact-erf GELU (esm/modules.py:17-24): 0.5*x*(1+erf(x/sqrt2)) = 0.5*x + 0.5*|x|*erf(|x|/sqrt2).
// erf via Abramowitz & Stegun 7.1.26 (abs error <= 1.5e-7; measured |gelu error| <= 4.7e-7, below torch's own fp32 gelu),
// branch-free: MUFU.RCP + MUFU.EX2 + FMA-pipe ops instead of erff()'s two divergent code paths. The polynomial is carried negated
// so that 1 - poly*e is a single FFMA.
__device__ __forceinline__ float gelu_erf(float x) {
  const float ax = fabsf(x);
  float t, e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(ax, 0.23164189f, 1.0f)));
  float npoly = fmaf(-1.061405429f, t, 1.453152027f);
  npoly = fmaf(npoly, t, -1.421413741f);
  npoly = fmaf(npoly, t, 0.284496736f);
  npoly = fmaf(npoly, t, -0.254829592f);
  npoly = npoly * t;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"((x * x) * -0.72134752044448170368f));
  return fmaf(ax * 0.5f, fmaf(npoly, e, 1.0f), x * 0.5f);
}

// tanh-approximated GELU of RITA (rita_modeling.py:24-26), with the reference's constants: x*0.5*(1+tanh(0.79788456*x*(1+0.044715*x^2))).
// tanhf is the accurate libdevice routine (<= 2 ulp; the library is built without fast math), not MUFU.TANH's ~2^-11 relative error.
__device__ __forceinline__ float gelu_tanh(float x) {
  return x * 0.5f * (1.0f + tanhf(0.79788456f * x * (1.0f + 0.044715f * x * x)));
}

// SiLU (ESM C SwiGLU, esm/layers/blocks.py:21-33): g / (1 + e^-g) with e^-g from MUFU.EX2 (ex2.approx.ftz, <= 2 ulp) and the quotient
// from MUFU.RCP (rcp.approx.ftz, <= 1 ulp): relative error <= ~4 ulp (5e-7) over the range; for g < -88 e^-g is inf and the result 0.
__device__ __forceinline__ float silu(float g) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(g * -1.4426950408889634074f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return g * r;
}

// Bias, activation and store of one consumer thread's fragment: rows row0 and row0 + 8, columns col0 + 8j (+1), j < 16.
template <int EPI>
__device__ __forceinline__ void epilogue(float (&acc)[64], const GemmKParams& p, long long row0, int col0) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const long long row = row0 + 8 * h;
    const long long trow = p.base_T > 0 ? row % p.base_T : 0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = col0 + 8 * j;
      if (col >= p.N) continue;
      const bool two = col + 1 < p.N;
      float& v0 = acc[4 * j + 2 * h];
      float& v1 = acc[4 * j + 2 * h + 1];
      if (p.bias != nullptr) {
        v0 += __ldg(p.bias + col);
        if (two) v1 += __ldg(p.bias + col + 1);
      }
      if (p.base_pre != nullptr) {  // delta-operand mode: the shared base row (W a0[t] + b) joins before the activation (N % 64 == 0)
        const float* bp = p.base_pre + trow * p.N + col;
        v0 += __ldg(bp);
        v1 += __ldg(bp + 1);
      }
      if (EPI == 1) {
        v0 = gelu_erf(v0);
        v1 = gelu_erf(v1);
        if (p.base_post != nullptr) {  // the output is again a difference, GELU(acc) - base_post[t]
          const __half* bq = p.base_post + trow * p.N + col;
          v0 -= __half2float(bq[0]);
          v1 -= __half2float(bq[1]);
        }
      } else if (EPI == 4) {  // squared ReLU (Tranception MLP, tranception/activations.py:79-84)
        const float a = fmaxf(v0, 0.f), b = fmaxf(v1, 0.f);
        v0 = a * a;
        v1 = b * b;
      } else if (EPI == 6) {
        v0 = gelu_tanh(v0);
        v1 = gelu_tanh(v1);
      }
    }
    if (EPI == 3 && p.rot_half == 64) {
      // the same over one 128-wide slot per N tile: blocks j and j + 8 hold columns c and c + 64; cos/sin[t, c] for c in [0, 64)
      const int t = static_cast<int>(row % p.rot_T);
      if (col0 - (col0 & 127) < 2 * p.rot_dim) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = (col0 & 127) + 8 * j + e;
            const float co = __ldg(p.rot_cos + static_cast<long long>(t) * 64 + c), s = __ldg(p.rot_sin + static_cast<long long>(t) * 64 + c);
            const float a = acc[4 * j + 2 * h + e], b = acc[4 * (j + 8) + 2 * h + e];
            acc[4 * j + 2 * h + e] = a * co - b * s;
            acc[4 * (j + 8) + 2 * h + e] = b * co + a * s;
          }
        }
      }
    } else if (EPI == 3) {
      // rotary: x*cos + rotate_half(x)*sin over each 64-wide head (blocks j and j + 4 of one head hold columns c and c + 32);
      // cos/sin[t, c] for c in [0,32) (both halves equal)
      const int t = static_cast<int>(row % p.rot_T);
#pragma unroll
      for (int hd = 0; hd < 2; ++hd) {
        if (col0 - (col0 & 63) + 64 * hd >= 2 * p.rot_dim) continue;
#pragma unroll
        for (int j = 8 * hd; j < 8 * hd + 4; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = (col0 & 63) + 8 * (j - 8 * hd) + e;
            const float co = __ldg(p.rot_cos + static_cast<long long>(t) * 32 + c), s = __ldg(p.rot_sin + static_cast<long long>(t) * 32 + c);
            const float a = acc[4 * j + 2 * h + e], b = acc[4 * (j + 4) + 2 * h + e];
            acc[4 * j + 2 * h + e] = a * co - b * s;
            acc[4 * (j + 4) + 2 * h + e] = b * co + a * s;
          }
        }
      }
    }
    if (row >= p.M) continue;
    if (EPI == 7) {
      // LM-head partials (K16): the four threads of a quad (lanes 4g .. 4g+3) hold the 128 columns of this row's N tile, 32 each; the
      // row, and so every branch below, is uniform over the quad. No logit leaves the registers unless lm_logits asks for them.
      const int t = static_cast<int>(row % p.lm_T);
      if (t + 1 >= __ldg(p.lm_lens + row / p.lm_T)) continue;
      const unsigned quad = 0xFu << (threadIdx.x & 28);
      float m = -INFINITY;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = col0 + 8 * j;
        if (col < p.N) m = fmaxf(m, acc[4 * j + 2 * h]);
        if (col + 1 < p.N) m = fmaxf(m, acc[4 * j + 2 * h + 1]);
      }
      m = fmaxf(m, __shfl_xor_sync(quad, m, 1));
      m = fmaxf(m, __shfl_xor_sync(quad, m, 2));
      float se = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = col0 + 8 * j;
        if (col < p.N) se += expf(acc[4 * j + 2 * h] - m);
        if (col + 1 < p.N) se += expf(acc[4 * j + 2 * h + 1] - m);
      }
      se += __shfl_xor_sync(quad, se, 1);
      se += __shfl_xor_sync(quad, se, 2);
      if ((threadIdx.x & 3) == 0) p.lm_part[row * p.tiles_n + col0 / BN] = make_float2(m, se);
      const int label = __ldg(p.lm_ids + row + 1);
      const int jl = label - col0;  // this thread's columns are col0 + 8j + e, j < 16, e < 2
      if (jl >= 0 && jl < 128 && (jl & 7) < 2 && label < p.N) {
        float v = 0.f;  // selected, not indexed: an index into acc that depends on the label would move acc to local memory
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float a0 = acc[4 * j + 2 * h], a1 = acc[4 * j + 2 * h + 1];
          v = (jl == 8 * j) ? a0 : ((jl == 8 * j + 1) ? a1 : v);
        }
        p.lm_tgt[row] = v;
      }
      if (p.lm_logits != nullptr) {
        float* lr = p.lm_logits + row * p.N;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = col0 + 8 * j;
          if (col < p.N) lr[col] = acc[4 * j + 2 * h];
          if (col + 1 < p.N) lr[col + 1] = acc[4 * j + 2 * h + 1];
        }
      }
    } else if (EPI == 2) {
      // the masked row of each copy is updated by the compact exact path instead (delta-operand mode)
      if (p.mask_pos != nullptr && trow == __ldg(p.mask_pos + row / p.base_T)) continue;
      float* r = p.resid + row * p.ldr;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = col0 + 8 * j;
        if (col >= p.N) continue;
        if (col + 1 < p.N && !(reinterpret_cast<uintptr_t>(r + col) & 7)) {
          float2 x = *reinterpret_cast<float2*>(r + col);
          x.x += acc[4 * j + 2 * h];
          x.y += acc[4 * j + 2 * h + 1];
          *reinterpret_cast<float2*>(r + col) = x;
        } else {
          r[col] += acc[4 * j + 2 * h];
          if (col + 1 < p.N) r[col + 1] += acc[4 * j + 2 * h + 1];
        }
      }
    } else if (EPI == 5) {
      // SwiGLU: W rows come interleaved in blocks of 8 (api.cu), so block j (even) of the fragment holds gate columns and block j + 1
      // the matching up columns. silu(gate) * up goes to output column (col / 16) * 8 + col % 8 of an N/2-wide operand row
      // (planes of N/2 columns at out_lo_off; N % 16 == 0).
      __half* o = p.out + row * p.ldo;
      const int nh = p.N >> 1;
      uint8_t* f8 = reinterpret_cast<uint8_t*>(o + p.out_lo_off);
      const float sh = p.out_scale, sl = p.out_scale * LO8_GAIN;
#pragma unroll
      for (int j = 0; j < 16; j += 2) {
        const int col = col0 + 8 * j;
        if (col >= p.N) continue;
        const int oc = ((col >> 4) << 3) + (col & 7);
        const float x0 = silu(acc[4 * j + 2 * h]) * acc[4 * (j + 1) + 2 * h];
        const float x1 = silu(acc[4 * j + 2 * h + 1]) * acc[4 * (j + 1) + 2 * h + 1];
        const uint32_t hi = cvt_f16x2_rn(x0, x1);
        const float2 hf = unpack_h2(hi);
        *reinterpret_cast<uint32_t*>(o + oc) = hi;
        if (p.out_fmt == 1) *reinterpret_cast<uint32_t*>(o + p.out_lo_off + oc) = cvt_f16x2_rn(x0 - hf.x, x1 - hf.y);
        else if (p.out_fmt == 2) {
          *reinterpret_cast<uint16_t*>(f8 + oc) = static_cast<uint16_t>(cvt_e4m3x2((x0 - hf.x) * sl, (x1 - hf.y) * sl));
          *reinterpret_cast<uint16_t*>(f8 + nh + oc) = static_cast<uint16_t>(cvt_e4m3x2(hf.x * sh, hf.y * sh));
        }
      }
    } else {
      // operand.cuh's column-pair store written out: through the helper the compiler no longer keeps the plane addresses and the
      // scales of a row in registers across the 16 column blocks (measured 1 % of the ESM-1v headline on an H100 at 700 W)
      __half* o = p.out + row * p.ldo;
      uint8_t* f8 = reinterpret_cast<uint8_t*>(o + p.out_lo_off);
      const float sh = p.out_scale, sl = p.out_scale * LO8_GAIN;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = col0 + 8 * j;
        if (col >= p.N) continue;
        const float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
        const uint32_t hi = cvt_f16x2_rn(x0, x1);
        const float2 hf = unpack_h2(hi);
        if (col + 1 < p.N) {
          *reinterpret_cast<uint32_t*>(o + col) = hi;
          if (p.out_fmt == 1) *reinterpret_cast<uint32_t*>(o + p.out_lo_off + col) = cvt_f16x2_rn(x0 - hf.x, x1 - hf.y);
          else if (p.out_fmt == 2) {  // lo8 plane: bytes [0, N) of the e4m3 region, hi8 plane: bytes [N, 2N)
            *reinterpret_cast<uint16_t*>(f8 + col) = static_cast<uint16_t>(cvt_e4m3x2((x0 - hf.x) * sl, (x1 - hf.y) * sl));
            *reinterpret_cast<uint16_t*>(f8 + p.N + col) = static_cast<uint16_t>(cvt_e4m3x2(hf.x * sh, hf.y * sh));
          }
        } else {  // odd N, last column (out_fmt 2 needs N % 64 == 0)
          o[col] = __ushort_as_half(static_cast<unsigned short>(hi & 0xFFFFu));
          if (p.out_fmt == 1) o[p.out_lo_off + col] = __float2half_rn(x0 - hf.x);
        }
      }
    }
  }
}

// One segment's k-blocks into the chunk accumulator. The wgmmas of a k-block stay in flight while the next block's are issued; a
// stage goes back to the producer once the wgmmas that read it are complete (`prev`: the stage still being read).
// A stage is released to the producers of both CTAs of a pair (each multicasts half of the W tile into it).
template <int CTA2>
__device__ __forceinline__ void release_stage(uint64_t* empty, int stage, int lane, uint32_t rank) {
  if (lane == 0) {
    mbar_arrive(&empty[stage]);
    if (CTA2) mbar_arrive_cluster(&empty[stage], rank ^ 1u);
  }
}

template <int KIND, int CTA2>
__device__ __forceinline__ void consume_seg(float (&cacc)[64], int nkb, uint32_t a_base, uint32_t b_base, uint64_t* full, uint64_t* empty,
                                            int& stage, uint32_t& phase, bool& fresh, int& prev, int lane, uint32_t rank) {
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait(&full[stage], phase);
    const uint64_t adesc = make_desc_sw128(a_base + stage * A_BYTES), bdesc = make_desc_sw128(b_base + stage * B_BYTES);
    wgmma_fence();
    wgmma_fence_regs(cacc);
#pragma unroll
    for (int k = 0; k < 4; ++k) {  // 4 x (K = 32 bytes of every row): 16 fp16 or 32 e4m3 per instruction
      const uint32_t sd = (fresh && k == 0) ? 0u : 1u;
      if (KIND) wgmma_m64n128k32_e4m3_ss(cacc, adesc + 2 * k, bdesc + 2 * k, sd);
      else wgmma_m64n128k16_f16_ss(cacc, adesc + 2 * k, bdesc + 2 * k, sd);
    }
    wgmma_commit();
    wgmma_fence_regs(cacc);
    fresh = false;
    wgmma_wait<1>();  // the previous k-block's wgmmas are done: its stage goes back to the producer
    if (prev >= 0) release_stage<CTA2>(empty, prev, lane, rank);
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
}

template <int EPI, int CTA2>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmA8, const __grid_constant__ CUtensorMap tmB8, const __grid_constant__ GemmKParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (base & 1023u)) & 1023u);
  uint8_t* smA = smem;
  uint8_t* smB = smem + OFF_B;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const uint32_t rank = CTA2 ? cluster_ctarank() : 0u;             // CTA2: rows [128 rank, 128 rank + 128) of the pair's 256-row tile
  const int ntiles = p.tiles_m * p.tiles_n;                         // CTA2: tiles_m counts 256-row tiles
  const int tile0 = CTA2 ? static_cast<int>(blockIdx.x >> 1) : static_cast<int>(blockIdx.x);
  const int tstep = CTA2 ? static_cast<int>(gridDim.x >> 1) : static_cast<int>(gridDim.x);
  constexpr int ROWS = CTA2 ? 2 * BM : BM;                          // rows of the output tile per (pair of) CTA(s)

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], CTA2 ? 2 * CONSUMER_WARPS : CONSUMER_WARPS);  // pair: the consumer warps of both CTAs
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (CTA2) cluster_sync_all();  // the peer's barriers are initialised before anything can signal them

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      // Optional L2 look-ahead cursor (p.prefetch k-blocks ahead of the loads, A operand only); off by default.
      int pf_tile = tile0, pf_s = 0, pf_kb = 0;
      auto pf_step = [&]() {
        if (pf_tile >= ntiles) return;
        const GemmSeg sg = p.seg[pf_s];
        tma_prefetch_l2_2d(sg.kind ? &tmA8 : &tmA, sg.a_col + pf_kb * (sg.kind ? 2 * BK : BK), (pf_tile / p.tiles_n) * ROWS + rank * BM);
        if (++pf_kb == sg.nkb) {
          pf_kb = 0;
          if (++pf_s == p.nsegs) { pf_s = 0; pf_tile += tstep; }
        }
      };
      for (int i = 0; i < p.prefetch; ++i) pf_step();
      for (int tile = tile0; tile < ntiles; tile += tstep) {
        const int m_blk = tile / p.tiles_n, n_blk = tile % p.tiles_n;
        const int a_row = m_blk * ROWS + static_cast<int>(rank) * BM;
        int b_row = n_blk * BN + (CTA2 ? static_cast<int>(rank) * (BN / 2) : 0);  // pair: this CTA's half of the W tile
        if (p.grp_rows_a) b_row += (m_blk * ROWS / p.grp_rows_a) * p.grp_rows_b;  // grouped: this group's block of W rows
        for (int s = 0; s < p.nsegs; ++s) {
          const GemmSeg sg = p.seg[s];
          const CUtensorMap* ma = sg.kind ? &tmA8 : &tmA;
          const CUtensorMap* mb = sg.kind ? &tmB8 : &tmB;
          const int step = sg.kind ? 2 * BK : BK;  // 128 B of a row: 64 fp16 or 128 e4m3
          for (int kb = 0; kb < sg.nkb; ++kb) {
            if (p.prefetch) pf_step();
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full[stage], A_BYTES + B_BYTES);
            tma_load_2d(smA + stage * A_BYTES, ma, &full[stage], sg.a_col + kb * step, a_row);
            if (CTA2)  // bytes of both halves complete on each CTA's own barrier
              tma_load_2d_mc(smB + stage * B_BYTES + rank * (B_BYTES / 2), mb, &full[stage], sg.b_col + kb * step, b_row, 3);
            else
              tma_load_2d(smB + stage * B_BYTES, mb, &full[stage], sg.b_col + kb * step, b_row);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int cw = wg - 1;                     // rows [64 cw, 64 cw + 64) of the tile
    const int g = lane >> 2, t = lane & 3;
    const uint32_t a_base = smem_u32(smA) + cw * 64 * 128, b_base = smem_u32(smB);
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = tile0; tile < ntiles; tile += tstep) {
      const int m_blk = tile / p.tiles_n, n_blk = tile % p.tiles_n;
      const long long row0 = static_cast<long long>(m_blk) * ROWS + rank * BM + cw * 64 + (warp & 3) * 16 + g;
      const int col0 = n_blk * BN + 2 * t;
      float acc[64], cacc[64];
      int ch = 0;
      bool fresh = true;
      int prev = -1;  // stage whose wgmmas may still be reading shared memory
      for (int s = 0; s < p.nsegs; ++s) {
        const GemmSeg sg = p.seg[s];
        // the operand kind selects the whole k-block loop: a branch between the wgmmas of one accumulator makes ptxas serialise them
        if (sg.kind) {
          // e4m3 cross terms. sm_90's e4m3 wgmma keeps only ~14 bits while it accumulates, so every k-block (128 products along K)
          // is its own chunk, folded into the fp32 accumulator with the scale 1 / (2^11 s_A t_n) applied
          for (int kb = 0; kb < sg.nkb; ++kb) {
            consume_seg<1, CTA2>(cacc, 1, a_base, b_base, full, empty, stage, phase, fresh, prev, lane, rank);
            wgmma_wait<0>();
            wgmma_fence_regs(cacc);
            release_stage<CTA2>(empty, prev, lane, rank);
            prev = -1;
            if (p.w_uniform) {  // one scale per weight matrix: a single factor for the whole tile
              const float f = p.a_inv * __ldg(p.w_inv);
#pragma unroll
              for (int i = 0; i < 64; ++i) acc[i] = (ch == 0 ? 0.f : acc[i]) + cacc[i] * f;
            } else {
#pragma unroll
              for (int i = 0; i < 64; ++i) {
                const int col = col0 + 8 * (i >> 2) + (i & 1);
                acc[i] = (ch == 0 ? 0.f : acc[i]) + cacc[i] * ((col < p.N) ? p.a_inv * __ldg(p.w_inv + col) : 0.f);
              }
            }
            ++ch;
            fresh = true;
          }
          continue;
        }
        consume_seg<0, CTA2>(cacc, sg.nkb, a_base, b_base, full, empty, stage, phase, fresh, prev, lane, rank);
        if (sg.commit) {
          wgmma_wait<0>();
          wgmma_fence_regs(cacc);
          release_stage<CTA2>(empty, prev, lane, rank);
          prev = -1;
#pragma unroll
          for (int i = 0; i < 64; ++i) acc[i] = (ch == 0 ? 0.f : acc[i]) + cacc[i];
          ++ch;
          fresh = true;
        }
      }
      epilogue<EPI>(acc, p, row0, col0);
    }
  }
  if (CTA2) cluster_sync_all();  // neither CTA may exit while its peer can still multicast into it or arrive on its barriers
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// Host-side cache of encoded tensor maps: the model issues the same few (buffer, shape) combinations thousands of times per
// assay. thread_local: one map per calling thread, so handles driven from different threads never share state.
struct TmapKey {
  const void* ptr; uint64_t rows, cols, ld; uint32_t box_rows, box_cols; int elem_bytes, swizzle;
  bool operator==(const TmapKey& o) const { return std::memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(TmapKey) / 8; ++i) h = (h ^ w[i]) * 1099511628211ull;
    return static_cast<size_t>(h);
  }
};
static_assert(sizeof(TmapKey) % 8 == 0, "TmapKey is hashed as 64-bit words");

}  // namespace

// 2D row-major tensor [rows, cols] with row pitch ld (elements); box = [box_rows, box_cols], out-of-bounds reads give zero,
// out-of-bounds parts of a store are clipped. elem_bytes 2 = fp16, 4 = fp32, 1 = bytes (e4m3 planes). swizzle in bytes: 128 or 64.
int make_tmap_2d(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, uint32_t box_cols,
                 int elem_bytes, int swizzle) {
  TmapKey key;
  std::memset(&key, 0, sizeof(key));
  key.ptr = ptr; key.rows = rows; key.cols = cols; key.ld = ld; key.box_rows = box_rows; key.box_cols = box_cols;
  key.elem_bytes = elem_bytes; key.swizzle = swizzle;
  static thread_local std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  auto it = cache.find(key);
  if (it != cache.end()) {
    *m = it->second;
    return PG_OK;
  }
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error(PG_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (ld * elem_bytes) % 16)
    return set_error(PG_ERR_ARG, "TMA operand must be 16-byte aligned with a 16-byte-multiple row pitch");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * elem_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                 : elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8;
  CUresult r = fn(m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(PG_ERR_CUDA, "cuTensorMapEncodeTiled failed: " + std::to_string(static_cast<int>(r)));
  if (cache.size() > 4096) cache.clear();
  cache.emplace(key, *m);
  return PG_OK;
}
int make_tmap_f16_2d(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                     uint32_t box_cols) {
  return make_tmap_2d(m, ptr, rows, cols, ld, box_rows, box_cols, 2, 128);
}

// Longest run of K one hi*hi chunk accumulates before it is folded into the fp32 accumulator (see the header). Default 1280; the
// environment variable PG_GEMM_KCHUNK or pg_set_tuning("gemm_kchunk", v) override it; 0 = no chunking (for the probe).
static int g_kchunk = -1, g_prefetch = -1, g_cta2 = -1;
int gemm_cta2() {
  if (g_cta2 < 0) {
    const char* e = getenv("PG_GEMM_CTA2");
    g_cta2 = e ? atoi(e) : 1;  // default: clusters of two CTAs sharing the W tile
  }
  return g_cta2;
}
void set_gemm_cta2(int v) { g_cta2 = v ? 1 : 0; }
int gemm_kchunk() {
  if (g_kchunk < 0) {
    const char* e = getenv("PG_GEMM_KCHUNK");
    g_kchunk = e ? atoi(e) : 1280;
  }
  return g_kchunk < BK ? (1 << 30) : g_kchunk;
}
void set_gemm_kchunk(int v) { g_kchunk = v < 0 ? 0 : v; }
int gemm_prefetch() {
  if (g_prefetch < 0) {
    const char* e = getenv("PG_GEMM_PREFETCH");
    g_prefetch = e ? atoi(e) : 0;
  }
  return g_prefetch;
}
void set_gemm_prefetch(int v) { g_prefetch = v < 0 ? 0 : (v > 64 ? 64 : v); }

int launch_gemm(const GemmLaunch& g, cudaStream_t s) {
  if (g.M <= 0 || g.N <= 0 || g.K <= 0) return set_error(PG_ERR_ARG, "gemm: empty problem");
  if (g.K % BK) return set_error(PG_ERR_ARG, "gemm: K must be a multiple of 64");
  if (g.nseg < 1 || g.nseg > 3) return set_error(PG_ERR_ARG, "gemm: nseg must be 1, 2 (fp16 + e4m3 cross terms) or 3");
  if (g.epi < 0 || g.epi > 7) return set_error(PG_ERR_ARG, "gemm: bad epilogue");
  if (g.epi == 7 && (!g.lm_part || !g.lm_tgt || !g.lm_ids || !g.lm_lens || g.lm_T <= 0 || g.M % g.lm_T || g.grp_rows_a || g.bias))
    return set_error(PG_ERR_ARG, "gemm: the LM-head epilogue needs partial, target, ids and lens buffers, rows a multiple of lm_T, no groups or bias");
  if (g.epi == 5 && (g.N % 16 || (g.out_fmt == 2 && (g.N / 2) % 64) || g.grp_rows_a || (g.out_fmt >= 1 && g.out_lo_off < g.N / 2)))
    return set_error(PG_ERR_ARG, "gemm: the SwiGLU epilogue needs N % 16 == 0 (N/2 % 64 == 0 for out_fmt 2), no groups, planes >= N/2 apart");
  if (g.epi != 7 && (g.epi == 2 ? !g.resid : !g.out)) return set_error(PG_ERR_ARG, "gemm: missing output");
  if (g.epi == 3 && (!g.rot_cos || !g.rot_sin || g.rot_T <= 0 || g.rot_dim % 64)) return set_error(PG_ERR_ARG, "gemm: bad rotary args");
  if (g.epi == 3 && ((g.rot_half != 32 && g.rot_half != 64) || g.rot_dim % (2 * g.rot_half)))
    return set_error(PG_ERR_ARG, "gemm: rotary slots must be 64 or 128 wide and divide rot_dim");
  if (g.nseg == 2 && (!g.w_inv || !(g.a_scale > 0.f))) return set_error(PG_ERR_ARG, "gemm: nseg 2 needs w_inv[N] and a_scale > 0");
  if (g.out_fmt < 0 || g.out_fmt > 2) return set_error(PG_ERR_ARG, "gemm: bad out_fmt");
  if ((g.base_pre || g.base_post || g.mask_pos) && (!g.base_pre || g.base_T <= 0 || g.N % 64 || g.M % g.base_T || g.grp_rows_a ||
                                                       (g.mask_pos && g.epi != 2) || (g.base_post && g.epi == 2)))
    return set_error(PG_ERR_ARG, "gemm: delta-operand mode needs base_pre, base_T > 0 dividing M, N % 64 == 0, no groups; mask_pos only with the residual epilogue");
  if (g.epi != 2 && g.out_fmt == 2 && (g.N % 64 || !(g.out_scale > 0.f)))
    return set_error(PG_ERR_ARG, "gemm: out_fmt 2 needs N % 64 == 0 and out_scale > 0");
  if (g.epi != 2 && g.out_fmt >= 1 && g.out_lo_off <= 0) return set_error(PG_ERR_ARG, "gemm: out_fmt 1/2 need out_lo_off > 0");
  if ((g.base_pre || g.base_post || g.mask_pos) && g.epi > 2)
    return set_error(PG_ERR_UNSUPPORTED, "gemm: the delta-operand form runs with epilogues 0, 1, 2");
  if (g.epi != 7 && (g.epi == 2 ? (g.ldr % 2 || (reinterpret_cast<uintptr_t>(g.resid) & 7)) : (g.ldo % 2 || (reinterpret_cast<uintptr_t>(g.out) & 3) || g.out_lo_off % 2)))
    return set_error(PG_ERR_ARG, "gemm: output pitches must be even and the output 8-byte (fp32) / 4-byte (fp16) aligned");
  int dev = 0;
  PG_CUDA_OK(cudaGetDevice(&dev));
  static bool attr_set[64] = {};
  if (dev < 64 && !attr_set[dev]) {
#define PG_SET_SMEM(E)                                                                                           \
  PG_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel<E, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM)); \
  PG_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel<E, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM))
    PG_SET_SMEM(0); PG_SET_SMEM(1); PG_SET_SMEM(2); PG_SET_SMEM(3); PG_SET_SMEM(4); PG_SET_SMEM(5); PG_SET_SMEM(6); PG_SET_SMEM(7);
#undef PG_SET_SMEM
    attr_set[dev] = true;
  }
  const uint64_t K = static_cast<uint64_t>(g.K);
  const uint64_t width = K * (g.nseg == 3 ? 2 : 1);
  const bool grouped = g.grp_rows_a > 0;
  // pairs work on 256-row tiles; a grouped problem whose groups are only a multiple of 128 rows runs the single-CTA form
  const int cta2 = gemm_cta2() && !(grouped && g.grp_rows_a % (2 * BM));
  const uint32_t wbox = cta2 ? BN / 2 : BN;  // rows of W one CTA loads per k-block
  CUtensorMap tmA, tmB, tmA8{}, tmB8{};
  int rc = make_tmap_2d(&tmA, g.a, g.M, width, g.lda, BM, BK, 2, 128);
  if (rc) return rc;
  if (grouped && (g.nseg == 2 || g.grp_rows_a % BM || g.grp_rows_b < g.N || g.M % g.grp_rows_a || g.bias || g.epi == 3))
    return set_error(PG_ERR_ARG, "gemm: grouped mode needs fp16 operands, A groups of a multiple of 128 rows, W groups of >= N rows, no bias");
  const uint64_t w_rows = grouped ? static_cast<uint64_t>(g.M / g.grp_rows_a) * g.grp_rows_b : static_cast<uint64_t>(g.N);
  rc = make_tmap_2d(&tmB, g.w, w_rows, width, g.ldw, wbox, BK, 2, 128);
  if (rc) return rc;
  if (g.nseg == 2) {  // e4m3 planes follow the fp16 hi plane of each row: bytes [2K, 4K) = K-concatenated [lo8 | hi8] / [hi8 | lo8]
    rc = make_tmap_2d(&tmA8, static_cast<const uint8_t*>(g.a) + 2 * K, g.M, 2 * K, static_cast<uint64_t>(g.lda) * 2, BM, 2 * BK, 1, 128);
    if (rc) return rc;
    rc = make_tmap_2d(&tmB8, static_cast<const uint8_t*>(g.w) + 2 * K, g.N, 2 * K, static_cast<uint64_t>(g.ldw) * 2, wbox, 2 * BK, 1, 128);
    if (rc) return rc;
  }
  GemmKParams p{};
  p.M = g.M; p.N = g.N; p.K = g.K;
  const int kblocks = g.K / BK;
  int ns = 0;
  auto push = [&](int a_col, int b_col, int nkb, int kind, int commit) {
    p.seg[ns].a_col = a_col; p.seg[ns].b_col = b_col; p.seg[ns].nkb = nkb;
    p.seg[ns].kind = static_cast<short>(kind); p.seg[ns].commit = static_cast<short>(commit);
    ++ns;
  };
  // hi*hi pieces: as equal as possible, each <= kchunk along K, at most what the segment table holds
  int pieces = (g.K + gemm_kchunk() - 1) / gemm_kchunk();
  if (pieces < 1) pieces = 1;
  if (pieces > MAX_SEGS - 2) pieces = MAX_SEGS - 2;
  if (pieces > kblocks) pieces = kblocks;
  if (g.nseg == 2) {
    push(0, 0, kblocks, 1, 1);  // [lo8 | hi8] x [hi8 | lo8]: 2K bytes = kblocks blocks of 128 B
    p.a_inv = 1.0f / (LO8_GAIN * g.a_scale);
    p.w_inv = g.w_inv;
    p.w_uniform = g.w_uniform;
  } else if (g.nseg == 3) {
    push(g.K, 0, kblocks, 0, 0);  // lo*hi
    push(0, g.K, kblocks, 0, 1);  // hi*lo
  }
  for (int i = 0, kb0 = 0; i < pieces; ++i) {
    const int nkb = kblocks / pieces + (i < kblocks % pieces ? 1 : 0);
    push(kb0 * BK, kb0 * BK, nkb, 0, 1);
    kb0 += nkb;
  }
  p.nsegs = ns;
  p.bias = g.bias;
  p.out = g.out; p.ldo = g.ldo; p.out_lo_off = g.out_lo_off;
  p.resid = g.resid; p.ldr = g.ldr;
  p.out_fmt = (g.epi == 2) ? 0 : g.out_fmt;
  p.out_scale = g.out_scale;
  p.rot_cos = g.rot_cos; p.rot_sin = g.rot_sin; p.rot_T = g.rot_T; p.rot_dim = g.rot_dim; p.rot_half = g.rot_half;
  p.tiles_m = cta2 ? (g.M + 2 * BM - 1) / (2 * BM) : (g.M + BM - 1) / BM;
  p.tiles_n = (g.N + BN - 1) / BN;
  p.prefetch = grouped ? 0 : gemm_prefetch();
  p.grp_rows_a = g.grp_rows_a; p.grp_rows_b = g.grp_rows_b;
  p.base_pre = g.base_pre; p.base_post = g.base_post; p.base_T = g.base_T; p.mask_pos = g.mask_pos;
  p.lm_part = g.lm_part; p.lm_tgt = g.lm_tgt; p.lm_logits = g.lm_logits; p.lm_ids = g.lm_ids; p.lm_lens = g.lm_lens; p.lm_T = g.lm_T;
  const int ntiles = p.tiles_m * p.tiles_n;
  cudaLaunchConfig_t cfg{};
  cudaLaunchAttribute attr[1];
  if (cta2) {  // clusters of two CTAs, one cluster per pair of SMs
    const int pairs = ntiles < num_sms() / 2 ? ntiles : num_sms() / 2;
    cfg.gridDim = dim3(2 * pairs);
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
  } else {
    cfg.gridDim = dim3(ntiles < num_sms() ? ntiles : num_sms());
  }
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = GEMM_SMEM;
  cfg.stream = s;
#define PG_LAUNCH(E) (cta2 ? cudaLaunchKernelEx(&cfg, gemm_tc_kernel<E, 1>, tmA, tmB, tmA8, tmB8, p) \
                           : cudaLaunchKernelEx(&cfg, gemm_tc_kernel<E, 0>, tmA, tmB, tmA8, tmB8, p))
  cudaError_t e;
  switch (g.epi) {
    case 0: e = PG_LAUNCH(0); break;
    case 1: e = PG_LAUNCH(1); break;
    case 2: e = PG_LAUNCH(2); break;
    case 3: e = PG_LAUNCH(3); break;
    case 4: e = PG_LAUNCH(4); break;
    case 5: e = PG_LAUNCH(5); break;
    case 6: e = PG_LAUNCH(6); break;
    default: e = PG_LAUNCH(7); break;
  }
#undef PG_LAUNCH
  PG_CUDA_OK(e);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

}  // namespace pg
