// K4 — wgmma/TMA attention, head width HD = 64 or 128: one warpgroup per CTA, 64-query tiles x 64-key blocks, flash-style online
// softmax. Optional causal + ALiBi + shared (wild-type) key/value prefix; NP = 2 runs the hi/lo three-product scheme.
//
// Per key block: S = Q K^T (wgmma, both operands from shared memory) -> online softmax on the register fragment -> O += P V (wgmma,
// P from registers: the S accumulator fragment of 16 keys is exactly the A fragment of one k16 step, so P never touches shared
// memory). K and V arrive by TMA into a two-slot ring (the next block loads while this one computes); several CTAs share an SM
// (NP = 2: 81 KB of shared memory each), so one CTA's softmax overlaps another's MMAs.
//   Work item = (sequence, head, 64-query tile); grid = items, tiles of one (sequence, head) adjacent so that K / V stay in L2.
// HD = 128 (ProGen2's 80- and 96-wide heads in 128-wide slots, api.cu): each of q, k and v is NB = 2 boxes of 64 columns (the TMA
// box stays at 128 B rows, SWIZZLE_128B); S = Q K^T runs 4 k16 steps per box, O += P V one n64 wgmma group per box into o[32 * NB].
// NP = 2 then needs ~160 KB of shared memory: one CTA per SM. The delta-operand and column (perm_C) forms are HD = 64 only.
#include <cstdlib>

#include "common.h"
#include "operand.cuh"

namespace pg {

namespace {

constexpr int QT = 64, KT = 64;
constexpr uint32_t TILE = 8192;  // 64 rows x 64 fp16
constexpr int NSLOT = 2;         // K/V smem ring
constexpr int ATT_THREADS = 128;

template <int NP, int HD>
struct SmemW {
  static constexpr int NB = HD / 64;                   // 64-column boxes per head
  static constexpr uint32_t Q = 0;                     // [NP][NB] tiles
  static constexpr uint32_t KV = NP * NB * TILE;       // [NSLOT][K planes NP x NB | V planes NP x NB]
  static constexpr uint32_t BAR = KV + NSLOT * 2 * NP * NB * TILE;
  static constexpr uint32_t TOTAL = BAR + 64 + 1024;   // barriers, alignment slack
};

struct AttnWParams {
  int B, T, heads, nqt, nkb;   // T = full sequence length (prefix + own rows); nqt = query tiles of the own rows; nkb = key blocks of T
  int Tq, s_blocks;            // own rows per sequence; shared-prefix length / 64 (0 = no prefix: Tq == T)
  int d;
  int dkv, grp;                // k / v width (kv_heads slots) and query heads per key / value head (grouped-query attention)
  long long lo_off;
  __half* out; long long ldo; long long out_lo_off;
  int causal;
  const float* alibi_slopes;
  int out_fmt; float out_scale;  // common.h operand formats: 1 = fp16 lo plane, 2 = e4m3 [lo8 | hi8] planes for the out_proj GEMM
  int perm_C;                    // > 0: sequence b is column (b / perm_C, b % perm_C) of an alignment; output rows go to (., r, c) order
  // delta-operand mode (common.h AttnLaunch): out = attention - base_o[row]; full-precision hi / lo copy of row mask_pos[b] to cout[b]
  const __half* base_o; const int* mask_pos; __half* cout; long long ldc; long long c_lo_off;
  int p_valid;            // prefix rows that exist (keys [p_valid, s_blocks * 64) are masked): s_blocks * 64 except in the memory form
  int head_major;         // work items ordered (head, sequence, tile) instead of (sequence, head, tile)
  const int* seg_start;   // segment-causal form (B == 1): first row of each row's segment, or null
};

__device__ __forceinline__ float ex2a(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// RNACC (memory form): each key block's P V goes to a fresh accumulator that is added to O in round-to-nearest fp32, as the GEMM's K
// chunks are (gemm_tc.cu): the tensor core's own fp32 accumulation does not round to nearest, and over the ~385 key blocks of a 24 640-row
// record its error grows with the number of blocks.
template <int NP, int DELTA, int HD, int RNACC = 0>
__global__ void __launch_bounds__(ATT_THREADS) attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tm,
                                                                 const __grid_constant__ CUtensorMap tmP, const AttnWParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (base & 1023u)) & 1023u);
  using L = SmemW<NP, HD>;
  constexpr int NB = L::NB;
  constexpr uint32_t PLANE = NB * TILE;  // one plane of one head: NB boxes
  uint8_t* sQ = smem + L::Q;
  uint8_t* sKV = smem + L::KV;
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + L::BAR);
  uint64_t* kv_full = q_full + 1;  // [NSLOT]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int item = blockIdx.x;
  const int qt_l = item % p.nqt, bh = item / p.nqt;
  const int qt = qt_l + p.s_blocks;  // tile index within the full sequence
  const int nb = p.B;
  const int h = p.head_major ? bh / nb : bh % p.heads, b = p.head_major ? bh % nb : bh / p.heads;
  const int row0 = b * p.Tq;
  const int hk = h / p.grp;
  const int cq = h * HD, ck = p.d + hk * HD, cv = p.d + p.dkv + hk * HD;
  // segment-causal: the tile's first row has the smallest segment start; blocks before it hold no visible key
  const int j0 = p.seg_start ? __ldg(p.seg_start + qt_l * QT) / KT : 0;
  const int nkb = (p.causal ? min(qt + 1, p.nkb) : p.nkb) - j0;  // causal: query tile qt needs key blocks 0 .. qt

  auto load_block = [&](int i) {  // K and V of key block j0 + i of the full sequence: shared prefix rows or this sequence's own rows
    const int j = j0 + i;
    const int slot = i % NSLOT;
    mbar_arrive_expect_tx(&kv_full[slot], 2 * NP * PLANE);
    const CUtensorMap* src = j < p.s_blocks ? &tmP : &tm;
    const int r = j < p.s_blocks ? j * KT : row0 + (j - p.s_blocks) * KT;
    uint8_t* dst = sKV + slot * 2 * NP * PLANE;
    for (int pl = 0; pl < NP; ++pl)
      for (int bx = 0; bx < NB; ++bx) {
        tma_load_2d(dst + pl * PLANE + bx * TILE, src, &kv_full[slot], ck + 64 * bx + pl * static_cast<int>(p.lo_off), r);
        tma_load_2d(dst + (NP + pl) * PLANE + bx * TILE, src, &kv_full[slot], cv + 64 * bx + pl * static_cast<int>(p.lo_off), r);
      }
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tm);
    mbar_init(q_full, 1);
    for (int i = 0; i < NSLOT; ++i) mbar_init(&kv_full[i], 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(q_full, NP * PLANE);
    for (int pl = 0; pl < NP; ++pl)
      for (int bx = 0; bx < NB; ++bx)
        tma_load_2d(sQ + pl * PLANE + bx * TILE, &tmQ, q_full, cq + 64 * bx + pl * static_cast<int>(p.lo_off), row0 + qt_l * QT);
    for (int j = 0; j < NSLOT && j < nkb; ++j) load_block(j);
  }
  __syncthreads();

  const float slope = p.alibi_slopes ? p.alibi_slopes[h] : 0.f;
  constexpr float LOG2E = 1.4426950408889634f;
  const float slope2 = slope * LOG2E;
  const int qrow = qt * QT + warp * 16 + g;  // this thread's rows qrow and qrow + 8 (full-sequence index)
  int sq[2] = {0, 0};                        // segment-causal: first visible key of rows qrow, qrow + 8
  if (p.seg_start)
    for (int r = 0; r < 2; ++r) sq[r] = qrow + 8 * r < p.T ? __ldg(p.seg_start + qrow + 8 * r) : 0;
  const int pad0 = p.p_valid, pad1 = p.s_blocks * KT;  // masked prefix rows [pad0, pad1) of the memory form
  float o[NB][32];  // o[bx]: head-dim columns [64 bx, 64 bx + 64)
#pragma unroll
  for (int bx = 0; bx < NB; ++bx)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[bx][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const uint32_t q_addr = smem_u32(sQ);
  mbar_wait(q_full, 0);

  for (int i = 0; i < nkb; ++i) {
    const int j = j0 + i;
    const int slot = i % NSLOT;
    mbar_wait(&kv_full[slot], (i / NSLOT) & 1);
    const uint32_t k_addr = smem_u32(sKV) + slot * 2 * NP * PLANE;
    const uint32_t v_addr = k_addr + NP * PLANE;
    // ---- S = Q K^T (64 x 64), hi*hi [+ lo*hi + hi*lo]; 4 k16 steps per 64-column box ----
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4 * NB; ++k) {
      const uint32_t bo = (k >> 2) * TILE;
      wgmma_m64n64k16_f16_ss(s, make_desc_sw128(q_addr + bo) + 2 * (k & 3), make_desc_sw128(k_addr + bo) + 2 * (k & 3), k > 0 ? 1u : 0u);
    }
    if (NP == 2) {
#pragma unroll
      for (int k = 0; k < 4 * NB; ++k) {
        const uint32_t bo = (k >> 2) * TILE;
        wgmma_m64n64k16_f16_ss(s, make_desc_sw128(q_addr + PLANE + bo) + 2 * (k & 3), make_desc_sw128(k_addr + bo) + 2 * (k & 3), 1u);
      }
#pragma unroll
      for (int k = 0; k < 4 * NB; ++k) {
        const uint32_t bo = (k >> 2) * TILE;
        wgmma_m64n64k16_f16_ss(s, make_desc_sw128(q_addr + bo) + 2 * (k & 3), make_desc_sw128(k_addr + PLANE + bo) + 2 * (k & 3), 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    // ---- scores to the log2 domain (+ ALiBi, masks), online softmax; s[4n + 2r + e] = S[row r][key 8n + 2t + e] ----
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int kidx = j * KT + n * 8 + 2 * t + (c & 1);
        const int qidx = qrow + (c >> 1) * 8;
        float v = fmaf(s[4 * n + c], LOG2E, slope2 * static_cast<float>(kidx));
        if (kidx >= p.T || (p.causal && kidx > qidx) || (kidx >= pad0 && kidx < pad1) || kidx < sq[c >> 1]) v = -INFINITY;
        s[4 * n + c] = v;
        mx[c >> 1] = fmaxf(mx[c >> 1], v);
      }
    }
    float alpha[2], mref[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float mn = fmaxf(m_run[r], mx[r]);
      mref[r] = (mn == -INFINITY) ? 0.f : mn;  // a row that has seen no key yet: every score is -inf -> P = 0
      alpha[r] = ex2a(m_run[r] - mref[r]);     // 0 for the first block (m_run = -inf)
      m_run[r] = mn;
      l[r] *= alpha[r];
    }
    if (!RNACC) {
#pragma unroll
      for (int bx = 0; bx < NB; ++bx)
#pragma unroll
        for (int i = 0; i < 32; ++i) o[bx][i] *= alpha[(i >> 1) & 1];
    }
    // ---- P = 2^(s - m) as fp16 hi [+ lo] A fragments, O += P V ----
    uint32_t ph[4][4], pl[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = 8 * kk + 2 * u;  // u: (block 2kk, row g), (2kk, g+8), (2kk+1, g), (2kk+1, g+8)
        const int r = u & 1;
        const float e0 = ex2a(s[i] - mref[r]), e1 = ex2a(s[i + 1] - mref[r]);
        l[r] += e0 + e1;
        ph[kk][u] = cvt_f16x2_rn_inf(e0, e1);
        if (NP == 2) {
          const float2 hf = unpack_h2(ph[kk][u]);
          pl[kk][u] = cvt_f16x2_rn_inf(e0 - hf.x, e1 - hf.y);
        }
      }
    }
    float pv[RNACC ? NB : 1][RNACC ? 32 : 1];
    auto& acc = [&]() -> float(&)[NB][32] {
      if constexpr (RNACC) return pv; else return o;
    }();
    wgmma_fence();
#pragma unroll
    for (int bx = 0; bx < NB; ++bx) wgmma_fence_regs(acc[bx]);
#pragma unroll
    for (int bx = 0; bx < NB; ++bx) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint64_t vh = make_desc_sw128(v_addr + bx * TILE + kk * 2048);  // 16 key rows of 128 B per k-step
        wgmma_m64n64k16_f16_rs_tb(acc[bx], ph[kk], vh, (RNACC && kk == 0) ? 0u : 1u);
        if (NP == 2) {
          wgmma_m64n64k16_f16_rs_tb(acc[bx], pl[kk], vh, 1u);
          wgmma_m64n64k16_f16_rs_tb(acc[bx], ph[kk], make_desc_sw128(v_addr + PLANE + bx * TILE + kk * 2048), 1u);
        }
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int bx = 0; bx < NB; ++bx) wgmma_fence_regs(acc[bx]);
    if (RNACC) {
#pragma unroll
      for (int bx = 0; bx < NB; ++bx)
#pragma unroll
        for (int i = 0; i < 32; ++i) o[bx][i] = __fmaf_rn(o[bx][i], alpha[(i >> 1) & 1], acc[bx][i]);
    }
    __syncthreads();  // every warp is done with this slot
    if (threadIdx.x == 0 && i + NSLOT < nkb) load_block(i + NSLOT);
  }

  // ---- epilogue: O / l -> fp16 hi [+ lo | + e4m3 planes]; rows qrow, qrow + 8, head-dim columns 8n + 2t (+1) ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    const int qidx = qrow + 8 * r;
    if (qidx >= p.T) continue;
    const float rl = 1.f / l[r];
    long long orow_idx = static_cast<long long>(b) * p.Tq + (qidx - p.s_blocks * KT);
    if (p.perm_C > 0) orow_idx = (static_cast<long long>(b / p.perm_C) * p.Tq + qidx) * p.perm_C + b % p.perm_C;
    // operand.cuh's column-pair store written out, for the same reason as in the GEMM epilogue (gemm_tc.cu)
    __half* orow = p.out + orow_idx * p.ldo + h * HD;
    uint8_t* f8 = reinterpret_cast<uint8_t*>(p.out + orow_idx * p.ldo + p.out_lo_off) + h * HD;
    const float sh = p.out_scale, sl = p.out_scale * LO8_GAIN;
    // delta-operand mode (DELTA): this row's exact value also goes to cout[b] when it is the masked row; base row to subtract
    const bool crow = DELTA && p.mask_pos != nullptr && qidx == __ldg(p.mask_pos + b);
    const __half* brow = (DELTA && p.base_o != nullptr) ? p.base_o + static_cast<long long>(qidx) * p.d + h * HD : nullptr;
#pragma unroll
    for (int n = 0; n < 8 * NB; ++n) {
      const int col = 8 * n + 2 * t;
      float x0 = o[n >> 3][4 * (n & 7) + 2 * r] * rl, x1 = o[n >> 3][4 * (n & 7) + 2 * r + 1] * rl;
      if (DELTA && crow) {  // rare (one row per sequence and head): fp16 hi / lo pair of the full value
        __half* cr = p.cout + static_cast<long long>(b) * p.ldc + h * HD + col;
        const uint32_t ch = cvt_f16x2_rn_inf(x0, x1);
        const float2 cf = unpack_h2(ch);
        *reinterpret_cast<uint32_t*>(cr) = ch;
        *reinterpret_cast<uint32_t*>(cr + p.c_lo_off) = cvt_f16x2_rn_inf(x0 - cf.x, x1 - cf.y);
      }
      if (DELTA && brow != nullptr) {
        const float2 bq = __half22float2(__ldg(reinterpret_cast<const __half2*>(brow + col)));
        x0 -= bq.x;
        x1 -= bq.y;
      }
      const uint32_t hi = cvt_f16x2_rn_inf(x0, x1);
      const float2 hf = unpack_h2(hi);
      *reinterpret_cast<uint32_t*>(orow + col) = hi;
      if (p.out_fmt == 1) {
        *reinterpret_cast<uint32_t*>(orow + p.out_lo_off + col) = cvt_f16x2_rn_inf(x0 - hf.x, x1 - hf.y);
      } else if (p.out_fmt == 2) {
        *reinterpret_cast<uint16_t*>(f8 + col) = static_cast<uint16_t>(cvt_e4m3x2((x0 - hf.x) * sl, (x1 - hf.y) * sl));
        *reinterpret_cast<uint16_t*>(f8 + p.d + col) = static_cast<uint16_t>(cvt_e4m3x2(hf.x * sh, hf.y * sh));
      }
    }
  }
}

}  // namespace

int launch_attention_wgmma(const AttnLaunch& a, cudaStream_t s) {
  if (a.B <= 0 || a.T <= 0) return PG_OK;
  if (a.nseg != 1 && a.nseg != 3) return set_error(PG_ERR_ARG, "attention: nseg must be 1 or 3");
  if (a.ld % 8 || a.lo_off % 8 || a.ldo % 8 || a.out_lo_off % 8 || (reinterpret_cast<uintptr_t>(a.out) & 15))
    return set_error(PG_ERR_ARG, "attention_wgmma: pitches must be multiples of 8 elements and out 16-byte aligned");
  if (a.q_begin != 0) return set_error(PG_ERR_ARG, "attention_wgmma: q_begin is only supported by the mma.sync kernel");
  if (a.prefix && (!a.causal || a.prefix_len <= 0 || (!a.prefix_mem && a.prefix_len % 128)))
    return set_error(PG_ERR_ARG, "attention_wgmma: a shared prefix needs causal attention and a length that is a multiple of 128");
  if ((a.prefix_mem && (!a.prefix || a.head_dim != 64)) || (a.seg_start && (a.B != 1 || a.prefix || !a.causal)))
    return set_error(PG_ERR_ARG, "attention_wgmma: the memory form needs a prefix and 64-wide heads; the segment-causal form one causal sequence");
  if (a.head_dim != 64 && a.head_dim != 128) return set_error(PG_ERR_ARG, "attention_wgmma: head width must be 64 or 128");
  const int HDw = a.head_dim;
  if (HDw == 128 && (a.base_o || a.mask_pos || a.perm_C))
    return set_error(PG_ERR_UNSUPPORTED, "attention_wgmma: the delta-operand and column-attention forms run on 64-wide heads only");
  AttnWParams p{};
  const int kvh = a.kv_heads ? a.kv_heads : a.heads;
  if (kvh <= 0 || a.heads % kvh || (kvh != a.heads && (a.prefix || a.perm_C || a.base_o || a.mask_pos || a.seg_start)))
    return set_error(PG_ERR_ARG, "attention_wgmma: kv_heads must divide heads; grouped-query attention runs the plain and causal forms");
  p.B = a.B; p.heads = a.heads; p.d = a.heads * HDw;
  p.dkv = kvh * HDw; p.grp = a.heads / kvh;
  p.Tq = a.T; p.s_blocks = a.prefix ? (a.prefix_len + KT - 1) / KT : 0;
  p.p_valid = a.prefix_mem ? a.prefix_len : p.s_blocks * KT;
  p.head_major = a.prefix_mem; p.seg_start = a.seg_start;
  p.T = a.T + p.s_blocks * KT;
  p.nqt = (a.T + QT - 1) / QT; p.nkb = (p.T + KT - 1) / KT;
  p.lo_off = a.lo_off; p.out = a.out; p.ldo = a.ldo; p.out_lo_off = a.out_lo_off;
  p.causal = a.causal; p.alibi_slopes = a.alibi_slopes;
  p.out_fmt = a.out_fmt;
  if (int rc = resolve_out_fmt(p.out_fmt, a.out_lo_off, a.out_scale, "attention_wgmma")) return rc;
  p.out_scale = a.out_scale;
  p.perm_C = a.perm_C;
  p.base_o = a.base_o; p.mask_pos = a.mask_pos; p.cout = a.cout; p.ldc = a.ldc; p.c_lo_off = a.c_lo_off;
  if ((a.base_o || a.mask_pos) && (a.prefix || a.perm_C || (a.mask_pos && (!a.cout || a.ldc % 2 || a.c_lo_off % 2 || a.c_lo_off <= 0))))
    return set_error(PG_ERR_ARG, "attention_wgmma: delta-operand mode needs plain sequences and, with mask_pos, a compact hi/lo output");
  if (a.perm_C < 0 || (a.perm_C > 0 && (a.prefix || a.B % a.perm_C))) return set_error(PG_ERR_ARG, "attention_wgmma: bad column-attention arguments");
  const int np = a.nseg == 3 ? 2 : 1;
  const uint64_t width = static_cast<uint64_t>(p.d + 2 * p.dkv) * np;
  if (np == 2 && a.lo_off != p.d + 2ll * p.dkv)
    return set_error(PG_ERR_ARG, "attention_wgmma: lo planes must follow the hi planes (lo_off == q + k + v width)");
  CUtensorMap tmQ, tm, tmP;
  int rc = make_tmap_f16_2d(&tmQ, a.qkv, static_cast<uint64_t>(a.B) * a.T, width, a.ld, QT, 64);
  if (rc) return rc;
  rc = make_tmap_f16_2d(&tm, a.qkv, static_cast<uint64_t>(a.B) * a.T, width, a.ld, KT, 64);
  if (rc) return rc;
  tmP = tm;
  if (a.prefix) {
    rc = make_tmap_f16_2d(&tmP, a.prefix, static_cast<uint64_t>(a.prefix_len), width, a.ld, KT, 64);
    if (rc) return rc;
  }
  const long long nitems = static_cast<long long>(a.B) * a.heads * p.nqt;
  if (nitems > 0x7FFFFFFFll) return set_error(PG_ERR_ARG, "attention_wgmma: grid too large");
  const int grid = static_cast<int>(nitems);
  int dev = 0;
  PG_CUDA_OK(cudaGetDevice(&dev));
  static bool attr_set[64] = {};
  if (dev < 64 && !attr_set[dev]) {
    PG_CUDA_OK(cudaFuncSetAttribute(attn_wgmma_kernel<1, 0, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemW<1, 64>::TOTAL));
    PG_CUDA_OK(cudaFuncSetAttribute(attn_wgmma_kernel<2, 0, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemW<2, 64>::TOTAL));
    PG_CUDA_OK(cudaFuncSetAttribute(attn_wgmma_kernel<2, 1, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemW<2, 64>::TOTAL));
    PG_CUDA_OK(cudaFuncSetAttribute(attn_wgmma_kernel<2, 0, 64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemW<2, 64>::TOTAL));
    PG_CUDA_OK(cudaFuncSetAttribute(attn_wgmma_kernel<1, 0, 64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemW<1, 64>::TOTAL));
    PG_CUDA_OK(cudaFuncSetAttribute(attn_wgmma_kernel<1, 0, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemW<1, 128>::TOTAL));
    PG_CUDA_OK(cudaFuncSetAttribute(attn_wgmma_kernel<2, 0, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemW<2, 128>::TOTAL));
    attr_set[dev] = true;
  }
  const bool delta = a.base_o != nullptr || a.mask_pos != nullptr;
  if (delta && np != 2) return set_error(PG_ERR_UNSUPPORTED, "attention_wgmma: the delta-operand form runs on fp16 hi/lo operands (nseg 3)");
  if (delta) attn_wgmma_kernel<2, 1, 64><<<grid, ATT_THREADS, SmemW<2, 64>::TOTAL, s>>>(tmQ, tm, tmP, p);
  else if (a.prefix_mem && np == 2) attn_wgmma_kernel<2, 0, 64, 1><<<grid, ATT_THREADS, SmemW<2, 64>::TOTAL, s>>>(tmQ, tm, tmP, p);
  else if (a.prefix_mem) attn_wgmma_kernel<1, 0, 64, 1><<<grid, ATT_THREADS, SmemW<1, 64>::TOTAL, s>>>(tmQ, tm, tmP, p);
  else if (HDw == 128 && np == 1) attn_wgmma_kernel<1, 0, 128><<<grid, ATT_THREADS, SmemW<1, 128>::TOTAL, s>>>(tmQ, tm, tmP, p);
  else if (HDw == 128) attn_wgmma_kernel<2, 0, 128><<<grid, ATT_THREADS, SmemW<2, 128>::TOTAL, s>>>(tmQ, tm, tmP, p);
  else if (np == 1) attn_wgmma_kernel<1, 0, 64><<<grid, ATT_THREADS, SmemW<1, 64>::TOTAL, s>>>(tmQ, tm, tmP, p);
  else attn_wgmma_kernel<2, 0, 64><<<grid, ATT_THREADS, SmemW<2, 64>::TOTAL, s>>>(tmQ, tm, tmP, p);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

}  // namespace pg
