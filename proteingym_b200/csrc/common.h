// Shared host-side declarations for libpgscore.so (internal; the public ABI is include/pgscore.h).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/pgscore.h"

namespace pg {

// Last error text for handle-less entry points (thread-local so concurrent per-GPU threads do not clobber each other).
std::string& tls_error();
int set_error(int code, const std::string& msg);

#define PG_CUDA_OK(expr)                                                                                   \
  do {                                                                                                     \
    cudaError_t _e = (expr);                                                                               \
    if (_e != cudaSuccess)                                                                                 \
      return ::pg::set_error(PG_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));             \
  } while (0)

int num_sms();

// Launch accounting + optional per-category CUDA-event timing (bench.py's roofline leg). Categories:
enum ProfCat { CAT_EMBED = 0, CAT_LN, CAT_GEMM_QKV, CAT_ATTN, CAT_GEMM_OUT, CAT_GEMM_FC1, CAT_GEMM_FC2, CAT_HEAD, CAT_SCORE, CAT_OTHER, CAT_TIED, CAT_REGROUP, CAT_COUNT };
struct ProfScope {  // records an event pair around the launches issued in its lifetime when profiling is on
  ProfScope(int cat, cudaStream_t s, int launches = 1);
  ~ProfScope();
  int cat; cudaStream_t s; int slot;
};

// ---- kernel launchers (each returns a pg_status) ----
// Operand row formats (pitches in fp16 elements; a "plane" is a column block of the row):
//   fmt 0  [hi fp16 (n)]
//   fmt 1  [hi fp16 (n) | lo fp16 (n)]                     lo at element offset lo_off
//   fmt 2  [hi fp16 (n) | lo8 (n bytes) | hi8 (n bytes)]   e4m3 planes start at element offset lo_off (= byte 2*lo_off);
//          lo8 = e4m3(lo * 2^11 * s), hi8 = e4m3(hi * s) with the power-of-two scale s of the consuming GEMM (gemm_tc.cu).
//          Weights use [hi fp16 | hi8 | lo8] with a per-row scale instead (api.cu pack_weight_f8_kernel).
// operand.cuh holds the device code that writes and reads these rows.
// Output format of a launcher: -1 = fmt 1 when there is a lo plane (lo_off > 0), else fmt 0. Resolves that default in place and
// rejects a format without its planes or its scale (`who` prefixes the error text).
inline int resolve_out_fmt(int& fmt, int64_t lo_off, float scale, const char* who) {
  if (fmt < 0) fmt = lo_off > 0 ? 1 : 0;
  if (fmt > 2 || (fmt >= 1 && lo_off <= 0) || (fmt == 2 && !(scale > 0.f))) return set_error(PG_ERR_ARG, std::string(who) + ": bad output format");
  return PG_OK;
}
struct GemmLaunch {
  const void* a; int64_t lda;
  const void* w; int64_t ldw;
  const float* bias;
  int M, N, K, nseg, epi;   // nseg: 1 fp16, 3 fp16 hi/lo x3, 2 fp16 hi*hi + e4m3 cross terms (a in fmt 2, w in weight fmt 2)
  __half* out; int64_t ldo; int64_t out_lo_off;
  float* resid; int64_t ldr;
  const float* rot_cos; const float* rot_sin; int rot_T; int rot_dim;
  int rot_half = 32;              // epi 3: half the head slot; 64 = 128-wide slots, tables [T, 64] (internal: pg_gemm keeps 32)
  float a_scale = 0.f;            // nseg 2: s used by the producer of a's e4m3 planes
  const float* w_inv = nullptr;   // nseg 2: [N] 1 / t_n of the weight rows
  int w_uniform = 0;              // nseg 2: all w_inv[n] are equal (one scale per matrix, as pg_load_weights / pg_pack_weight produce)
  int out_fmt = 0;                // epi != 2: 0, 1 or 2 (see above); planes at out_lo_off
  float out_scale = 0.f;          // out_fmt 2: s of the GEMM that will consume `out`
  // Grouped (block-diagonal) form, nseg 1 / 3 only: rows [g*grp_rows_a, (g+1)*grp_rows_a) of A (M = groups * grp_rows_a, a multiple of
  // 128 per group) are multiplied with rows [g*grp_rows_b, g*grp_rows_b + N) of w; outputs keep A's row index. 0 = plain GEMM.
  int grp_rows_a = 0, grp_rows_b = 0;
  // Delta-operand mode (api.cu forward_rows_delta): A holds the difference of each row to a shared base row t = row % base_T.
  //   base_pre  [base_T, N] fp32: added to the accumulator before the activation (W * base row + bias, computed once)
  //   base_post [base_T, N] fp16: subtracted after the activation (the base row's own activated output, rounded to fp16: any fixed
  //                               reference works as long as the next layer's base_pre was computed from the same values), so that
  //                               `out` is again a difference; null = `out` holds full values
  //   mask_pos  [M / base_T] (device): epi 2 only — row (row / base_T) * base_T + mask_pos[row / base_T] receives no update (its
  //                               exact value comes from the compact full-precision path)
  const float* base_pre = nullptr; const __half* base_post = nullptr; int base_T = 0; const int32_t* mask_pos = nullptr;
  // LM-head log-softmax partials (epi 7, K16; internal): the accumulator holds the logits of rows (b, t) = (row / lm_T, row % lm_T)
  // against N vocabulary columns, and no logit is stored. For every row with t + 1 < lm_lens[b] and every 128-column N tile the tile's
  // (max, sum exp(l - max)) goes to lm_part[row * tiles_n + tile] (columns >= N count as -inf), and the logit of column
  // lm_ids[row + 1] to lm_tgt[row]; lm_logits (optional, [M, N] fp32) receives every logit of those rows.
  float2* lm_part = nullptr; float* lm_tgt = nullptr; float* lm_logits = nullptr;
  const int32_t* lm_ids = nullptr; const int32_t* lm_lens = nullptr; int lm_T = 0;
};
int launch_gemm(const GemmLaunch& g, cudaStream_t s);
constexpr int GEMM_BN = 128;  // N tile of launch_gemm (the granularity of the epi 7 partials)
void set_gemm_kchunk(int v);    // tuning: see gemm_tc.cu
void set_gemm_prefetch(int v);
void set_gemm_cta2(int v);      // 1: clusters of two CTAs sharing the W tile (TMA multicast)

// fmt / scale as above (fmt 0 when lo_off == 0).
// base (optional, fp16 [base_T, d]): the output is LN(x[row]) - base[row % base_T] (delta-operand mode).
// dp: width of each output plane (0 = d); columns [d, dp) of every plane are written as zeros.
int launch_layernorm_f16(const float* x, int64_t ldx, const float* gamma, const float* beta, int rows, int d, __half* out,
                         int64_t ldo, int64_t lo_off, cudaStream_t s, int fmt = -1, float scale = 0.f, int perm_R = 0, int perm_C = 0,
                         const __half* base = nullptr, int base_T = 0, int dp = 0);
// dst row (b * T + row_sel[b]) <- src row b, row_bytes each (a multiple of 16): the compact exact rows back into the full buffers
int launch_scatter_rows(const void* src, int64_t src_pitch_bytes, void* dst, int64_t dst_pitch_bytes, const int32_t* row_sel, int B, int T,
                        int row_bytes, cudaStream_t s);

struct AttnLaunch {
  const __half* qkv; int64_t ld; int64_t lo_off;
  __half* out; int64_t ldo; int64_t out_lo_off;
  int B, T, heads, nseg, causal;
  const float* alibi_slopes;
  int q_begin = 0;  // first query row handled by this launch (mma.sync kernel only): rows [q_begin, T)
  int out_fmt = -1;        // -1: 1 if out_lo_off > 0 else 0; 2: e4m3 planes with out_scale (wgmma kernel only)
  float out_scale = 0.f;
  // Exact prefix reuse (causal, wgmma kernel only): the B sequences hold rows [prefix_len, prefix_len + T) of longer sequences
  // whose first prefix_len rows (a multiple of 128) are shared; their K and V live in `prefix` (one sequence, same pitch / planes).
  const __half* prefix = nullptr;
  int prefix_len = 0;
  // Column attention of an alignment (wgmma kernel only): the B sequences are the columns (b, c) of [R = T, C = perm_C] alignments;
  // output row (sequence (b, c), position r) is written to row (b, r, c) of `out`.
  int perm_C = 0;
  // Delta-operand mode: base_o (fp16 [T, heads*64]) is subtracted from every output row t before rounding (out = attention - base);
  // the full-precision value of row mask_pos[b] of sequence b is additionally written as an fp16 hi / lo pair to row b of `cout`.
  const __half* base_o = nullptr; const int32_t* mask_pos = nullptr; __half* cout = nullptr; int64_t ldc = 0; int64_t c_lo_off = 0;
  // Width of a head's q / k / v / output slot (wgmma kernel): 64, or 128 for the 128-wide slots of ProGen2's 80- and 96-wide heads.
  int head_dim = 64;
};
int launch_attention(const AttnLaunch& a, cudaStream_t s);

// x[row, :] = token embedding (mask row zeroed, token-dropout rescale) + learned position; optional LayerNorm-before.
struct EmbedLaunch {
  const int32_t* tokens; int n_tokens;
  const int32_t* positions;  // [P] masked token index or -1
  const int32_t* win_start;  // [P] or null
  int P, T, d;
  const float* embed;        // [vocab, d] fp32 (mask row as loaded)
  const float* pos_table;    // [max_pos+2, d] or null (ESM2)
  const float* lnb_gamma; const float* lnb_beta;  // emb_layer_norm_before or null
  int token_dropout; int mask_idx; int p_offset;  // p_offset: first row index p of this chunk
  int force_mask_scale = 0;  // 1: token-dropout rescale of a copy holding ONE mask even though no token is masked (the shared base row)
  float* x;                  // [P*T, d]
};
int launch_embed(const EmbedLaunch& e, cudaStream_t s);

// LM head on selected rows (esm/modules.py:322-328) + log_softmax: out [P, vocab].
struct HeadLaunch {
  const float* x; int d; int T;          // residual stream [P*T, d]
  const int32_t* row_in_seq;             // [P] token index within the window to emit (device) or null when all rows
  int P;                                 // number of output rows
  int all_rows;                          // 1: emit every row of x (P == rows), row_in_seq ignored
  const float* lna_g; const float* lna_b;    // emb_layer_norm_after
  const float* dense_w; const float* dense_b;  // [d, d], [d]
  const float* ln_g; const float* ln_b;      // lm_head.layer_norm
  const float* out_w; const float* out_b;    // [vocab, d] tied embedding, [vocab]
  int vocab;
  float* scratch_a; float* scratch_b;    // [P, d] each
  float* out;                            // [P, vocab]
};
int launch_head(const HeadLaunch& h, cudaStream_t s);

int launch_score(const float* table, int n_rows, int vocab, const int32_t* site_row, const int32_t* site_wt,
                 const int32_t* site_mt, const int32_t* row_offsets, int M, float* out, cudaStream_t s);

}  // namespace pg

namespace pg {
// 2D fp16 row-major tensor map [rows, cols] (pitch ld elements), box [box_rows, box_cols], SWIZZLE_128B, OOB -> 0.
int make_tmap_f16_2d(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                     uint32_t box_cols);
// General form: elem_bytes 2 (fp16) / 4 (fp32) / 1 (bytes), swizzle 128 or 64 bytes. Encoded maps are cached per host thread.
int make_tmap_2d(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, uint32_t box_cols,
                 int elem_bytes, int swizzle);
int launch_attention_wgmma(const AttnLaunch& a, cudaStream_t s);  // the model's attention: wgmma/TMA, 64-query x 64-key blocks
}  // namespace pg

namespace pg {
int launch_attn_single_query(const __half* qkv, int64_t ld, int64_t lo_off, const int32_t* row_sel, int B, int T, int heads,
                             __half* out, int64_t ldo, int64_t out_lo_off, cudaStream_t s, int out_fmt = -1, float out_scale = 0.f);
int launch_gather_rows(const float* x, const int32_t* row_sel, int B, int T, int d, float* xc, cudaStream_t s);
// ESM C: in place on q/k rows (q at column 0, k at heads*64, fp16 hi [+ lo at lo_off]): weight-only LayerNorm over the full width, then
// rotary per 64-wide head (t = row % T, cos/sin [T, 32]) and q *= 1/8 (elementwise.cu).
int launch_qk_ln_rotary(__half* qkv, int64_t ld, int64_t lo_off, int rows, int heads, const float* q_gamma, const float* k_gamma,
                        const float* rot_cos, const float* rot_sin, int T, cudaStream_t s);
// x[row] = wte[ids[row]] (+ wpe[row % T + pos_off] when a position table is given; null keeps the token embedding alone)
int launch_gather_embed(const int32_t* ids, const float* wte, long long rows, int d, int vocab, float* x, cudaStream_t s,
                        const float* wpe = nullptr, int T = 1, int pos_off = 0);
int launch_qkv_conv(const __half* in, __half* out, int64_t ld, int64_t lo_off, int B, int T, int heads, const float* taps,
                    float qscale, cudaStream_t s, const __half* prefix = nullptr);
// Retrieval-prior fusion arguments of the autoregressive head (device pointers; see pg_ar_fusion in include/pgscore.h).
struct ArFusion {
  const float* log_prior = nullptr; const int32_t* prior_row = nullptr; float alpha = 0.f;
  const float* log_prior2 = nullptr; const int32_t* prior_row2 = nullptr; float beta = 0.f;
  int first_col = 0;
  float* out_logprobs = nullptr;
};
// wte: the head [vocab, d]; bias: [vocab] or null; the label of token id v is head column v - label_off.
int launch_ar_head(const float* x, int d, int B, int T, int vocab, const int32_t* ids, const int32_t* lens, const float* lnf_g,
                   const float* lnf_b, const float* wte, const float* bias, int label_off, const ArFusion& fusion, float* tok_logp,
                   float* out_sum, cudaStream_t s);
// After a GEMM epi 7 pass over B sequences of T rows: tok_logp[r] = lm_tgt[r] - logsumexp of the row's `tiles` partials combined in
// tile order (0 for t >= lens[b] - 1, NaN for a next token outside [0, vocab)); out_logprobs (optional, [B*T, vocab], holding the logits
// epi 7 wrote) becomes the log-softmax rows in place; out_sum[b] = the sequence sums (seq_sum_kernel).
int launch_lm_head_combine(const float2* part, int tiles, const float* tgt, const int32_t* ids, const int32_t* lens, int B, int T, int vocab,
                           float* out_logprobs, float* tok_logp, float* out_sum, cudaStream_t s);
}  // namespace pg

namespace pg {
// MSA Transformer (msa_transformer.cu): embedding of B masked copies of an [R, Cfull] alignment window, and the regroupings /
// softmax of the tied row attention.
struct MsaEmbedLaunch {
  const int32_t* tokens; int R, Cfull;   // [R, Cfull] alignment tokens (BOS column included)
  const int32_t* positions;              // [P] masked column of row 0
  const int32_t* win_start;              // [P] first column of the window, or null (0)
  int p_offset, B, Cw, d;                // this chunk: positions [p_offset, p_offset + B), windows of Cw columns
  const float* embed; const float* pos_table; const float* row_pos;  // [vocab, d], [max_pos + 2, d], [1024, d] or null
  const float* gamma; const float* beta; // emb_layer_norm_before
  int mask_idx;
  float* x;                              // [B * R * Cw, d]
};
int launch_msa_embed(const MsaEmbedLaunch& e, cudaStream_t s);
int launch_tied_gather_qk(const __half* qkv, int64_t ldq, int64_t lo_off, int B, int R, int C, int H, int Cp, __half* tq, __half* tk,
                          int64_t ldt, cudaStream_t s);
int launch_tied_transpose_v(const __half* qkv, int64_t ldq, int64_t lo_off, int B, int R, int C, int H, int Kp, __half* tv, int64_t ldv,
                            cudaStream_t s);
int launch_tied_softmax(const float* S, int64_t lds, int G, int C, int Cp, int Kp, float scale, __half* P, int64_t ldp, int np, cudaStream_t s);
int launch_tied_scatter_out(const __half* ot, int64_t ldo_t, __half* out, int64_t ldo, int fmt, int B, int R, int C, int H, int Cp,
                            cudaStream_t s);
// Last layer: tied row attention for the single query column sel[b] of every alignment -> context rows (b, r) in operand format
// (S1: [B, H, C] fp32 scratch); and the residual rows of that column.
int launch_tied_col_attention(const __half* qkv, int64_t ldq, int64_t lo_off, const int32_t* sel, int B, int R, int C, int H, float scale,
                              float* S1, __half* out, int64_t ldo, int64_t out_lo_off, int out_fmt, float out_scale, cudaStream_t s);
int launch_msa_gather_col(const float* x, const int32_t* sel, int B, int R, int C, int d, float* xr, cudaStream_t s);
}  // namespace pg
