/*
 * pgscore.h — C ABI of libpgscore.so, the H100 (sm_90a) scorer for ProteinGym's PLM log-likelihood hot path.
 *
 * ProteinGym has no FFI/plugin API; its "operator interface" for this path is the Python call sequence in
 * proteingym/baselines/esm/compute_fitness.py (reference root: OATML-Markslab/ProteinGym). Each entry point below
 * names the reference code it replaces. All buffers are plain device pointers owned by the caller (PyTorch
 * allocations in our host code); the library never frees caller memory and keeps its own workspace inside the handle.
 * Calls are asynchronous on the given stream; the caller synchronises. Errors: non-zero return code + pg_last_error().
 * No C++ exceptions cross this boundary. A handle is bound to one device and is not thread-safe.
 */
#ifndef PGSCORE_H
#define PGSCORE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pg_handle_s* pg_handle;
typedef void* pg_stream; /* cudaStream_t */

enum pg_status { PG_OK = 0, PG_ERR_ARG = 1, PG_ERR_CUDA = 2, PG_ERR_STATE = 3, PG_ERR_UNSUPPORTED = 4 };

enum pg_arch {
  PG_ARCH_ESM1B = 0, /* ESM-1b / ESM-1v: learned positions (esm/model/esm1.py:83-102) */
  PG_ARCH_ESM2 = 1,  /* ESM2: rotary (esm/model/esm2.py:40-74) */
  PG_ARCH_TRANCEPTION = 2, /* Tranception decoder: grouped ALiBi, depthwise-conv q/k/v, relu^2 MLP
                              (tranception/model_pytorch.py:90-632); max_positions = n_ctx, vocab = 25 */
  PG_ARCH_MSA = 3,         /* MSA Transformer: tied row attention + column attention + FFN per layer, learned column positions and
                              (when the state holds "msa_position_embedding") row positions (esm/model/msa_transformer.py:100-222,
                              esm/axial_attention.py) */
  PG_ARCH_ESMC = 4,        /* ESM C (evoscale esm/models/esmc.py:117-173): pre-LN blocks without linear biases, q/k LayerNorm over the
                              full width + rotary, SwiGLU MLP (ffn_dim = the SwiGLU hidden width f; fc1 is [2f, d]), residual branches
                              divided by sqrt(layers / 36), untied 64-way output head; vocab 64, heads = embed_dim / 64, token_dropout
                              = emb_ln_before = 0, max_positions unused. Weights: the reference state-dict keys verbatim plus
                              "rotary.cos" / "rotary.sin" [T, 32]. Windows (compute_fitness.py:346-409 re-tokenises each one as
                              <cls> slice <eos>) are the caller's: pass one token row per distinct window, concatenated, with
                              win_start[p] = that row's offset and positions[p] = offset + index within the row. */
  PG_ARCH_RITA = 5,        /* RITA S / M / L causal decoder (proteingym/baselines/rita/rita_modeling.py:129-252): pre-LN blocks, separate
                              q/k/v Linear with bias, rotate-half rotary over 64-wide heads, no attention bias, tanh-GELU MLP (ffn_dim =
                              ff_ratio * d), final LayerNorm, head without bias; heads = embed_dim / 64 (RITA XL's 128-wide heads are
                              refused), max_positions = rows of the rotary tables = the longest token row a call may pass. Scored through
                              the pg_ar_* entry points without retrieval fusion. Weights: the HF state-dict keys without "transformer."
                              ("layers.{i}.self_attention.{query,key,value,proj}.{weight,bias}", "layers.{i}.{attn_norm,mlp_norm}.*",
                              "layers.{i}.mlp.{0,2}.*", "embedding.weight", "final_norm.*"), "lm_head.weight" [vocab, d] only for an
                              untied head (absent = the embedding), plus "rotary.cos" / "rotary.sin" [T, 32] = cos / sin(t * inv_freq[c])
                              from the checkpoint's rotary_embedding.inv_freq. */
  PG_ARCH_PROGEN2 = 6,     /* ProGen2 small / medium / base / large causal decoder (proteingym/baselines/progen2/models/progen/
                              modeling_progen.py:60-282, 389-401, 541-548): parallel residual x + attn(ln_1(x)) + mlp(ln_1(x)), bias-free
                              fused qkv_proj in 8 [q | v | k] shards (heads % 8 == 0), interleaved (rotate_every_two) rotary on the first
                              rotary_dim dims of q and k, bias-free out_proj, tanh-GELU MLP (ffn_dim = n_inner or 4d) with biases, ln_f, and
                              lm_head WITH bias of which only rows 5..29 are scored (compute_fitness.py:71-77: token ids 5..29, vocab =
                              the embedding rows, >= 30). head_dim 64 runs in 64-wide head slots, 66..128 (even) in 128-wide slots; head_dim
                              > 128 (progen2-xlarge) and PG_PREC_F16D are refused. max_positions = the longest token row a call may pass.
                              Scored through the pg_ar_* entry points without retrieval fusion: token ids are the full vocabulary's, a
                              next token outside 5..29 gives a NaN log-probability, and out_logprobs rows are 25 wide. Weights: the HF
                              state-dict keys without "transformer." ("h.{i}.ln_1.*", "h.{i}.attn.qkv_proj.weight" [3d, d],
                              "h.{i}.attn.out_proj.weight", "h.{i}.mlp.{fc_in,fc_out}.{weight,bias}", "wte.weight", "ln_f.*",
                              "lm_head.weight" [vocab, d], "lm_head.bias" [vocab]) plus "rotary.cos" / "rotary.sin" [T, S/2] with S the
                              slot width: column i < rotary_dim / 2 holds cos / sin(t * 10000^(-2i / rotary_dim)) in fp32 as
                              fixed_pos_embedding computes it (rotary_dim = head_dim when the config has none), later columns cos = 1,
                              sin = 0. ln_1 / ln_f use eps 1e-5. */
  PG_ARCH_PROTGPT2 = 7     /* ProtGPT2 = GPT-2 large causal decoder (proteingym/baselines/protgpt2/compute_fitness.py; transformers
                              modeling_gpt2.py GPT2LMHeadModel): learned absolute positions (wpe) added to the token embedding, pre-LN blocks
                              with c_attn / c_proj biases, causal attention without bias, tanh-GELU ("gelu_new") MLP (ffn_dim = n_inner or
                              4d), ln_f, and the head tied to wte: a log-softmax over all `vocab` columns (50 257) that runs as one
                              tensor-core GEMM whose epilogue keeps only per-tile (max, sum exp) partials (no logits are stored), in
                              fp16 hi/lo x3 under PG_PREC_F16X3 and PG_PREC_F16F8 and single fp16 under PG_PREC_F16. head_dim 64 only;
                              PG_PREC_F16D is refused. max_positions = the rows of wpe (n_positions); a row at position t of a call, or
                              start + t after a recorded prefix, adds wpe[t] / wpe[start + t]. Scored through the pg_ar_* entry points
                              without retrieval fusion; out_logprobs rows are `vocab` wide. Weights: the HF state-dict keys without
                              "transformer." ("h.{i}.ln_{1,2}.*", "h.{i}.attn.c_attn.{weight [d, 3d], bias [3d]}", "h.{i}.attn.c_proj.*",
                              "h.{i}.mlp.c_fc.{weight [d, ffn], bias}", "h.{i}.mlp.c_proj.{weight [ffn, d], bias}", "wte.weight" [vocab, d],
                              "wpe.weight" [max_positions, d], "ln_f.*"): Conv1D weights are [in, out] as for PG_ARCH_TRANCEPTION, and
                              no "lm_head.weight" (tied). LayerNorms use eps 1e-5. */
};

/* Tensor-core operand precision. The reference is strict fp32 (SURVEY.md §0.4). Every operand is an fp16 pair hi + lo.
 *  PG_PREC_F16X3: three fp16 wgmma passes (hi*hi + lo*hi + hi*lo), fp32 accumulate — ~22-bit operands, 3 tensor-pipe
 *                 units per product; the most accurate mode.
 *  PG_PREC_F16F8: linear layers = one fp16 wgmma pass hi*hi + one e4m3 wgmma pass holding BOTH cross terms as e4m3
 *                 ([lo8 | hi8] x [hi8 | lo8] along K, 2x the fp16 rate) = 2 units; attention keeps the x3 scheme. ~16-bit
 *                 operands; meets the 1e-3 abs per-mutant parity target (DESIGN.md §2). Default of the host code.
 *  PG_PREC_F16D : delta operands (ESM-1b / ESM-1v masked-marginals on one shared window): every linear layer = the shared unmasked
 *                 row at F16X3 precision, computed once per window, + ONE fp16 pass on the per-copy difference to it; the row that
 *                 holds the mask takes an exact (F16X3) compact path. 1 tensor-pipe unit per algorithmic FLOP; every other entry
 *                 point of such a handle behaves as F16X3.
 *  PG_PREC_F16  : single fp16 pass; fastest, |error| ~1e-2 on scores of std ~6 (Spearman > 0.999) — not a parity mode.
 * In all modes the hi*hi accumulation is cut into K chunks that the epilogue adds in round-to-nearest fp32 (gemm_tc.cu). */
enum pg_precision { PG_PREC_F16 = 0, PG_PREC_F16X3 = 1, PG_PREC_F16F8 = 2, PG_PREC_F16D = 3 };

typedef struct {
  int32_t arch;            /* pg_arch */
  int32_t layers;          /* args.layers / cfg.encoder_layers */
  int32_t embed_dim;       /* args.embed_dim */
  int32_t heads;           /* args.attention_heads; head_dim = embed_dim / heads must be 64, except ESM2: any even head_dim <= 64 */
  int32_t ffn_dim;         /* args.ffn_embed_dim (ESM2: 4*embed_dim, esm2.py:52) */
  int32_t vocab;           /* 33 */
  int32_t max_positions;   /* learned-position table rows - 2 (ESM-1b: 1024) */
  int32_t token_dropout;   /* esm1.py:125 / esm2.py:85 */
  int32_t emb_ln_before;   /* esm1.py:135-136; decided by key presence in the checkpoint (pretrained.py:80-82) */
  int32_t precision;       /* pg_precision */
  int32_t device;          /* CUDA device ordinal */
  int32_t max_rows;        /* workspace capacity in token rows (sequences x window length) per pass; 0 = default */
} pg_model_desc;

typedef struct {
  const char* name;   /* reference state_dict key after prefix stripping, e.g. "layers.0.self_attn.q_proj.weight" */
  const void* data;   /* device pointer, fp32, contiguous */
  int64_t shape[2];   /* [rows, cols]; 1-D tensors use shape[1] = 1 */
} pg_tensor;

/* Replaces pretrained.load_model_and_alphabet + model.cuda() (compute_fitness.py:349-353; esm/pretrained.py:24-218):
 * create a model instance, then hand it the (already key-normalised) fp32 state dict; the library repacks into its own
 * operand buffers (q scaling folded in, multihead_attention.py:261). pg_load_weights is SYNCHRONOUS: it runs on the default
 * stream and returns after the repack has finished, so the caller may free its tensors immediately.
 * Limits of one handle: head_dim 64; a pass holds at most max_rows token rows and 8192 sequences (longer inputs are processed
 * in several passes inside the call; results do not depend on the split). */
int pg_create(const pg_model_desc* desc, pg_handle* out);
int pg_load_weights(pg_handle h, const pg_tensor* tensors, int32_t n);
int pg_destroy(pg_handle h);
const char* pg_last_error(pg_handle h); /* h may be NULL: returns the last creation error */

/* Replaces the masked-marginals loop (compute_fitness.py:486-504) — L+2 batch-1 forwards of
 * ProteinBertModel/ESM2.forward (esm1.py:116-193 / esm2.py:76-143) + log_softmax + row pick — by one batched pass.
 *   tokens     [n_tokens] int32 (device): <cls> seq <eos> of the FULL sequence
 *   positions  [P] int32 (device): token index i to mask for row p; -1 = no mask (wt-marginals row)
 *   win_start  [P] int32 (device) or NULL (= all 0): first token of row p's window (get_optimal_window, utils/scoring_utils.py:43-52)
 *   out_row    [P] int32 (device) or NULL: which token index of the window to emit for row p, relative to the full
 *              sequence; NULL = positions[p]
 *   T          window length (<= 1024 for ESM-1b; tokens per row)
 *   out_logprobs [P, vocab] fp32 (device): log_softmax(logits)[out_row - win_start]
 * All rows share T (no padding exists on this path). */
int pg_masked_marginals(pg_handle h, const int32_t* tokens, int32_t n_tokens, const int32_t* positions,
                        const int32_t* win_start, const int32_t* out_row, int32_t P, int32_t T, float* out_logprobs,
                        pg_stream stream);

/* Replaces the MSA Transformer masked-marginals loop (compute_fitness.py:383-399; model call msa_transformer.py:150-222): `tokens` is
 * the sampled alignment as [R, C_full] token ids (BOS column included, row 0 = the target, no padding); for every p the token at
 * (row 0, column positions[p]) is replaced by <mask>, the whole alignment — or its window of Cw columns starting at win_start[p] when
 * C_full > 1024 (win_start null: 0) — is forwarded, and out_logprobs[p, :] = log_softmax(logits[row 0, column positions[p]]).
 * PG_ARCH_MSA handles only. All pointers are device memory. Several positions are processed per pass (max_rows / (R * Cw), at least 1
 * alignment must fit). */
int pg_msa_masked_marginals(pg_handle h, const int32_t* tokens, int32_t R, int32_t C_full, const int32_t* positions,
                            const int32_t* win_start, int32_t P, int32_t Cw, float* out_logprobs, pg_stream stream);

/* Full-table variant used by wt-marginals (compute_fitness.py:475): one unmasked (or arbitrarily masked) forward of
 * `T` tokens starting at `win_start`, emitting log_softmax for every token: out [T, vocab]. mask_pos = -1 for none. */
int pg_forward_logprobs(pg_handle h, const int32_t* tokens, int32_t n_tokens, int32_t win_start, int32_t T,
                        int32_t mask_pos, float* out_logprobs, pg_stream stream);

/* Replaces one batch of get_tranception_scores_mutated_sequences (tranception/utils/scoring_utils.py:97-128): forward of B
 * right-padded sequences + shifted token log-likelihood summed over the real tokens of each sequence.
 *   ids   [B, T] int32 (device): [CLS] seq [SEP] then [PAD]; lens [B]: number of real tokens (len(seq) + 2)
 *   log_prior [Lp, vocab] fp32 + prior_row [B, T] int32 (device) or both NULL: retrieval fusion of
 *             model_pytorch.py:806-830 — for row (b, t) with prior_row >= 0 the predicted distribution becomes
 *             (1 - alpha) * log_softmax + alpha * log_prior[prior_row]  (the host computes the slice/flip index arithmetic)
 *   out_sum_logp [B] fp32: sum_{t < len-1} log p(ids[b, t+1] | ids[b, <= t])
 * Weights for a PG_ARCH_TRANCEPTION handle use the HF names without the "transformer." prefix (Conv1D weights [in, out]),
 * plus "h.{i}.attn.conv_taps" [768, 8] (look-back taps + bias per q/k/v, head group, channel) and "alibi_slopes" [heads, 1]. */
/* A PG_ARCH_RITA handle runs the same entry points on its own token ids (any vocabulary, no [CLS] / [SEP] assumed): out_sum_logp[b] =
 * sum_{t < lens[b]-1} log p(ids[b, t+1] | ids[b, <= t]); a retrieval prior is refused with PG_ERR_ARG (f->out_logprobs is allowed). */
int pg_ar_loglik(pg_handle h, const int32_t* ids, const int32_t* lens, int32_t B, int32_t T, const float* log_prior,
                 const int32_t* prior_row, float alpha, float* out_sum_logp, pg_stream stream);

/* Retrieval fusion arguments of pg_ar_loglik_fused — the per-position mixing the reference does inside forward():
 *   Tranception   (tranception/model_pytorch.py:806-830):  fused = (1-alpha)*logp + alpha*log_prior            on ALL columns
 *   TranceptEVE   (trancepteve/model_pytorch.py:1100-1116): fused = (1-beta)*((1-alpha)*logp + alpha*log_prior) + beta*log_prior2
 *                                                          on the amino-acid columns (>= 5) only
 * The host does the slice / flip index arithmetic and hands the kernel one table row index per token row:
 *   prior_row  [B, T] int32: row of log_prior for (b, t); -1 = no fusion; -2 = keep only the (1-alpha) factor (the reference's
 *              fallback for non-focus columns that its coordinate arithmetic places outside the MSA, :1131-1133)
 *   prior_row2 [B, T] int32: row of log_prior2 (EVE) or -1 (= two-way fusion with log_prior only, :1129-1130)
 *   first_col  fusion applies to vocabulary columns >= first_col (0 Tranception, 5 TranceptEVE)
 *   out_logprobs optional [B, T, vocab] fp32: the fused log-probabilities of every column for t < len-1 (what
 *              get_transformer_log_softmax, trancepteve/model_pytorch.py:821-874, returns; used for prior recalibration)
 * All pointers are device pointers; tables are [rows, vocab] fp32. */
typedef struct pg_ar_fusion {
  const float* log_prior;
  const int32_t* prior_row;
  float alpha;
  const float* log_prior2;
  const int32_t* prior_row2;
  float beta;
  int32_t first_col;
  float* out_logprobs;
} pg_ar_fusion;

/* pg_ar_loglik with the full fusion argument block (f may be NULL = no retrieval). pg_ar_loglik(h, ..., log_prior, prior_row,
 * alpha, ...) is the same call with only the first prior set and first_col = 0. */
int pg_ar_loglik_fused(pg_handle h, const int32_t* ids, const int32_t* lens, int32_t B, int32_t T, const pg_ar_fusion* f,
                       float* out_sum_logp, pg_stream stream);

/* Exact wild-type-prefix reuse (north_star: "positions share a single prefix/KV pass"; the reference carries the layer_past /
 * use_cache plumbing, model_pytorch.py:209-237, 441-458, and never uses it in scoring_utils.py:89-132). In a causal decoder with
 * causal depthwise convolutions every hidden state of a mutant before its first changed token equals the wild type's, so only rows
 * >= start need the transformer; keys / values of rows < start and the 6 rows of conv look-back come from the wild type's pass.
 *   pg_ar_prefix_begin : forward of ONE sequence ids[T] (the wild type in the window being scored), recording every layer's raw and
 *                        conv'd q/k/v rows inside the handle. out_tok_logp [T] fp32 (device): log p(ids[t+1] | ids[<=t]) for
 *                        t < T-1 (0 at T-1), fused with the priors in f like pg_ar_loglik_fused (f->prior_row is [1, T]);
 *                        f->out_logprobs [T, vocab] receives the full fused rows when non-NULL (the host needs row start-1 to score
 *                        a mutant whose first changed token sits exactly at `start`).
 *   pg_ar_loglik_prefix: B right-padded suffixes ids[B, T] = tokens start .. start+T-1 of sequences that share tokens 0 .. start-1
 *                        with the recorded wild type; lens[B] = real tokens in each suffix; start = a positive multiple of 128 (the
 *                        attention tile), < the recorded length. out_sum_logp[b] = sum over the suffix rows of
 *                        log p(token t+1 | tokens <= t), t >= start. Rows are bit-identical to what pg_ar_loglik computes for the
 *                        same sequences; only the summation is split (prefix part from the wild type's rows + this suffix part).
 * The record lives until the next pg_ar_prefix_begin on the handle. */
int pg_ar_prefix_begin(pg_handle h, const int32_t* ids, int32_t T, const pg_ar_fusion* f, float* out_tok_logp, pg_stream stream);
int pg_ar_loglik_prefix(pg_handle h, const int32_t* ids, const int32_t* lens, int32_t B, int32_t T, int32_t start,
                        const pg_ar_fusion* f, float* out_sum_logp, pg_stream stream);

/* Replaces label_row over the whole DMS frame (compute_fitness.py:240-250, :505-514):
 *   score[m] = sum_{s in [row_offsets[m], row_offsets[m+1])} table[site_row[s], site_mt[s]] - table[site_row[s], site_wt[s]]
 * table [n_rows, vocab] fp32; site_* int32 CSR arrays (device); out_scores [M] fp32. Fixed summation order per mutant. */
int pg_score_mutants(const float* table, int32_t n_rows, int32_t vocab, const int32_t* site_row, const int32_t* site_wt,
                     const int32_t* site_mt, const int32_t* row_offsets, int32_t M, float* out_scores,
                     pg_stream stream);

/* ---- kernel-level entry points (used by the parity tests and bench roofline legs; same kernels as above) ---- */

/* C = epilogue(A[M,K] * W[N,K]^T + bias). Operand rows (pitches lda/ldw/ldo in fp16 elements):
 *   nseg 1: [hi fp16 (K)]        nseg 3: [hi fp16 (K) | lo fp16 (K)]
 *   nseg 2: a = [hi fp16 (K) | lo8 (K bytes) | hi8 (K bytes)] with lo8 = e4m3(lo * 2^11 * a_scale), hi8 = e4m3(hi * a_scale);
 *           w = [hi fp16 (K) | hi8 (K bytes) | lo8 (K bytes)] with the per-row scale t_n, w_inv[n] = 1/t_n (pg_pack_weight fmt 2)
 *   out_fmt (epi != 2): 0 = auto (1 if out_lo_off > 0), 1 = fp16 lo plane at column out_lo_off, 2 = e4m3 planes
 *           [lo8 (N bytes) | hi8 (N bytes)] at column out_lo_off scaled by out_scale (i.e. an `a` operand for an nseg-2 GEMM)
 *   epi 0: out_h[M, ldo] = fp16(acc + bias) (+ second plane(s) per out_fmt)
 *   epi 1: same with exact-erf GELU (esm/modules.py:17-24)
 *   epi 2: resid[M, ldr] (fp32) += acc + bias
 *   epi 3: as 0, with rotary applied to the first 2*rot_dim columns ([q | k], heads of 64; esm/rotary_embedding.py:11-20),
 *          token index = row % rot_T, cos/sin tables [rot_T, 32] fp32 in rot_cos/rot_sin.
 *   epi 4: as 0 with squared ReLU relu(x)^2 (tranception/activations.py:79-84). bias may be NULL (no bias).
 *   epi 5: SwiGLU silu(g) * v (esm/layers/blocks.py:21-43): w rows interleaved in blocks of 8 (rows 16i..16i+7 = gate rows 8i..8i+7,
 *          rows 16i+8..16i+15 = up rows 8i..8i+7; N % 16 == 0); the output is N/2 columns wide (planes of N/2 columns at out_lo_off,
 *          out_fmt 2 needs N/2 % 64 == 0), column 8i + c = silu(acc[16i + c]) * acc[16i + 8 + c]. */
typedef struct {
  const void* a; int64_t lda;
  const void* w; int64_t ldw;
  const float* bias;
  int32_t M, N, K, nseg, epi;
  void* out_h; int64_t ldo; int64_t out_lo_off;
  float* resid; int64_t ldr;
  const float* rot_cos; const float* rot_sin; int32_t rot_T; int32_t rot_dim;
  float a_scale; const float* w_inv; /* nseg 2 */
  int32_t out_fmt; float out_scale;
  /* grouped (block-diagonal) form, nseg 1 / 3, no bias: rows [g*grp_rows_a, (g+1)*grp_rows_a) of a (M = groups * grp_rows_a, a multiple
   * of 128 per group) meet rows [g*grp_rows_b, g*grp_rows_b + N) of w; outputs keep a's row index. The tied row attention of the MSA
   * Transformer runs its two products this way (esm/axial_attention.py:140,176). 0 = plain GEMM. */
  int32_t grp_rows_a, grp_rows_b;
  /* delta-operand form (PG_PREC_F16D): `a` holds differences to shared base rows t = row % base_T (M a multiple of base_T, N % 64 == 0);
   * base_pre [base_T, N] fp32 is added to the accumulator before the activation, base_post [base_T, N] fp16 (or NULL) subtracted after
   * it, and with epi 2 the rows (row / base_T) * base_T + mask_pos[row / base_T] receive no update (mask_pos device int32, or NULL). */
  const float* base_pre; const void* base_post; int32_t base_T; const int32_t* mask_pos;
} pg_gemm_args;
int pg_gemm(const pg_gemm_args* args, pg_stream stream);

/* fp32 weights [N, K] (nn.Linear layout) -> the operand format of pg_gemm's `w`: fmt 0 = nseg 1, fmt 1 = nseg 3,
 * fmt 2 = nseg 2 (writes w_inv[N]). out has N rows of K (fmt 0) or 2K (fmt 1, 2) fp16 elements. */
int pg_pack_weight(const float* w, int32_t N, int32_t K, int32_t fmt, void* out, float* w_inv, pg_stream stream);

/* LayerNorm (eps 1e-5, esm/modules.py:68-81) of fp32 rows -> fp16 hi, and at column offset lo_off (if > 0) the second
 * plane(s): fmt 0 = auto (fp16 lo), 1 = fp16 lo, 2 = e4m3 [lo8 | hi8] scaled by `scale` (an nseg-2 `a` operand). */
int pg_layernorm_f16(const float* x, int64_t ldx, const float* gamma, const float* beta, int32_t rows, int32_t d,
                     void* out, int64_t ldo, int64_t lo_off, int32_t fmt, float scale, pg_stream stream);

/* Multi-head self-attention over equal-length sequences (multihead_attention.py:357-394), head_dim 64, q pre-scaled.
 *   qkv [B*T, ld] fp16 with q at column 0, k at column d, v at 2d (d = heads*64); lo parts at +lo_off when nseg == 3.
 *   out [B*T, ldo] fp16 (lo at +out_lo_off). causal/alibi are for the Tranception path (model_pytorch.py:155-183). */
typedef struct {
  const void* qkv; int64_t ld; int64_t lo_off;
  void* out; int64_t ldo; int64_t out_lo_off;
  int32_t B, T, heads, nseg;
  int32_t causal; const float* alibi_slopes; /* NULL = none */
  int32_t impl; /* 0 = the model's kernel (wgmma/TMA, 64x64 blocks), 1 = mma.sync cross-check kernel */
  int32_t out_fmt; float out_scale; /* as pg_gemm_args (0 = auto); 2 only with impl 0 */
  /* delta-operand form (impl 0): out = attention - base_o[t] (base_o fp16 [T, heads*64], or NULL); the full-precision value of row
   * mask_pos[b] of every sequence b goes to row b of cout as an fp16 hi / lo pair (pitch ldc, lo plane at +c_lo_off), or NULL. */
  const void* base_o; const int32_t* mask_pos; void* cout; int64_t ldc; int64_t c_lo_off;
} pg_attn_args;
int pg_attention(const pg_attn_args* args, pg_stream stream);

/* ---- MSA pre-processing for the Tranception retrieval prior (SURVEY.md §8f rank 2) ----
 * pg_msa_cluster_neighbors replaces calc_num_cluster_members_nogaps[_parallel] (proteingym/utils/weights.py:114-216):
 *   tokens [N, ld] uint8 (device), 0 = gap/invalid; min_matches[i] = smallest pair_matches for which the reference's float64 test
 *   `pair_matches / L_non_gaps[i] > identity_threshold` holds; out_neighbors[i] = 1 + #{j != i : matches(i, j) >= min_matches[i]}
 *   where matches counts positions with tokens[i,k] == tokens[j,k] != 0. Sequence weight = 1 / neighbors (weights.py:51-52).
 * pg_msa_prior replaces the frequency computation of get_msa_prior (tranception/utils/msa_utils.py:118-128):
 *   tokens_t [L, N] uint8 (device, column-major MSA; id >= vocab = letter outside the vocabulary), weights [N] fp64;
 *   out [L, vocab] fp64 = (sum_i w_i [tok == k] + base_rate * W) / (sum_i w_i [tok in vocab] + vocab * base_rate * W). */
int pg_msa_cluster_neighbors(const uint8_t* tokens, int64_t ld, int32_t N, int32_t L, const int32_t* min_matches,
                             int32_t* out_neighbors, pg_stream stream);
int pg_msa_prior(const uint8_t* tokens_t, const double* weights, int32_t N, int32_t L, int32_t vocab, double base_rate, double* out,
                 pg_stream stream);

/* EVE log-prior pre-step of TranceptEVE (trancepteve/model_pytorch.py:969-1001 -> EVE/VAE_decoder.py:118-169). The dense layers of
 * the encoder / Bayesian decoder run through pg_gemm (fp16 hi/lo operand rows from pg_pack_weight fmt 1, nseg 3, fp32 reduce-add
 * epilogue); this entry is the one op of the batched sampler that is not a GEMM with shared weights: the decoder's 1x1 output
 * convolution (VAE_decoder.py:139-147) with one weight draw PER SAMPLE,
 *   y[s, j*C + c] = sum_a x[s, j*A + a] * conv[s, c*A + a]      x [S, J*A], conv [S, C*A], y [S, J*C], all fp32 on the device. */
int pg_eve_output_conv(const float* x, const float* conv, int32_t S, int32_t J, int32_t A, int32_t C, float* y, pg_stream stream);

/* Launch accounting and per-category device timing (bench.py's roofline leg).
 * pg_launch_count: kernels launched by this library since load. pg_profile_begin/end: CUDA-event pairs are recorded on
 * the launching stream around every kernel; _end (after the caller synchronised) returns summed ms and scope counts
 * for categories {0 embed, 1 layernorm, 2 gemm_qkv, 3 attention, 4 gemm_out, 5 gemm_fc1, 6 gemm_fc2, 7 head, 8 score, 9 other}. */
long long pg_launch_count(void);
int pg_profile_begin(void);
int pg_profile_end(float* ms, int32_t* counts, int32_t ncat);

/* Process-wide tuning knobs (benchmarks / numerics probes; defaults are the measured-best values):
 *   "gemm_kchunk"  longest run of K (elements) a hi*hi accumulation chunk covers before it is added to the accumulator in RN fp32
 *                  (default 1280; 0 = no chunking). Also settable through the environment variable PG_GEMM_KCHUNK.
 *   "gemm_cta2"    1 (default): the GEMM runs as clusters of two CTAs that share the W tile (each loads half and multicasts it
 *                  to both); 0: one CTA per 128 x 128 tile. PG_GEMM_CTA2.
 *   "gemm_prefetch" k-blocks of L2 look-ahead the GEMM's TMA producer issues for the streamed A operand (default 0 = off: measured
 *                  neutral-to-negative in the model; PG_GEMM_PREFETCH). */
int pg_set_tuning(const char* key, int32_t value);


/* Build/version probe (also what the CPU-only test suite calls to check the library loads). */
int pg_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* PGSCORE_H */
