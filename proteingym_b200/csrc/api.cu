// C-ABI of libpgscore.so (include/pgscore.h): model handle, weight repacking, and the batched masked-marginal forward.
#include <cmath>
#include <cstdlib>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "common.h"
#include "operand.cuh"
#include "reduce.cuh"

namespace pg {

std::string& tls_error() {
  static thread_local std::string e;
  return e;
}
int set_error(int code, const std::string& msg) {
  tls_error() = msg;
  return code;
}

int num_sms() {  // of the current device (cached per ordinal: one process may hold handles on several GPUs)
  static int n[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return 132;
  if (!n[dev]) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[dev] = v > 0 ? v : 132;
  }
  return n[dev];
}

// ---- launch accounting / profiling -------------------------------------------------------------------------------
namespace {
struct ProfState {
  bool on = false;
  std::vector<cudaEvent_t> ev;      // pairs
  std::vector<int> ev_cat;
  size_t used = 0;
  long long launches[CAT_COUNT] = {};
};
ProfState& prof() {
  static ProfState p;
  return p;
}
std::mutex& prof_mu() {
  static std::mutex m;
  return m;
}
}  // namespace

ProfScope::ProfScope(int c, cudaStream_t st, int launches) : cat(c), s(st), slot(-1) {
  std::lock_guard<std::mutex> lk(prof_mu());
  ProfState& p = prof();
  p.launches[c] += launches;
  if (!p.on) return;
  if (p.used + 2 > p.ev.size()) {
    for (int i = 0; i < 2; ++i) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      p.ev.push_back(e);
    }
    p.ev_cat.push_back(c);
  }
  slot = static_cast<int>(p.used);
  p.ev_cat[slot / 2] = c;
  p.used += 2;
  cudaEventRecord(p.ev[slot], s);
}
ProfScope::~ProfScope() {
  if (slot < 0) return;
  std::lock_guard<std::mutex> lk(prof_mu());
  cudaEventRecord(prof().ev[slot + 1], s);
}

namespace {

// Element (n, k) of a source weight is w[n * sn + k * sk]: sk = 1 for nn.Linear ([out = N, in = K]), sn = 1 for Conv1D ([in, out],
// x @ W). Both are packed to the K-major [N, np*K] operand layout, scaled by `scale` (the q scaling fold).
// fp16 formats: hi at [n, 0:K] and (np == 2) lo at [n, K:2K].
__global__ void pack_weight_kernel(const float* __restrict__ w, int N, int K, long long sn, long long sk, float scale, __half* __restrict__ out,
                                   int np) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(N) * K) return;
  const int n = static_cast<int>(i / K), k = static_cast<int>(i % K);
  store_operand_one(out + static_cast<long long>(n) * K * np, K, 0, np == 2 ? 1 : 0, 0.f, k, w[n * sn + k * sk] * scale);
}
// Weights in the fp16 + e4m3 format of gemm_tc.cu (nseg 2): row n = [hi fp16 (K) | hi8 (K bytes) | lo8 (K bytes)], pitch 4K bytes,
// hi8 = e4m3(hi * t), lo8 = e4m3(lo * 2^11 * t) with ONE power of two t per matrix: the one that puts the largest |hi| of the matrix in
// (112, 224]. e4m3 is a floating-point format (2^-4 relative precision over 15 binades), so rows much smaller than the largest one
// keep their precision; a per-row scale would only cost the epilogue a load per output column. w_inv[n] = 1 / t for every n.
// Two kernels: matrix |hi| maximum, then pack.
__global__ void weight_absmax_kernel(const float* __restrict__ w, int N, int K, long long sn, long long sk, float scale,
                                     unsigned int* __restrict__ amax_bits) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  float a = 0.f;
  if (i < static_cast<long long>(N) * K) a = fabsf(__half2float(f2h_sat(w[(i / K) * sn + (i % K) * sk] * scale)));
  a = warp_max(a);
  if ((threadIdx.x & 31) == 0 && a > 0.f) atomicMax(amax_bits, __float_as_uint(a));  // non-negative floats order like their bit patterns
}
__global__ void pack_weight_f8_kernel(const float* __restrict__ w, int N, int K, long long sn, long long sk, float scale,
                                      const unsigned int* __restrict__ amax_bits, __half* __restrict__ out, float* __restrict__ w_inv) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  const float amax = __uint_as_float(*amax_bits);
  float t = 1.f;
  if (amax > 0.f) {
    int e;
    frexpf(amax, &e);                 // amax = m * 2^e, m in [0.5, 1)
    t = ldexpf(1.f, 8 - e);           // amax * t in [128, 256)
    if (amax * t > 224.f) t *= 0.5f;  // -> (112, 224]: one binade of headroom below the e4m3 maximum of 448
  }
  const float* wr = w + static_cast<long long>(n) * sn;
  __half* orow = out + static_cast<long long>(n) * K * 2;
  for (int k = lane; k < K; k += 32) store_weight_f8_one(orow, K, t, k, wr[k * sk] * scale);
  if (lane == 0) w_inv[n] = 1.f / t;
}
// Packs a group of [N, K] weights (w[i] scaled by scale[i]) into consecutive blocks of N operand rows of `out` on stream s, in fp16
// format (np 1 / 2) or, with `f8_scratch`, in the fp16 + e4m3 format (np 2) with ONE scale t for the whole group: a group is one
// GEMM operand (q, k and v). w_inv[i * N + n] = 1 / t. `f8_scratch` is one device word per call (kept alive by the caller).
struct PackSrc {
  PackSrc(const float* w_, float scale_ = 1.f) : w(w_), scale(scale_) {}
  const float* w;
  float scale;
};
void pack_weights(std::initializer_list<PackSrc> group, int N, int K, long long sn, long long sk, int np, unsigned int* f8_scratch,
                  __half* out, float* w_inv, cudaStream_t s) {
  const long long tot = static_cast<long long>(N) * K;
  const unsigned blocks = static_cast<unsigned>((tot + 255) / 256);
  if (!f8_scratch) {
    for (const PackSrc& m : group) {
      pack_weight_kernel<<<blocks, 256, 0, s>>>(m.w, N, K, sn, sk, m.scale, out, np);
      out += tot * np;
    }
    return;
  }
  cudaMemsetAsync(f8_scratch, 0, sizeof(unsigned int), s);
  for (const PackSrc& m : group) weight_absmax_kernel<<<blocks, 256, 0, s>>>(m.w, N, K, sn, sk, m.scale, f8_scratch);
  for (const PackSrc& m : group) {
    pack_weight_f8_kernel<<<(N + 7) / 8, 256, 0, s>>>(m.w, N, K, sn, sk, m.scale, f8_scratch, out, w_inv);
    out += tot * 2;
    w_inv += N;
  }
}
__global__ void scale_copy_kernel(const float* __restrict__ src, float* __restrict__ dst, int n, float scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i] * scale;
}

struct Layer {
  __half *wqkv = nullptr, *wo = nullptr, *w1 = nullptr, *w2 = nullptr;
  float *bqkv = nullptr, *bo = nullptr, *b1 = nullptr, *b2 = nullptr;
  float *ln1g = nullptr, *ln1b = nullptr, *ln2g = nullptr, *ln2b = nullptr;
  float *iqkv = nullptr, *io = nullptr, *i1 = nullptr, *i2 = nullptr;  // PG_PREC_F16F8: 1 / t_n per weight row
  float* conv_taps = nullptr;  // Tranception: [3][4][64][8]
  float *qlng = nullptr, *klng = nullptr;  // ESM C: q_ln / k_ln weights [d]
};

// Power-of-two scales the producers of A operands apply to their e4m3 planes (PG_PREC_F16F8; gemm_tc.cu header). e4m3 keeps
// ~2^-4 relative precision from 2^-6 to 448 (scaled), so the scale only places the window: values above 448/s saturate (their
// cross-term contribution degrades towards single-fp16 accuracy, nothing worse), values below 2^-9/s vanish from the cross term.
// Measured insensitive between 1 and 16 (scripts/precision_f8.py).
constexpr float S_LN = 4.f;     // LayerNorm output            -> QKV / fc1 GEMM     (|x| up to 112)
constexpr float S_ATT = 4.f;    // attention output            -> out_proj GEMM
constexpr float S_GELU = 2.f;   // GELU(fc1) (ESM)             -> fc2 GEMM           (up to 224)
constexpr float S_RELU2 = 1.f;  // relu(fc1)^2 (Tranception)   -> fc2 GEMM           (up to 448)
constexpr float S_SWIGLU = 2.f; // silu(g) * v (ESM C)         -> fc2 GEMM           (up to 224)

// Operand formats of a precision mode (common.h fmt 0 / 1 / 2), fixed at pg_create. Pitches and offsets in fp16 elements.
// Widths (DESIGN.md §3): residual rows d; GEMM-input rows of width d (LayerNorm outputs) dk = d rounded up to 64, zero-padded; q/k/v
// and attention outputs da = heads * S, head h in the slot [Sh, Sh + S), zeros after its head_dim columns. S = 64, except ProGen2's
// 80- and 96-wide heads: S = 128. All d for hd 64.
struct OpFmt {
  int np = 1;    // operand row pitch in units of the fp16 hi plane: 1 (fp16) or 2 (hi | lo, or hi | e4m3 planes)
  int nseg = 1;  // GEMM operand mode: 1 fp16, 3 fp16 hi/lo x3, 2 fp16 + e4m3 cross terms
  int afmt = 0;  // GEMM inputs (LayerNorm, attention and fc1 outputs): 2 under nseg 2, else 1 when np == 2
  int qfmt = 0;  // q/k/v rows, read by the attention kernels: fp16 hi [| lo]
  int pseg = 1;  // nseg of the operands that are fp16 hi [| lo] in every mode (attention, the MSA tied GEMMs): 3 when np == 2
  int slot = 64;                               // head slot width S
  int dk = 0, da = 0;                          // plane widths of GEMM-input rows of width d, and of attention rows (see above)
  int64_t ldd = 0, ldf = 0, ldat = 0, ldq = 0;  // pitches of dk-, ffn-, da- and 3da-wide rows
  int64_t lo_d = 0, lo_at = 0, lo_q = 0;        // offset of the planes after the hi plane in dk-, da- and 3da-wide rows (0: none)
};
OpFmt op_fmt(const pg_model_desc& D) {
  OpFmt o;
  o.np = D.precision == PG_PREC_F16 ? 1 : 2;
  o.nseg = D.precision == PG_PREC_F16 ? 1 : (D.precision == PG_PREC_F16F8 ? 2 : 3);  // F16D: the fp16 hi/lo x3 plumbing + delta GEMMs
  o.afmt = o.nseg == 2 ? 2 : o.np - 1;
  o.qfmt = o.np - 1;
  o.pseg = o.np == 2 ? 3 : 1;
  o.dk = (D.embed_dim + 63) / 64 * 64;
  o.slot = D.arch == PG_ARCH_PROGEN2 && D.embed_dim / D.heads > 64 ? 128 : 64;
  o.da = D.heads * o.slot;
  o.ldd = static_cast<int64_t>(o.dk) * o.np;
  o.ldf = static_cast<int64_t>(D.ffn_dim) * o.np;
  o.ldat = static_cast<int64_t>(o.da) * o.np;
  o.ldq = 3 * o.ldat;
  o.lo_d = o.np == 2 ? o.dk : 0;
  o.lo_at = o.np == 2 ? o.da : 0;
  o.lo_q = 3 * o.lo_at;
  return o;
}

// Slot maps: index i of a padded width -> source index, or -1 (zero); S = the slot width (64 or 128). SL_PAD: i < n (dk columns).
// SL_HEAD: dim c of head h at Sh + c (v rows, out_proj columns). SL_ROT (q/k rows): dims c < hd/2 at Sh + c, the others at
// Sh + S/2 + (c - hd/2), so ESM2's rotate-half partners (c, c + hd/2) sit on the pair (c', c' + S/2) the GEMM's rotary epilogue
// rotates; q.k is unchanged.
// ProGen2's fused qkv_proj [3d, d] (modeling_progen.py:157-168) is 8 shards of [q | v | k] rows, d/8 each; head h is sub-head
// h % (heads/8) of shard h / (heads/8). SL_PGQ / SL_PGK place its q / k rows with each rotate_every_two pair (2i, 2i+1) on the slot
// pair (Sh + i, Sh + S/2 + i), i < hd/2, which turns the interleaved rotation into the epilogue's rotate-half; SL_PGV places v dim c
// at Sh + c. For these maps n = d.
enum SlotMap { SL_PAD = 0, SL_HEAD, SL_ROT, SL_PGQ, SL_PGK, SL_PGV };
__device__ __forceinline__ int slot_src(int i, int map, int n, int hd, int S) {
  if (map == SL_PAD) return i < n ? i : -1;
  const int h = i / S, c = i % S, half = hd >> 1, hs = S >> 1;
  if (map == SL_HEAD) return c < hd ? h * hd + c : -1;
  if (map == SL_ROT) {
    if (c < half) return h * hd + c;
    if (c >= hs && c < hs + half) return h * hd + half + (c - hs);
    return -1;
  }
  const int per = n / hd / 8;  // heads per shard
  const int base = (h / per) * (3 * n / 8) + (h % per) * hd;
  if (map == SL_PGV) return c < hd ? base + n / 8 + c : -1;
  const int part = map == SL_PGQ ? 0 : 2 * n / 8;
  if (c < half) return base + part + 2 * c;
  if (c >= hs && c < hs + half) return base + part + 2 * (c - hs) + 1;
  return -1;
}
// dst [N, K] = src [*, k_src] (row-major) with its rows placed by map rmap (over rn source rows) and its columns by cmap (over kn
// source columns), zeros elsewhere.
__global__ void expand_slots_kernel(const float* __restrict__ src, int rn, int k_src, float* __restrict__ dst, int N, int K, int rmap,
                                    int cmap, int hd, int S, int kn) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(N) * K) return;
  const int r = slot_src(static_cast<int>(i / K), rmap, rn, hd, S), c = slot_src(static_cast<int>(i % K), cmap, kn, hd, S);
  dst[i] = (r >= 0 && c >= 0) ? src[static_cast<long long>(r) * k_src + c] : 0.f;
}

// ESM C fc1 [2f, K] = [gate (f rows) ; up (f rows)] -> rows interleaved in blocks of 8 (rows 16i..16i+7 = gate rows 8i..8i+7, rows
// 16i+8..16i+15 = up rows 8i..8i+7): the SwiGLU epilogue (gemm_tc.cu, epi 5) then finds each gate column and its up column in one
// thread's fragment. A row permutation, so one e4m3 scale per matrix still covers it.
__global__ void interleave_gate_up_kernel(const float* __restrict__ src, int f, int K, float* __restrict__ dst) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= 2LL * f * K) return;
  const int r = static_cast<int>(i / K), k = static_cast<int>(i % K);
  const int blk = r >> 4, c = r & 15;
  const int sr = c < 8 ? 8 * blk + c : f + 8 * blk + (c - 8);
  dst[i] = src[static_cast<long long>(sr) * K + k];
}

}  // namespace
}  // namespace pg

struct pg_handle_s {
  pg_model_desc desc{};
  pg::OpFmt op;
  bool loaded = false;
  std::string err;
  std::vector<void*> allocs;
  std::vector<pg::Layer> layers;
  float *embed = nullptr, *pos = nullptr, *lnbg = nullptr, *lnbb = nullptr, *lnag = nullptr, *lnab = nullptr;
  float *hdw = nullptr, *hdb = nullptr, *hlng = nullptr, *hlnb = nullptr, *hbias = nullptr;
  float* outw = nullptr;  // untied output matrix [vocab, d] (ESM C sequence_head.3); null = the tied embedding
  int head_vocab = 0, label_off = 0;  // autoregressive head: columns (ProGen2: 25, vocabulary rows 5..29) and token id of column 0
  // ProtGPT2's fused LM head (K16): the tied wte packed as a [vocab, dk] GEMM operand in fp16 hi [| lo] (never e4m3), and per pass the
  // (max, sum exp) partials [max_rows, ceil(vocab / 128)] and target logits [max_rows] of GEMM epi 7
  __half* lmw = nullptr;
  float2* lm_part = nullptr;
  float* lm_tgt = nullptr;
  float *rot_cos = nullptr, *rot_sin = nullptr;
  int rot_rows = 0;
  // workspace
  long long max_rows = 0;
  int head_cap = 0;
  float* x = nullptr;
  __half *abuf = nullptr, *qkv = nullptr, *fbuf = nullptr;
  float *hs_a = nullptr, *hs_b = nullptr;
  int32_t* row_sel = nullptr;  // [head_cap] token index within the window to emit
  // Tranception
  __half* qkv2 = nullptr;
  float *tok_logp = nullptr, *slopes = nullptr;
  // exact wild-type-prefix reuse (pg_ar_prefix_begin / pg_ar_loglik_prefix): per layer, the wild type's raw q/k/v rows (conv
  // look-back) and conv'd q/k/v rows (keys / values of the shared prefix), [layers][prefix_T][3d*np] fp16 each
  unsigned int* pack_scratch = nullptr;  // one word per packed matrix (absmax of the matrix), [layers * 6]
  int pack_used = 0;
  __half *raw_cache = nullptr, *kv_cache = nullptr;
  int prefix_T = 0;        // rows recorded by the last pg_ar_prefix_begin (0 = none)
  int prefix_cap = 0;      // rows the caches can hold
  // MSA Transformer: column-attention blocks (ln1*, wqkv, wo of a Layer), row-position table, tied-attention workspace
  std::vector<pg::Layer> col_layers;
  float* row_pos = nullptr;         // [1024, d] or null
  void* tied_ws = nullptr;          // one allocation, regrown on demand (not in `allocs`)
  size_t tied_bytes = 0;
  // compact buffers for the pruned last layer (one row per sequence)
  float* xc = nullptr;
  __half *cabuf = nullptr, *cfbuf = nullptr;
  // delta-operand mode (PG_PREC_F16D): per-layer base rows of the unmasked window (one allocation, regrown on demand, not in
  // `allocs`) and the compact exact q/k/v rows of the masked positions
  bool delta = false;
  float* base = nullptr;
  size_t base_alloc_bytes = 0;  // allocated for `base`
  int base_T = 0;
  __half* cq = nullptr;
};

namespace pg {
namespace {

bool is_ar(int arch) {
  return arch == PG_ARCH_TRANCEPTION || arch == PG_ARCH_RITA || arch == PG_ARCH_PROGEN2 || arch == PG_ARCH_PROTGPT2;
}

int fail(pg_handle h, int code, const std::string& msg) {
  if (h) h->err = msg;
  return set_error(code, msg);
}

template <typename T>
int dev_alloc(pg_handle h, T** p, size_t count) {
  void* q = nullptr;
  cudaError_t e = cudaMalloc(&q, count * sizeof(T) + 256);
  if (e != cudaSuccess) return fail(h, PG_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e));
  h->allocs.push_back(q);
  *p = static_cast<T*>(q);
  return PG_OK;
}

__global__ void row_select_kernel(const int32_t* positions, const int32_t* win_start, const int32_t* out_row, int p_offset, int n,
                                  int32_t* sel) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int gp = p_offset + i;
  const int tok = out_row ? out_row[gp] : positions[gp];
  sel[i] = tok - (win_start ? win_start[gp] : 0);
}

// ---- block helpers: every operand they write or read is in the handle's formats (h->op) ------------------------------------

// ESM embedding of the copies [p_offset, p_offset + P) of a window of T tokens into h->x (force_mask_scale: see EmbedLaunch).
int embed(pg_handle h, const int32_t* tokens, int n_tokens, const int32_t* positions, const int32_t* win_start, int p_offset, int P,
          int T, cudaStream_t s, int force_mask_scale = 0) {
  const pg_model_desc& D = h->desc;
  EmbedLaunch e{};
  e.tokens = tokens; e.n_tokens = n_tokens; e.positions = positions; e.win_start = win_start;
  e.P = P; e.T = T; e.d = D.embed_dim; e.embed = h->embed; e.pos_table = h->pos;  // null for ESM2 (rotary)
  e.lnb_gamma = D.emb_ln_before ? h->lnbg : nullptr; e.lnb_beta = D.emb_ln_before ? h->lnbb : nullptr;
  e.token_dropout = D.token_dropout; e.mask_idx = 32; e.p_offset = p_offset; e.x = h->x; e.force_mask_scale = force_mask_scale;
  ProfScope ps(CAT_EMBED, s);
  return launch_embed(e, s);
}

// LayerNorm of M fp32 rows x (pitch d) into operand rows `out` in the GEMM-input format (perm_R / perm_C: launch_layernorm_f16).
int ln(pg_handle h, const float* x, const float* g, const float* b, int M, __half* out, cudaStream_t s, int perm_R = 0, int perm_C = 0) {
  const int d = h->desc.embed_dim;
  ProfScope ps(CAT_LN, s);
  return launch_layernorm_f16(x, d, g, b, M, d, out, h->op.ldd, h->op.lo_d, s, h->op.afmt, S_LN, perm_R, perm_C, nullptr, 0, h->op.dk);
}

// The projections of a Layer, each profiled in its own GEMM category.
enum Proj { QKV = CAT_GEMM_QKV, OUT = CAT_GEMM_OUT, FC1 = CAT_GEMM_FC1, FC2 = CAT_GEMM_FC2 };
// Projection p of layer L on M operand rows `a` in the GEMM-input format (a_scale: the e4m3 scale their producer applied).
GemmLaunch proj_gemm(pg_handle h, const Layer& L, Proj p, const __half* a, float a_scale, int M) {
  const int d = h->desc.embed_dim, f = h->desc.ffn_dim, dk = h->op.dk, da = h->op.da;
  GemmLaunch g{};
  switch (p) {
    case QKV: g.w = L.wqkv; g.w_inv = L.iqkv; g.bias = L.bqkv; g.N = 3 * da; g.K = dk; break;
    case OUT: g.w = L.wo; g.w_inv = L.io; g.bias = L.bo; g.N = d; g.K = da; break;
    case FC1: g.w = L.w1; g.w_inv = L.i1; g.bias = L.b1; g.N = h->desc.arch == PG_ARCH_ESMC ? 2 * f : f; g.K = dk; break;  // ESM C: gate|up
    case FC2: g.w = L.w2; g.w_inv = L.i2; g.bias = L.b2; g.N = d; g.K = f; break;
  }
  g.a = a; g.lda = static_cast<int64_t>(g.K) * h->op.np; g.ldw = g.lda; g.M = M; g.nseg = h->op.nseg;
  g.a_scale = a_scale; g.w_uniform = 1;  // pg_load_weights: one e4m3 scale per (fused) weight matrix
  return g;
}
// ... written as operand rows to `out` through epilogue `epi`: q/k/v in the q/k/v format (epi 0, or 3: rotary embedding over windows of
// rot_T rows, row t of a window at position rot_start + t), fc1 in the GEMM-input format (epi: the MLP's activation, out_scale: the e4m3
// scale of its output; SwiGLU, epi 5, writes half as many columns as the GEMM has).
int lin(pg_handle h, const Layer& L, Proj p, const __half* a, float a_scale, int M, __half* out, cudaStream_t s, int epi = 0,
        float out_scale = 0.f, int rot_T = 0, int rot_start = 0) {
  GemmLaunch g = proj_gemm(h, L, p, a, a_scale, M);
  const int n_out = epi == 5 ? g.N / 2 : g.N;
  g.epi = epi;
  g.out = out; g.ldo = static_cast<int64_t>(n_out) * h->op.np; g.out_fmt = p == QKV ? h->op.qfmt : h->op.afmt;
  g.out_lo_off = g.out_fmt ? n_out : 0; g.out_scale = out_scale;
  if (epi == 3) {  // q and k slots; tables [T, S/2]
    const int hs = h->op.slot / 2;
    g.rot_cos = h->rot_cos + static_cast<int64_t>(rot_start) * hs; g.rot_sin = h->rot_sin + static_cast<int64_t>(rot_start) * hs;
    g.rot_T = rot_T; g.rot_dim = h->op.da; g.rot_half = hs;
  }
  ProfScope ps(p, s);
  return launch_gemm(g, s);
}
// ... added into the fp32 rows `resid` (pitch N): out_proj and fc2 into the residual stream, and the base rows of the delta mode.
int lin_add(pg_handle h, const Layer& L, Proj p, const __half* a, float a_scale, int M, float* resid, cudaStream_t s) {
  GemmLaunch g = proj_gemm(h, L, p, a, a_scale, M);
  g.epi = 2; g.resid = resid; g.ldr = g.N;
  ProfScope ps(p, s);
  return launch_gemm(g, s);
}

// MLP block on M fp32 residual rows x: x += fc2(act(fc1(LN2(x)))), through operand rows `ab` (LayerNorm output) and `fb` (hidden
// layer). act: fc1's activation epilogue (1 GELU, 4 relu^2, 5 SwiGLU, 6 tanh-GELU); act_scale: the e4m3 scale of its output (S_GELU,
// S_RELU2, S_SWIGLU).
int mlp(pg_handle h, const Layer& L, float* x, int M, __half* ab, __half* fb, int act, float act_scale, cudaStream_t s) {
  int rc = ln(h, x, L.ln2g, L.ln2b, M, ab, s);
  if (!rc) rc = lin(h, L, FC1, ab, S_LN, M, fb, s, act, act_scale);
  if (!rc) rc = lin_add(h, L, FC2, fb, act_scale, M, x, s);
  return rc;
}

// The activation of the ESM-family MLPs (fc1 epilogue) and the e4m3 scale of its output: erf-GELU, or SwiGLU for ESM C.
struct Act { int epi; float scale; };
Act esm_act(pg_handle h) { return h->desc.arch == PG_ARCH_ESMC ? Act{5, S_SWIGLU} : Act{1, S_GELU}; }

// ESM C after the QKV projection of M rows in h->qkv (windows of T rows): q/k LayerNorm + rotary + q scaling, in place.
int qk_norm(pg_handle h, const Layer& L, int M, int T, cudaStream_t s) {
  ProfScope ps(CAT_LN, s);
  return launch_qk_ln_rotary(h->qkv, h->op.ldq, h->op.lo_q, M, h->desc.heads, L.qlng, L.klng, h->rot_cos, h->rot_sin, T, s);
}

// Attention over B sequences of T rows, q/k/v rows `qkv` -> operand rows `out` in the GEMM-input format; bidirectional and without
// bias. The caller sets the causal / ALiBi / prefix / column (perm_C) / delta-operand fields.
AttnLaunch attn_args(pg_handle h, const __half* qkv, __half* out, int B, int T) {
  const OpFmt& o = h->op;
  AttnLaunch a{};
  a.qkv = qkv; a.ld = o.ldq; a.lo_off = o.lo_q;
  a.out = out; a.ldo = o.ldat; a.out_lo_off = o.lo_at; a.out_fmt = o.afmt; a.out_scale = S_ATT;
  a.B = B; a.T = T; a.heads = h->desc.heads; a.nseg = o.pseg; a.causal = 0; a.alibi_slopes = nullptr; a.head_dim = o.slot;
  return a;
}

// Exact pruning of the final ESM layer, after its q/k/v projection into h->qkv: one query row per sequence (emit_rows[b] of sequence b)
// from here on; out_proj and the MLP run on the Bc compact residual rows h->xc. `gather`: fill h->xc from h->x first (otherwise the
// caller already holds those rows there).
int last_layer(pg_handle h, const Layer& L, const int32_t* emit_rows, int Bc, int T, bool gather, cudaStream_t s) {
  const OpFmt& o = h->op;
  int rc;
  { ProfScope ps(CAT_ATTN, s, gather ? 2 : 1);
    rc = launch_attn_single_query(h->qkv, o.ldq, o.lo_q, emit_rows, Bc, T, h->desc.heads, h->cabuf, o.ldat, o.lo_at, s, o.afmt, S_ATT);
    if (!rc && gather) rc = launch_gather_rows(h->x, emit_rows, Bc, T, h->desc.embed_dim, h->xc, s); }
  if (!rc) rc = lin_add(h, L, OUT, h->cabuf, S_ATT, Bc, h->xc, s);
  if (!rc) rc = mlp(h, L, h->xc, Bc, h->cabuf, h->cfbuf, esm_act(h).epi, esm_act(h).scale, s);
  return rc;
}

// `emit_rows` (device, [Bc]) = the one row per sequence the caller will read, or null when every row is needed. When given,
// the last layer runs its attention-output / out_proj / LayerNorm / MLP for those rows only and leaves them in h->xc [Bc, d].
int forward_rows(pg_handle h, const int32_t* tokens, int n_tokens, const int32_t* positions, const int32_t* win_start,
                 int p_offset, int Bc, int T, cudaStream_t s, const int32_t* emit_rows = nullptr) {
  const pg_model_desc& D = h->desc;
  const int rows = Bc * T;
  const bool rotary = (D.arch == PG_ARCH_ESM2);
  int rc = embed(h, tokens, n_tokens, positions, win_start, p_offset, Bc, T, s);
  if (rc) return rc;
  for (int l = 0; l < D.layers; ++l) {
    const Layer& L = h->layers[l];
    if ((rc = ln(h, h->x, L.ln1g, L.ln1b, rows, h->abuf, s))) return rc;
    if ((rc = lin(h, L, QKV, h->abuf, S_LN, rows, h->qkv, s, rotary ? 3 : 0, 0.f, T))) return rc;
    if (D.arch == PG_ARCH_ESMC && (rc = qk_norm(h, L, rows, T, s))) return rc;  // every row: the pruned layer reads all keys
    if (emit_rows && l == D.layers - 1) return last_layer(h, L, emit_rows, Bc, T, true, s);
    const AttnLaunch a = attn_args(h, h->qkv, h->abuf, Bc, T);
    { ProfScope ps(CAT_ATTN, s); rc = launch_attention_wgmma(a, s); }
    if (rc) return rc;
    if ((rc = lin_add(h, L, OUT, h->abuf, S_ATT, rows, h->x, s))) return rc;
    if ((rc = mlp(h, L, h->x, rows, h->abuf, h->fbuf, esm_act(h).epi, esm_act(h).scale, s))) return rc;
  }
  return PG_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------
// Delta-operand mode (PG_PREC_F16D) of the masked-marginal pass. The P masked copies of a window differ from the unmasked window
// by a perturbation: every GEMM input is a = a0[t] + D with the base row a0[t] shared by all copies. The linear layers then are
//   W a + b = (W a0[t] + b)  +  W D
// with the first term computed ONCE per window at the fp16 hi/lo x3 precision (forward_base: T rows) and the second per copy in a
// SINGLE fp16 pass on D = rn16(a - a0[t]) — the products' error scales with |D|, which is 6-10 % of |a| on the rows that do not
// hold the mask (scripts/precision_delta.py, true ESM-1v 650M size: max score error 5.7e-4 at L = 96 against 1.5e-2 for a plain
// single pass). The row that holds the mask (|D| ~ |a|) takes the compact exact path: P rows per layer through the x3 GEMMs, like
// the pruned last layer. One tensor-pipe unit per algorithmic FLOP instead of two (fp16 + e4m3 cross terms) or three.
//   base rows per layer, T rows each. Inputs of the four GEMMs, as ONE fp16 plane (any fixed reference works as long as the matching
//   output rows were computed from exactly these values): a0 = rn16(LN1 output), o0 = rn16(attention output), b0 = rn16(LN2 output),
//   f0 = rn16(GELU output). Their images, fp32: bqkv = Wqkv a0 + b, bout = Wo o0 + b, bfc1 = W1 b0 + b (pre-GELU), bfc2 = W2 f0 + b.
struct BaseRows { float *bqkv, *bout, *bfc1, *bfc2; __half *a0, *o0, *b0, *f0; };
size_t base_bytes(const pg_model_desc& D, int T) {
  const size_t d = D.embed_dim, f = D.ffn_dim;
  return static_cast<size_t>(D.layers) * T * (4 * (5 * d + f) + 2 * (3 * d + f));
}
BaseRows base_rows(pg_handle h, int l) {
  const long long T = h->base_T, d = h->desc.embed_dim, f = h->desc.ffn_dim;
  float* p = h->base + static_cast<long long>(l) * T * (5 * d + f);
  __half* q = reinterpret_cast<__half*>(h->base + static_cast<long long>(h->desc.layers) * T * (5 * d + f)) +
              static_cast<long long>(l) * T * (3 * d + f);
  BaseRows b;
  b.bqkv = p; b.bout = p + T * 3 * d; b.bfc1 = p + T * 4 * d; b.bfc2 = p + T * (4 * d + f);
  b.a0 = q; b.o0 = q + T * d; b.b0 = q + T * 2 * d; b.f0 = q + T * 3 * d;
  return b;
}

// The unmasked window (with the token-dropout scale of a copy that holds one mask) through the model at x3 precision, recording
// the base rows of every layer. Uses the pass workspace (T rows of it) before the passes start.
int forward_base(pg_handle h, const int32_t* tokens, int n_tokens, int T, cudaStream_t s) {
  const pg_model_desc& D = h->desc;
  const OpFmt& o = h->op;
  const int d = D.embed_dim, f = D.ffn_dim;
  const size_t need = base_bytes(D, T);
  if (need > h->base_alloc_bytes) {
    if (h->base) cudaFree(h->base);
    h->base = nullptr; h->base_alloc_bytes = 0;
    cudaError_t e = cudaMalloc(&h->base, need);
    if (e != cudaSuccess) return set_error(PG_ERR_CUDA, std::string("forward_base: cudaMalloc: ") + cudaGetErrorString(e));
    h->base_alloc_bytes = need;
  }
  h->base_T = T;
  PG_CUDA_OK(cudaMemsetAsync(h->base, 0, need, s));  // the tap GEMMs reduce-add into zero
  int rc = embed(h, tokens, n_tokens, nullptr, nullptr, 0, 1, T, s, 1);
  if (rc) return rc;
  // The base row of a GEMM input is its fp16 hi plane: zero the lo plane of the T rows (the tap GEMM, lin_add into the base rows,
  // then multiplies exactly that plane by the full hi/lo weights) and keep a copy of the hi plane.
  auto fix_base = [&](__half* buf, int64_t ld, int n, __half* dst) -> int {
    ProfScope ps(CAT_OTHER, s);
    PG_CUDA_OK(cudaMemset2DAsync(buf + n, ld * 2, 0, static_cast<size_t>(n) * 2, T, s));
    PG_CUDA_OK(cudaMemcpy2DAsync(dst, static_cast<size_t>(n) * 2, buf, ld * 2, static_cast<size_t>(n) * 2, T, cudaMemcpyDeviceToDevice, s));
    return PG_OK;
  };
  for (int l = 0; l < D.layers; ++l) {
    const Layer& L = h->layers[l];
    const BaseRows B = base_rows(h, l);
    if ((rc = ln(h, h->x, L.ln1g, L.ln1b, T, h->abuf, s))) return rc;
    if ((rc = lin(h, L, QKV, h->abuf, S_LN, T, h->qkv, s))) return rc;
    if ((rc = fix_base(h->abuf, o.ldd, d, B.a0))) return rc;
    if ((rc = lin_add(h, L, QKV, h->abuf, S_LN, T, B.bqkv, s))) return rc;
    const AttnLaunch a = attn_args(h, h->qkv, h->abuf, 1, T);
    { ProfScope ps(CAT_ATTN, s); rc = launch_attention_wgmma(a, s); }
    if (rc) return rc;
    if ((rc = lin_add(h, L, OUT, h->abuf, S_ATT, T, h->x, s))) return rc;
    if ((rc = fix_base(h->abuf, o.ldd, d, B.o0))) return rc;
    if ((rc = lin_add(h, L, OUT, h->abuf, S_ATT, T, B.bout, s))) return rc;
    if ((rc = ln(h, h->x, L.ln2g, L.ln2b, T, h->abuf, s))) return rc;
    if ((rc = lin(h, L, FC1, h->abuf, S_LN, T, h->fbuf, s, 1, S_GELU))) return rc;
    if ((rc = fix_base(h->abuf, o.ldd, d, B.b0))) return rc;
    if ((rc = lin_add(h, L, FC1, h->abuf, S_LN, T, B.bfc1, s))) return rc;
    if ((rc = lin_add(h, L, FC2, h->fbuf, S_GELU, T, h->x, s))) return rc;
    if ((rc = fix_base(h->fbuf, o.ldf, f, B.f0))) return rc;
    if ((rc = lin_add(h, L, FC2, h->fbuf, S_GELU, T, B.bfc2, s))) return rc;
  }
  return PG_OK;
}

// One single-pass GEMM on difference rows: C = epi(base_pre[t] + A_delta * W_hi^T) [- base_post[t]].
int run_lin_delta(pg_handle h, int cat, const __half* a, int64_t lda, const __half* w, int M, int N, int K, int epi, const float* base_pre,
                  const __half* base_post, int T, const int32_t* mask_pos, __half* out, int64_t ldo, int out_fmt, float* resid,
                  cudaStream_t s) {
  GemmLaunch g{};
  g.a = a; g.lda = lda; g.w = w; g.ldw = static_cast<int64_t>(K) * h->op.np; g.bias = nullptr;  // W: the hi plane of the hi/lo rows
  g.M = M; g.N = N; g.K = K; g.nseg = 1; g.epi = epi;
  g.base_pre = base_pre; g.base_post = base_post; g.base_T = T; g.mask_pos = mask_pos;
  if (epi == 2) {
    g.resid = resid; g.ldr = N;
  } else {
    g.out = out; g.ldo = ldo; g.out_fmt = out_fmt; g.out_lo_off = out_fmt ? N : 0;
  }
  ProfScope ps(cat, s);
  return launch_gemm(g, s);
}

// forward_rows in delta-operand mode (single window: every copy sees tokens [0, T); emit_rows[b] = the masked token of copy b).
int forward_rows_delta(pg_handle h, const int32_t* tokens, int n_tokens, const int32_t* positions, const int32_t* win_start,
                       int p_offset, int Bc, int T, cudaStream_t s, const int32_t* emit_rows) {
  const pg_model_desc& D = h->desc;
  const OpFmt& o = h->op;
  const int d = D.embed_dim, f = D.ffn_dim;
  const int rows = Bc * T;
  int rc = embed(h, tokens, n_tokens, positions, win_start, p_offset, Bc, T, s);
  if (rc) return rc;
  { ProfScope ps(CAT_OTHER, s); rc = launch_gather_rows(h->x, emit_rows, Bc, T, d, h->xc, s); }  // xc = the masked rows, kept exact
  if (rc) return rc;
  // The masked rows (h->xc, through h->cabuf / h->cfbuf) take the compact exact path of the block helpers: in this mode their
  // operand formats are the fp16 hi / lo pairs (fmt 1) and the e4m3 scales are unread.
  auto ln_delta = [&](const float* g, const float* b, const __half* base) {   // all rows: LN(x) - base[t] -> abuf (fp16, pitch ldd)
    ProfScope ps(CAT_LN, s);
    return launch_layernorm_f16(h->x, d, g, b, rows, d, h->abuf, o.ldd, 0, s, 0, 0.f, 0, 0, base, T);
  };
  auto put_back = [&]() {                                                    // x[masked rows] <- xc
    ProfScope ps(CAT_OTHER, s);
    return launch_scatter_rows(h->xc, static_cast<int64_t>(d) * 4, h->x, static_cast<int64_t>(d) * 4, emit_rows, Bc, T, d * 4, s);
  };
  for (int l = 0; l < D.layers; ++l) {
    const Layer& L = h->layers[l];
    const BaseRows B = base_rows(h, l);
    // q/k/v: all rows from the difference, the masked rows exactly
    if ((rc = ln_delta(L.ln1g, L.ln1b, B.a0))) return rc;
    if ((rc = run_lin_delta(h, CAT_GEMM_QKV, h->abuf, o.ldd, L.wqkv, rows, 3 * d, d, 0, B.bqkv, nullptr, T, nullptr, h->qkv, o.ldq, 1, nullptr, s)))
      return rc;
    if ((rc = ln(h, h->xc, L.ln1g, L.ln1b, Bc, h->cabuf, s))) return rc;
    if ((rc = lin(h, L, QKV, h->cabuf, S_LN, Bc, h->cq, s))) return rc;
    { ProfScope ps(CAT_OTHER, s);
      rc = launch_scatter_rows(h->cq, o.ldq * 2, h->qkv, o.ldq * 2, emit_rows, Bc, T, static_cast<int>(o.ldq * 2), s); }
    if (rc) return rc;
    if (l == D.layers - 1) return last_layer(h, L, emit_rows, Bc, T, false, s);
    // attention on full-value q/k/v; output as difference rows (one fp16 plane), the masked rows' exact output to cabuf
    AttnLaunch a = attn_args(h, h->qkv, h->abuf, Bc, T);
    a.out_lo_off = 0; a.out_fmt = 0;
    a.base_o = B.o0; a.mask_pos = emit_rows; a.cout = h->cabuf; a.ldc = o.ldd; a.c_lo_off = d;
    { ProfScope ps(CAT_ATTN, s); rc = launch_attention_wgmma(a, s); }
    if (rc) return rc;
    if ((rc = run_lin_delta(h, CAT_GEMM_OUT, h->abuf, o.ldd, L.wo, rows, d, d, 2, B.bout, nullptr, T, emit_rows, nullptr, 0, 0, h->x, s))) return rc;
    if ((rc = lin_add(h, L, OUT, h->cabuf, S_ATT, Bc, h->xc, s))) return rc;
    if ((rc = put_back())) return rc;
    // MLP
    if ((rc = ln_delta(L.ln2g, L.ln2b, B.b0))) return rc;
    if ((rc = run_lin_delta(h, CAT_GEMM_FC1, h->abuf, o.ldd, L.w1, rows, f, d, 1, B.bfc1, B.f0, T, nullptr, h->fbuf, o.ldf, 0, nullptr, s))) return rc;
    if ((rc = ln(h, h->xc, L.ln2g, L.ln2b, Bc, h->cabuf, s))) return rc;
    if ((rc = lin(h, L, FC1, h->cabuf, S_LN, Bc, h->cfbuf, s, 1, S_GELU))) return rc;
    if ((rc = run_lin_delta(h, CAT_GEMM_FC2, h->fbuf, o.ldf, L.w2, rows, d, f, 2, B.bfc2, nullptr, T, emit_rows, nullptr, 0, 0, h->x, s))) return rc;
    if ((rc = lin_add(h, L, FC2, h->cfbuf, S_GELU, Bc, h->xc, s))) return rc;
    if ((rc = put_back())) return rc;
  }
  return PG_OK;
}

// Causal decoder stack over B right-padded sequences of T tokens: no padding mask is needed because pads sit to the right of every real
// token and attention is causal.
//   Tranception (model_pytorch.py:526-612): grouped ALiBi, depthwise-conv q/k/v, relu^2 MLP.
//   RITA (rita_modeling.py:129-210, 244-252): rotary q/k (GEMM epilogue 3, q pre-scaled by 1/8 at load), no attention bias, tanh-GELU
//   MLP (epilogue 6).
//   ProGen2 (modeling_progen.py:244-282): RITA's rotary attention and tanh-GELU MLP as a parallel residual, x + attn(h) + mlp(h) with
//   h = ln_1(x): fc_in runs on ln_1's output before attention overwrites it, then out_proj and fc_out add into x in that order (the
//   reference adds (attn + mlp) + x: an fp32 reassociation).
//   ProtGPT2 (GPT-2, transformers modeling_gpt2.py GPT2Model / GPT2Block): learned absolute positions added to the token embedding,
//   c_attn with bias (q pre-scaled by 1/8 at load), causal attention without bias, c_proj, and RITA's tanh-GELU MLP.
// mode 0: plain forward. mode 1 (B == 1): also record every layer's keys / values (Tranception: the raw q/k/v rows for the conv
// look-back and the conv'd rows; the others: the (rotated) rows) into the prefix caches.
// mode 2: the B sequences are rows [start, start + T) of sequences whose first `start` rows (multiple of 128) equal the recorded
// wild type's: the keys / values of the prefix (and Tranception's conv look-back) come from the caches, and the rotary or learned
// positions are the absolute positions start + t.
int forward_ar(pg_handle h, const int32_t* ids, int B, int T, cudaStream_t s, int mode = 0, int start = 0) {
  const pg_model_desc& D = h->desc;
  const bool progen2 = D.arch == PG_ARCH_PROGEN2;
  const bool tranception = D.arch == PG_ARCH_TRANCEPTION;  // conv'd q/k/v, grouped ALiBi, relu^2; the others: tanh-GELU, no attention bias
  const bool rotary = D.arch == PG_ARCH_RITA || progen2;
  const int64_t ldq = h->op.ldq;
  const int rows = B * T;
  int rc;
  { ProfScope ps(CAT_EMBED, s);
    rc = launch_gather_embed(ids, h->embed, rows, D.embed_dim, D.vocab, h->x, s, h->pos, T, mode == 2 ? start : 0); }  // pos: ProtGPT2's wpe
  if (rc) return rc;
  for (int l = 0; l < D.layers; ++l) {
    const Layer& L = h->layers[l];
    if ((rc = ln(h, h->x, L.ln1g, L.ln1b, rows, h->abuf, s))) return rc;
    if ((rc = lin(h, L, QKV, h->abuf, S_LN, rows, h->qkv, s, rotary ? 3 : 0, 0.f, T, mode == 2 ? start : 0))) return rc;
    if (progen2 && (rc = lin(h, L, FC1, h->abuf, S_LN, rows, h->fbuf, s, 6, S_GELU))) return rc;
    const size_t layer_off = static_cast<size_t>(l) * h->prefix_cap * ldq;
    const __half* kv = h->qkv;  // the q/k/v rows attention reads
    if (tranception) {
      if (mode == 1)
        PG_CUDA_OK(cudaMemcpyAsync(h->raw_cache + layer_off, h->qkv, static_cast<size_t>(T) * ldq * sizeof(__half), cudaMemcpyDeviceToDevice, s));
      { ProfScope ps(CAT_OTHER, s);
        rc = launch_qkv_conv(h->qkv, h->qkv2, ldq, h->op.lo_q, B, T, D.heads, L.conv_taps, 0.125f, s,
                             mode == 2 ? h->raw_cache + layer_off + static_cast<size_t>(start - 6) * ldq : nullptr); }
      if (rc) return rc;
      kv = h->qkv2;
    }
    if (mode == 1)
      PG_CUDA_OK(cudaMemcpyAsync(h->kv_cache + layer_off, kv, static_cast<size_t>(T) * ldq * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    AttnLaunch a = attn_args(h, kv, h->abuf, B, T);
    a.causal = 1; a.alibi_slopes = tranception ? h->slopes : nullptr;
    if (mode == 2) { a.prefix = h->kv_cache + layer_off; a.prefix_len = start; }
    { ProfScope ps(CAT_ATTN, s); rc = launch_attention_wgmma(a, s); }
    if (rc) return rc;
    if ((rc = lin_add(h, L, OUT, h->abuf, S_ATT, rows, h->x, s))) return rc;
    if (progen2) rc = lin_add(h, L, FC2, h->fbuf, S_GELU, rows, h->x, s);
    else rc = mlp(h, L, h->x, rows, h->abuf, h->fbuf, tranception ? 4 : 6, tranception ? S_RELU2 : S_GELU, s);
    if (rc) return rc;
  }
  return PG_OK;
}

// MSA Transformer stack (msa_transformer.py:150-222) over Bc masked copies of an [R, Cw] alignment window; token rows are (b, r, c)
// with c fastest. Per layer (AxialTransformerLayer, modules.py:205-235): tied row attention, column attention, FFN, each a pre-LN
// residual block. The tied attention's two products run as grouped GEMMs on regrouped operands (msa_transformer.cu), always with fp16
// hi/lo pairs when the handle has them (x3: they are < 10 % of the FLOPs); the column attention is the wgmma attention kernel over
// the B*Cw columns as sequences of R rows, fed by a LayerNorm that writes its rows in (b, c, r) order.
// `sel` (device, [Bc]): the window column of each alignment whose (row 0) output the caller reads. The last layer then runs exactly
// what that output depends on — the full q/k/v projection of its row attention, one row of each tied attention map, and the rest on
// the Bc*R rows of column sel[b] (column attention) and on Bc rows (FFN); the result is left in h->xc [Bc, d].
int forward_msa(pg_handle h, const int32_t* tokens, int R, int Cfull, const int32_t* positions, const int32_t* win_start, int p_offset,
                int Bc, int Cw, cudaStream_t s, const int32_t* sel) {
  const pg_model_desc& D = h->desc;
  const OpFmt& o = h->op;
  const int d = D.embed_dim, np = o.np, H = D.heads;
  const int rows = Bc * R * Cw;
  // tied-attention workspace: Q' / K' [G*Cp, Nt*np] (Q' doubles as the context buffer), V' [G*Nt, Kp*np], S fp32 [G*Cp, Kp], P [G*Cp, Kp*np]
  const int G = Bc * H, Cp = (Cw + 127) / 128 * 128, Kp = (Cw + 63) / 64 * 64, Nt = R * 64;
  const int64_t ldt = static_cast<int64_t>(Nt) * np, ldv = static_cast<int64_t>(Kp) * np, lds = Kp, ldp = static_cast<int64_t>(Kp) * np;
  auto al = [](size_t b) { return (b + 255) / 256 * 256; };
  const size_t b_q = al(static_cast<size_t>(G) * Cp * ldt * 2), b_v = al(static_cast<size_t>(G) * Nt * ldv * 2);
  const size_t b_s = al(static_cast<size_t>(G) * Cp * lds * 4), b_p = al(static_cast<size_t>(G) * Cp * ldp * 2);
  const size_t need = 2 * b_q + b_v + b_s + b_p;
  if (need > h->tied_bytes) {
    if (h->tied_ws) cudaFree(h->tied_ws);
    h->tied_ws = nullptr; h->tied_bytes = 0;
    PG_CUDA_OK(cudaMalloc(&h->tied_ws, need));
    h->tied_bytes = need;
    PG_CUDA_OK(cudaMemsetAsync(h->tied_ws, 0, need, s));
  }
  uint8_t* ws = static_cast<uint8_t*>(h->tied_ws);
  __half* tq = reinterpret_cast<__half*>(ws);
  __half* tk = reinterpret_cast<__half*>(ws + b_q);
  __half* tv = reinterpret_cast<__half*>(ws + 2 * b_q);
  float* S = reinterpret_cast<float*>(ws + 2 * b_q + b_v);
  __half* P = reinterpret_cast<__half*>(ws + 2 * b_q + b_v + b_s);
  int rc;
  MsaEmbedLaunch e{};
  e.tokens = tokens; e.R = R; e.Cfull = Cfull; e.positions = positions; e.win_start = win_start; e.p_offset = p_offset;
  e.B = Bc; e.Cw = Cw; e.d = d; e.embed = h->embed; e.pos_table = h->pos; e.row_pos = h->row_pos;
  e.gamma = h->lnbg; e.beta = h->lnbb; e.mask_idx = 32; e.x = h->x;
  { ProfScope ps(CAT_EMBED, s); rc = launch_msa_embed(e, s); }
  if (rc) return rc;
  const float row_scale = 1.0f / sqrtf(static_cast<float>(R));  // align_scaling (axial_attention.py:78-80); head_dim^-1/2 is in the weights
  for (int l = 0; l < D.layers; ++l) {
    const Layer& L = h->layers[l];
    const Layer& CL = h->col_layers[l];
    // ---- tied row attention
    if ((rc = ln(h, h->x, L.ln1g, L.ln1b, rows, h->abuf, s))) return rc;
    if ((rc = lin(h, L, QKV, h->abuf, S_LN, rows, h->qkv, s))) return rc;
    if (l == D.layers - 1) {
      // ---- pruned last layer (exact)
      const int BR = Bc * R;
      uint8_t* fb = reinterpret_cast<uint8_t*>(h->fbuf);  // the MLP hidden buffer is idle here: compact residual / operand / q-k-v rows
      float* xr = reinterpret_cast<float*>(fb);
      __half* cab = reinterpret_cast<__half*>(fb + al(static_cast<size_t>(BR) * d * 4));
      __half* cqkv = reinterpret_cast<__half*>(fb + al(static_cast<size_t>(BR) * d * 4) + al(static_cast<size_t>(BR) * o.ldd * 2));
      { ProfScope ps(CAT_TIED, s, 3);
        rc = launch_tied_col_attention(h->qkv, o.ldq, o.lo_q, sel, Bc, R, Cw, H, row_scale, S, cab, o.ldd, o.lo_d, o.afmt, S_ATT, s); }
      if (rc) return rc;
      { ProfScope ps(CAT_REGROUP, s);
        rc = launch_msa_gather_col(h->x, sel, Bc, R, Cw, d, xr, s); }
      if (rc) return rc;
      if ((rc = lin_add(h, L, OUT, cab, S_ATT, BR, xr, s))) return rc;
      if ((rc = ln(h, xr, CL.ln1g, CL.ln1b, BR, cab, s))) return rc;
      if ((rc = lin(h, CL, QKV, cab, S_LN, BR, cqkv, s))) return rc;
      const AttnLaunch a = attn_args(h, cqkv, cab, Bc, R);
      { ProfScope ps(CAT_ATTN, s); rc = launch_attention_wgmma(a, s); }
      if (rc) return rc;
      if ((rc = lin_add(h, CL, OUT, cab, S_ATT, BR, xr, s))) return rc;
      rc = launch_gather_rows(xr, h->row_sel + h->head_cap, Bc, R, d, h->xc, s);  // row 0 of every alignment (counted by the head)
      if (rc) return rc;
      return mlp(h, L, h->xc, Bc, h->cabuf, h->cfbuf, 1, S_GELU, s);
    }
    { ProfScope ps(CAT_REGROUP, s, 2);
      rc = launch_tied_gather_qk(h->qkv, o.ldq, o.lo_q, Bc, R, Cw, H, Cp, tq, tk, ldt, s);
      if (!rc) rc = launch_tied_transpose_v(h->qkv, o.ldq, o.lo_q, Bc, R, Cw, H, Kp, tv, ldv, s); }
    if (rc) return rc;
    PG_CUDA_OK(cudaMemsetAsync(S, 0, b_s, s));
    { GemmLaunch g{};
      g.a = tq; g.lda = ldt; g.w = tk; g.ldw = ldt; g.M = G * Cp; g.N = Cw; g.K = Nt; g.nseg = o.pseg; g.epi = 2;
      g.resid = S; g.ldr = lds; g.grp_rows_a = Cp; g.grp_rows_b = Cp;
      ProfScope ps(CAT_TIED, s);
      rc = launch_gemm(g, s); }
    if (rc) return rc;
    { ProfScope ps(CAT_REGROUP, s);
      rc = launch_tied_softmax(S, lds, G, Cw, Cp, Kp, row_scale, P, ldp, np, s); }
    if (rc) return rc;
    { GemmLaunch g{};
      g.a = P; g.lda = ldp; g.w = tv; g.ldw = ldv; g.M = G * Cp; g.N = Nt; g.K = Kp; g.nseg = o.pseg; g.epi = 0;
      g.out = tq; g.ldo = ldt; g.out_fmt = o.afmt; g.out_lo_off = o.afmt ? Nt : 0; g.out_scale = S_ATT;
      g.grp_rows_a = Cp; g.grp_rows_b = Nt;
      ProfScope ps(CAT_TIED, s);
      rc = launch_gemm(g, s); }
    if (rc) return rc;
    { ProfScope ps(CAT_REGROUP, s);
      rc = launch_tied_scatter_out(tq, ldt, h->abuf, o.ldd, o.afmt, Bc, R, Cw, H, Cp, s); }
    if (rc) return rc;
    if ((rc = lin_add(h, L, OUT, h->abuf, S_ATT, rows, h->x, s))) return rc;
    // ---- column attention: rows regrouped to (b, c, r) by the LayerNorm, back to (b, r, c) by the attention kernel
    if ((rc = ln(h, h->x, CL.ln1g, CL.ln1b, rows, h->abuf, s, R, Cw))) return rc;
    if ((rc = lin(h, CL, QKV, h->abuf, S_LN, rows, h->qkv, s))) return rc;
    AttnLaunch a = attn_args(h, h->qkv, h->abuf, Bc * Cw, R);
    a.perm_C = Cw;
    { ProfScope ps(CAT_ATTN, s); rc = launch_attention_wgmma(a, s); }
    if (rc) return rc;
    if ((rc = lin_add(h, CL, OUT, h->abuf, S_ATT, rows, h->x, s))) return rc;
    // ---- feed-forward
    if ((rc = mlp(h, L, h->x, rows, h->abuf, h->fbuf, 1, S_GELU, s))) return rc;
  }
  return PG_OK;
}

HeadLaunch head_args(pg_handle h, int T) {
  HeadLaunch hl{};
  hl.x = h->x; hl.d = h->desc.embed_dim; hl.T = T;
  hl.lna_g = h->lnag; hl.lna_b = h->lnab; hl.dense_w = h->hdw; hl.dense_b = h->hdb;
  hl.ln_g = h->hlng; hl.ln_b = h->hlnb; hl.out_w = h->outw ? h->outw : h->embed; hl.out_b = h->hbias; hl.vocab = h->desc.vocab;
  hl.scratch_a = h->hs_a; hl.scratch_b = h->hs_b;
  return hl;
}

// Sequences per pass: as many as the workspace holds, then evened out over the passes that needs — 512 copies of a 514-token window
// against the default 131 072-row workspace are 171 + 171 + 170, not 255 + 255 + 2 (a 2-sequence pass pays all 33 layers' launch
// latencies and partial waves for 0.4 % of the rows). Results do not depend on the split (rows are independent; tested).
long long balanced_per(long long total, long long cap) {
  if (cap < 1) cap = 1;
  if (total <= cap) return total > 0 ? total : 1;
  const long long passes = (total + cap - 1) / cap;
  return (total + passes - 1) / passes;
}

// LM head on the Bc rows a pruned last layer left compacted in h->xc -> out [Bc, vocab]. `launches`: the head's own and the pass's
// launches no other scope counts.
int compact_head(pg_handle h, int T, int Bc, float* out, int launches, cudaStream_t s) {
  ProfScope ps(CAT_HEAD, s, launches);
  HeadLaunch hl = head_args(h, T);
  hl.x = h->xc; hl.P = Bc; hl.all_rows = 1;
  hl.out = out;
  return launch_head(hl, s);
}

// ProtGPT2's 50 257-way head on B sequences of T rows in h->x: ln_f into fp16 hi [| lo] operand rows (fmt 1 in both parity modes: no
// LayerNorm follows the head, so it runs the x3 scheme, or single fp16 in PG_PREC_F16), the GEMM against the packed wte with the
// log-softmax partial epilogue (epi 7, K16: no logit is stored unless f.out_logprobs asks for the rows), then the combine + sums.
int lm_head_fused(pg_handle h, const int32_t* ids, const int32_t* lens, int B, int T, const ArFusion& f, float* tok_logp, float* out_sum,
                  cudaStream_t s) {
  const OpFmt& o = h->op;
  const int d = h->desc.embed_dim, V = h->desc.vocab, rows = B * T;
  int rc = launch_layernorm_f16(h->x, d, h->lnag, h->lnab, rows, d, h->abuf, o.ldd, o.lo_d, s, o.qfmt, 0.f, 0, 0, nullptr, 0, o.dk);
  if (rc) return rc;
  GemmLaunch g{};
  g.a = h->abuf; g.lda = o.ldd; g.w = h->lmw; g.ldw = o.ldd; g.bias = nullptr;
  g.M = rows; g.N = V; g.K = o.dk; g.nseg = o.pseg; g.epi = 7;
  g.lm_part = h->lm_part; g.lm_tgt = h->lm_tgt; g.lm_logits = f.out_logprobs; g.lm_ids = ids; g.lm_lens = lens; g.lm_T = T;
  if ((rc = launch_gemm(g, s))) return rc;
  return launch_lm_head_combine(h->lm_part, (V + GEMM_BN - 1) / GEMM_BN, h->lm_tgt, ids, lens, B, T, V, f.out_logprobs, tok_logp, out_sum, s);
}

// The autoregressive head (ln_f, the handle's head matrix and bias, log-softmax) on B sequences of T rows in h->x.
int ar_head(pg_handle h, const int32_t* ids, const int32_t* lens, int B, int T, const ArFusion& f, float* tok_logp, float* out_sum,
            cudaStream_t s) {
  if (h->desc.arch == PG_ARCH_PROTGPT2) return lm_head_fused(h, ids, lens, B, T, f, tok_logp, out_sum, s);
  return launch_ar_head(h->x, h->desc.embed_dim, B, T, h->head_vocab, ids, lens, h->lnag, h->lnab, h->outw ? h->outw : h->embed,
                        h->desc.arch == PG_ARCH_PROGEN2 ? h->hbias : nullptr, h->label_off, f, tok_logp, out_sum, s);
}

// The decoder passes over B sequences of T rows (forward_ar mode 0, or mode 2 after the recorded prefix at `start`), as many sequences
// per pass as the workspace holds, each followed by the head on its rows (the tied embedding, or RITA's untied lm_head).
int ar_passes(pg_handle h, const int32_t* ids, const int32_t* lens, int B, int T, int mode, int start, const ArFusion& fusion,
              float* out_sum_logp, cudaStream_t s) {
  const long long per = balanced_per(B, h->max_rows / T);
  for (int b0 = 0; b0 < B; b0 += static_cast<int>(per)) {
    const int Bc = (B - b0) < per ? (B - b0) : static_cast<int>(per);
    const long long off = static_cast<long long>(b0) * T;
    int rc = forward_ar(h, ids + off, Bc, T, s, mode, start);
    if (rc) return fail(h, rc, tls_error());
    ProfScope ps(CAT_HEAD, s, h->desc.arch == PG_ARCH_PROTGPT2 ? 4 : 2);
    ArFusion fc = fusion;
    if (fc.prior_row) fc.prior_row += off;
    if (fc.prior_row2) fc.prior_row2 += off;
    if (fc.out_logprobs) fc.out_logprobs += off * h->head_vocab;
    rc = ar_head(h, ids + off, lens + b0, Bc, T, fc, h->tok_logp, out_sum_logp + b0, s);
    if (rc) return fail(h, rc, tls_error());
  }
  return PG_OK;
}

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" {

int pg_abi_version(void) { return 5; }

long long pg_launch_count(void) {
  std::lock_guard<std::mutex> lk(prof_mu());
  long long t = 0;
  for (int i = 0; i < CAT_COUNT; ++i) t += prof().launches[i];
  return t;
}

int pg_profile_begin(void) {
  std::lock_guard<std::mutex> lk(prof_mu());
  prof().on = true;
  prof().used = 0;
  return PG_OK;
}

// Stops profiling and returns, per category, the summed device time (ms) and number of timed scopes.
// The caller must have synchronised the stream(s) first.
int pg_profile_end(float* ms, int32_t* counts, int32_t ncat) {
  std::lock_guard<std::mutex> lk(prof_mu());
  ProfState& p = prof();
  p.on = false;
  for (int i = 0; i < ncat; ++i) { ms[i] = 0.f; counts[i] = 0; }
  for (size_t i = 0; i + 1 < p.used; i += 2) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, p.ev[i], p.ev[i + 1]) != cudaSuccess) continue;
    const int c = p.ev_cat[i / 2];
    if (c < ncat) { ms[c] += t; counts[c] += 1; }
  }
  p.used = 0;
  return PG_OK;
}

const char* pg_last_error(pg_handle h) {
  if (h && !h->err.empty()) return h->err.c_str();
  return tls_error().c_str();
}

int pg_create(const pg_model_desc* desc, pg_handle* out) {
  if (!desc || !out) return set_error(PG_ERR_ARG, "pg_create: null argument");
  const pg_model_desc& D = *desc;
  if (D.layers <= 0 || D.embed_dim <= 0 || D.heads <= 0 || D.ffn_dim <= 0 || D.vocab <= 0)
    return set_error(PG_ERR_ARG, "pg_create: non-positive model dimension");
  if (D.arch == PG_ARCH_PROGEN2) {  // head_dim 64 in 64-wide slots, 65..128 in 128-wide slots (OpFmt)
    const int hd = D.embed_dim % D.heads ? 0 : D.embed_dim / D.heads;
    if (hd > 128)
      return set_error(PG_ERR_UNSUPPORTED, "pg_create: ProGen2 head_dim " + std::to_string(hd) +
                                               " > 128 (progen2-xlarge, 4096 / 16 = 256) has no attention tile");
    if (hd < 64 || hd % 2) return set_error(PG_ERR_UNSUPPORTED, "pg_create: ProGen2 needs an even head_dim from 64 to 128");
    if (D.heads % 8) return set_error(PG_ERR_UNSUPPORTED, "pg_create: ProGen2 needs heads % 8 == 0 (qkv_proj is 8 shards, modeling_progen.py:157-168)");
    if (D.embed_dim % 64 || D.ffn_dim % 64) return set_error(PG_ERR_UNSUPPORTED, "pg_create: embed_dim and ffn_dim must be multiples of 64");
    if (D.vocab < 30) return set_error(PG_ERR_UNSUPPORTED, "pg_create: ProGen2 scores vocabulary columns 5..29 (vocab >= 30)");
  } else if (D.arch == PG_ARCH_ESM2) {  // narrow heads in 64-wide slots, widths padded to 64 (OpFmt)
    if (D.embed_dim % D.heads || (D.embed_dim / D.heads) % 2 || D.embed_dim / D.heads > 64)
      return set_error(PG_ERR_UNSUPPORTED, "pg_create: ESM2 head_dim must be even and at most 64");
    if (D.embed_dim % 4 || D.ffn_dim % 64) return set_error(PG_ERR_UNSUPPORTED, "pg_create: ESM2 needs embed_dim % 4 == 0 and ffn_dim % 64 == 0");
  } else {
    if (D.arch == PG_ARCH_RITA && D.embed_dim != D.heads * 64)  // RITA XL (2048 / 16) has 128-wide heads
      return set_error(PG_ERR_UNSUPPORTED, "pg_create: RITA needs head_dim 64 (RITA S / M / L); 128-wide heads (RITA XL) have no attention tile");
    if (D.arch == PG_ARCH_PROTGPT2 && D.embed_dim != D.heads * 64)  // the 1/8 q fold and the attention tile are for 64-wide heads
      return set_error(PG_ERR_UNSUPPORTED, "pg_create: ProtGPT2 needs head_dim 64 (GPT-2 large: 1280 / 20)");
    if (D.arch == PG_ARCH_PROTGPT2 && D.max_positions <= 0)
      return set_error(PG_ERR_ARG, "pg_create: ProtGPT2 needs max_positions = the rows of the position table (n_positions)");
    if (D.embed_dim != D.heads * 64) return set_error(PG_ERR_UNSUPPORTED, "pg_create: head_dim must be 64");
    if (D.embed_dim % 64 || D.ffn_dim % 64) return set_error(PG_ERR_UNSUPPORTED, "pg_create: embed_dim and ffn_dim must be multiples of 64");
  }
  if (D.arch != PG_ARCH_ESM1B && D.arch != PG_ARCH_ESM2 && D.arch != PG_ARCH_TRANCEPTION && D.arch != PG_ARCH_MSA && D.arch != PG_ARCH_ESMC &&
      D.arch != PG_ARCH_RITA && D.arch != PG_ARCH_PROGEN2 && D.arch != PG_ARCH_PROTGPT2)
    return set_error(PG_ERR_UNSUPPORTED, "pg_create: unknown arch");
  if (D.arch == PG_ARCH_ESMC && D.heads > 24) return set_error(PG_ERR_UNSUPPORTED, "pg_create: the ESM C q/k LayerNorm kernel holds at most 24 heads");
  if (D.arch == PG_ARCH_TRANCEPTION && D.heads % 4) return set_error(PG_ERR_UNSUPPORTED, "pg_create: Tranception needs heads % 4 == 0 (model_pytorch.py:129-131)");
  if (D.precision != PG_PREC_F16 && D.precision != PG_PREC_F16X3 && D.precision != PG_PREC_F16F8 && D.precision != PG_PREC_F16D)
    return set_error(PG_ERR_ARG, "pg_create: unknown precision");
  if (D.precision == PG_PREC_F16D && D.arch != PG_ARCH_ESM1B)
    return set_error(PG_ERR_UNSUPPORTED, "pg_create: PG_PREC_F16D (delta operands) is built for the ESM-1b / ESM-1v masked-marginal path");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return set_error(PG_ERR_CUDA, "pg_create: no CUDA device (the library has no CPU fallback)");
  if (D.device < 0 || D.device >= ndev) return set_error(PG_ERR_ARG, "pg_create: bad device ordinal");
  PG_CUDA_OK(cudaSetDevice(D.device));
  cudaDeviceProp prop;
  PG_CUDA_OK(cudaGetDeviceProperties(&prop, D.device));
  if (prop.major != 9 || prop.minor != 0) return set_error(PG_ERR_UNSUPPORTED, "pg_create: device is not sm_90 (the kernels are built for sm_90a: wgmma, TMA)");
  pg_handle h = new pg_handle_s();
  h->desc = D;
  h->op = op_fmt(D);
  h->delta = (D.precision == PG_PREC_F16D);
  h->max_rows = D.max_rows > 0 ? D.max_rows : 131072;
  h->head_cap = 8192;
  h->head_vocab = D.arch == PG_ARCH_PROGEN2 ? 25 : D.vocab;
  h->label_off = D.arch == PG_ARCH_PROGEN2 ? 5 : 0;
  const int d = D.embed_dim, f = D.ffn_dim, np = h->op.np, dk = h->op.dk, da = h->op.da;
  const int dw = dk > da ? dk : da;  // abuf / cabuf hold both LayerNorm outputs (dk) and attention outputs (da)
  int rc = PG_OK;
  auto A = [&](auto** p, size_t n) { if (!rc) rc = dev_alloc(h, p, n); };
  h->layers.resize(D.layers);
  const bool esmc = D.arch == PG_ARCH_ESMC;
  const int f1 = esmc ? 2 * f : f;  // rows of fc1: ESM C holds the SwiGLU gate and up halves
  for (auto& L : h->layers) {
    A(&L.wqkv, static_cast<size_t>(3) * da * dk * np); A(&L.wo, static_cast<size_t>(d) * da * np);
    A(&L.w1, static_cast<size_t>(f1) * dk * np); A(&L.w2, static_cast<size_t>(d) * f * np);
    if (!esmc && D.arch != PG_ARCH_PROGEN2) { A(&L.bqkv, 3 * da); A(&L.bo, d); }  // ESM C and ProGen2 attention: no bias (null = none)
    if (!esmc) { A(&L.b1, f); A(&L.b2, d); }  // ESM C MLP: no bias
    A(&L.ln1g, d); A(&L.ln1b, d); A(&L.ln2g, d); A(&L.ln2b, d);
    if (h->op.nseg == 2) { A(&L.iqkv, 3 * da); A(&L.io, d); A(&L.i1, f1); A(&L.i2, d); }
    if (D.arch == PG_ARCH_TRANCEPTION) A(&L.conv_taps, 3 * 4 * 64 * 8);
    if (esmc) { A(&L.qlng, d); A(&L.klng, d); }
  }
  if (esmc || D.arch == PG_ARCH_RITA || D.arch == PG_ARCH_PROGEN2) A(&h->outw, static_cast<size_t>(D.vocab) * d);
  if (D.arch == PG_ARCH_MSA) {
    h->col_layers.resize(D.layers);
    for (auto& L : h->col_layers) {
      A(&L.wqkv, static_cast<size_t>(3) * da * dk * np); A(&L.wo, static_cast<size_t>(d) * da * np);
      A(&L.bqkv, 3 * da); A(&L.bo, d); A(&L.ln1g, d); A(&L.ln1b, d);
      if (h->op.nseg == 2) { A(&L.iqkv, 3 * da); A(&L.io, d); }
    }
    A(&h->row_pos, static_cast<size_t>(1024) * d);
  }
  if (D.arch == PG_ARCH_TRANCEPTION) {
    A(&h->qkv2, static_cast<size_t>(h->max_rows) * 3 * d * np);
    A(&h->slopes, D.heads);
  }
  if (is_ar(D.arch)) A(&h->tok_logp, static_cast<size_t>(h->max_rows));
  if (D.arch == PG_ARCH_PROTGPT2) {  // 8 B per row and N tile: 412 MB at the default 131 072 rows and 50 257 columns
    A(&h->lmw, static_cast<size_t>(D.vocab) * dk * np);
    A(&h->lm_part, static_cast<size_t>(h->max_rows) * ((D.vocab + GEMM_BN - 1) / GEMM_BN));
    A(&h->lm_tgt, static_cast<size_t>(h->max_rows));
    A(&h->pos, static_cast<size_t>(D.max_positions) * d);
  }
  if (h->op.nseg == 2) A(&h->pack_scratch, static_cast<size_t>(D.layers) * 6);
  A(&h->embed, static_cast<size_t>(D.vocab) * d);
  if (D.arch == PG_ARCH_ESM1B || D.arch == PG_ARCH_MSA) A(&h->pos, static_cast<size_t>(D.max_positions + 2) * d);
  A(&h->lnbg, d); A(&h->lnbb, d); A(&h->lnag, d); A(&h->lnab, d);
  A(&h->hdw, static_cast<size_t>(d) * d); A(&h->hdb, d); A(&h->hlng, d); A(&h->hlnb, d); A(&h->hbias, D.vocab);
  A(&h->x, static_cast<size_t>(h->max_rows) * d);
  A(&h->abuf, static_cast<size_t>(h->max_rows) * dw * np);
  A(&h->qkv, static_cast<size_t>(h->max_rows) * 3 * da * np);
  A(&h->fbuf, static_cast<size_t>(h->max_rows) * f * np);
  A(&h->hs_a, static_cast<size_t>(h->head_cap) * d);
  A(&h->hs_b, static_cast<size_t>(h->head_cap) * d);
  A(&h->row_sel, 2 * static_cast<size_t>(h->head_cap));  // second half: zeros (row 0 of every compacted sequence)
  A(&h->xc, static_cast<size_t>(h->head_cap) * d);
  A(&h->cabuf, static_cast<size_t>(h->head_cap) * dw * np);
  A(&h->cfbuf, static_cast<size_t>(h->head_cap) * f * np);
  if (h->delta) A(&h->cq, static_cast<size_t>(h->head_cap) * 3 * d * np);
  if (rc) {
    std::string m = h->err;
    pg_destroy(h);
    return set_error(rc, m);
  }
  cudaMemset(h->row_sel, 0, 2 * static_cast<size_t>(h->head_cap) * sizeof(int32_t));
  *out = h;
  return PG_OK;
}

int pg_destroy(pg_handle h) {
  if (!h) return PG_OK;
  cudaSetDevice(h->desc.device);
  for (void* p : h->allocs) cudaFree(p);
  if (h->tied_ws) cudaFree(h->tied_ws);
  if (h->base) cudaFree(h->base);
  delete h;
  return PG_OK;
}

int pg_load_weights(pg_handle h, const pg_tensor* tensors, int32_t n) {
  if (!h || !tensors) return set_error(PG_ERR_ARG, "pg_load_weights: null argument");
  PG_CUDA_OK(cudaSetDevice(h->desc.device));
  const pg_model_desc& D = h->desc;
  const int d = D.embed_dim, f = D.ffn_dim, np = h->op.np;
  std::map<std::string, const pg_tensor*> by_name;
  for (int i = 0; i < n; ++i) by_name[tensors[i].name] = &tensors[i];
  std::string missing;
  auto get = [&](const std::string& name, int64_t r, int64_t c) -> const float* {
    auto it = by_name.find(name);
    if (it == by_name.end()) { missing += name + " "; return nullptr; }
    if (it->second->shape[0] != r || it->second->shape[1] != c) { missing += name + "(shape) "; return nullptr; }
    return static_cast<const float*>(it->second->data);
  };
  struct Scratch {  // weights expanded to the padded operand layout (ESM2 head slots); cudaFree waits for the packing kernels
    std::vector<float*> p;
    ~Scratch() { for (float* q : p) cudaFree(q); }
  } expanded;
  cudaError_t exp_err = cudaSuccess;
  auto copy = [&](float* dst, const float* src, size_t cnt, float scale = 1.f) {
    if (!src) return;
    scale_copy_kernel<<<static_cast<unsigned>((cnt + 255) / 256), 256>>>(src, dst, static_cast<int>(cnt), scale);
  };
  // A group of [N, K] weights that form one GEMM operand, packed into dst (inv: where the per-row 1/t of PG_PREC_F16F8 go).
  // Conv1D weights are stored [in = K, out = N]; conv_ld: their row pitch when the N columns are a slice of a wider matrix.
  auto pack = [&](__half* dst, float* inv, std::initializer_list<PackSrc> group, int N, int K, bool conv1d = false, long long conv_ld = 0) {
    for (const PackSrc& m : group)
      if (!m.w) return;
    unsigned int* f8_scratch = h->op.nseg == 2 ? h->pack_scratch + (h->pack_used++ % (D.layers * 6)) : nullptr;
    pack_weights(group, N, K, conv1d ? 1 : K, conv1d ? (conv_ld ? conv_ld : N) : 1, np, f8_scratch, dst, inv, 0);
  };
  // "rotary.cos" / "rotary.sin" [T, S/2] (ESM C, RITA: [T, 32]; ProGen2: half its slot width) -> the tables of the rotary GEMM epilogue
  auto rotary32 = [&]() -> int {
    const int hs = h->op.slot / 2;
    auto it = by_name.find("rotary.cos");
    auto is = by_name.find("rotary.sin");
    if (it == by_name.end() || is == by_name.end() || it->second->shape[1] != hs || is->second->shape[1] != hs ||
        is->second->shape[0] != it->second->shape[0]) {
      missing += "rotary.cos/rotary.sin[T," + std::to_string(hs) + "] ";
      return PG_OK;
    }
    h->rot_rows = static_cast<int>(it->second->shape[0]);
    int rc = dev_alloc(h, &h->rot_cos, static_cast<size_t>(h->rot_rows) * hs);
    if (!rc) rc = dev_alloc(h, &h->rot_sin, static_cast<size_t>(h->rot_rows) * hs);
    if (rc) return rc;
    copy(h->rot_cos, static_cast<const float*>(it->second->data), static_cast<size_t>(h->rot_rows) * hs);
    copy(h->rot_sin, static_cast<const float*>(is->second->data), static_cast<size_t>(h->rot_rows) * hs);
    return PG_OK;
  };
  const int hd = d / D.heads;
  // A [n_src, k_src] source weight placed in the padded operand layout [N, K] (OpFmt, slot maps rmap / cmap), in a scratch buffer
  // freed on return; the source itself when the layout is unpadded. The ProGen2 maps read rows of the fused [3d, d] qkv_proj.
  auto slots = [&](const float* w, int n_src, int k_src, int N, int K, int rmap, int cmap) -> const float* {
    if (!w || (N == n_src && K == k_src)) return w;
    float* p = nullptr;
    const cudaError_t e = cudaMalloc(&p, static_cast<size_t>(N) * K * sizeof(float));
    if (e != cudaSuccess) {
      if (!exp_err) exp_err = e;
      return nullptr;
    }
    expanded.p.push_back(p);
    const long long tot = static_cast<long long>(N) * K;
    const int rn = rmap >= SL_PGQ ? n_src / 3 : n_src;
    expand_slots_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256>>>(w, rn, k_src, p, N, K, rmap, cmap, hd, h->op.slot, k_src);
    return p;
  };
  if (D.arch == PG_ARCH_TRANCEPTION) {
    // HF GPT2-style names with the "transformer." prefix stripped by the host
    for (int l = 0; l < D.layers; ++l) {
      Layer& L = h->layers[l];
      const std::string p = "h." + std::to_string(l) + ".";
      pack(L.wqkv, L.iqkv, {get(p + "attn.c_attn.weight", d, 3 * d)}, 3 * d, d, true);
      copy(L.bqkv, get(p + "attn.c_attn.bias", 3 * d, 1), 3 * d);
      pack(L.wo, L.io, {get(p + "attn.c_proj.weight", d, d)}, d, d, true);
      copy(L.bo, get(p + "attn.c_proj.bias", d, 1), d);
      pack(L.w1, L.i1, {get(p + "mlp.c_fc.weight", d, f)}, f, d, true);
      copy(L.b1, get(p + "mlp.c_fc.bias", f, 1), f);
      pack(L.w2, L.i2, {get(p + "mlp.c_proj.weight", f, d)}, d, f, true);
      copy(L.b2, get(p + "mlp.c_proj.bias", d, 1), d);
      copy(L.ln1g, get(p + "ln_1.weight", d, 1), d);
      copy(L.ln1b, get(p + "ln_1.bias", d, 1), d);
      copy(L.ln2g, get(p + "ln_2.weight", d, 1), d);
      copy(L.ln2b, get(p + "ln_2.bias", d, 1), d);
      copy(L.conv_taps, get(p + "attn.conv_taps", 3 * 4 * 64, 8), 3 * 4 * 64 * 8);
    }
    copy(h->embed, get("wte.weight", D.vocab, d), static_cast<size_t>(D.vocab) * d);
    copy(h->lnag, get("ln_f.weight", d, 1), d);
    copy(h->lnab, get("ln_f.bias", d, 1), d);
    copy(h->slopes, get("alibi_slopes", D.heads, 1), D.heads);
  } else if (D.arch == PG_ARCH_ESMC) {
    // evoscale key names (esm/models/esmc.py:63-76, layers/blocks.py:35-43,95-110, layers/attention.py:28-39). Residual branches are
    // divided by s = sqrt(layers / 36) (transformer_stack.py:48-50, blocks.py:150-160): 1/s is folded into out_proj and fc2 here.
    const float rs = static_cast<float>(1.0 / std::sqrt(static_cast<double>(D.layers) / 36.0));
    for (int l = 0; l < D.layers; ++l) {
      Layer& L = h->layers[l];
      const std::string p = "transformer.blocks." + std::to_string(l) + ".";
      copy(L.ln1g, get(p + "attn.layernorm_qkv.0.weight", d, 1), d);
      copy(L.ln1b, get(p + "attn.layernorm_qkv.0.bias", d, 1), d);
      pack(L.wqkv, L.iqkv, {get(p + "attn.layernorm_qkv.1.weight", 3 * d, d)}, 3 * d, d);
      copy(L.qlng, get(p + "attn.q_ln.weight", d, 1), d);
      copy(L.klng, get(p + "attn.k_ln.weight", d, 1), d);
      pack(L.wo, L.io, {{get(p + "attn.out_proj.weight", d, d), rs}}, d, d);
      copy(L.ln2g, get(p + "ffn.0.weight", d, 1), d);
      copy(L.ln2b, get(p + "ffn.0.bias", d, 1), d);
      const float* w1 = get(p + "ffn.1.weight", 2 * f, d);
      if (w1) {  // gate / up rows interleaved in blocks of 8 for the SwiGLU epilogue
        float* t = nullptr;
        const cudaError_t e = cudaMalloc(&t, static_cast<size_t>(2) * f * d * sizeof(float));
        if (e != cudaSuccess) {
          if (!exp_err) exp_err = e;
        } else {
          expanded.p.push_back(t);
          const long long tot = 2LL * f * d;
          interleave_gate_up_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256>>>(w1, f, d, t);
          pack(L.w1, L.i1, {t}, 2 * f, d);
        }
      }
      pack(L.w2, L.i2, {{get(p + "ffn.3.weight", d, f), rs}}, d, f);
    }
    copy(h->embed, get("embed.weight", D.vocab, d), static_cast<size_t>(D.vocab) * d);
    copy(h->lnag, get("transformer.norm.weight", d, 1), d);
    PG_CUDA_OK(cudaMemset(h->lnab, 0, static_cast<size_t>(d) * sizeof(float)));  // the final norm has no bias
    copy(h->hdw, get("sequence_head.0.weight", d, d), static_cast<size_t>(d) * d);
    copy(h->hdb, get("sequence_head.0.bias", d, 1), d);
    copy(h->hlng, get("sequence_head.2.weight", d, 1), d);
    copy(h->hlnb, get("sequence_head.2.bias", d, 1), d);
    copy(h->outw, get("sequence_head.3.weight", D.vocab, d), static_cast<size_t>(D.vocab) * d);
    copy(h->hbias, get("sequence_head.3.bias", D.vocab, 1), D.vocab);
    if (int rc = rotary32()) return rc;
  } else if (D.arch == PG_ARCH_RITA) {
    // HF names without the "transformer." prefix (rita_modeling.py:113-121, 185-194, 222-224). q, k and v form one GEMM operand with
    // 1/sqrt(64) = 0.125 folded into the q rows and bias: exact (a power of two), and it commutes with the (linear) rotary.
    for (int l = 0; l < D.layers; ++l) {
      Layer& L = h->layers[l];
      const std::string p = "layers." + std::to_string(l) + ".";
      const std::string a = p + "self_attention.";
      pack(L.wqkv, L.iqkv, {{get(a + "query.weight", d, d), 0.125f}, get(a + "key.weight", d, d), get(a + "value.weight", d, d)}, d, d);
      copy(L.bqkv, get(a + "query.bias", d, 1), d, 0.125f);
      copy(L.bqkv + d, get(a + "key.bias", d, 1), d);
      copy(L.bqkv + 2 * d, get(a + "value.bias", d, 1), d);
      pack(L.wo, L.io, {get(a + "proj.weight", d, d)}, d, d);
      copy(L.bo, get(a + "proj.bias", d, 1), d);
      copy(L.ln1g, get(p + "attn_norm.weight", d, 1), d);
      copy(L.ln1b, get(p + "attn_norm.bias", d, 1), d);
      pack(L.w1, L.i1, {get(p + "mlp.0.weight", f, d)}, f, d);
      copy(L.b1, get(p + "mlp.0.bias", f, 1), f);
      pack(L.w2, L.i2, {get(p + "mlp.2.weight", d, f)}, d, f);
      copy(L.b2, get(p + "mlp.2.bias", d, 1), d);
      copy(L.ln2g, get(p + "mlp_norm.weight", d, 1), d);
      copy(L.ln2b, get(p + "mlp_norm.bias", d, 1), d);
    }
    copy(h->embed, get("embedding.weight", D.vocab, d), static_cast<size_t>(D.vocab) * d);
    copy(h->lnag, get("final_norm.weight", d, 1), d);
    copy(h->lnab, get("final_norm.bias", d, 1), d);
    // the output head: "lm_head.weight" when the caller passes it (an untied checkpoint), else the embedding matrix
    if (by_name.count("lm_head.weight")) copy(h->outw, get("lm_head.weight", D.vocab, d), static_cast<size_t>(D.vocab) * d);
    else copy(h->outw, get("embedding.weight", D.vocab, d), static_cast<size_t>(D.vocab) * d);
    if (int rc = rotary32()) return rc;
    if (h->rot_rows && h->rot_rows < D.max_positions) missing += "rotary.cos/rotary.sin(fewer than max_positions rows) ";
  } else if (D.arch == PG_ARCH_PROTGPT2) {
    // GPT-2 names without the "transformer." prefix (transformers modeling_gpt2.py GPT2Attention / GPT2MLP / GPT2Model), Conv1D weights
    // [in, out]. c_attn's q, k and v column blocks form one GEMM operand with 1/sqrt(64) = 0.125 folded into the q columns and bias
    // (exact: a power of two). The head is wte itself (tied), packed once more as a [vocab, d] operand for K16.
    for (int l = 0; l < D.layers; ++l) {
      Layer& L = h->layers[l];
      const std::string p = "h." + std::to_string(l) + ".";
      const float* wa = get(p + "attn.c_attn.weight", d, 3 * d);
      pack(L.wqkv, L.iqkv, {{wa, 0.125f}, wa ? wa + d : nullptr, wa ? wa + 2 * d : nullptr}, d, d, true, 3 * d);
      const float* ba = get(p + "attn.c_attn.bias", 3 * d, 1);
      copy(L.bqkv, ba, d, 0.125f);
      copy(L.bqkv + d, ba ? ba + d : nullptr, 2 * d);
      pack(L.wo, L.io, {get(p + "attn.c_proj.weight", d, d)}, d, d, true);
      copy(L.bo, get(p + "attn.c_proj.bias", d, 1), d);
      pack(L.w1, L.i1, {get(p + "mlp.c_fc.weight", d, f)}, f, d, true);
      copy(L.b1, get(p + "mlp.c_fc.bias", f, 1), f);
      pack(L.w2, L.i2, {get(p + "mlp.c_proj.weight", f, d)}, d, f, true);
      copy(L.b2, get(p + "mlp.c_proj.bias", d, 1), d);
      copy(L.ln1g, get(p + "ln_1.weight", d, 1), d);
      copy(L.ln1b, get(p + "ln_1.bias", d, 1), d);
      copy(L.ln2g, get(p + "ln_2.weight", d, 1), d);
      copy(L.ln2b, get(p + "ln_2.bias", d, 1), d);
    }
    const float* wte = get("wte.weight", D.vocab, d);
    copy(h->embed, wte, static_cast<size_t>(D.vocab) * d);
    if (wte) pack_weights({wte}, D.vocab, d, d, 1, np, nullptr, h->lmw, nullptr, 0);  // fp16 hi [| lo] in every mode
    copy(h->pos, get("wpe.weight", D.max_positions, d), static_cast<size_t>(D.max_positions) * d);
    copy(h->lnag, get("ln_f.weight", d, 1), d);
    copy(h->lnab, get("ln_f.bias", d, 1), d);
  } else if (D.arch == PG_ARCH_PROGEN2) {
    // HF names without the "transformer." prefix (modeling_progen.py:84-95, 209-226, 389-401, 541-548). qkv_proj [3d, d] is placed
    // into the head slots by SL_PGQ / SL_PGK / SL_PGV (one GEMM operand, no bias) with head_dim^-1/2 folded into the q rows: exact
    // for head_dim 64, one fp32 rounding for 80 and 96. out_proj's columns take the SL_HEAD slots. The head is rows 5..29 of
    // lm_head (weight and bias): the reference's log-softmax runs over exactly those columns (compute_fitness.py:71-77).
    const int da = h->op.da;
    const float qscale = static_cast<float>(1.0 / std::sqrt(static_cast<double>(hd)));
    for (int l = 0; l < D.layers; ++l) {
      Layer& L = h->layers[l];
      const std::string p = "h." + std::to_string(l) + ".";
      const float* wqkv = get(p + "attn.qkv_proj.weight", 3 * d, d);
      pack(L.wqkv, L.iqkv, {{slots(wqkv, 3 * d, d, da, d, SL_PGQ, SL_PAD), qscale}, slots(wqkv, 3 * d, d, da, d, SL_PGK, SL_PAD),
                            slots(wqkv, 3 * d, d, da, d, SL_PGV, SL_PAD)}, da, d);
      pack(L.wo, L.io, {slots(get(p + "attn.out_proj.weight", d, d), d, d, d, da, SL_PAD, SL_HEAD)}, d, da);
      copy(L.ln1g, get(p + "ln_1.weight", d, 1), d);
      copy(L.ln1b, get(p + "ln_1.bias", d, 1), d);
      pack(L.w1, L.i1, {get(p + "mlp.fc_in.weight", f, d)}, f, d);
      copy(L.b1, get(p + "mlp.fc_in.bias", f, 1), f);
      pack(L.w2, L.i2, {get(p + "mlp.fc_out.weight", d, f)}, d, f);
      copy(L.b2, get(p + "mlp.fc_out.bias", d, 1), d);
    }
    copy(h->embed, get("wte.weight", D.vocab, d), static_cast<size_t>(D.vocab) * d);
    copy(h->lnag, get("ln_f.weight", d, 1), d);
    copy(h->lnab, get("ln_f.bias", d, 1), d);
    const float* hw = get("lm_head.weight", D.vocab, d);
    const float* hb = get("lm_head.bias", D.vocab, 1);
    copy(h->outw, hw ? hw + static_cast<size_t>(h->label_off) * d : nullptr, static_cast<size_t>(h->head_vocab) * d);
    copy(h->hbias, hb ? hb + h->label_off : nullptr, h->head_vocab);
    if (int rc = rotary32()) return rc;
    if (h->rot_rows && h->rot_rows < D.max_positions) missing += "rotary.cos/rotary.sin(fewer than max_positions rows) ";
  } else {
    const int dk = h->op.dk, da = h->op.da;
    // head_dim^-1/2 (multihead_attention.py:103,261), folded into the fp32 q weights and bias: 0.125 (exact) for head_dim 64
    const float qscale = static_cast<float>(1.0 / std::sqrt(static_cast<double>(hd)));
    // one attention block: q/k/v/out projections at `pa` ("...self_attn." / "...row_self_attention.layer."), its LayerNorm at `pl`
    auto load_attn = [&](Layer& L, const std::string& pa, const std::string& pl) {
      // q, k, v form ONE GEMM operand: one common e4m3 scale (matrix maximum over the three, q already scaled)
      const float* wq = slots(get(pa + "q_proj.weight", d, d), d, d, da, dk, SL_ROT, SL_PAD);
      const float* wk = slots(get(pa + "k_proj.weight", d, d), d, d, da, dk, SL_ROT, SL_PAD);
      const float* wv = slots(get(pa + "v_proj.weight", d, d), d, d, da, dk, SL_HEAD, SL_PAD);
      pack(L.wqkv, L.iqkv, {{wq, qscale}, wk, wv}, da, dk);
      copy(L.bqkv, slots(get(pa + "q_proj.bias", d, 1), d, 1, da, 1, SL_ROT, SL_PAD), da, qscale);
      copy(L.bqkv + da, slots(get(pa + "k_proj.bias", d, 1), d, 1, da, 1, SL_ROT, SL_PAD), da);
      copy(L.bqkv + 2 * da, slots(get(pa + "v_proj.bias", d, 1), d, 1, da, 1, SL_HEAD, SL_PAD), da);
      pack(L.wo, L.io, {slots(get(pa + "out_proj.weight", d, d), d, d, d, da, SL_PAD, SL_HEAD)}, d, da);
      copy(L.bo, get(pa + "out_proj.bias", d, 1), d);
      copy(L.ln1g, get(pl + "weight", d, 1), d);
      copy(L.ln1b, get(pl + "bias", d, 1), d);
    };
    auto load_ffn = [&](Layer& L, const std::string& pf, const std::string& pl) {
      pack(L.w1, L.i1, {slots(get(pf + "fc1.weight", f, d), f, d, f, dk, SL_PAD, SL_PAD)}, f, dk);
      copy(L.b1, get(pf + "fc1.bias", f, 1), f);
      pack(L.w2, L.i2, {get(pf + "fc2.weight", d, f)}, d, f);
      copy(L.b2, get(pf + "fc2.bias", d, 1), d);
      copy(L.ln2g, get(pl + "weight", d, 1), d);
      copy(L.ln2b, get(pl + "bias", d, 1), d);
    };
    for (int l = 0; l < D.layers; ++l) {
      const std::string p = "layers." + std::to_string(l) + ".";
      if (D.arch == PG_ARCH_MSA) {  // AxialTransformerLayer (modules.py:194-196): three NormalizedResidualBlocks {layer, layer_norm}
        load_attn(h->layers[l], p + "row_self_attention.layer.", p + "row_self_attention.layer_norm.");
        load_attn(h->col_layers[l], p + "column_self_attention.layer.", p + "column_self_attention.layer_norm.");
        load_ffn(h->layers[l], p + "feed_forward_layer.layer.", p + "feed_forward_layer.layer_norm.");
      } else {
        load_attn(h->layers[l], p + "self_attn.", p + "self_attn_layer_norm.");
        load_ffn(h->layers[l], p, p + "final_layer_norm.");
      }
    }
    if (D.arch == PG_ARCH_MSA) {
      auto it = by_name.find("msa_position_embedding");  // host-expanded to [1024, d] (the first release stores a 1-wide table)
      if (it != by_name.end()) {
        if (it->second->shape[0] != 1024 || it->second->shape[1] != d) missing += "msa_position_embedding(shape) ";
        else copy(h->row_pos, static_cast<const float*>(it->second->data), static_cast<size_t>(1024) * d);
      } else {
        h->row_pos = nullptr;  // embed_positions_msa off (msa_transformer.py:106-114)
      }
    }
    copy(h->embed, get("embed_tokens.weight", D.vocab, d), static_cast<size_t>(D.vocab) * d);
    if (D.arch == PG_ARCH_ESM1B || D.arch == PG_ARCH_MSA)
      copy(h->pos, get("embed_positions.weight", D.max_positions + 2, d), static_cast<size_t>(D.max_positions + 2) * d);
    if (D.emb_ln_before || D.arch == PG_ARCH_MSA) {
      copy(h->lnbg, get("emb_layer_norm_before.weight", d, 1), d);
      copy(h->lnbb, get("emb_layer_norm_before.bias", d, 1), d);
    }
    copy(h->lnag, get("emb_layer_norm_after.weight", d, 1), d);
    copy(h->lnab, get("emb_layer_norm_after.bias", d, 1), d);
    copy(h->hdw, get("lm_head.dense.weight", d, d), static_cast<size_t>(d) * d);
    copy(h->hdb, get("lm_head.dense.bias", d, 1), d);
    copy(h->hlng, get("lm_head.layer_norm.weight", d, 1), d);
    copy(h->hlnb, get("lm_head.layer_norm.bias", d, 1), d);
    copy(h->hbias, get("lm_head.bias", D.vocab, 1), D.vocab);
    if (D.arch == PG_ARCH_ESM2) {
      // cos / sin [T, hd/2] (checkpoint.rotary_tables) or [T, 32] -> device tables [T, 32], zero after column hd/2
      auto it = by_name.find("rotary.cos");
      auto is = by_name.find("rotary.sin");
      const int64_t rw = it == by_name.end() ? 0 : it->second->shape[1];
      if (it == by_name.end() || is == by_name.end() || (rw != 32 && rw != hd / 2) || is->second->shape[1] != rw ||
          is->second->shape[0] != it->second->shape[0]) {
        missing += "rotary.cos/rotary.sin[T,head_dim/2] ";
      } else {
        h->rot_rows = static_cast<int>(it->second->shape[0]);
        int rc = dev_alloc(h, &h->rot_cos, static_cast<size_t>(h->rot_rows) * 32);
        if (!rc) rc = dev_alloc(h, &h->rot_sin, static_cast<size_t>(h->rot_rows) * 32);
        if (rc) return rc;
        for (auto [dst, src] : {std::make_pair(h->rot_cos, it->second->data), std::make_pair(h->rot_sin, is->second->data)})
          expand_slots_kernel<<<(h->rot_rows * 32 + 255) / 256, 256>>>(static_cast<const float*>(src), h->rot_rows, static_cast<int>(rw), dst,
                                                                       h->rot_rows, 32, SL_PAD, SL_PAD, hd, 64, static_cast<int>(rw));
      }
    }
  }
  if (exp_err != cudaSuccess) return fail(h, PG_ERR_CUDA, std::string("pg_load_weights: cudaMalloc: ") + cudaGetErrorString(exp_err));
  if (!missing.empty()) return fail(h, PG_ERR_ARG, "pg_load_weights: missing or mis-shaped tensors: " + missing);
  PG_CUDA_OK(cudaGetLastError());
  PG_CUDA_OK(cudaDeviceSynchronize());  // caller may free its tensors on return
  h->loaded = true;
  return PG_OK;
}

int pg_masked_marginals(pg_handle h, const int32_t* tokens, int32_t n_tokens, const int32_t* positions, const int32_t* win_start,
                        const int32_t* out_row, int32_t P, int32_t T, float* out_logprobs, pg_stream stream) {
  if (!h) return set_error(PG_ERR_ARG, "pg_masked_marginals: null handle");
  if (!h->loaded) return fail(h, PG_ERR_STATE, "pg_masked_marginals: weights not loaded");
  if (is_ar(h->desc.arch)) return fail(h, PG_ERR_STATE, "pg_masked_marginals: handle is an autoregressive model (use pg_ar_loglik)");
  if (h->desc.arch == PG_ARCH_MSA) return fail(h, PG_ERR_STATE, "pg_masked_marginals: handle is an MSA Transformer (use pg_msa_masked_marginals)");
  if (!tokens || !positions || !out_logprobs) return fail(h, PG_ERR_ARG, "pg_masked_marginals: null buffer");
  if (P < 0 || T <= 0 || T > n_tokens) return fail(h, PG_ERR_ARG, "pg_masked_marginals: bad P/T");
  if (h->desc.arch == PG_ARCH_ESM1B && T > h->desc.max_positions)
    return fail(h, PG_ERR_ARG, "pg_masked_marginals: window longer than the learned position table (modules.py:256-260)");
  if ((h->desc.arch == PG_ARCH_ESM2 || h->desc.arch == PG_ARCH_ESMC) && T > h->rot_rows)
    return fail(h, PG_ERR_ARG, "pg_masked_marginals: window longer than rotary tables");
  if (T > h->max_rows) return fail(h, PG_ERR_ARG, "pg_masked_marginals: window longer than workspace (raise max_rows)");
  PG_CUDA_OK(cudaSetDevice(h->desc.device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  long long per = h->max_rows / T;
  if (per > h->head_cap) per = h->head_cap;
  per = balanced_per(P, per);
  // delta-operand mode needs one shared window (every copy sees all n_tokens tokens) and the masked row as the emitted row
  const bool delta = h->delta && T == n_tokens && out_row == nullptr && P > 0;
  if (delta) {
    int rc = forward_base(h, tokens, n_tokens, T, s);
    if (rc) return fail(h, rc, tls_error());
  }
  for (int p0 = 0; p0 < P; p0 += static_cast<int>(per)) {
    const int Bc = (P - p0) < per ? (P - p0) : static_cast<int>(per);
    row_select_kernel<<<(Bc + 255) / 256, 256, 0, s>>>(positions, win_start, out_row, p0, Bc, h->row_sel);
    int rc = delta ? forward_rows_delta(h, tokens, n_tokens, positions, win_start, p0, Bc, T, s, h->row_sel)
                   : forward_rows(h, tokens, n_tokens, positions, win_start, p0, Bc, T, s, h->row_sel);
    if (rc) return fail(h, rc, tls_error());
    rc = compact_head(h, T, Bc, out_logprobs + static_cast<long long>(p0) * h->desc.vocab, 4, s);  // + row_select_kernel
    if (rc) return fail(h, rc, tls_error());
  }
  return PG_OK;
}

int pg_msa_masked_marginals(pg_handle h, const int32_t* tokens, int32_t R, int32_t C_full, const int32_t* positions,
                            const int32_t* win_start, int32_t P, int32_t Cw, float* out_logprobs, pg_stream stream) {
  if (!h) return set_error(PG_ERR_ARG, "pg_msa_masked_marginals: null handle");
  if (!h->loaded) return fail(h, PG_ERR_STATE, "pg_msa_masked_marginals: weights not loaded");
  if (h->desc.arch != PG_ARCH_MSA) return fail(h, PG_ERR_STATE, "pg_msa_masked_marginals: handle is not an MSA Transformer");
  if (!tokens || !positions || !out_logprobs) return fail(h, PG_ERR_ARG, "pg_msa_masked_marginals: null buffer");
  if (P < 0 || R <= 0 || Cw <= 0 || Cw > C_full) return fail(h, PG_ERR_ARG, "pg_msa_masked_marginals: bad P/R/Cw");
  if (Cw > h->desc.max_positions) return fail(h, PG_ERR_ARG, "pg_msa_masked_marginals: window longer than the learned position table");
  if (R > 1024 && h->row_pos) return fail(h, PG_ERR_ARG, "pg_msa_masked_marginals: the row-position table covers 1024 alignment rows (msa_transformer.py:163-168)");
  if (Cw < C_full && !win_start) return fail(h, PG_ERR_ARG, "pg_msa_masked_marginals: windows need win_start");
  const long long per_msa = static_cast<long long>(R) * Cw;
  if (per_msa > h->max_rows) return fail(h, PG_ERR_ARG, "pg_msa_masked_marginals: one alignment exceeds the workspace (raise max_rows)");
  PG_CUDA_OK(cudaSetDevice(h->desc.device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  long long per = h->max_rows / per_msa;
  if (per > h->head_cap) per = h->head_cap;
  per = balanced_per(P, per);
  for (int p0 = 0; p0 < P; p0 += static_cast<int>(per)) {
    const int Bc = (P - p0) < per ? (P - p0) : static_cast<int>(per);
    row_select_kernel<<<(Bc + 255) / 256, 256, 0, s>>>(positions, win_start, nullptr, p0, Bc, h->row_sel);
    int rc = forward_msa(h, tokens, R, C_full, positions, win_start, p0, Bc, Cw, s, h->row_sel);
    if (rc) return fail(h, rc, tls_error());
    rc = compact_head(h, 1, Bc, out_logprobs + static_cast<long long>(p0) * h->desc.vocab, 5, s);  // + row_select_kernel, row-0 gather
    if (rc) return fail(h, rc, tls_error());
  }
  return PG_OK;
}

int pg_forward_logprobs(pg_handle h, const int32_t* tokens, int32_t n_tokens, int32_t win_start, int32_t T, int32_t mask_pos,
                        float* out_logprobs, pg_stream stream) {
  if (!h) return set_error(PG_ERR_ARG, "pg_forward_logprobs: null handle");
  if (!h->loaded) return fail(h, PG_ERR_STATE, "pg_forward_logprobs: weights not loaded");
  if (is_ar(h->desc.arch)) return fail(h, PG_ERR_STATE, "pg_forward_logprobs: handle is an autoregressive model (use pg_ar_loglik)");
  if (h->desc.arch == PG_ARCH_MSA) return fail(h, PG_ERR_STATE, "pg_forward_logprobs: handle is an MSA Transformer (use pg_msa_masked_marginals)");
  if (!tokens || !out_logprobs || T <= 0 || win_start < 0 || win_start + T > n_tokens) return fail(h, PG_ERR_ARG, "pg_forward_logprobs: bad arguments");
  if (h->desc.arch == PG_ARCH_ESM1B && T > h->desc.max_positions) return fail(h, PG_ERR_ARG, "pg_forward_logprobs: sequence longer than the learned position table");
  if ((h->desc.arch == PG_ARCH_ESM2 || h->desc.arch == PG_ARCH_ESMC) && T > h->rot_rows)
    return fail(h, PG_ERR_ARG, "pg_forward_logprobs: sequence longer than rotary tables");
  if (T > h->max_rows) return fail(h, PG_ERR_ARG, "pg_forward_logprobs: sequence longer than workspace");
  PG_CUDA_OK(cudaSetDevice(h->desc.device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // one row: positions / win_start as 1-element device arrays kept in row_sel scratch
  int32_t hostv[2] = {mask_pos, win_start};
  PG_CUDA_OK(cudaMemcpyAsync(h->row_sel, hostv, sizeof(hostv), cudaMemcpyHostToDevice, s));
  int rc = forward_rows(h, tokens, n_tokens, h->row_sel, h->row_sel + 1, 0, 1, T, s);
  if (rc) return fail(h, rc, tls_error());
  for (int r0 = 0; r0 < T; r0 += h->head_cap) {
    HeadLaunch hl = head_args(h, T);
    hl.x = h->x + static_cast<long long>(r0) * h->desc.embed_dim;
    hl.P = (T - r0) < h->head_cap ? (T - r0) : h->head_cap; hl.all_rows = 1;
    hl.out = out_logprobs + static_cast<long long>(r0) * h->desc.vocab;
    { ProfScope ps(CAT_HEAD, s, 3); rc = launch_head(hl, s); }
    if (rc) return fail(h, rc, tls_error());
  }
  return PG_OK;
}

static int ar_fusion_args(pg_handle h, const pg_ar_fusion* f, ArFusion* base) {
  if (!f) return PG_OK;
  if ((f->log_prior == nullptr) != (f->prior_row == nullptr)) return fail(h, PG_ERR_ARG, "pg_ar_loglik: log_prior and prior_row go together");
  if ((f->log_prior2 == nullptr) != (f->prior_row2 == nullptr)) return fail(h, PG_ERR_ARG, "pg_ar_loglik: log_prior2 and prior_row2 go together");
  if (f->log_prior2 && !f->log_prior) return fail(h, PG_ERR_ARG, "pg_ar_loglik: the second prior needs the first (it is fused inside the MSA overlap)");
  if (f->first_col < 0 || f->first_col > h->desc.vocab) return fail(h, PG_ERR_ARG, "pg_ar_loglik: first_col outside the vocabulary");
  if (h->desc.arch == PG_ARCH_RITA && (f->log_prior || f->log_prior2))
    return fail(h, PG_ERR_ARG, "pg_ar_loglik: RITA has no retrieval fusion (pass no log_prior / log_prior2)");
  if (h->desc.arch == PG_ARCH_PROGEN2 && (f->log_prior || f->log_prior2))
    return fail(h, PG_ERR_ARG, "pg_ar_loglik: ProGen2 has no retrieval fusion (pass no log_prior / log_prior2)");
  if (h->desc.arch == PG_ARCH_PROTGPT2 && (f->log_prior || f->log_prior2))
    return fail(h, PG_ERR_ARG, "pg_ar_loglik: ProtGPT2 has no retrieval fusion (pass no log_prior / log_prior2)");
  base->log_prior = f->log_prior; base->prior_row = f->prior_row; base->alpha = f->alpha;
  base->log_prior2 = f->log_prior2; base->prior_row2 = f->prior_row2; base->beta = f->beta;
  base->first_col = f->first_col; base->out_logprobs = f->out_logprobs;
  return PG_OK;
}

int pg_ar_loglik_fused(pg_handle h, const int32_t* ids, const int32_t* lens, int32_t B, int32_t T, const pg_ar_fusion* f,
                       float* out_sum_logp, pg_stream stream) {
  if (!h) return set_error(PG_ERR_ARG, "pg_ar_loglik: null handle");
  if (!h->loaded) return fail(h, PG_ERR_STATE, "pg_ar_loglik: weights not loaded");
  if (!is_ar(h->desc.arch)) return fail(h, PG_ERR_STATE, "pg_ar_loglik: handle is not an autoregressive model (Tranception, RITA, ProGen2)");
  if (B < 0 || T <= 0) return fail(h, PG_ERR_ARG, "pg_ar_loglik: bad B/T");
  if (B == 0) return PG_OK;
  if (!ids || !lens || !out_sum_logp) return fail(h, PG_ERR_ARG, "pg_ar_loglik: null buffer");
  ArFusion base;
  { int frc = ar_fusion_args(h, f, &base); if (frc) return frc; }
  if (T > h->desc.max_positions) return fail(h, PG_ERR_ARG, "pg_ar_loglik: sequence longer than n_ctx");
  if (T > h->max_rows) return fail(h, PG_ERR_ARG, "pg_ar_loglik: sequence longer than workspace");
  PG_CUDA_OK(cudaSetDevice(h->desc.device));
  return ar_passes(h, ids, lens, B, T, 0, 0, base, out_sum_logp, static_cast<cudaStream_t>(stream));
}

int pg_ar_prefix_begin(pg_handle h, const int32_t* ids, int32_t T, const pg_ar_fusion* f, float* out_tok_logp, pg_stream stream) {
  if (!h) return set_error(PG_ERR_ARG, "pg_ar_prefix_begin: null handle");
  if (!h->loaded) return fail(h, PG_ERR_STATE, "pg_ar_prefix_begin: weights not loaded");
  if (!is_ar(h->desc.arch))
    return fail(h, PG_ERR_STATE, "pg_ar_prefix_begin: handle is not an autoregressive model (Tranception, RITA, ProGen2)");
  if (!ids || !out_tok_logp || T < 2) return fail(h, PG_ERR_ARG, "pg_ar_prefix_begin: bad arguments");
  if (T > h->desc.max_positions || T > h->max_rows) return fail(h, PG_ERR_ARG, "pg_ar_prefix_begin: sequence longer than n_ctx / workspace");
  ArFusion fu;
  int rc = ar_fusion_args(h, f, &fu);
  if (rc) return rc;
  PG_CUDA_OK(cudaSetDevice(h->desc.device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t ldq = static_cast<size_t>(h->op.ldq);
  if (h->prefix_cap < h->desc.max_positions) {  // first use: [layers][n_ctx][3da*np] fp16, twice (RITA, ProGen2: once, no conv look-back)
    const size_t n = static_cast<size_t>(h->desc.layers) * h->desc.max_positions * ldq;
    rc = h->desc.arch == PG_ARCH_TRANCEPTION ? dev_alloc(h, &h->raw_cache, n) : PG_OK;
    if (!rc) rc = dev_alloc(h, &h->kv_cache, n);
    if (rc) return rc;
    h->prefix_cap = h->desc.max_positions;
  }
  h->prefix_T = 0;
  rc = forward_ar(h, ids, 1, T, s, 1, 0);
  if (rc) return fail(h, rc, tls_error());
  // per-token log p(ids[t+1] | ids[<=t]) of the wild type, t = 0 .. T-2 (and the fused rows in f->out_logprobs when asked for)
  int32_t* len_dev = h->row_sel;
  PG_CUDA_OK(cudaMemcpyAsync(len_dev, &T, sizeof(int32_t), cudaMemcpyHostToDevice, s));
  { ProfScope ps(CAT_HEAD, s, h->desc.arch == PG_ARCH_PROTGPT2 ? 4 : 2);
    rc = ar_head(h, ids, len_dev, 1, T, fu, out_tok_logp, h->tok_logp, s); }
  if (rc) return fail(h, rc, tls_error());
  h->prefix_T = T;
  return PG_OK;
}

int pg_ar_loglik_prefix(pg_handle h, const int32_t* ids, const int32_t* lens, int32_t B, int32_t T, int32_t start, const pg_ar_fusion* f,
                        float* out_sum_logp, pg_stream stream) {
  if (!h) return set_error(PG_ERR_ARG, "pg_ar_loglik_prefix: null handle");
  if (!h->loaded) return fail(h, PG_ERR_STATE, "pg_ar_loglik_prefix: weights not loaded");
  if (!is_ar(h->desc.arch))
    return fail(h, PG_ERR_STATE, "pg_ar_loglik_prefix: handle is not an autoregressive model (Tranception, RITA, ProGen2)");
  if (h->prefix_T <= 0) return fail(h, PG_ERR_STATE, "pg_ar_loglik_prefix: no wild-type prefix recorded (call pg_ar_prefix_begin first)");
  if (start <= 0 || start % 128 || start >= h->prefix_T) return fail(h, PG_ERR_ARG, "pg_ar_loglik_prefix: start must be a positive multiple of 128 below the recorded length");
  if (B < 0 || T <= 0) return fail(h, PG_ERR_ARG, "pg_ar_loglik_prefix: bad B/T");
  if (B == 0) return PG_OK;
  if (!ids || !lens || !out_sum_logp) return fail(h, PG_ERR_ARG, "pg_ar_loglik_prefix: null buffer");
  if (start + T > h->desc.max_positions) return fail(h, PG_ERR_ARG, "pg_ar_loglik_prefix: sequence longer than n_ctx");
  if (T > h->max_rows) return fail(h, PG_ERR_ARG, "pg_ar_loglik_prefix: suffix longer than workspace");
  ArFusion base;
  int rc = ar_fusion_args(h, f, &base);
  if (rc) return rc;
  PG_CUDA_OK(cudaSetDevice(h->desc.device));
  return ar_passes(h, ids, lens, B, T, 2, start, base, out_sum_logp, static_cast<cudaStream_t>(stream));
}

int pg_ar_loglik(pg_handle h, const int32_t* ids, const int32_t* lens, int32_t B, int32_t T, const float* log_prior,
                 const int32_t* prior_row, float alpha, float* out_sum_logp, pg_stream stream) {
  pg_ar_fusion f = {};
  f.log_prior = log_prior; f.prior_row = prior_row; f.alpha = alpha;
  return pg_ar_loglik_fused(h, ids, lens, B, T, &f, out_sum_logp, stream);
}

int pg_score_mutants(const float* table, int32_t n_rows, int32_t vocab, const int32_t* site_row, const int32_t* site_wt,
                     const int32_t* site_mt, const int32_t* row_offsets, int32_t M, float* out_scores, pg_stream stream) {
  if (M < 0 || n_rows < 0 || vocab <= 0) return set_error(PG_ERR_ARG, "pg_score_mutants: bad sizes");
  if (M == 0) return PG_OK;
  if (!table || !site_row || !site_wt || !site_mt || !row_offsets || !out_scores) return set_error(PG_ERR_ARG, "pg_score_mutants: null buffer");
  ProfScope ps(CAT_SCORE, static_cast<cudaStream_t>(stream));
  return launch_score(table, n_rows, vocab, site_row, site_wt, site_mt, row_offsets, M, out_scores, static_cast<cudaStream_t>(stream));
}

int pg_set_tuning(const char* key, int32_t value) {
  if (!key) return set_error(PG_ERR_ARG, "pg_set_tuning: null key");
  if (std::string(key) == "gemm_kchunk") { set_gemm_kchunk(value); return PG_OK; }
  if (std::string(key) == "gemm_prefetch") { set_gemm_prefetch(value); return PG_OK; }
  if (std::string(key) == "gemm_cta2") { set_gemm_cta2(value); return PG_OK; }
  return set_error(PG_ERR_ARG, std::string("pg_set_tuning: unknown key ") + key);
}

int pg_gemm(const pg_gemm_args* a, pg_stream stream) {
  if (!a) return set_error(PG_ERR_ARG, "pg_gemm: null args");
  GemmLaunch g{};
  g.a = a->a; g.lda = a->lda; g.w = a->w; g.ldw = a->ldw; g.bias = a->bias;
  g.M = a->M; g.N = a->N; g.K = a->K; g.nseg = a->nseg; g.epi = a->epi;
  g.out = static_cast<__half*>(a->out_h); g.ldo = a->ldo; g.out_lo_off = a->out_lo_off;
  g.resid = a->resid; g.ldr = a->ldr;
  g.rot_cos = a->rot_cos; g.rot_sin = a->rot_sin; g.rot_T = a->rot_T; g.rot_dim = a->rot_dim;
  g.a_scale = a->a_scale; g.w_inv = a->w_inv; g.out_scale = a->out_scale;
  g.out_fmt = a->out_fmt ? a->out_fmt : (a->out_lo_off > 0 ? 1 : 0);
  g.grp_rows_a = a->grp_rows_a; g.grp_rows_b = a->grp_rows_b;
  g.base_pre = a->base_pre; g.base_post = static_cast<const __half*>(a->base_post); g.base_T = a->base_T; g.mask_pos = a->mask_pos;
  ProfScope ps(CAT_OTHER, static_cast<cudaStream_t>(stream));
  return launch_gemm(g, static_cast<cudaStream_t>(stream));
}

int pg_layernorm_f16(const float* x, int64_t ldx, const float* gamma, const float* beta, int32_t rows, int32_t d, void* out,
                     int64_t ldo, int64_t lo_off, int32_t fmt, float scale, pg_stream stream) {
  if (!x || !gamma || !beta || !out) return set_error(PG_ERR_ARG, "pg_layernorm_f16: null buffer");
  return launch_layernorm_f16(x, ldx, gamma, beta, rows, d, static_cast<__half*>(out), ldo, lo_off, static_cast<cudaStream_t>(stream),
                              fmt ? fmt : -1, scale);
}

int pg_pack_weight(const float* w, int32_t N, int32_t K, int32_t fmt, void* out, float* w_inv, pg_stream stream) {
  if (!w || !out || N <= 0 || K <= 0) return set_error(PG_ERR_ARG, "pg_pack_weight: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (fmt == 2) {
    if (!w_inv) return set_error(PG_ERR_ARG, "pg_pack_weight: fmt 2 needs w_inv[N]");
    // the matrix maximum is accumulated in w_inv[0]'s storage (as bits) before the pack kernel overwrites it with 1 / t... a separate
    // word is cleaner: the last row's slot is written last by its own warp only, so use a small static scratch per device instead
    static unsigned int* scratch[64] = {};
    int dev = 0;
    PG_CUDA_OK(cudaGetDevice(&dev));
    if (dev >= 64) return set_error(PG_ERR_UNSUPPORTED, "pg_pack_weight: device ordinal >= 64");
    if (!scratch[dev]) PG_CUDA_OK(cudaMalloc(&scratch[dev], 256));
    pack_weights({w}, N, K, K, 1, 2, scratch[dev], static_cast<__half*>(out), w_inv, s);
  } else if (fmt == 0 || fmt == 1) {
    pack_weights({w}, N, K, K, 1, fmt + 1, nullptr, static_cast<__half*>(out), nullptr, s);
  } else {
    return set_error(PG_ERR_ARG, "pg_pack_weight: fmt must be 0, 1 or 2");
  }
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int pg_attention(const pg_attn_args* a, pg_stream stream) {
  if (!a || !a->qkv || !a->out) return set_error(PG_ERR_ARG, "pg_attention: null args");
  AttnLaunch l{};
  l.qkv = static_cast<const __half*>(a->qkv); l.ld = a->ld; l.lo_off = a->lo_off;
  l.out = static_cast<__half*>(a->out); l.ldo = a->ldo; l.out_lo_off = a->out_lo_off;
  l.B = a->B; l.T = a->T; l.heads = a->heads; l.nseg = a->nseg; l.causal = a->causal; l.alibi_slopes = a->alibi_slopes;
  l.out_fmt = a->out_fmt ? a->out_fmt : -1; l.out_scale = a->out_scale;
  l.base_o = static_cast<const __half*>(a->base_o); l.mask_pos = a->mask_pos; l.cout = static_cast<__half*>(a->cout); l.ldc = a->ldc; l.c_lo_off = a->c_lo_off;
  if ((l.base_o || l.mask_pos) && a->impl != 0) return set_error(PG_ERR_UNSUPPORTED, "pg_attention: the delta-operand form needs impl 0");
  ProfScope ps(CAT_OTHER, static_cast<cudaStream_t>(stream));
  if (a->impl == 0) return launch_attention_wgmma(l, static_cast<cudaStream_t>(stream));   // the model's kernel
  if (a->impl != 1) return set_error(PG_ERR_ARG, "pg_attention: impl must be 0 (the model's wgmma kernel) or 1 (mma.sync cross-check)");
  if (l.out_fmt == 2) return set_error(PG_ERR_UNSUPPORTED, "pg_attention: the mma.sync cross-check kernel writes fp16 planes only");
  return launch_attention(l, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
