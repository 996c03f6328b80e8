// ProGen3's sparse mixture-of-experts half of a layer (progen3/model/moe.py:62-134) around the ragged grouped GEMM (gemm_tc.cu):
//
//   rms_router_kernel    RMSNorm (flash-attn rms_norm_fn: x * rsqrt(mean(x^2) + eps) * w, fp32) of one token row -> the GEMM operand
//                        row; with a gate: E fp32 router logits of the fp32 normalised row (not on the tensor cores: routing is a
//                        discrete decision), softmax, top-k, renormalisation -> (expert, weight) per (token, k)
//   moe_rank_kernel      per block of 1024 (token, k) entries in token order: each entry's rank among the block's entries of its expert
//                        and the block's per-expert counts (warp match + per-warp counts: no atomics, so the order is fixed)
//   moe_scan_kernel      one block: per-expert block offsets, segment sizes padded to the GEMM tile height, segment starts and the
//                        tile table (expert of every tile) with its length, all on the device
//   moe_permute_kernel   every entry's operand row into its slot of the expert-grouped buffer (slot = segment start + block offset + rank)
//   moe_combine_kernel   x[t] += ((0 + w_a * y_a) + w_b * y_b) + ... over the token's experts in increasing index order, as index_add_
//                        accumulates them; one thread per element, so the result does not depend on how rows are split into passes
// All arithmetic is fp32; products and sums are rounded separately (no FMA contraction) where they mirror the reference's tensor ops.
#include "common.h"
#include "operand.cuh"
#include "reduce.cuh"

namespace pg {

namespace {

constexpr int RANK_BLOCK = 1024;  // entries per moe_rank_kernel block

// torch.topk(p, K) on the CPU (ATen TopKImpl.h, largest, sorted), reproduced step for step so that equal probabilities pick the same
// experts: (value, index) pairs compared by value only (a > b); K * 64 <= E: std::partial_sort to K; otherwise std::nth_element to
// K - 1 (libstdc++ introselect: median-of-three pivot, unguarded partition, heap select past the depth limit, insertion sort below four
// elements) and std::sort of the first K - 1 (insertion sort: K <= 8). For example, eight equal probabilities give experts 6, 5, 4, 7.
// One thread; x = value, y = index bits.
struct TopKSelect {
  float2 v[64];
  __device__ static bool gt(float2 a, float2 b) { return a.x > b.x; }
  __device__ void sw(int i, int j) { const float2 t = v[i]; v[i] = v[j]; v[j] = t; }
  __device__ void push_heap(int first, int hole, int top, float2 val) {
    int parent = (hole - 1) / 2;
    while (hole > top && gt(v[first + parent], val)) { v[first + hole] = v[first + parent]; hole = parent; parent = (hole - 1) / 2; }
    v[first + hole] = val;
  }
  __device__ void adjust_heap(int first, int hole, int len, float2 val) {
    const int top = hole;
    int child = hole;
    while (child < (len - 1) / 2) {
      child = 2 * (child + 1);
      if (gt(v[first + child], v[first + child - 1])) --child;
      v[first + hole] = v[first + child];
      hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
      child = 2 * (child + 1);
      v[first + hole] = v[first + child - 1];
      hole = child - 1;
    }
    push_heap(first, hole, top, val);
  }
  __device__ void heap_select(int first, int middle, int last) {
    const int len = middle - first;
    if (len >= 2)
      for (int parent = (len - 2) / 2;; --parent) {
        adjust_heap(first, parent, len, v[first + parent]);
        if (parent == 0) break;
      }
    for (int i = middle; i < last; ++i)
      if (gt(v[i], v[first])) {  // pop_heap(first, middle, i)
        const float2 val = v[i];
        v[i] = v[first];
        adjust_heap(first, 0, len, val);
      }
  }
  __device__ void insertion_sort(int first, int last) {
    for (int i = first + 1; i < last; ++i) {
      const float2 val = v[i];
      if (gt(val, v[first])) {
        for (int j = i; j > first; --j) v[j] = v[j - 1];
        v[first] = val;
      } else {
        int j = i;
        while (gt(val, v[j - 1])) { v[j] = v[j - 1]; --j; }
        v[j] = val;
      }
    }
  }
  __device__ void select(int n, int k) {
    if (k * 64 <= n) {  // std::partial_sort(0, k, n): heap select, then sort_heap (k == 1 here: a one-element heap)
      heap_select(0, k, n);
      return;
    }
    const int nth = k - 1;
    int first = 0, last = n, depth = 2 * (31 - __clz(n));
    bool heap = false;
    while (last - first > 3) {
      if (depth == 0) {
        heap_select(first, nth + 1, last);
        sw(first, nth);
        heap = true;
        break;
      }
      --depth;
      const int a = first + 1, b = first + (last - first) / 2, c = last - 1;  // median of three to `first`
      if (gt(v[a], v[b])) {
        if (gt(v[b], v[c])) sw(first, b);
        else if (gt(v[a], v[c])) sw(first, c);
        else sw(first, a);
      } else if (gt(v[a], v[c])) sw(first, a);
      else if (gt(v[b], v[c])) sw(first, c);
      else sw(first, b);
      int lo = first + 1, hi = last;  // unguarded partition around v[first]
      while (true) {
        while (gt(v[lo], v[first])) ++lo;
        --hi;
        while (gt(v[first], v[hi])) --hi;
        if (!(lo < hi)) break;
        sw(lo, hi);
        ++lo;
      }
      if (lo <= nth) first = lo;
      else last = lo;
    }
    if (!heap) insertion_sort(first, last);
    insertion_sort(0, k - 1);  // std::sort of the first k - 1
  }
};

// One block (128 threads) per token row; dynamic shared memory: the fp32 normalised row [d] and the logits [E].
__global__ void __launch_bounds__(128) rms_router_kernel(MoeRouteLaunch r) {
  extern __shared__ float dyn[];
  __shared__ float sh[33];
  float* y = dyn;
  float* lg = dyn + r.d;
  const long long row = blockIdx.x;
  const float* xr = r.x + row * r.d;
  float ss = 0.f;
  for (int j = threadIdx.x; j < r.d; j += blockDim.x) ss += xr[j] * xr[j];
  ss = block_sum(ss, sh);
  const float rstd = rsqrtf(ss / r.d + r.eps);
  __half* orow = r.out + row * r.ldo;
  for (int j = threadIdx.x * 4; j < r.d; j += blockDim.x * 4) {
    float v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      v[i] = __fmul_rn(__fmul_rn(xr[j + i], rstd), r.gamma[j + i]);
      y[j + i] = v[i];
    }
    store_operand_quad(orow, r.lo_off, r.d, r.fmt, r.scale, j, v);
  }
  if (!r.route_e) return;
  const int E = r.E, K = r.K;
  __syncthreads();
  if (E > 1) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int e = warp; e < E; e += blockDim.x >> 5) {
      const float* w = r.gate + static_cast<long long>(e) * r.d;
      float a = 0.f;
      for (int j = lane; j < r.d; j += 32) a = fmaf(y[j], w[j], a);
      a = warp_sum(a);
      if (lane == 0) lg[e] = a;
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  int32_t* oe = r.route_e + row * K;
  float* ow = r.route_w + row * K;
  if (E == 1) {  // no gate: the single expert with weight 1 (moe.py:81-88)
    oe[0] = 0;
    ow[0] = 1.f;
    return;
  }
  // softmax in fp32 (SoftmaxMixIn), then torch.topk's CPU selection (TopKSelect below), then renormalisation
  float m = -INFINITY;
  for (int e = 0; e < E; ++e) m = fmaxf(m, lg[e]);
  float s = 0.f;
  for (int e = 0; e < E; ++e) {
    lg[e] = expf(lg[e] - m);
    s += lg[e];
  }
  TopKSelect q;
  for (int e = 0; e < E; ++e) q.v[e] = make_float2(lg[e] / s, __int_as_float(e));
  q.select(E, K);
  float tot = 0.f;
  for (int k = 0; k < K; ++k) {
    oe[k] = __float_as_int(q.v[k].y);
    ow[k] = q.v[k].x;
    tot += q.v[k].x;
  }
  for (int k = 0; k < K; ++k) ow[k] = ow[k] / tot;  // renormalised to sum 1 (moe.py:95)
}

__global__ void __launch_bounds__(RANK_BLOCK) moe_rank_kernel(const int32_t* __restrict__ route_e, int n, int E, int32_t* __restrict__ rank,
                                                              int32_t* __restrict__ hist) {
  __shared__ int32_t cnt[32][64];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 32 * 64; i += blockDim.x) cnt[i / 64][i % 64] = 0;
  __syncthreads();
  const long long i = static_cast<long long>(blockIdx.x) * RANK_BLOCK + threadIdx.x;
  const int e = i < n ? route_e[i] : -1;
  const unsigned peers = __match_any_sync(0xffffffffu, e);
  const int rw = __popc(peers & ((1u << lane) - 1u));
  if (e >= 0 && rw == 0) cnt[warp][e] = __popc(peers);
  __syncthreads();
  if (threadIdx.x < E) {  // exclusive prefix over the warps, per expert
    int run = 0;
    for (int w = 0; w < 32; ++w) {
      const int c = cnt[w][threadIdx.x];
      cnt[w][threadIdx.x] = run;
      run += c;
    }
    hist[static_cast<long long>(blockIdx.x) * E + threadIdx.x] = run;
  }
  __syncthreads();
  if (e >= 0) rank[i] = cnt[warp][e] + rw;
}

// One block of 64 threads. hist [nblk][E] in: block counts; out: exclusive block offsets within each expert's segment.
__global__ void moe_scan_kernel(int32_t* __restrict__ hist, int nblk, int E, int pad, int32_t* __restrict__ seg_start,
                                int32_t* __restrict__ tile_expert, int32_t* __restrict__ n_tiles) {
  __shared__ int32_t padded[64];
  const int e = threadIdx.x;
  int run = 0;
  if (e < E) {
    for (int b = 0; b < nblk; ++b) {
      const int c = hist[static_cast<long long>(b) * E + e];
      hist[static_cast<long long>(b) * E + e] = run;
      run += c;
    }
    padded[e] = (run + pad - 1) / pad * pad;
  }
  __syncthreads();
  if (e >= E) return;
  int start = 0;
  for (int j = 0; j < e; ++j) start += padded[j];
  seg_start[e] = start;
  for (int t = 0; t < padded[e] / pad; ++t) tile_expert[start / pad + t] = e;
  if (e == E - 1) *n_tiles = (start + padded[e]) / pad;
}

// One block per entry: 16-byte copies of the token's operand row into the entry's slot row.
__global__ void moe_permute_kernel(const int32_t* __restrict__ route_e, const int32_t* __restrict__ rank, const int32_t* __restrict__ hist,
                                   const int32_t* __restrict__ seg_start, int E, int K, const uint4* __restrict__ src, long long src_pitch,
                                   uint4* __restrict__ dst, int row_vecs, int32_t* __restrict__ slot_of) {
  const long long i = blockIdx.x;
  const int e = route_e[i];
  const int slot = seg_start[e] + hist[(i / RANK_BLOCK) * E + e] + rank[i];
  if (threadIdx.x == 0) slot_of[i] = slot;
  const uint4* s = src + (i / K) * src_pitch;
  uint4* o = dst + static_cast<long long>(slot) * src_pitch;
  for (int j = threadIdx.x; j < row_vecs; j += blockDim.x) o[j] = s[j];
}

constexpr int MAX_TOPK = 8;
__global__ void moe_combine_kernel(const float* __restrict__ y, int d, const int32_t* __restrict__ route_e, const float* __restrict__ route_w,
                                   const int32_t* __restrict__ slot_of, int K, float* __restrict__ x) {
  const long long t = blockIdx.x;
  int ex[MAX_TOPK], sl[MAX_TOPK];
  float wt[MAX_TOPK];
#pragma unroll
  for (int k = 0; k < MAX_TOPK; ++k) {
    if (k >= K) break;
    int e = route_e[t * K + k], s = slot_of[t * K + k];
    float w = route_w[t * K + k];
    int j = k;
    for (; j > 0 && ex[j - 1] > e; --j) { ex[j] = ex[j - 1]; sl[j] = sl[j - 1]; wt[j] = wt[j - 1]; }
    ex[j] = e; sl[j] = s; wt[j] = w;
  }
  float* xr = x + t * d;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float acc = 0.f;
    for (int k = 0; k < K; ++k) acc = __fadd_rn(acc, __fmul_rn(y[static_cast<long long>(sl[k]) * d + c], wt[k]));
    xr[c] = __fadd_rn(xr[c], acc);
  }
}

}  // namespace

int launch_moe_route(const MoeRouteLaunch& r, cudaStream_t s) {
  if (r.rows <= 0) return PG_OK;
  if (r.d % 4 || (r.route_e && (r.E < 1 || r.E > 64 || r.K < 1 || r.K > MAX_TOPK || r.K > r.E || (r.E > 1 && !r.gate))))
    return set_error(PG_ERR_ARG, "moe: d % 4 == 0, 1 <= top_k <= min(experts, 8), experts <= 64 and a gate when experts > 1");
  const size_t smem = (static_cast<size_t>(r.d) + 64) * sizeof(float);
  if (smem > 48 * 1024) PG_CUDA_OK(cudaFuncSetAttribute(rms_router_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  rms_router_kernel<<<static_cast<unsigned>(r.rows), 128, smem, s>>>(r);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int moe_ws_blocks(long long entries) { return static_cast<int>((entries + RANK_BLOCK - 1) / RANK_BLOCK); }

int launch_moe_dispatch(const MoeDispatchLaunch& m, cudaStream_t s) {
  const long long n = m.rows * m.K;
  if (n <= 0) return PG_OK;
  if ((m.pad != 128 && m.pad != 256) || m.row_bytes % 16 || m.pitch_bytes % 16)
    return set_error(PG_ERR_ARG, "moe: segments pad to 128 or 256 rows; operand rows are 16-byte multiples");
  const int nblk = moe_ws_blocks(n);
  moe_rank_kernel<<<nblk, RANK_BLOCK, 0, s>>>(m.route_e, static_cast<int>(n), m.E, m.rank, m.hist);
  moe_scan_kernel<<<1, 64, 0, s>>>(m.hist, nblk, m.E, m.pad, m.seg_start, m.tile_expert, m.n_tiles);
  moe_permute_kernel<<<static_cast<unsigned>(n), 128, 0, s>>>(m.route_e, m.rank, m.hist, m.seg_start, m.E, m.K,
                                                              static_cast<const uint4*>(m.src), m.pitch_bytes / 16, static_cast<uint4*>(m.dst),
                                                              m.row_bytes / 16, m.slot_of);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

int launch_moe_combine(const float* y, int d, const int32_t* route_e, const float* route_w, const int32_t* slot_of, long long rows, int K,
                       float* x, cudaStream_t s) {
  if (rows <= 0) return PG_OK;
  if (K < 1 || K > MAX_TOPK) return set_error(PG_ERR_ARG, "moe_combine: top_k must be 1..8");
  moe_combine_kernel<<<static_cast<unsigned>(rows), 256, 0, s>>>(y, d, route_e, route_w, slot_of, K, x);
  PG_CUDA_OK(cudaGetLastError());
  return PG_OK;
}

}  // namespace pg
