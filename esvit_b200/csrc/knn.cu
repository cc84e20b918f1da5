// Exact weighted k-NN classifier over frozen features (eval_knn.py:193-232): bf16 tensor-core similarities, exact fp32
// neighbours.
//
//   esvit_knn_prep    fp32 features -> bf16 copy (zero-padded rows) + fp32 row norms + their maximum, one read
//   (similarities)    S = test . train^T through esvit_gemm_bf16 (bf16 out), chunked by the caller
//   esvit_knn_select  per test row: k-th largest bf16 similarity tau by a two-pass radix select on the 16-bit key,
//                     every column with S >= tau - 2 delta_i collected, rescored in fp32 from the fp32 rows, top-k by
//                     (value desc, index asc)
//   esvit_knn_vote    per test row: sum of exp(s / T) per class in neighbour-rank order, rank of the true class by
//                     (score desc, class asc) -> top-1 / top-5 hit counts (integer atomics)
//
// delta_i = (3u + 4u^2 + D 2^-23) ||a_i|| max_j ||b_j||, u = 2^-8, bounds |S_bf16 - a_i . b_j| (DESIGN.md §4.4), so the
// candidate set holds every true top-k member.  No floating-point atomics: results are bit-reproducible.
#include "common.cuh"

namespace {

constexpr int PREP_THREADS = 256;  // one warp per row
constexpr int SEL_THREADS = 512;
constexpr int SEL_WARPS = SEL_THREADS / 32;
constexpr int RANK_TILE = 1024;    // candidates staged in shared memory per pass of the rank count
constexpr int VOTE_THREADS = 256;
constexpr int MAX_CLASSES = 11264; // class scores: 44 KB of shared memory, under the 48 KB that needs no opt-in

// order-preserving 16-bit key of a bf16 bit pattern (larger key = larger value) and back
__device__ __forceinline__ unsigned key16(unsigned h) { return (h & 0x8000u) ? (~h & 0xffffu) : (h | 0x8000u); }
__device__ __forceinline__ float key_to_float(unsigned k) {
  const unsigned h = (k & 0x8000u) ? (k & 0x7fffu) : (~k & 0xffffu);
  return __uint_as_float(h << 16);
}

__global__ void __launch_bounds__(PREP_THREADS) prep_kernel(const float* __restrict__ x, bf16* __restrict__ xb,
                                                            float* __restrict__ norm, unsigned* __restrict__ max_bits,
                                                            long long R, long long R_pad, int D) {
  const int lane = threadIdx.x & 31;
  const long long nw = (long long)gridDim.x * (PREP_THREADS / 32);
  for (long long r = (long long)blockIdx.x * (PREP_THREADS / 32) + (threadIdx.x >> 5); r < R_pad; r += nw) {
    uint2* yr = reinterpret_cast<uint2*>(xb + r * D);
    if (r >= R) {  // the GEMM's N % 8 padding rows
      for (int e = 4 * lane; e < D; e += 128) yr[e / 4] = make_uint2(0u, 0u);
      continue;
    }
    const float4* xr = reinterpret_cast<const float4*>(x + r * D);
    float s = 0.f;
    for (int e = 4 * lane; e < D; e += 128) {
      const float4 v = xr[e / 4];
      s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
      yr[e / 4] = make_uint2(pack_bf162(v.x, v.y), pack_bf162(v.z, v.w));
    }
    s = warp_sum(s);
    if (lane == 0) {
      const float nr = sqrtf(s);
      norm[r] = nr;
      atomicMax(max_bits, __float_as_uint(nr));  // non-negative floats order like their bit patterns
    }
  }
}

// histogram of 8 bits of the keys of one bf16 row into per-warp bins, optionally only over keys whose high byte is `hi`
template <bool LOW>
__device__ __forceinline__ void row_hist(const uint4* __restrict__ row, int N, unsigned hi, unsigned (*hist)[256],
                                         unsigned* tot) {
  const int warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < SEL_WARPS * 256; i += SEL_THREADS) (&hist[0][0])[i] = 0u;
  __syncthreads();
  const int nv = (N + 7) / 8;
  for (int v = threadIdx.x; v < nv; v += SEL_THREADS) {
    const uint4 q = row[v];
    const unsigned w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < 8; j++) {
      if (8 * v + j >= N) break;
      const unsigned key = key16((w[j / 2] >> (16 * (j & 1))) & 0xffffu);
      if (!LOW) atomicAdd(&hist[warp][key >> 8], 1u);
      else if ((key >> 8) == hi) atomicAdd(&hist[warp][key & 255u], 1u);
    }
  }
  __syncthreads();
  if (threadIdx.x < 256) {
    unsigned s = 0;
    for (int w = 0; w < SEL_WARPS; w++) s += hist[w][threadIdx.x];
    tot[threadIdx.x] = s;
  }
  __syncthreads();
}

// the bin holding the `rank`-th largest key (1-based) and the rank inside it
__device__ __forceinline__ void pick_bin(const unsigned* tot, unsigned rank, int* bin, unsigned* rem) {
  unsigned above = 0;
  int b = 255;
  for (; b > 0; b--) {
    if (above + tot[b] >= rank) break;
    above += tot[b];
  }
  *bin = b;
  *rem = rank - above;
}

// One CTA per test row r = rows ? rows[blockIdx.x] : blockIdx.x.  Scratch cand_idx / cand_val hold `cap` slots per CTA.
// count[r] = number of candidates; when it exceeds cap the row's sims / idx are left unwritten (the host reruns it).
__global__ void __launch_bounds__(SEL_THREADS, 2)
select_kernel(const bf16* __restrict__ S, long long ld, const float* __restrict__ a, const float* __restrict__ b,
              const float* __restrict__ a_norm, const float* __restrict__ max_norm, const int* __restrict__ rows,
              int N, int D, int k, int cap, float coef, int* __restrict__ cand_idx, float* __restrict__ cand_val,
              int* __restrict__ count, float* __restrict__ sims, long long* __restrict__ idx) {
  __shared__ unsigned hist[SEL_WARPS][256];
  __shared__ unsigned tot[256];
  __shared__ float tile_v[RANK_TILE];
  __shared__ int tile_i[RANK_TILE];
  __shared__ int s_bin;
  __shared__ unsigned s_rem;
  __shared__ int s_cnt;
  const int r = rows ? rows[blockIdx.x] : blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint4* row = reinterpret_cast<const uint4*>(S + (long long)r * ld);

  // 1. tau = the k-th largest bf16 value: high byte, then low byte inside the chosen bin
  row_hist<false>(row, N, 0u, hist, tot);
  if (tid == 0) { int bn; unsigned rem; pick_bin(tot, (unsigned)k, &bn, &rem); s_bin = bn; s_rem = rem; }
  __syncthreads();
  const unsigned hi = (unsigned)s_bin;
  row_hist<true>(row, N, hi, hist, tot);
  if (tid == 0) { int bn; unsigned rem; pick_bin(tot, s_rem, &bn, &rem); s_bin = bn; s_cnt = 0; }
  __syncthreads();
  const float tau = key_to_float((hi << 8) | (unsigned)s_bin);
  const float thr = tau - 2.f * (coef * a_norm[r] * max_norm[0]);

  // 2. collect every column with S >= tau - 2 delta (warp-aggregated slot allocation)
  int* ci = cand_idx + (long long)blockIdx.x * cap;
  float* cv = cand_val + (long long)blockIdx.x * cap;
  const int nv = (N + 7) / 8;
  for (int v0 = 0; v0 < nv; v0 += SEL_THREADS) {
    const int v = v0 + tid;
    uint4 q = make_uint4(0u, 0u, 0u, 0u);
    if (v < nv) q = row[v];
    const unsigned w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const int col = 8 * v + j;
      const bool take = v < nv && col < N && __uint_as_float(((w[j / 2] >> (16 * (j & 1))) & 0xffffu) << 16) >= thr;
      const unsigned m = __ballot_sync(0xffffffffu, take);
      if (m == 0u) continue;
      const int leader = __ffs(m) - 1;
      int base = 0;
      if (lane == leader) base = atomicAdd(&s_cnt, __popc(m));
      base = __shfl_sync(0xffffffffu, base, leader);
      const int pos = base + __popc(m & ((1u << lane) - 1u));
      if (take && pos < cap) ci[pos] = col;
    }
  }
  __syncthreads();
  const int cnt = s_cnt;
  if (tid == 0) count[r] = cnt;
  if (cnt > cap) return;

  // 3. rescore in fp32 from the fp32 rows: one warp per candidate, fixed lane order and reduction tree
  const float4* ar = reinterpret_cast<const float4*>(a + (long long)r * D);
  for (int c = warp; c < cnt; c += SEL_WARPS) {
    const float4* br = reinterpret_cast<const float4*>(b + (long long)ci[c] * D);
    float s = 0.f;
    for (int e = 4 * lane; e < D; e += 128) {
      const float4 x = ar[e / 4], y = br[e / 4];
      s = fmaf(x.x, y.x, s); s = fmaf(x.y, y.y, s); s = fmaf(x.z, y.z, s); s = fmaf(x.w, y.w, s);
    }
    s = warp_sum(s);
    if (lane == 0) cv[c] = s;
  }
  __syncthreads();

  // 4. top-k: a candidate's output slot is the number of candidates ahead of it by (value desc, index asc)
  for (int c0 = 0; c0 < cnt; c0 += SEL_THREADS) {
    const int c = c0 + tid;
    const bool mine = c < cnt;
    const float val = mine ? cv[c] : 0.f;
    const int col = mine ? ci[c] : 0;
    int ahead = 0;
    for (int t0 = 0; t0 < cnt; t0 += RANK_TILE) {
      const int nt = min(RANK_TILE, cnt - t0);
      __syncthreads();
      for (int t = tid; t < nt; t += SEL_THREADS) { tile_v[t] = cv[t0 + t]; tile_i[t] = ci[t0 + t]; }
      __syncthreads();
      for (int t = 0; t < nt; t++) {
        const float u = tile_v[t];
        ahead += (u > val) || (u == val && tile_i[t] < col);
      }
    }
    if (mine && ahead < k) {
      sims[(long long)r * k + ahead] = val;
      idx[(long long)r * k + ahead] = col;
    }
  }
}

__global__ void __launch_bounds__(VOTE_THREADS) vote_kernel(const float* __restrict__ sims,
                                                            const long long* __restrict__ idx,
                                                            const long long* __restrict__ train_labels,
                                                            const long long* __restrict__ test_labels, int k, float T,
                                                            int C, unsigned long long* __restrict__ hits) {
  extern __shared__ float score[];
  __shared__ float w_t[VOTE_THREADS];
  __shared__ int lab_t[VOTE_THREADS];
  __shared__ int red[VOTE_THREADS / 32];
  const long long r = blockIdx.x;
  const int tid = threadIdx.x;
  for (int c = tid; c < C; c += VOTE_THREADS) score[c] = 0.f;
  // weights exp(s / T) added per class in neighbour-rank order (one thread: a fixed summation order)
  for (int j0 = 0; j0 < k; j0 += VOTE_THREADS) {
    const int j = j0 + tid;
    if (j < k) {
      w_t[tid] = expf(sims[r * k + j] / T);
      lab_t[tid] = (int)train_labels[idx[r * k + j]];
    }
    __syncthreads();
    if (tid == 0) {
      const int n = min(VOTE_THREADS, k - j0);
      for (int t = 0; t < n; t++) score[lab_t[t]] += w_t[t];
    }
    __syncthreads();
  }
  // rank of the true class by (score desc, class asc): the order of a stable descending sort
  const int tc = (int)test_labels[r];
  const float st = score[tc];
  int ahead = 0;
  for (int c = tid; c < C; c += VOTE_THREADS) {
    const float u = score[c];
    ahead += (u > st) || (u == st && c < tc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ahead += __shfl_xor_sync(0xffffffffu, ahead, o);
  if ((tid & 31) == 0) red[tid >> 5] = ahead;
  __syncthreads();
  if (tid == 0) {
    int a = 0;
    for (int w = 0; w < VOTE_THREADS / 32; w++) a += red[w];
    if (a < 1) atomicAdd(&hits[0], 1ull);
    if (a < 5) atomicAdd(&hits[1], 1ull);
  }
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

}  // namespace

// ---- C ABI ----------------------------------------------------------------------------------------------------------
ESVIT_API int esvit_knn_prep(const float* x, void* xb, float* norm, float* max_norm, long long R, long long R_pad, int D,
                             void* stream) {
  if (R <= 0 || R_pad < R || D <= 0 || (D % 8) || !x || !xb || !norm || !max_norm || !aligned16(x) || !aligned16(xb))
    return ESVIT_ERR_BAD_ARG;
  const long long blocks = (R_pad + PREP_THREADS / 32 - 1) / (PREP_THREADS / 32);
  const int grid = (int)(blocks < 8LL * esvit_num_sms() ? blocks : 8LL * esvit_num_sms());
  prep_kernel<<<grid, PREP_THREADS, 0, (cudaStream_t)stream>>>(x, (bf16*)xb, norm, (unsigned*)max_norm, R, R_pad, D);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_knn_select(const void* S, long long ld, const float* a, const float* b, const float* a_norm,
                               const float* max_norm, const int* rows, int nrows, int N, int D, int k, int cap,
                               int* cand_idx, float* cand_val, int* count, float* sims, long long* idx, void* stream) {
  if (nrows <= 0 || N <= 0 || D <= 0 || (D % 8) || k <= 0 || k > N || cap < k || ld < N || (ld % 8) || !S || !a || !b ||
      !a_norm || !max_norm || !cand_idx || !cand_val || !count || !sims || !idx || !aligned16(S) || !aligned16(a) ||
      !aligned16(b))
    return ESVIT_ERR_BAD_ARG;
  const double u = 1.0 / 256.0;  // bf16 unit roundoff
  const float coef = (float)(3.0 * u + 4.0 * u * u + (double)D * 0x1p-23);
  select_kernel<<<nrows, SEL_THREADS, 0, (cudaStream_t)stream>>>((const bf16*)S, ld, a, b, a_norm, max_norm, rows, N, D,
                                                                 k, cap, coef, cand_idx, cand_val, count, sims, idx);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_knn_vote(const float* sims, const long long* idx, const long long* train_labels,
                             const long long* test_labels, long long M, int k, float T, int num_classes,
                             long long* hits, void* stream) {
  if (M <= 0 || M > 0x7fffffffLL || k <= 0 || !(T > 0.f) || num_classes <= 0 || num_classes > MAX_CLASSES || !sims ||
      !idx || !train_labels || !test_labels || !hits)
    return ESVIT_ERR_BAD_ARG;
  vote_kernel<<<(unsigned)M, VOTE_THREADS, num_classes * sizeof(float), (cudaStream_t)stream>>>(
      sims, idx, train_labels, test_labels, k, T, num_classes, (unsigned long long*)hits);
  ESVIT_LAUNCH_CHECK();
}
