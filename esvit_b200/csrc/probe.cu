// Linear-probe cross-entropy (eval_linear.py:244-304 with utils.accuracy, utils.py:468-475): one pass over each fp32
// logit row for the loss, the logit gradient and the top-1 / top-5 hits, then a fixed-order batch reduction.
//
//   probe_ce_row_kernel   one CTA per row: the row staged once in shared memory; max, sum exp, lse, the target's rank
//                         by (value desc, index asc); dlogits = (softmax - onehot) / B_valid (bf16); loss and rank to
//                         per-row scratch
//   probe_ce_sum_kernel   one CTA: the batch's loss sum in row order (fp64), its mean, and the running accumulators
//
// B_valid is the number of rows with a label >= 0, counted on the device: rows labelled -1 are padding and contribute no
// loss, no hit and a zero gradient, so one captured graph serves any batch up to its captured size.  Classes [C, ld)
// are padding of the GEMMs' N % 8: they never enter the max, the sum, a rank or a gradient.  No floating-point atomics.
#include "common.cuh"

namespace {

constexpr int CE_THREADS = 256;
constexpr int CE_WARPS = CE_THREADS / 32;
constexpr int MAX_CLASSES = 12288;  // one row in shared memory: 48 KB, the limit that needs no opt-in

// block reductions in a fixed order: per-thread partials, a warp butterfly, then the warps' results in warp order
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < CE_WARPS; w++) r = fmaxf(r, red[w]);
  return r;
}
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < CE_WARPS; w++) r += red[w];
  return r;
}
__device__ __forceinline__ int block_count(int v, int* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int r = 0;
#pragma unroll
  for (int w = 0; w < CE_WARPS; w++) r += red[w];
  return r;
}

__global__ void __launch_bounds__(CE_THREADS) probe_ce_row_kernel(const float* __restrict__ logits, int ld,
                                                                  const long long* __restrict__ labels, int B, int C,
                                                                  bf16* __restrict__ dlogits,
                                                                  float* __restrict__ row_loss,
                                                                  int* __restrict__ row_rank) {
  extern __shared__ float row[];  // [C]
  __shared__ float redf[CE_WARPS];
  __shared__ int redi[CE_WARPS];
  const int r = blockIdx.x;
  int nv = 0;
  for (int i = threadIdx.x; i < B; i += CE_THREADS) nv += labels[i] >= 0;
  const int n_valid = block_count(nv, redi);
  const long long t = labels[r];
  bf16* dl = dlogits ? dlogits + (long long)r * ld : nullptr;
  if (t < 0 || t >= C) {  // padding row (labels >= C are rejected by the host wrapper): no loss, no rank, zero gradient
    if (dl)
      for (int j = threadIdx.x; j < ld; j += CE_THREADS) dl[j] = __float2bfloat16_rn(0.f);
    if (threadIdx.x == 0) { row_loss[r] = 0.f; row_rank[r] = -1; }
    return;
  }
  const float* x = logits + (long long)r * ld;
  float m = -INFINITY;
  for (int j = threadIdx.x; j < C; j += CE_THREADS) {
    const float v = x[j];
    row[j] = v;
    m = fmaxf(m, v);
  }
  m = block_max(m, redf);  // its barriers also publish row[]
  const float lt = row[t];
  float s = 0.f;
  int ahead = 0;
  for (int j = threadIdx.x; j < C; j += CE_THREADS) {
    const float v = row[j];
    s += expf(v - m);
    ahead += (v > lt) || (v == lt && j < t);
  }
  s = block_sum(s, redf);
  const int rank = block_count(ahead, redi);
  const float lse = m + logf(s);
  if (dl) {
    const float inv_b = __frcp_rn((float)n_valid);
    for (int j = threadIdx.x; j < ld; j += CE_THREADS) {
      float g = 0.f;
      if (j < C) g = (expf(row[j] - lse) - (j == t ? 1.f : 0.f)) * inv_b;
      dl[j] = __float2bfloat16_rn(g);
    }
  }
  if (threadIdx.x == 0) { row_loss[r] = lse - lt; row_rank[r] = rank; }
}

// acc: fp64 [1] += this batch's mean loss;  counts int64 [4] += {1 batch, B_valid images, top-1 hits, top-5 hits}
__global__ void __launch_bounds__(CE_THREADS) probe_ce_sum_kernel(const float* __restrict__ row_loss,
                                                                  const int* __restrict__ row_rank, int B,
                                                                  float* __restrict__ loss_out,
                                                                  double* __restrict__ acc,
                                                                  long long* __restrict__ counts) {
  __shared__ double redd[CE_THREADS];
  __shared__ int redi[3][CE_THREADS];
  double s = 0.0;
  int nv = 0, h1 = 0, h5 = 0;
  for (int i = threadIdx.x; i < B; i += CE_THREADS) {
    const int k = row_rank[i];
    if (k < 0) continue;
    s += (double)row_loss[i];
    nv++;
    h1 += k < 1;
    h5 += k < 5;
  }
  redd[threadIdx.x] = s;
  redi[0][threadIdx.x] = nv; redi[1][threadIdx.x] = h1; redi[2][threadIdx.x] = h5;
  __syncthreads();
  for (int o = CE_THREADS / 2; o > 0; o >>= 1) {  // fixed pairwise tree
    if (threadIdx.x < o) {
      redd[threadIdx.x] += redd[threadIdx.x + o];
      for (int q = 0; q < 3; q++) redi[q][threadIdx.x] += redi[q][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int n = redi[0][0];
    const float mean = n > 0 ? (float)(redd[0] / n) : 0.f;
    loss_out[0] = mean;
    if (n > 0 && acc) {
      acc[0] += (double)mean;
      counts[0] += 1;
      counts[1] += n;
      counts[2] += redi[1][0];
      counts[3] += redi[2][0];
    }
  }
}

}  // namespace

// logits fp32 [B, ld] (classes [0, C) used), labels int64 [B] in [0, C) or -1 (padding row).  dlogits bf16 [B, ld] or
// NULL (no gradient: validation); row_loss fp32 [B] and row_rank int32 [B] scratch; loss_out fp32 [1] = the batch's mean
// loss over its labelled rows; acc fp64 [1] and counts int64 [4] ACCUMULATE (mean loss | batches, images, top-1 hits,
// top-5 hits), or NULL.  C <= 12288, C <= ld, ld % 8 == 0.
ESVIT_API int esvit_probe_ce(const float* logits, int ld, const long long* labels, int B, int C, void* dlogits,
                             float* row_loss, int* row_rank, float* loss_out, double* acc, long long* counts,
                             void* stream) {
  if (B <= 0 || C <= 0 || C > MAX_CLASSES || ld < C || (ld % 8) || !logits || !labels || !row_loss || !row_rank ||
      !loss_out || (!acc) != (!counts))
    return ESVIT_ERR_BAD_ARG;
  probe_ce_row_kernel<<<B, CE_THREADS, (size_t)C * sizeof(float), (cudaStream_t)stream>>>(
      logits, ld, labels, B, C, (bf16*)dlogits, row_loss, row_rank);
  probe_ce_sum_kernel<<<1, CE_THREADS, 0, (cudaStream_t)stream>>>(row_loss, row_rank, B, loss_out, acc, counts);
  ESVIT_LAUNCH_CHECK();
}
