// Hopper-native bf16 GEMM family: every Linear of the training step - forward, input gradient and weight gradient - on
// wgmma tensor cores with TMA-staged operands and register accumulators.
//
//   D[M,N] = epi( opA(A) . opB(B) )        fp32 accumulation in registers
//
//   * warp specialisation: one producer warpgroup (one thread issues the TMA loads of a STAGES-deep ring of
//     [A | B] tiles, mbarrier-synchronised) and WG = 1 or 2 consumer warpgroups, each owning 64 rows of the
//     (64 * WG) x BN tile (wgmma m64nBNk16).  setmaxnreg moves registers from the producer to the consumers.
//   * operands K-major (nn.Linear forward: A[M,K], W[N,K]) or MN-major (a_mn / b_mn): the SAME row-major matrices
//     read "transposed" by TMA boxes of [64 contiguous MN elements x 64 K rows] and wgmma's transpose bits, so
//     the input-gradient GEMM dX = dY . W reads W[N,K] as it lies and the weight-gradient GEMM dW = dY^T . X reads
//     dY[T,N] and X[T,K] as they lie: no transposed copies exist anywhere.
//   * epilogues (template EPI), straight from the accumulator registers: bias -> bf16 | bias + GELU (+ gelu' for the
//     backward) | accumulator * multiplier + column sums (fc2 dgrad fused with GELU' and the fc1 bias gradient) |
//     fp32 split-K partials for the weight gradients (deterministic: partial tiles + fold kernel, no atomics).
// Persistent: one CTA per SM, static round-robin over (split, m tile, n tile) work items; the producer runs ahead into
// the next item's K blocks while the consumers store the previous one.
#include <cuda.h>

#include "common.cuh"

namespace hg {

constexpr int BK = 64;
constexpr int FOLD_THREADS = 64;                 // EPI_MUL: producer-warpgroup threads that fold the column sums
constexpr int SMEM_LIMIT = 232448;               // 227 KB opt-in dynamic shared memory per CTA
enum { EPI_BIAS = 0, EPI_GELU = 1, EPI_MUL = 2, EPI_F32 = 3 };

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
// bounded spin: a mis-programmed pipeline traps after ~2 s of wall time instead of hanging the GPU
__device__ __forceinline__ uint64_t global_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;\n" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t a = smem_u32(bar);
  uint32_t done = 0;
  uint64_t t0 = 0;
  for (uint32_t it = 0;; ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(a), "r"(parity)
        : "memory");
    if (done) return;
    if ((it & 1023u) == 1023u) {
      const uint64_t t = global_ns();
      if (t0 == 0) t0 = t;
      else if (t - t0 > 2000000000ull) __trap();
    }
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n" ::"r"(smem_dst),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// wgmma shared-memory matrix descriptor, 128B swizzle:
// start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | layout SWIZZLE_128B = 1 [62,64)
//   K-major tile : rows of 128 B (64 bf16 along K), 8-row swizzle atoms 1024 B apart (SBO); LBO unused (1);
//                  one wgmma (K = 16) advances the start address by 32 B.
//   MN-major tile: TMA boxes of [64 K rows][64 MN elements = 128 B]: 8-K-row atoms 1024 B apart (SBO), the next 64 MN
//                  elements (next box) 8192 B further (LBO); one wgmma (K = 16 rows) advances the start by 2048 B.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, bool mn_major) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)(mn_major ? (8192 >> 4) : 1) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A[64 x 16] . B[16 x N], both from shared memory; TA / TB: operand is MN-major
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, %131, %132;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BN == 256) wgmma_n256<TA, TB>(d, da, db, scale_d);
  else wgmma_n128<TA, TB>(d, da, db, scale_d);
}

// GELU in the epilogue: Phi(x) = 0.5 + 0.5 tanh(x (a + b x^2)) with ONE MUFU (tanh.approx);
// |gelu - x Phi_erf(x)| < 1e-3 absolute at |x| ~ 4 and < 3e-4 for |x| < 3 - below the bf16 resolution of the stored value
// (0.4 % relative).  The stored derivative is the derivative of THIS function, so forward and backward are consistent.
constexpr float GELU_A = 0.7978845608028654f, GELU_B = 0.7978845608028654f * 0.044715f;
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;\n" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_fwd(float x) {
  const float x2 = x * x;
  const float th = tanh_approx(x * fmaf(GELU_B, x2, GELU_A));
  const float hx = 0.5f * x;
  return fmaf(hx, th, hx);
}
__device__ __forceinline__ float gelu_fwd_grad(float x, float& dy) {
  const float x2 = x * x;
  const float th = tanh_approx(x * fmaf(GELU_B, x2, GELU_A));
  const float hx = 0.5f * x;
  // d/dx [0.5 x (1 + th)] = 0.5 (1 + th) + 0.5 x (1 - th^2) (a + 3 b x^2) = 0.5 (1 + th) + [0.5 x (th^2 - 1)] [-(a + 3 b x^2)]
  const float m = fmaf(th, th, -1.f);
  const float nc = fmaf(-3.f * GELU_B, x2, -GELU_A);
  dy = fmaf(hx * m, nc, fmaf(0.5f, th, 0.5f));
  return fmaf(hx, th, hx);
}

struct Params {
  const float* bias;  // [N] or nullptr (EPI_BIAS / EPI_GELU)
  bf16* out;          // [M][N] bf16 (EPI_BIAS / EPI_GELU / EPI_MUL)
  bf16* aux;          // EPI_GELU: gelu'(pre-activation) out [M][N] or nullptr; EPI_MUL: multiplier in [M][N]
  float* colsum;      // EPI_MUL: [gridDim.x][N] per-CTA column sums of out (zeroed by the launcher)
  float* part;        // EPI_F32: [splits][M][N] fp32 partial products
  int M, N, K;
  int splits;         // K splits (EPI_F32 only; 1 otherwise)
  int kb_per_split;   // 64-wide K blocks per split
};

template <int WG, int BN, int EPI>
struct Cfg {
  static constexpr int BM = 64 * WG;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_BYTES = 256;
  static constexpr int STAGES_RAW = (SMEM_LIMIT - 1024 /*alignment slack*/ - BAR_BYTES) / STAGE_BYTES;
  static constexpr int STAGES_MAX = STAGES_RAW > 6 ? 6 : STAGES_RAW;
  // EPI_MUL: one row of column partials per consumer warp.  Its stages are cut so that the CTA takes no more shared
  // memory than the other epilogues: a larger shared-memory carve-out shrinks L1, through which the epilogue reads the
  // multiplier (measured on H100: the partials on top of the full stage count cost 1.5 ms per Swin-T step, one stage
  // fewer costs nothing measurable).
  static constexpr int CS_BYTES = EPI == EPI_MUL ? 4 * WG * BN * 4 : 0;
  static constexpr int STAGES = (STAGES_MAX * STAGE_BYTES - CS_BYTES) / STAGE_BYTES;
  static constexpr int SMEM = 1024 + STAGES * STAGE_BYTES + CS_BYTES + BAR_BYTES;
  static constexpr int NTHREADS = 128 * (WG + 1);
  static_assert(STAGES >= 2, "pipeline needs at least two stages");
};

template <int WG, int BN, int EPI, int AMN, int BMN>
__global__ void __launch_bounds__(128 * (WG + 1), 1) gemm_kernel(const __grid_constant__ CUtensorMap map_a,
                                                                 const __grid_constant__ CUtensorMap map_b,
                                                                 const Params p) {
  using C = Cfg<WG, BN, EPI>;
  constexpr int STAGES = C::STAGES, BM = C::BM;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // [STAGES][A | B], every tile 1024-byte aligned in the SHARED address space (swizzle-128B)
  uint8_t* tiles = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* cs_part = reinterpret_cast<float*>(tiles + STAGES * C::STAGE_BYTES);   // [4 WG][BN]
  uint64_t* full = reinterpret_cast<uint64_t*>(tiles + STAGES * C::STAGE_BYTES + C::CS_BYTES);
  uint64_t* empty = full + STAGES;
  uint64_t* cs_full = empty + STAGES;     // EPI_MUL: every consumer warp has written its partials of a tile
  uint64_t* cs_empty = cs_full + 1;       // ... and the fold threads have consumed them

  const int wg = threadIdx.x >> 7;
  const int m_tiles = (p.M + BM - 1) / BM, n_tiles = (p.N + BN - 1) / BN;
  const int tiles_mn = m_tiles * n_tiles, num_items = tiles_mn * p.splits;
  const int k_blocks = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(&map_b) : "memory");
    for (int i = 0; i < STAGES; i++) { mbar_init(&full[i], 1); mbar_init(&empty[i], 128 * WG); }
    mbar_init(cs_full, 4 * WG);
    mbar_init(cs_empty, FOLD_THREADS);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (wg == WG) {
    // ===================== TMA producer (one thread of the last warpgroup) and, for EPI_MUL, the column-sum fold =====
    if constexpr (WG == 2) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (threadIdx.x == 128 * WG) {
      int stage = 0;
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const int tile = item % tiles_mn, split = item / tiles_mn;
        const int m0 = (tile / n_tiles) * BM, n0 = (tile % n_tiles) * BN;
        const int kb0 = split * p.kb_per_split;
        int kb1 = kb0 + p.kb_per_split; kb1 = kb1 < k_blocks ? kb1 : k_blocks;
        for (int kb = kb0; kb < kb1; kb++) {
          mbar_wait(&empty[stage], phase ^ 1);
          const uint32_t sa = smem_u32(tiles + stage * C::STAGE_BYTES), sb = sa + C::A_BYTES;
          mbar_expect_tx(&full[stage], C::STAGE_BYTES);
          if (!AMN) {
            tma_load_2d(sa, &map_a, &full[stage], kb * BK, m0);                          // box [64 K][BM rows]
          } else {
#pragma unroll
            for (int j = 0; j < BM / 64; j++)
              tma_load_2d(sa + j * 8192, &map_a, &full[stage], m0 + j * 64, kb * BK);    // box [64 M][64 K rows]
          }
          if (!BMN) {
            tma_load_2d(sb, &map_b, &full[stage], kb * BK, n0);                          // box [64 K][BN rows]
          } else {
#pragma unroll
            for (int j = 0; j < BN / 64; j++)
              tma_load_2d(sb + j * 8192, &map_b, &full[stage], n0 + j * 64, kb * BK);    // box [64 N][64 K rows]
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    } else if (EPI == EPI_MUL && threadIdx.x >= 128 * WG + 32 && threadIdx.x < 128 * WG + 32 + FOLD_THREADS) {
      // EPI_MUL column sums: fixed-order fold of the consumer warps' partials of each tile into this CTA's private
      // workspace row, off the consumers' path.  Column c of a tile is always folded by thread c % FOLD_THREADS, whose
      // adds to one address land in program order, and the CTA walks the same items in the same order on every run:
      // the column sums (the fc1 bias gradient) are bit-reproducible.
      const int t = threadIdx.x - 128 * WG - 32;
      float* dst = p.colsum + (long long)blockIdx.x * p.N;
      int local = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x, local++) {
        const int n0 = ((item % tiles_mn) % n_tiles) * BN;
        mbar_wait(cs_full, local & 1);
        for (int c = t; c < BN && n0 + c < p.N; c += FOLD_THREADS) {
          float sum = 0.f;
#pragma unroll
          for (int w = 0; w < 4 * WG; w++) sum += cs_part[w * BN + c];
          atomicAdd(dst + n0 + c, sum);
        }
        mbar_arrive(cs_empty);
      }
    }
  } else {
    // ===================== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile =====================
    if constexpr (WG == 2) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
    const int frag_row = wg * 64 + warp * 16 + (lane >> 2);   // tile row of acc[4i], acc[4i + 1]; +8 for acc[4i + 2 / 3]
    const int frag_col = 2 * (lane & 3);                      // + 8 i
    constexpr uint32_t KSTEP_A = AMN ? (2048 >> 4) : (32 >> 4), KSTEP_B = BMN ? (2048 >> 4) : (32 >> 4);
    int stage = 0;
    uint32_t phase = 0;
    int local = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x, local++) {
      const int tile = item % tiles_mn, split = item / tiles_mn;
      const int m0 = (tile / n_tiles) * BM, n0 = (tile % n_tiles) * BN;
      const int kb0 = split * p.kb_per_split;
      int kb1 = kb0 + p.kb_per_split; kb1 = kb1 < k_blocks ? kb1 : k_blocks;
      float acc[BN / 2];
      int prev = -1;
      for (int kb = kb0; kb < kb1; kb++) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(tiles + stage * C::STAGE_BYTES) + wg * 8192;   // this warpgroup's 64 rows of A
        const uint64_t da = make_smem_desc(sa, AMN), db = make_smem_desc(smem_u32(tiles + stage * C::STAGE_BYTES) + C::A_BYTES, BMN);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; k++)
          wgmma_tile<BN, AMN, BMN>(acc, da + k * KSTEP_A, db + k * KSTEP_B, (kb > kb0 || k != 0) ? 1u : 0u);
        wgmma_commit();
        // keep one K block of wgmma in flight: the previous block's stage is free once its group has retired
        wgmma_wait<1>();
        if (prev >= 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0) mbar_arrive(&empty[prev]);

      // ---- epilogue from registers ----
      if constexpr (EPI == EPI_MUL) mbar_wait(cs_empty, (local & 1) ^ 1);   // the previous tile's partials are folded
#pragma unroll
      for (int i = 0; i < BN / 8; i++) {
        float cs0 = 0.f, cs1 = 0.f;
        const int col = n0 + i * 8 + frag_col;
        if (col >= p.N) continue;  // N % 8 == 0: col + 1 < N as well, and the test is uniform over the warp
        float b0 = 0.f, b1 = 0.f;
        if constexpr (EPI == EPI_BIAS || EPI == EPI_GELU) {
          if (p.bias) { const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col)); b0 = bb.x; b1 = bb.y; }
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int row = m0 + frag_row + 8 * h;
          if (row >= p.M) continue;
          float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
          const long long off = (long long)row * p.N + col;
          if constexpr (EPI == EPI_F32) {
            *reinterpret_cast<float2*>(p.part + (long long)split * p.M * p.N + off) = make_float2(v0, v1);
          } else if constexpr (EPI == EPI_MUL) {
            const float2 m = __bfloat1622float2(*reinterpret_cast<const bf162*>(p.aux + off));
            const bf162 o = __floats2bfloat162_rn(v0 * m.x, v1 * m.y);
            *reinterpret_cast<bf162*>(p.out + off) = o;
            const float2 of = __bfloat1622float2(o);   // column sums of the STORED (bf16) values
            cs0 += of.x; cs1 += of.y;
          } else if constexpr (EPI == EPI_GELU) {
            v0 += b0; v1 += b1;
            if (p.aux) {
              float d0, d1;
              const float y0 = gelu_fwd_grad(v0, d0), y1 = gelu_fwd_grad(v1, d1);
              *reinterpret_cast<bf162*>(p.out + off) = __floats2bfloat162_rn(y0, y1);
              *reinterpret_cast<bf162*>(p.aux + off) = __floats2bfloat162_rn(d0, d1);
            } else {
              *reinterpret_cast<bf162*>(p.out + off) = __floats2bfloat162_rn(gelu_fwd(v0), gelu_fwd(v1));
            }
          } else {
            *reinterpret_cast<bf162*>(p.out + off) = __floats2bfloat162_rn(v0 + b0, v1 + b1);
          }
        }
        if constexpr (EPI == EPI_MUL) {
          // reduce over the 8 row groups of the warp (lanes with equal lane % 4) into this warp's row of partials
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            cs0 += __shfl_xor_sync(0xffffffffu, cs0, o);
            cs1 += __shfl_xor_sync(0xffffffffu, cs1, o);
          }
          if (lane < 4) *reinterpret_cast<float2*>(cs_part + (wg * 4 + warp) * BN + i * 8 + frag_col) = make_float2(cs0, cs1);
        }
      }
      if constexpr (EPI == EPI_MUL) {
        __syncwarp();   // the warp's partials (lanes 0-3) are written before lane 0 releases them to the fold warps
        if (lane == 0) mbar_arrive(cs_full);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeFn)ptr;
  }
  return fn;
}

// row-major [rows, cols] bf16 matrix, box = [box_rows, 64 cols], 128B swizzle, zero fill out of bounds
static bool make_map(CUtensorMap* map, const void* ptr, long long rows, long long cols, int box_rows) {
  EncodeFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {64u, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// colsum[n] += sum over the CTAs' private rows
__global__ void __launch_bounds__(256) colsum_fold_kernel(const float* __restrict__ ws, int rows, int N, float* __restrict__ colsum) {
  const int n = blockIdx.x * 256 + threadIdx.x;
  if (n >= N) return;
  float s = 0.f;
  for (int r = 0; r < rows; r++) s += ws[(long long)r * N + n];
  colsum[n] += s;
}

// out[i] (+)= sum_s part[s][i]  (deterministic fold of the split-K partials)
__global__ void __launch_bounds__(256) split_fold_kernel(const float* __restrict__ part, int splits, long long n4,
                                                         float* __restrict__ out, int accumulate) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n4) return;
  float4 s = accumulate ? reinterpret_cast<const float4*>(out)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  for (int k = 0; k < splits; k++) {
    const float4 t = reinterpret_cast<const float4*>(part)[(long long)k * n4 + i];
    s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
  }
  reinterpret_cast<float4*>(out)[i] = s;
}

constexpr int MAX_GRID = 160;  // rows of the column-sum workspace (callers allocate MAX_GRID * N floats): bound on the EPI_MUL grid

struct Call {
  const void* a; const void* b;
  int a_mn, b_mn;
  Params p;
};

template <int WG, int BN, int EPI, int AMN, int BMN>
static int launch_cfg(const Call& c, void* stream, int* rows_out) {
  using C = Cfg<WG, BN, EPI>;
  Params p = c.p;
  CUtensorMap ma, mb;
  // A: K-major [M,K] box [64 K][BM rows] | MN-major [K,M] box [64 M][64 K rows]
  if (!(AMN ? make_map(&ma, c.a, p.K, p.M, 64) : make_map(&ma, c.a, p.M, p.K, C::BM))) return ESVIT_ERR_BAD_ARG;
  // B: K-major [N,K] box [64 K][BN rows] | MN-major [K,N] box [64 N][64 K rows]
  if (!(BMN ? make_map(&mb, c.b, p.K, p.N, 64) : make_map(&mb, c.b, p.N, p.K, BN))) return ESVIT_ERR_BAD_ARG;
  auto kernel = gemm_kernel<WG, BN, EPI, AMN, BMN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  const int m_tiles = (p.M + C::BM - 1) / C::BM, n_tiles = (p.N + BN - 1) / BN;
  const long long items = (long long)m_tiles * n_tiles * p.splits;
  int grid = esvit_num_sms();
  if (EPI == EPI_MUL && grid > MAX_GRID) grid = MAX_GRID;   // one private workspace row per CTA
  if ((long long)grid > items) grid = (int)items;
  if (EPI == EPI_MUL) {
    cudaError_t e = cudaMemsetAsync(p.colsum, 0, (size_t)grid * p.N * sizeof(float), (cudaStream_t)stream);
    if (e != cudaSuccess) return (int)e;
  }
  if (rows_out) *rows_out = grid;
  kernel<<<grid, C::NTHREADS, C::SMEM, (cudaStream_t)stream>>>(ma, mb, p);
  return (int)cudaGetLastError();
}

template <int WG, int BN, int EPI>
static int launch_majors(const Call& c, void* stream, int* rows_out) {
  if constexpr (EPI == EPI_F32) {  // weight gradient: both operands MN-major
    if (c.a_mn && c.b_mn) return launch_cfg<WG, BN, EPI, 1, 1>(c, stream, rows_out);
  } else if constexpr (EPI == EPI_MUL) {
    if (!c.a_mn) return c.b_mn ? launch_cfg<WG, BN, EPI, 0, 1>(c, stream, rows_out) : launch_cfg<WG, BN, EPI, 0, 0>(c, stream, rows_out);
  } else {
    if (!c.a_mn) return c.b_mn ? launch_cfg<WG, BN, EPI, 0, 1>(c, stream, rows_out) : launch_cfg<WG, BN, EPI, 0, 0>(c, stream, rows_out);
    return c.b_mn ? launch_cfg<WG, BN, EPI, 1, 1>(c, stream, rows_out) : launch_cfg<WG, BN, EPI, 1, 0>(c, stream, rows_out);
  }
  return ESVIT_ERR_BAD_ARG;
}

template <int EPI>
static int launch_epi(const Call& c, int wg, int bn, void* stream, int* rows_out) {
  if (wg == 2 && bn == 256) return launch_majors<2, 256, EPI>(c, stream, rows_out);
  if (wg == 2 && bn == 128) return launch_majors<2, 128, EPI>(c, stream, rows_out);
  if (wg == 1 && bn == 256) return launch_majors<1, 256, EPI>(c, stream, rows_out);
  if (wg == 1 && bn == 128) return launch_majors<1, 128, EPI>(c, stream, rows_out);
  return ESVIT_ERR_BAD_ARG;
}

static int launch(const Call& c, int epi, int wg, int bn, void* stream, int* rows_out = nullptr) {
  switch (epi) {
    case EPI_BIAS: return launch_epi<EPI_BIAS>(c, wg, bn, stream, rows_out);
    case EPI_GELU: return launch_epi<EPI_GELU>(c, wg, bn, stream, rows_out);
    case EPI_MUL: return launch_epi<EPI_MUL>(c, wg, bn, stream, rows_out);
    case EPI_F32: return launch_epi<EPI_F32>(c, wg, bn, stream, rows_out);
  }
  return ESVIT_ERR_BAD_ARG;
}

// Tile shape policy; overridable per call through `tile` = forced_splits * 10000 + wg * 1000 + bn (0 = automatic), wg =
// consumer warpgroups (tile rows = 64 wg).  The largest tile that still gives every SM a work item: 128 x 256 tiles read
// the fewest operand bytes per MAC, but a GEMM with fewer tiles than SMs leaves SMs idle.
static void pick_tile(long long M, int N, int tile, int* wg, int* bn) {
  tile %= 10000;
  if (tile > 0) { *wg = tile / 1000; *bn = tile % 1000; return; }
  const int sms = esvit_num_sms();
  const int cand[4][2] = {{2, 256}, {2, 128}, {1, 256}, {1, 128}};
  for (const auto& cd : cand) {
    if (cd[1] == 256 && N <= 128) continue;
    const long long items = ((M + 64 * cd[0] - 1) / (64 * cd[0])) * ((N + cd[1] - 1) / cd[1]);
    if (items >= sms) { *wg = cd[0]; *bn = cd[1]; return; }
  }
  *wg = 1; *bn = 128;
}
// weight gradient (GEMM M = out features, N = in features, contraction over tokens): split-K supplies the parallelism
static void pick_tile_wgrad(int Nout, int Kin, int tile, int* wg, int* bn) {
  tile %= 10000;
  if (tile > 0) { *wg = tile / 1000; *bn = tile % 1000; return; }
  *bn = Kin > 128 ? 256 : 128;
  *wg = Nout > 64 ? 2 : 1;
}

}  // namespace hg

// ---- C ABI ----------------------------------------------------------------------------------------------------------
// out[M,N] (bf16) = act( opA(a) . opB(b) + bias[N] )
//   a: a_mn = 0: [M,K] row-major (K contiguous) | a_mn = 1: [K,M] row-major (M contiguous)
//   b: b_mn = 0: [N,K] row-major (nn.Linear weight layout) | b_mn = 1: [K,N] row-major (N contiguous)
//   act 0: identity; act 1: GELU (pre != NULL also receives gelu'(pre-activation) for the backward)
//   M, N, K multiples of 8; bias fp32 or NULL.  tile = 0 (automatic) or warpgroups * 1000 + BN (1128, 1256, 2128, 2256).
ESVIT_API int esvit_gemm_bf16(const void* a, const void* b, const float* bias, void* out, void* pre, long long M, int N,
                              int K, int a_mn, int b_mn, int act, int tile, void* stream) {
  if (M <= 0 || N <= 0 || K <= 0 || (N % 8) || (K % 8) || M > 0x7fffffffLL || (a_mn && (M % 8)) || act < 0 || act > 1)
    return ESVIT_ERR_BAD_ARG;
  hg::Call c;
  c.a = a; c.b = b; c.a_mn = a_mn ? 1 : 0; c.b_mn = b_mn ? 1 : 0;
  c.p.bias = bias; c.p.out = (bf16*)out; c.p.aux = (act == 1) ? (bf16*)pre : nullptr; c.p.colsum = nullptr; c.p.part = nullptr;
  c.p.M = (int)M; c.p.N = N; c.p.K = K; c.p.splits = 1; c.p.kb_per_split = (K + hg::BK - 1) / hg::BK;
  int wg, bn;
  hg::pick_tile(M, N, tile, &wg, &bn);
  return hg::launch(c, act ? hg::EPI_GELU : hg::EPI_BIAS, wg, bn, stream);
}

// out[M,N] (bf16) = (a[M,K] . opB(b)) * mult[M,N];  colsum[N] (fp32) += column sums of out.
// The input-gradient GEMM of fc2 fused with the GELU backward of fc1: a = dy, b = W2 ([K,N] row-major = the Linear weight
// as it lies, b_mn = 1; or a pre-transposed [N,K] copy, b_mn = 0), mult = gelu'(pre-activation) saved by the forward,
// out = d(pre-activation), colsum = fc1 bias gradient (caller zero-fills); ws fp32 [160 * N] scratch.
ESVIT_API int esvit_gemm_mul_colsum2(const void* a, const void* b, const void* mult, void* out, float* colsum, float* ws,
                                     long long M, int N, int K, int b_mn, int tile, void* stream) {
  if (M <= 0 || N <= 0 || K <= 0 || (N % 8) || (K % 8) || M > 0x7fffffffLL || !mult || !colsum || !ws) return ESVIT_ERR_BAD_ARG;
  hg::Call c;
  c.a = a; c.b = b; c.a_mn = 0; c.b_mn = b_mn ? 1 : 0;
  c.p.bias = nullptr; c.p.out = (bf16*)out; c.p.aux = (bf16*)mult; c.p.colsum = ws; c.p.part = nullptr;
  c.p.M = (int)M; c.p.N = N; c.p.K = K; c.p.splits = 1; c.p.kb_per_split = (K + hg::BK - 1) / hg::BK;
  int wg, bn, rows = 0;
  hg::pick_tile(M, N, tile, &wg, &bn);
  const int rc = hg::launch(c, hg::EPI_MUL, wg, bn, stream, &rows);
  if (rc != 0) return rc;
  hg::colsum_fold_kernel<<<(N + 255) / 256, 256, 0, (cudaStream_t)stream>>>(ws, rows, N, colsum);
  ESVIT_LAUNCH_CHECK();
}

// Weight gradient of a Linear: dw[N,K] (fp32) (+)= dy[T,N]^T . x[T,K]   (dy, x bf16 row-major, read as they lie through
// MN-major TMA boxes; any T).  Split over T across the persistent CTAs; partial tiles go to ws (fp32, esvit_gemm_wgrad_ws_floats
// elements) and are folded in a fixed order: bit-reproducible, no atomics.  N, K multiples of 8.
static long long wgrad_ws_floats(int N, int K) {
  const int tiles = ((N + 127) / 128) * ((K + 255) / 256);   // the fewest output tiles any tile shape yields
  long long splits = (2LL * 160 + tiles - 1) / tiles;
  if (splits > 96) splits = 96;                              // bound on the workspace: 96 partial copies of dw
  if (splits < 1) splits = 1;
  return splits * (long long)N * K;
}
// number of fp32 elements of workspace esvit_gemm_wgrad needs for an [N,K] weight (returned as the status-free int)
ESVIT_API int esvit_gemm_wgrad_ws_floats(int N, int K) {
  const long long n = wgrad_ws_floats(N, K);
  return n > 0x7fffffffLL ? -1 : (int)n;
}
ESVIT_API int esvit_gemm_wgrad(const void* dy, const void* x, float* dw, float* ws, long long T, int N, int K,
                               int accumulate, int tile, void* stream) {
  if (T <= 0 || N <= 0 || K <= 0 || (N % 8) || (K % 8) || T > 0x7fffffffLL || !ws) return ESVIT_ERR_BAD_ARG;
  // GEMM view: M = N (out features), N = K (in features), contraction = T
  int wg, bn;
  hg::pick_tile_wgrad(N, K, tile, &wg, &bn);
  const int m_tiles = (N + 64 * wg - 1) / (64 * wg), n_tiles = (K + bn - 1) / bn;
  const int tiles = m_tiles * n_tiles;
  const int k_blocks = (int)((T + hg::BK - 1) / hg::BK);
  const int ctas = esvit_num_sms();
  // one wave of work items: every CTA gets (at most) one K-slice of one output tile, slices of >= 8 K blocks
  int splits = tiles >= ctas ? 1 : ctas / tiles;
  if (splits > k_blocks / 8) splits = k_blocks / 8;
  if (tile >= 10000) splits = tile / 10000;                   // forced (tests / tuning)
  const long long cap = wgrad_ws_floats(N, K) / ((long long)N * K);
  if (splits > cap) splits = (int)cap;
  if (splits > k_blocks) splits = k_blocks;
  if (splits < 1) splits = 1;
  int kbs = (k_blocks + splits - 1) / splits;
  splits = (k_blocks + kbs - 1) / kbs;                         // no empty split
  hg::Call c;
  c.a = dy; c.b = x; c.a_mn = 1; c.b_mn = 1;
  c.p.bias = nullptr; c.p.out = nullptr; c.p.aux = nullptr; c.p.colsum = nullptr; c.p.part = ws;
  c.p.M = N; c.p.N = K; c.p.K = (int)T; c.p.splits = splits; c.p.kb_per_split = kbs;
  const int rc = hg::launch(c, hg::EPI_F32, wg, bn, stream);
  if (rc != 0) return rc;
  const long long n4 = (long long)N * K / 4;
  hg::split_fold_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(ws, splits, n4, dw, accumulate);
  ESVIT_LAUNCH_CHECK();
}

// ---- first-generation entry points, served by the same kernel family ------------------------------------------------
// out[M,N] (bf16) = act(a[M,K] @ w[N,K]^T + bias[N]); act 1 = GELU (pre, if not NULL, receives gelu'(pre-activation)).
ESVIT_API int esvit_gemm_bias_act(const void* a, const void* w, const float* bias, void* out, void* pre, long long M,
                                  int N, int K, int act, void* stream) {
  return esvit_gemm_bf16(a, w, bias, out, pre, M, N, K, 0, 0, act, 0, stream);
}
// out[M,N] (bf16) = (a[M,K] @ w[N,K]^T) * mult[M,N];  colsum[N] (fp32) += column sums of out; ws fp32 [160 * N].
ESVIT_API int esvit_gemm_mul_colsum(const void* a, const void* w, const void* mult, void* out, float* colsum, float* ws,
                                    long long M, int N, int K, void* stream) {
  return esvit_gemm_mul_colsum2(a, w, mult, out, colsum, ws, M, N, K, 0, 0, stream);
}
