// Hopper-native bf16 GEMM family: every Linear of the training step - forward, input gradient and weight gradient - on
// wgmma tensor cores with TMA-staged operands and register accumulators.
//
//   D[M,N] = epi( opA(A) . opB(B) )        fp32 accumulation in registers
//
//   * warp specialisation: one producer warpgroup (one thread issues the TMA loads of a STAGES-deep ring of
//     [A | B] tiles, mbarrier-synchronised) and two consumer warpgroups (wgmma m64nBNk16); setmaxnreg moves registers
//     from the producer to the consumers.  128-row tiles (WG = 2): cooperative, each consumer owns 64 rows of every
//     tile.  64-row tiles (WG = 1): ping-pong, the consumers take the CTA's items alternately, the mainloops run in
//     item order (a pair of mbarriers passes the turn), and one warpgroup's epilogue overlaps the other's mainloop.
//   * operands K-major (nn.Linear forward: A[M,K], W[N,K]) or MN-major (a_mn / b_mn): the SAME row-major matrices
//     read "transposed" by TMA boxes of [64 contiguous MN elements x 64 K rows] and wgmma's transpose bits, so
//     the input-gradient GEMM dX = dY . W reads W[N,K] as it lies and the weight-gradient GEMM dW = dY^T . X reads
//     dY[T,N] and X[T,K] as they lie: no transposed copies exist anywhere.
//   * epilogues (template EPI): bias -> bf16 | bias + GELU (+ gelu' for the backward) | accumulator * multiplier +
//     column sums (fc2 dgrad fused with GELU' and the fc1 bias gradient) | fp32 split-K partials for the weight
//     gradients (deterministic: partial tiles + fold kernel, no atomics).  The bf16 results go out in 64-column chunks:
//     stmatrix into a 128B-swizzled shared buffer, then one TMA tile store per chunk and consumer warpgroup (full
//     32-byte sectors, clipped at M / N by the TMA); the multiplier comes in by TMA, issued by the producer during the
//     mainloop.  The fp32 partials are stored from the registers.
// Persistent: one CTA per SM, static round-robin over (split, m tile, n tile) work items; the producer runs ahead into
// the next item's K blocks while the consumers store the previous one.  Neither schedule changes an element's k16
// accumulation order: the bf16 results of every tile shape are bit-identical.
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
// shared -> global tile store; the box is clipped at the tensor's bounds (nothing is written past row M / column N)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];\n" ::"l"(map), "r"(smem_src),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
// at most N of this thread's committed store groups still read shared memory
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;\n" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;\n" ::: "memory"); }
// this thread's generic-proxy shared-memory writes become visible to the TMA (async proxy)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
__device__ __forceinline__ void named_barrier(int id, int threads) {
  asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(threads) : "memory");
}
// four 8x8 bf16 matrices; lane l addresses row l % 8 of matrix l / 8 and holds row l / 4, columns 2 (l % 4) + {0, 1} of
// each (the mma accumulator fragment layout)
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};\n" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2),
               "r"(r3)
               : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr)
               : "memory");
}
__device__ __forceinline__ float2 unpack_bf162(uint32_t u) { return __bfloat1622float2(*reinterpret_cast<const bf162*>(&u)); }

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

// D[64 x 64] (+)= A[64 x 16] . B[16 x 64], both K-major from shared memory
__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
// D[64 x N] (+)= A[64 x 16] . B[16 x N]: A from registers (the m64k16 fragment, four bf16 pairs per thread), B K-major
// from shared memory; N = 2 * size of d (the back-to-back MLP's fc2 at N = C)
__device__ __forceinline__ void wgmma_rs(float (&d)[48], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %53, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
      "{%48, %49, %50, %51}, %52, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_rs(float (&d)[96], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %101, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, "
      "{%96, %97, %98, %99}, %100, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
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
// QuickGELU x sigmoid(1.702 x) (CvT's act_layer, models/cvt_v4_transformer.py:44-46) and its derivative
// s (1 + 1.702 x (1 - s)), s = sigmoid(1.702 x)
constexpr float QGELU_A = 1.702f;
__device__ __forceinline__ float qgelu_fwd(float x) { return x * __frcp_rn(1.f + __expf(-QGELU_A * x)); }
__device__ __forceinline__ float qgelu_fwd_grad(float x, float& dy) {
  const float s = __frcp_rn(1.f + __expf(-QGELU_A * x));
  dy = s * fmaf(QGELU_A * x, 1.f - s, 1.f);
  return x * s;
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

// Two consumer warpgroups either way.  WG = 2 (cooperative): both work on one 128-row tile, warpgroup wg on rows
// [64 wg, 64 wg + 64).  WG = 1 (ping-pong, PP): each warpgroup owns whole 64-row items, the CTA's items alternately, with
// its own epilogue buffers and barriers, so one warpgroup's epilogue runs while the other's mainloop keeps the tensor
// cores busy.
template <int WG, int BN, int EPI>
struct Cfg {
  static constexpr bool PP = WG == 1;
  static constexpr int NEP = PP ? 2 : 1;         // sets of epilogue buffers and epilogue mbarriers
  static constexpr int BM = 64 * WG;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_BYTES = PP ? 512 : 256;
  // bf16 epilogue staging: 64-column chunks of the tile, [BM rows][128 B] each, 128B-swizzled like a [64 x 64] TMA box
  // (cooperative: consumer warpgroup wg owns the 8 KB at wg * 8192).  EPI_BIAS: two chunk buffers; EPI_GELU: two
  // (out, gelu') pairs; EPI_MUL: one buffer per chunk of the tile, loaded with the multiplier by TMA and overwritten in
  // place by the result.  Ping-pong: one such set per consumer warpgroup.
  static constexpr int NCHUNK = BN / 64;
  static constexpr int CHUNK_BYTES = BM * 128;
  static constexpr int EP_WG_BYTES = EPI == EPI_BIAS ? 2 * CHUNK_BYTES
                                   : EPI == EPI_GELU ? 4 * CHUNK_BYTES
                                   : EPI == EPI_MUL  ? NCHUNK * CHUNK_BYTES : 0;
  static constexpr int EP_BYTES = NEP * EP_WG_BYTES;
  // EPI_MUL: one row of column partials per consumer warp
  static constexpr int CS_BYTES = EPI == EPI_MUL ? 8 * BN * 4 : 0;
  static constexpr int STAGES_RAW = (SMEM_LIMIT - 1024 /*alignment slack*/ - BAR_BYTES - EP_BYTES - CS_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 6 ? 6 : STAGES_RAW;
  static constexpr int SMEM = 1024 + STAGES * STAGE_BYTES + EP_BYTES + CS_BYTES + BAR_BYTES;
  static constexpr int NTHREADS = 384;
  // 64 x 256 multiplier items keep three 40 KB stages beside two warpgroups' 32 KB of multiplier chunks
  static_assert(STAGES >= (BN == 256 && (WG == 2 || EPI == EPI_MUL) ? 3 : 4), "operand ring too shallow");
  static_assert(SMEM <= SMEM_LIMIT, "shared memory budget");
  static_assert((2 * STAGES + 2 * NEP + 2 * NEP * NCHUNK + 2) * 8 <= BAR_BYTES, "mbarrier area");
};

// map_o: out, map_x: gelu' out (EPI_GELU) or the multiplier in (EPI_MUL); both [64 columns x 64 rows] boxes, 128B swizzle.
// QUICK (EPI_GELU only): QuickGELU instead of the tanh GELU
template <int WG, int BN, int EPI, int AMN, int BMN, bool QUICK = false>
__global__ void __launch_bounds__(384, 1) gemm_kernel(const __grid_constant__ CUtensorMap map_a,
                                                      const __grid_constant__ CUtensorMap map_b,
                                                      const __grid_constant__ CUtensorMap map_o,
                                                      const __grid_constant__ CUtensorMap map_x,
                                                      const Params p) {
  using C = Cfg<WG, BN, EPI>;
  constexpr int STAGES = C::STAGES, BM = C::BM, NCHUNK = C::NCHUNK;
  constexpr bool PP = C::PP;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // [STAGES][A | B] | [NEP] epilogue chunks | column partials | mbarriers; every tile and chunk 1024-byte aligned in the
  // SHARED address space (swizzle-128B)
  uint8_t* tiles = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* ep = tiles + STAGES * C::STAGE_BYTES;
  float* cs_part = reinterpret_cast<float*>(ep + C::EP_BYTES);   // [8 consumer warps][BN]
  uint64_t* full = reinterpret_cast<uint64_t*>(ep + C::EP_BYTES + C::CS_BYTES);
  uint64_t* empty = full + STAGES;
  uint64_t* cs_full = empty + STAGES;             // [NEP] EPI_MUL: every consumer warp has written its partials of a tile
  uint64_t* cs_empty = cs_full + C::NEP;          // ... and the fold threads have consumed them
  uint64_t* mul_full = cs_empty + C::NEP;         // [NEP][NCHUNK] EPI_MUL, per chunk: the multiplier has landed
  uint64_t* mul_empty = mul_full + C::NEP * NCHUNK;  // ... and the TMA store of the result has read it back out
  uint64_t* turn = mul_empty + C::NEP * NCHUNK;   // PP, per warpgroup: the CTA's previous item has issued its mainloop

  const int wg = threadIdx.x >> 7;
  const int m_tiles = (p.M + BM - 1) / BM, n_tiles = (p.N + BN - 1) / BN;
  const int tiles_mn = m_tiles * n_tiles, num_items = tiles_mn * p.splits;
  const int k_blocks = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(&map_b) : "memory");
    // every count holds for both schedules: a stage, a tile's partials and a multiplier chunk are consumed by the WG
    // warpgroups of one item
    for (int i = 0; i < STAGES; i++) { mbar_init(&full[i], 1); mbar_init(&empty[i], 128 * WG); }
    for (int e = 0; e < C::NEP; e++) { mbar_init(&cs_full[e], 4 * WG); mbar_init(&cs_empty[e], FOLD_THREADS); }
    if constexpr (EPI == EPI_MUL)
      for (int i = 0; i < C::NEP * NCHUNK; i++) { mbar_init(&mul_full[i], 1); mbar_init(&mul_empty[i], WG); }
    if constexpr (PP) { mbar_init(&turn[0], 128); mbar_init(&turn[1], 128); }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (wg == 2) {
    // ===================== TMA producer (one thread of the last warpgroup) and, for EPI_MUL, the column-sum fold =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (threadIdx.x == 256) {
      int stage = 0;
      uint32_t phase = 0;
      int local = 0;
      if constexpr (EPI == EPI_MUL) asm volatile("prefetch.tensormap [%0];\n" ::"l"(&map_x) : "memory");
      for (int item = blockIdx.x; item < num_items; item += gridDim.x, local++) {
        const int tile = item % tiles_mn, split = item / tiles_mn;
        const int m0 = (tile / n_tiles) * BM, n0 = (tile % n_tiles) * BN;
        const int kb0 = split * p.kb_per_split;
        int kb1 = kb0 + p.kb_per_split; kb1 = kb1 < k_blocks ? kb1 : k_blocks;
        // EPI_MUL: multiplier chunk j of this tile, issued after K block kb0 + j so that it lands during the mainloop
        // while the first operand stages go out ahead of it; its buffer is free once the result chunk j of the
        // previous tile that used the same buffer set (PP: the same warpgroup's previous item) has been stored
        const int e = PP ? (local & 1) : 0, use = PP ? local >> 1 : local;
        auto load_mul = [&](int j) {
          mbar_wait(&mul_empty[e * NCHUNK + j], (use & 1) ^ 1);
          const uint32_t dst = smem_u32(ep + e * C::EP_WG_BYTES + j * C::CHUNK_BYTES);
          mbar_expect_tx(&mul_full[e * NCHUNK + j], C::CHUNK_BYTES);
#pragma unroll
          for (int h = 0; h < WG; h++)
            tma_load_2d(dst + h * 8192, &map_x, &mul_full[e * NCHUNK + j], n0 + 64 * j, m0 + 64 * h);
        };
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
          if constexpr (EPI == EPI_MUL) if (kb - kb0 < NCHUNK) load_mul(kb - kb0);
        }
        if constexpr (EPI == EPI_MUL)
          for (int j = kb1 - kb0; j < NCHUNK; j++) load_mul(j);
      }
    } else if (EPI == EPI_MUL && threadIdx.x >= 256 + 32 && threadIdx.x < 256 + 32 + FOLD_THREADS) {
      // EPI_MUL column sums: fixed-order fold of the consumer warps' partials of each tile into this CTA's private
      // workspace row, off the consumers' path.  Column c of a tile is always folded by thread c % FOLD_THREADS, whose
      // adds to one address land in program order, and the CTA walks the same items in the same order on every run
      // (PP: in item order, alternating between the two warpgroups' partial rows): the column sums (the fc1 bias
      // gradient) are bit-reproducible.
      const int t = threadIdx.x - 256 - 32;
      float* dst = p.colsum + (long long)blockIdx.x * p.N;
      int local = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x, local++) {
        const int n0 = ((item % tiles_mn) % n_tiles) * BN;
        const int e = PP ? (local & 1) : 0, use = PP ? local >> 1 : local;
        mbar_wait(&cs_full[e], use & 1);
        for (int c = t; c < BN && n0 + c < p.N; c += FOLD_THREADS) {
          float sum = 0.f;
#pragma unroll
          for (int w = 0; w < 4 * WG; w++) sum += cs_part[(4 * e + w) * BN + c];
          atomicAdd(dst + n0 + c, sum);
        }
        mbar_arrive(&cs_empty[e]);
      }
    }
  } else {
    // ===================== consumers: cooperative, warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile; ========
    // ===================== ping-pong, warpgroup wg owns the whole 64-row items local % 2 == wg of the CTA  ========
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
    const int row0 = PP ? 0 : 64 * wg;                        // this warpgroup's first row of the tile
    const int frag_row = row0 + warp * 16 + (lane >> 2);      // tile row of acc[4i], acc[4i + 1]; +8 for acc[4i + 2 / 3]
    const int frag_col = 2 * (lane & 3);                      // + 8 i
    const uint32_t rows_off = PP ? 0u : (uint32_t)wg * 8192u; // byte offset of those rows in an A tile / a chunk buffer
    const int e = PP ? wg : 0;                                // this warpgroup's set of epilogue buffers and barriers
    uint8_t* const my_ep = ep + e * C::EP_WG_BYTES;
    constexpr uint32_t KSTEP_A = AMN ? (2048 >> 4) : (32 >> 4), KSTEP_B = BMN ? (2048 >> 4) : (32 >> 4);
    int stage = 0;
    uint32_t phase = 0;
    int local = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x, local++) {
      const int tile = item % tiles_mn, split = item / tiles_mn;
      const int m0 = (tile / n_tiles) * BM, n0 = (tile % n_tiles) * BN;
      const int kb0 = split * p.kb_per_split;
      int kb1 = kb0 + p.kb_per_split; kb1 = kb1 < k_blocks ? kb1 : k_blocks;
      if constexpr (PP) {
        if ((local & 1) != wg) {   // the other warpgroup's item: its K blocks pass through the ring in between
          stage += kb1 - kb0;
          while (stage >= STAGES) { stage -= STAGES; phase ^= 1; }
          continue;
        }
        // the mainloops go in item order: wait until the previous item's wgmma have been issued
        if (local > 0) mbar_wait(&turn[wg], ((local - 1) >> 1) & 1);
      }
      const int use = PP ? local >> 1 : local;   // this warpgroup's items so far: parity of its epilogue barriers
      float acc[BN / 2];
      int prev = -1;
      for (int kb = kb0; kb < kb1; kb++) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(tiles + stage * C::STAGE_BYTES) + rows_off;   // this warpgroup's 64 rows of A
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
      if constexpr (PP) mbar_arrive(&turn[wg ^ 1]);   // the other warpgroup's next mainloop may go
      wgmma_wait<0>();
      if (prev >= 0) mbar_arrive(&empty[prev]);

      if constexpr (EPI == EPI_F32) {
        // ---- fp32 split-K partials straight from the registers (+ bias: the unsplit esvit_gemm_f32 only) ----
#pragma unroll
        for (int i = 0; i < BN / 8; i++) {
          const int col = n0 + i * 8 + frag_col;
          if (col >= p.N) continue;  // N % 8 == 0: col + 1 < N as well, and the test is uniform over the warp
          const float2 bb = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + col)) : make_float2(0.f, 0.f);
#pragma unroll
          for (int h = 0; h < 2; h++) {
            const int row = m0 + frag_row + 8 * h;
            if (row >= p.M) continue;
            const long long off = (long long)row * p.N + col;
            float2 v = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
            if (p.bias) { v.x += bb.x; v.y += bb.y; }   // no bias: the partials as accumulated, signed zeros included
            *reinterpret_cast<float2*>(p.part + (long long)split * p.M * p.N + off) = v;
          }
        }
        continue;
      }

      // ---- bf16 epilogue: 64-column chunks through swizzled shared memory, one TMA tile store per chunk and warpgroup.
      // Rows >= M and columns >= N of a box are clipped by the TMA, so there is no bounds test on the stores; the
      // operands' out-of-bounds rows / columns were zero-filled, so those accumulators (and multipliers) are 0.
      // ldmatrix / stmatrix lane address: row (lane & 15) of the warp's 16, 16-byte column block (lane >> 4) of a pair;
      // the 128B swizzle puts 16-byte block c of row r at block c ^ (r & 7): the 8 rows of a matrix hit distinct banks.
      if constexpr (EPI == EPI_MUL) mbar_wait(&cs_empty[e], (use & 1) ^ 1);   // the previous tile's partials are folded
      const uint32_t lrow = (uint32_t)(warp * 16 + (lane & 15)) * 128u, lsw = lane & 7, lblk = lane >> 4;
      const bool leader = t == 0;   // issues this warpgroup's stores and waits for them
#pragma unroll
      for (int c = 0; c < NCHUNK; c++) {
        uint32_t buf;   // this warpgroup's [64 rows][128 B] of the chunk buffer
        if constexpr (EPI == EPI_MUL) {
          buf = smem_u32(my_ep + c * C::CHUNK_BYTES) + rows_off;
          mbar_wait(&mul_full[e * NCHUNK + c], use & 1);
        } else {
          buf = smem_u32(my_ep + (c & 1) * (EPI == EPI_GELU ? 2 : 1) * C::CHUNK_BYTES) + rows_off;
        }
#pragma unroll
        for (int jj = 0; jj < 8; jj += 2) {
          const int i = c * 8 + jj;   // 8-column blocks i, i + 1 of the tile
          const uint32_t addr = buf + lrow + (((jj + lblk) ^ lsw) << 4);
          const float* a0 = acc + 4 * i;
          if constexpr (EPI == EPI_MUL) {
            uint32_t m[4];
            ldmatrix_x4(addr, m[0], m[1], m[2], m[3]);
            uint32_t o[4];
            float cs[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
            for (int q = 0; q < 4; q++) {   // matrix q: column block i + q / 2, rows + 8 (q % 2)
              const float2 mf = unpack_bf162(m[q]);
              o[q] = pack_bf162(a0[2 * q] * mf.x, a0[2 * q + 1] * mf.y);
              const float2 of = unpack_bf162(o[q]);   // column sums of the STORED (bf16) values
              cs[q >> 1][0] += of.x; cs[q >> 1][1] += of.y;
            }
            stmatrix_x4(addr, o[0], o[1], o[2], o[3]);
            // reduce over the 8 row groups of the warp (lanes with equal lane % 4) into this warp's row of partials
#pragma unroll
            for (int s = 0; s < 2; s++) {
              float cs0 = cs[s][0], cs1 = cs[s][1];
#pragma unroll
              for (int o2 = 4; o2 < 32; o2 <<= 1) {
                cs0 += __shfl_xor_sync(0xffffffffu, cs0, o2);
                cs1 += __shfl_xor_sync(0xffffffffu, cs1, o2);
              }
              if (lane < 4)
                *reinterpret_cast<float2*>(cs_part + (wg * 4 + warp) * BN + (i + s) * 8 + frag_col) = make_float2(cs0, cs1);
            }
          } else {
            float b[4] = {0.f, 0.f, 0.f, 0.f};
            if (p.bias) {
#pragma unroll
              for (int s = 0; s < 2; s++) {
                const int col = n0 + (i + s) * 8 + frag_col;
                if (col < p.N) {   // N % 8 == 0: col + 1 < N as well
                  const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col));
                  b[2 * s] = bb.x; b[2 * s + 1] = bb.y;
                }
              }
            }
            uint32_t o[4], d[4];
#pragma unroll
            for (int q = 0; q < 4; q++) {
              const float v0 = a0[2 * q] + b[2 * (q >> 1)], v1 = a0[2 * q + 1] + b[2 * (q >> 1) + 1];
              if constexpr (EPI == EPI_GELU) {
                if (p.aux) {
                  float d0, d1;
                  float y0, y1;
                  if constexpr (QUICK) {
                    y0 = qgelu_fwd_grad(v0, d0); y1 = qgelu_fwd_grad(v1, d1);
                  } else {
                    y0 = gelu_fwd_grad(v0, d0); y1 = gelu_fwd_grad(v1, d1);
                  }
                  o[q] = pack_bf162(y0, y1);
                  d[q] = pack_bf162(d0, d1);
                } else if constexpr (QUICK) {
                  o[q] = pack_bf162(qgelu_fwd(v0), qgelu_fwd(v1));
                } else {
                  o[q] = pack_bf162(gelu_fwd(v0), gelu_fwd(v1));
                }
              } else {
                o[q] = pack_bf162(v0, v1);
              }
            }
            stmatrix_x4(addr, o[0], o[1], o[2], o[3]);
            if constexpr (EPI == EPI_GELU)
              if (p.aux) stmatrix_x4(addr + C::CHUNK_BYTES, d[0], d[1], d[2], d[3]);
          }
        }
        fence_proxy_async();
        // EPI_BIAS / EPI_GELU: the next chunk reuses the buffer of the previous one, whose store must have read it out
        if constexpr (EPI != EPI_MUL)
          if (leader) bulk_wait_read<0>();
        named_barrier(1 + wg, 128);
        if (leader) {
          const int gc = n0 + 64 * c, gr = m0 + row0;
          if (gc < p.N && gr < p.M) {
            tma_store_2d(&map_o, buf, gc, gr);
            if constexpr (EPI == EPI_GELU)
              if (p.aux) tma_store_2d(&map_x, buf + C::CHUNK_BYTES, gc, gr);
          }
          bulk_commit();
          if constexpr (EPI == EPI_MUL) {
            // chunk c - 1's buffer has been stored: the producer may load the next tile's multiplier into it
            if (c > 0) { bulk_wait_read<1>(); mbar_arrive(&mul_empty[e * NCHUNK + c - 1]); }
            if (c == NCHUNK - 1) { bulk_wait_read<0>(); mbar_arrive(&mul_empty[e * NCHUNK + c]); }
          }
        }
      }
      if constexpr (EPI == EPI_MUL) {
        __syncwarp();   // the warp's partials (lanes 0-3) are written before lane 0 releases them to the fold warps
        if (lane == 0) mbar_arrive(&cs_full[e]);
      }
    }
    if constexpr (EPI != EPI_F32)
      if (t == 0) bulk_wait_all();   // the CTA's last stores have completed before it exits
  }
}

// ---- back-to-back MLP forward: y = GELU(x . W1^T + b1) . W2^T + b2, the hidden activation never re-read from HBM ------
// x [M, C], W1 [4C, C], W2 [C, 4C] bf16.  Persistent over 128-row items; the producer TMA-loads an item's x tile once
// (double buffered across items) and streams the weights through the ring in chunks of 64 hidden units (W1 rows j*64..,
// W2 columns j*64..).  Each consumer warpgroup owns 64 rows and, per chunk in ascending order:
//   acc1 = x . W1_chunk^T          C/16 k16 steps of wgmma m64n64k16 (both operands from shared memory)
//   h    = GELU(acc1 + b1)         the gemm_kernel EPI_GELU arithmetic, packed to bf16: the m64n64 accumulator fragment
//                                  of 8-column blocks 2s, 2s + 1 IS the m64k16 A-register fragment of k16 step s
//   acc2 += h . W2_chunk^T         4 k16 steps of wgmma m64nCk16 with A from registers
// so fc1 runs the same k16 sequence as gemm_kernel over K = C and fc2 the same k16 sequence over K = 4C as its BK = 64
// mainloop: y, h and gelu' equal the two-launch chain's.  With STORE (the student) h and gelu' of each chunk leave
// through the bf16 staging path for the backward; y = acc2 + b2 leaves the same way at the end of the item.  acc2 [64 x C]
// lives in registers for the whole item, which bounds C: C = 256 fits neither the registers nor (with a double-buffered
// x tile) the shared memory.
template <int C>
struct MlpCfg {
  static constexpr int BM = 128, HB = 64;               // rows per item, hidden units per chunk
  static constexpr int KB = (C + 63) / 64;              // 64-column TMA boxes across C (the last zero-filled past C)
  static constexpr int NH = 4 * C / HB;                 // hidden chunks per item
  static constexpr int X_BYTES = KB * BM * 128;         // x tile: KB boxes of [128 rows][128 B]
  static constexpr int W1_BYTES = KB * HB * 128;        // W1 chunk: KB boxes of [64 hidden rows][128 B]
  static constexpr int W2_BYTES = C * 128;              // W2 chunk: one box of [C rows][64 hidden = 128 B]
  static constexpr int STAGE_BYTES = W1_BYTES + W2_BYTES;
  static constexpr int CHUNK_BYTES = BM * 128;          // one [128 rows x 64 columns] bf16 output chunk, 128B-swizzled
  static constexpr int EP_BYTES = 2 * CHUNK_BYTES;      // (h, gelu') of a hidden chunk; y chunks alternate over both
  static constexpr int BAR_BYTES = 128;
  static constexpr int STAGES_RAW = (SMEM_LIMIT - 1024 - BAR_BYTES - 2 * X_BYTES - EP_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 4 ? 4 : STAGES_RAW;
  static constexpr int SMEM = 1024 + 2 * X_BYTES + STAGES * STAGE_BYTES + EP_BYTES + BAR_BYTES;
  static_assert(C % 32 == 0 && C <= 192, "acc2 [64 x C] must fit the consumer registers; C / 8 even");
  static_assert(STAGES >= 2, "weight ring too shallow");
  static_assert(SMEM <= SMEM_LIMIT, "shared memory budget");
  static_assert((2 * STAGES + 4) * 8 <= BAR_BYTES, "mbarrier area");
};

struct MlpParams {
  const float* b1;  // [4C] or nullptr
  const float* b2;  // [C] or nullptr
  int M;
};

// map_x: x box [64 cols][128 rows]; map_w1: [64 cols][64 rows]; map_w2: [64 cols][C rows]; map_y / map_h / map_g: output
// boxes [64 cols][64 rows] (map_h / map_g unused without STORE)
template <int C, bool STORE>
__global__ void __launch_bounds__(384, 1) mlp_fwd_kernel(const __grid_constant__ CUtensorMap map_x,
                                                         const __grid_constant__ CUtensorMap map_w1,
                                                         const __grid_constant__ CUtensorMap map_w2,
                                                         const __grid_constant__ CUtensorMap map_y,
                                                         const __grid_constant__ CUtensorMap map_h,
                                                         const __grid_constant__ CUtensorMap map_g, const MlpParams p) {
  using G = MlpCfg<C>;
  constexpr int BM = G::BM, KB = G::KB, NH = G::NH, STAGES = G::STAGES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // x[2] | [STAGES][W1 | W2] | (h, gelu') staging | mbarriers; every tile 1024-byte aligned in the shared address space
  uint8_t* xs = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* ws = xs + 2 * G::X_BYTES;
  uint8_t* ep = ws + STAGES * G::STAGE_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(ep + G::EP_BYTES);
  uint64_t* empty = full + STAGES;
  uint64_t* x_full = empty + STAGES;
  uint64_t* x_empty = x_full + 2;

  const int wg = threadIdx.x >> 7;
  const int num_items = (p.M + BM - 1) / BM;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(&map_x) : "memory");
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(&map_w1) : "memory");
    asm volatile("prefetch.tensormap [%0];\n" ::"l"(&map_w2) : "memory");
    for (int i = 0; i < STAGES; i++) { mbar_init(&full[i], 1); mbar_init(&empty[i], 256); }
    for (int i = 0; i < 2; i++) { mbar_init(&x_full[i], 1); mbar_init(&x_empty[i], 256); }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (wg == 2) {
    // ===================== TMA producer: one thread of the last warpgroup =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (threadIdx.x == 256) {
      int stage = 0;
      uint32_t phase = 0;
      int local = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x, local++) {
        const int m0 = item * BM, xb = local & 1;
        // x buffer xb was last read by the fc1 of item local - 2
        mbar_wait(&x_empty[xb], ((local >> 1) & 1) ^ 1);
        mbar_expect_tx(&x_full[xb], G::X_BYTES);
#pragma unroll
        for (int kb = 0; kb < KB; kb++)
          tma_load_2d(smem_u32(xs + xb * G::X_BYTES + kb * BM * 128), &map_x, &x_full[xb], kb * 64, m0);
        for (int j = 0; j < NH; j++) {
          mbar_wait(&empty[stage], phase ^ 1);
          const uint32_t sw = smem_u32(ws + stage * G::STAGE_BYTES);
          mbar_expect_tx(&full[stage], G::STAGE_BYTES);
#pragma unroll
          for (int kb = 0; kb < KB; kb++) tma_load_2d(sw + kb * 8192, &map_w1, &full[stage], kb * 64, j * 64);
          tma_load_2d(sw + G::W1_BYTES, &map_w2, &full[stage], j * 64, 0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the item =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
    const int frag_col = 2 * (lane & 3);
    const uint32_t lrow = (uint32_t)(warp * 16 + (lane & 15)) * 128u, lsw = lane & 7, lblk = lane >> 4;
    const bool leader = t == 0;   // issues this warpgroup's stores and waits for them
    const uint32_t hbuf = smem_u32(ep) + wg * 8192;   // this warpgroup's rows of the h staging chunk (+ CHUNK_BYTES: gelu')
    int stage = 0;
    uint32_t phase = 0;
    int local = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x, local++) {
      const int m0 = item * BM, xb = local & 1;
      const uint64_t da = make_smem_desc(smem_u32(xs + xb * G::X_BYTES) + wg * 8192, false);   // this warpgroup's 64 rows
      float acc1[32], acc2[C / 2];
      mbar_wait(&x_full[xb], (local >> 1) & 1);
      for (int j = 0; j < NH; j++) {
        // fc1: acc1 = x . W1_chunk^T
        {
          const uint64_t db = make_smem_desc(smem_u32(ws + stage * G::STAGE_BYTES), false);
          mbar_wait(&full[stage], phase);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < C / 16; k++)   // descriptor units of 16 B: k16 step = 32 B, x box = BM * 128 B, W1 box = 8 KB
            wgmma_ss_n64(acc1, da + (k >> 2) * (BM * 128 >> 4) + (k & 3) * 2, db + (k >> 2) * (8192 >> 4) + (k & 3) * 2,
                         k ? 1u : 0u);
          wgmma_commit();
        }
        wgmma_wait<0>();   // fc1 of chunk j has retired
        if (j == NH - 1) mbar_arrive(&x_empty[xb]);   // the item's last fc1 has read x
        if constexpr (STORE) {
          // the previous chunk's stores have read the staging buffers before they are overwritten
          if (leader) bulk_wait_read<0>();
          named_barrier(1 + wg, 128);
        }
        // bias + GELU (+ gelu' to the staging buffer) -> bf16 A fragments of the 4 k16 steps of fc2
        uint32_t af[4][4];
#pragma unroll
        for (int s = 0; s < 4; s++) {
          const float* a0 = acc1 + 8 * s;   // 8-column blocks 2s, 2s + 1 of the chunk
          float b[4] = {0.f, 0.f, 0.f, 0.f};
          if (p.b1) {
#pragma unroll
            for (int u = 0; u < 2; u++) {
              const float2 bb = __ldg(reinterpret_cast<const float2*>(p.b1 + j * 64 + (2 * s + u) * 8 + frag_col));
              b[2 * u] = bb.x; b[2 * u + 1] = bb.y;
            }
          }
          uint32_t d[4];
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const float v0 = a0[2 * q] + b[2 * (q >> 1)], v1 = a0[2 * q + 1] + b[2 * (q >> 1) + 1];
            if constexpr (STORE) {
              float d0, d1;
              const float y0 = gelu_fwd_grad(v0, d0), y1 = gelu_fwd_grad(v1, d1);
              af[s][q] = pack_bf162(y0, y1);
              d[q] = pack_bf162(d0, d1);
            } else {
              af[s][q] = pack_bf162(gelu_fwd(v0), gelu_fwd(v1));
            }
          }
          if constexpr (STORE) {
            const uint32_t addr = hbuf + lrow + (((2 * s + lblk) ^ lsw) << 4);
            stmatrix_x4(addr, af[s][0], af[s][1], af[s][2], af[s][3]);
            stmatrix_x4(addr + G::CHUNK_BYTES, d[0], d[1], d[2], d[3]);
          }
        }
        if constexpr (STORE) fence_proxy_async();
        // fc2: acc2 += h_chunk . W2_chunk^T.  It retires before the next fc1 is issued, so acc1 and the A fragments are
        // never live at once: at C = 192 acc2 (96) + acc1 (32) + the fragments (16) would not fit next to the addressing.
        const uint64_t d2 = make_smem_desc(smem_u32(ws + stage * G::STAGE_BYTES) + G::W1_BYTES, false);
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < 4; s++) wgmma_rs(acc2, af[s], d2 + s * 2, (j > 0 || s > 0) ? 1u : 0u);
        wgmma_commit();
        if constexpr (STORE) {
          named_barrier(1 + wg, 128);
          if (leader) {
            const int gr = m0 + 64 * wg;
            if (gr < p.M) {
              tma_store_2d(&map_h, hbuf, j * 64, gr);
              tma_store_2d(&map_g, hbuf + G::CHUNK_BYTES, j * 64, gr);
            }
            bulk_commit();
          }
        }
        wgmma_wait<0>();   // fc2 of chunk j has retired: its stage is free
        mbar_arrive(&empty[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      // ---- y = acc2 + b2: 64-column chunks alternating over the two staging buffers (the gemm_kernel EPI_BIAS path)
#pragma unroll
      for (int c = 0; c < KB; c++) {
        const uint32_t buf = smem_u32(ep + (c & 1) * G::CHUNK_BYTES) + wg * 8192;
        if (leader) bulk_wait_read<0>();
        named_barrier(1 + wg, 128);
#pragma unroll
        for (int jj = 0; jj < 8; jj += 2) {
          const int i = c * 8 + jj;   // 8-column blocks i, i + 1 of y
          if (i >= C / 8) continue;
          const float* a0 = acc2 + 4 * i;
          float b[4] = {0.f, 0.f, 0.f, 0.f};
          if (p.b2) {
#pragma unroll
            for (int u = 0; u < 2; u++) {
              const float2 bb = __ldg(reinterpret_cast<const float2*>(p.b2 + (i + u) * 8 + frag_col));
              b[2 * u] = bb.x; b[2 * u + 1] = bb.y;
            }
          }
          uint32_t o[4];
#pragma unroll
          for (int q = 0; q < 4; q++) o[q] = pack_bf162(a0[2 * q] + b[2 * (q >> 1)], a0[2 * q + 1] + b[2 * (q >> 1) + 1]);
          stmatrix_x4(buf + lrow + (((jj + lblk) ^ lsw) << 4), o[0], o[1], o[2], o[3]);
        }
        fence_proxy_async();
        named_barrier(1 + wg, 128);
        if (leader) {
          const int gr = m0 + 64 * wg;
          if (gr < p.M) tma_store_2d(&map_y, buf, c * 64, gr);
          bulk_commit();
        }
      }
    }
    if (t == 0) bulk_wait_all();   // the CTA's last stores have completed before it exits
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
  auto encode = [&]() {
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  };
  CUresult r = encode();
  if (r == CUDA_ERROR_INVALID_CONTEXT) {
    // a driver-API call in a thread that has made no runtime call yet (e.g. the first GEMM of autograd's backward
    // thread): the runtime binds its context to a thread lazily, so bind the current device's primary context and retry
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaSetDevice(dev) == cudaSuccess) r = encode();
  }
  return r == CUDA_SUCCESS;
}

template <int C, bool STORE>
static int mlp_launch(const void* x, const void* w1, const float* b1, const void* w2, const float* b2, void* y, void* h,
                      void* g, int M, void* stream) {
  using G = MlpCfg<C>;
  CUtensorMap mx, m1, m2, my, mh = {}, mg = {};
  if (!make_map(&mx, x, M, C, G::BM) || !make_map(&m1, w1, 4 * C, C, 64) || !make_map(&m2, w2, C, 4 * C, C) ||
      !make_map(&my, y, M, C, 64))
    return ESVIT_ERR_BAD_ARG;
  if (STORE && (!make_map(&mh, h, M, 4 * C, 64) || !make_map(&mg, g, M, 4 * C, 64))) return ESVIT_ERR_BAD_ARG;
  auto kernel = mlp_fwd_kernel<C, STORE>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, G::SMEM);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  const int items = (M + G::BM - 1) / G::BM;
  int grid = esvit_num_sms();
  if (grid > items) grid = items;
  MlpParams p;
  p.b1 = b1; p.b2 = b2; p.M = M;
  kernel<<<grid, 384, G::SMEM, (cudaStream_t)stream>>>(mx, m1, m2, my, mh, mg, p);
  return (int)cudaGetLastError();
}

template <int C>
static int mlp_launch_c(const void* x, const void* w1, const float* b1, const void* w2, const float* b2, void* y, void* h,
                        void* g, int M, void* stream) {
  return h ? mlp_launch<C, true>(x, w1, b1, w2, b2, y, h, g, M, stream)
           : mlp_launch<C, false>(x, w1, b1, w2, b2, y, h, g, M, stream);
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

template <int WG, int BN, int EPI, int AMN, int BMN, bool QUICK = false>
static int launch_cfg(const Call& c, void* stream, int* rows_out) {
  using C = Cfg<WG, BN, EPI>;
  Params p = c.p;
  CUtensorMap ma, mb;
  // A: K-major [M,K] box [64 K][BM rows] | MN-major [K,M] box [64 M][64 K rows]
  if (!(AMN ? make_map(&ma, c.a, p.K, p.M, 64) : make_map(&ma, c.a, p.M, p.K, C::BM))) return ESVIT_ERR_BAD_ARG;
  // B: K-major [N,K] box [64 K][BN rows] | MN-major [K,N] box [64 N][64 K rows]
  if (!(BMN ? make_map(&mb, c.b, p.K, p.N, 64) : make_map(&mb, c.b, p.N, p.K, BN))) return ESVIT_ERR_BAD_ARG;
  // bf16 epilogues: out (and gelu' / the multiplier) [M,N] as [64 columns x 64 rows] boxes; the TMA needs 16-byte aligned
  // base addresses (the row pitch N * 2 B is a multiple of 16 because N % 8 == 0)
  CUtensorMap mo = {}, mx = {};
  if (EPI != EPI_F32) {
    auto aligned = [](const void* q) { return ((uintptr_t)q & 15u) == 0; };
    if (!p.out || !aligned(p.out) || (p.aux && !aligned(p.aux))) return ESVIT_ERR_BAD_ARG;
    if (!make_map(&mo, p.out, p.M, p.N, 64)) return ESVIT_ERR_BAD_ARG;
    if (p.aux && !make_map(&mx, p.aux, p.M, p.N, 64)) return ESVIT_ERR_BAD_ARG;
  }
  auto kernel = gemm_kernel<WG, BN, EPI, AMN, BMN, QUICK>;
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
  kernel<<<grid, C::NTHREADS, C::SMEM, (cudaStream_t)stream>>>(ma, mb, mo, mx, p);
  return (int)cudaGetLastError();
}

template <int WG, int BN, int EPI>
static int launch_majors(const Call& c, void* stream, int* rows_out) {
  if constexpr (EPI == EPI_F32) {  // weight gradient: both operands MN-major; fp32 forward (esvit_gemm_f32): both K-major
    if (c.a_mn && c.b_mn) return launch_cfg<WG, BN, EPI, 1, 1>(c, stream, rows_out);
    if (!c.a_mn && !c.b_mn) return launch_cfg<WG, BN, EPI, 0, 0>(c, stream, rows_out);
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

// QuickGELU forward GEMM (K-major operands only: the CvT fc1)
static int launch_quick(const Call& c, int wg, int bn, void* stream) {
  if (c.a_mn || c.b_mn) return ESVIT_ERR_BAD_ARG;
  if (wg == 2 && bn == 256) return launch_cfg<2, 256, EPI_GELU, 0, 0, true>(c, stream, nullptr);
  if (wg == 2 && bn == 128) return launch_cfg<2, 128, EPI_GELU, 0, 0, true>(c, stream, nullptr);
  if (wg == 1 && bn == 256) return launch_cfg<1, 256, EPI_GELU, 0, 0, true>(c, stream, nullptr);
  if (wg == 1 && bn == 128) return launch_cfg<1, 128, EPI_GELU, 0, 0, true>(c, stream, nullptr);
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
// the fewest operand bytes per MAC, but a GEMM with fewer tiles than SMs leaves SMs idle.  fit_n (the bf16 bias / GELU
// epilogues): no 256-wide tile where it pads N further than 128-wide ones (N = 288, 384, 576, 1152 of the Swin step),
// whose wasted wgmma columns and half-empty last tile cost more than the extra B reads, nor at K <= 256 (4 K blocks or
// fewer: the item is mostly epilogue, and 128-wide items overlap it better; the 65 536-wide last layers).  Measured at
// the step's shapes, DESIGN §4.1.  The multiplier epilogue keeps 256-wide tiles: at 128 x 128 it runs slowest of the
// four shapes.
static bool pads_more(long long n, int wide, int narrow) {
  return (n + wide - 1) / wide * wide > (n + narrow - 1) / narrow * narrow;
}
static void pick_tile(long long M, int N, int K, int tile, bool fit_n, int* wg, int* bn) {
  tile %= 10000;
  if (tile > 0) { *wg = tile / 1000; *bn = tile % 1000; return; }
  const int sms = esvit_num_sms();
  const bool narrow = fit_n && (pads_more(N, 256, 128) || K <= 256);
  const int cand[4][2] = {{2, 256}, {2, 128}, {1, 256}, {1, 128}};
  for (const auto& cd : cand) {
    if (cd[1] == 256 && (N <= 128 || narrow)) continue;
    const long long items = ((M + 64 * cd[0] - 1) / (64 * cd[0])) * ((N + cd[1] - 1) / cd[1]);
    if (items >= sms) { *wg = cd[0]; *bn = cd[1]; return; }
  }
  *wg = 1; *bn = 128;
}
// weight gradient (GEMM M = out features, N = in features, contraction over tokens): split-K supplies the parallelism.
// Tiles as large as the weight allows without padding it further than the smaller shape would: 64-row (ping-pong) tiles
// where 128-row ones pad the out features (192, 288, 576), 128-wide ones where 256-wide pad the in features (384).
static void pick_tile_wgrad(int Nout, int Kin, int tile, int* wg, int* bn) {
  tile %= 10000;
  if (tile > 0) { *wg = tile / 1000; *bn = tile % 1000; return; }
  *bn = Kin > 128 && !pads_more(Kin, 256, 128) ? 256 : 128;
  *wg = Nout > 64 && !pads_more(Nout, 128, 64) ? 2 : 1;
}

}  // namespace hg

// ---- C ABI ----------------------------------------------------------------------------------------------------------
// out[M,N] (bf16) = act( opA(a) . opB(b) + bias[N] )
//   a: a_mn = 0: [M,K] row-major (K contiguous) | a_mn = 1: [K,M] row-major (M contiguous)
//   b: b_mn = 0: [N,K] row-major (nn.Linear weight layout) | b_mn = 1: [K,N] row-major (N contiguous)
//   act 0: identity; act 1: GELU (pre != NULL also receives gelu'(pre-activation) for the backward); act 2: QuickGELU
//   x sigmoid(1.702 x) (pre likewise receives its derivative; a_mn = b_mn = 0 only)
//   M, N, K multiples of 8; bias fp32 or NULL.  tile = 0 (automatic) or warpgroups * 1000 + BN (1128, 1256, 2128, 2256).
ESVIT_API int esvit_gemm_bf16(const void* a, const void* b, const float* bias, void* out, void* pre, long long M, int N,
                              int K, int a_mn, int b_mn, int act, int tile, void* stream) {
  if (M <= 0 || N <= 0 || K <= 0 || (N % 8) || (K % 8) || M > 0x7fffffffLL || (a_mn && (M % 8)) || act < 0 || act > 2)
    return ESVIT_ERR_BAD_ARG;
  hg::Call c;
  c.a = a; c.b = b; c.a_mn = a_mn ? 1 : 0; c.b_mn = b_mn ? 1 : 0;
  c.p.bias = bias; c.p.out = (bf16*)out; c.p.aux = act ? (bf16*)pre : nullptr; c.p.colsum = nullptr; c.p.part = nullptr;
  c.p.M = (int)M; c.p.N = N; c.p.K = K; c.p.splits = 1; c.p.kb_per_split = (K + hg::BK - 1) / hg::BK;
  int wg, bn;
  hg::pick_tile(M, N, K, tile, true, &wg, &bn);
  if (act == 2) return hg::launch_quick(c, wg, bn, stream);
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
  hg::pick_tile(M, N, K, tile, false, &wg, &bn);
  const int rc = hg::launch(c, hg::EPI_MUL, wg, bn, stream, &rows);
  if (rc != 0) return rc;
  hg::colsum_fold_kernel<<<(N + 255) / 256, 256, 0, (cudaStream_t)stream>>>(ws, rows, N, colsum);
  ESVIT_LAUNCH_CHECK();
}

// out[M,N] (fp32) = a[M,K] . b[N,K]^T + bias[N]: a Linear forward with fp32 output (the linear probe's logits, whose
// top-5 order bf16 could not resolve).  The fp32 epilogue of the weight gradient with one K split, so every output is
// one tile's accumulator (+ bias) written once: bit-reproducible.  N, K multiples of 8; bias fp32 [N] or NULL; out
// 8-byte aligned.  tile as esvit_gemm_bf16.
ESVIT_API int esvit_gemm_f32(const void* a, const void* b, const float* bias, float* out, long long M, int N, int K,
                             int tile, void* stream) {
  if (M <= 0 || N <= 0 || K <= 0 || (N % 8) || (K % 8) || M > 0x7fffffffLL || !out || ((uintptr_t)out & 7) ||
      ((uintptr_t)bias & 7))
    return ESVIT_ERR_BAD_ARG;
  hg::Call c;
  c.a = a; c.b = b; c.a_mn = 0; c.b_mn = 0;
  c.p.bias = bias; c.p.out = nullptr; c.p.aux = nullptr; c.p.colsum = nullptr; c.p.part = out;
  c.p.M = (int)M; c.p.N = N; c.p.K = K; c.p.splits = 1; c.p.kb_per_split = (K + hg::BK - 1) / hg::BK;
  int wg, bn;
  hg::pick_tile(M, N, K, tile, false, &wg, &bn);
  return hg::launch(c, hg::EPI_F32, wg, bn, stream);
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
  if (T <= 0 || N <= 0 || K <= 0 || (N % 8) || (K % 8) || T > 0x7fffffffLL || !dw || !ws) return ESVIT_ERR_BAD_ARG;
  // the fold reads and writes dw and reads ws as float4
  auto aligned = [](const void* q) { return ((uintptr_t)q & 15u) == 0; };
  if (!aligned(dw) || !aligned(ws)) return ESVIT_ERR_BAD_ARG;
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

// y[M,C] (bf16) = GELU(x[M,C] . w1[4C,C]^T + b1) . w2[C,4C]^T + b2 in one kernel (hg::mlp_fwd_kernel): bit-identical to
// esvit_gemm_bf16 act 1 followed by esvit_gemm_bf16 act 0.  h, gelu_grad [M,4C] bf16: both NULL (no-grad forward), or both
// set to receive GELU(pre-activation) and gelu'(pre-activation) for the backward.  C in {96, 128, 192}; biases fp32 or NULL;
// every matrix 16-byte aligned.
ESVIT_API int esvit_mlp_fwd(const void* x, const void* w1, const float* b1, const void* w2, const float* b2, void* y,
                            void* h, void* gelu_grad, long long M, int C, void* stream) {
  auto aligned = [](const void* q, uintptr_t a) { return ((uintptr_t)q & (a - 1)) == 0; };
  if (M <= 0 || M > 0x7fffffffLL || !x || !w1 || !w2 || !y || (h == nullptr) != (gelu_grad == nullptr)) return ESVIT_ERR_BAD_ARG;
  if (!aligned(x, 16) || !aligned(w1, 16) || !aligned(w2, 16) || !aligned(y, 16) || !aligned(h, 16) ||
      !aligned(gelu_grad, 16) || !aligned(b1, 8) || !aligned(b2, 8))
    return ESVIT_ERR_BAD_ARG;
  switch (C) {
    case 96: return hg::mlp_launch_c<96>(x, w1, b1, w2, b2, y, h, gelu_grad, (int)M, stream);
    case 128: return hg::mlp_launch_c<128>(x, w1, b1, w2, b2, y, h, gelu_grad, (int)M, stream);
    case 192: return hg::mlp_launch_c<192>(x, w1, b1, w2, b2, y, h, gelu_grad, (int)M, stream);
  }
  return ESVIT_ERR_BAD_ARG;
}
