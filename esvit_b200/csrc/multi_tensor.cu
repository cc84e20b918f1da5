// Multi-tensor teacher EMA and per-tensor gradient clipping: one launch per <=64 tensors, no host sync.
//
// Reference semantics:
//   EMA   main_esvit.py:587-590   param_k.mul_(m).add_((1 - m) * param_q)   -> fl(fl(k*m) + fl(q*(1-m))), NO fma
//   clip  utils.py:106-115        per-parameter L2 norm; coef = clip / (norm + 1e-6); if coef < 1: grad *= coef
#include "common.cuh"

namespace {

constexpr int MT_MAX = 64;
struct MTList {
  void* a[MT_MAX];
  const void* b[MT_MAX];
  long long n[MT_MAX];
};

__global__ void __launch_bounds__(256) ema_kernel(MTList L, float m, float om) {
  float* k = (float*)L.a[blockIdx.y];
  const float* q = (const float*)L.b[blockIdx.y];
  const long long n = L.n[blockIdx.y];
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  const bool vec = ((((uintptr_t)k) | ((uintptr_t)q)) & 15) == 0;
  const long long n4 = vec ? n / 4 : 0;
  for (long long i = tid; i < n4; i += nt) {
    float4 a = reinterpret_cast<float4*>(k)[i];
    const float4 b = reinterpret_cast<const float4*>(q)[i];
    a.x = __fadd_rn(__fmul_rn(a.x, m), __fmul_rn(b.x, om));
    a.y = __fadd_rn(__fmul_rn(a.y, m), __fmul_rn(b.y, om));
    a.z = __fadd_rn(__fmul_rn(a.z, m), __fmul_rn(b.z, om));
    a.w = __fadd_rn(__fmul_rn(a.w, m), __fmul_rn(b.w, om));
    reinterpret_cast<float4*>(k)[i] = a;
  }
  for (long long i = n4 * 4 + tid; i < n; i += nt) k[i] = __fadd_rn(__fmul_rn(k[i], m), __fmul_rn(q[i], om));
}

__global__ void __launch_bounds__(256) sumsq_kernel(MTList L, double* __restrict__ sumsq, int base) {
  const float* g = (const float*)L.a[blockIdx.y];
  const long long n = L.n[blockIdx.y];
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  if ((long long)blockIdx.x * blockDim.x >= n) return;
  const bool vec = (((uintptr_t)g) & 15) == 0;
  const long long n4 = vec ? n / 4 : 0;
  float s = 0.f;
  for (long long i = tid; i < n4; i += nt) {
    const float4 a = reinterpret_cast<const float4*>(g)[i];
    s += (a.x * a.x + a.y * a.y) + (a.z * a.z + a.w * a.w);
  }
  for (long long i = n4 * 4 + tid; i < n; i += nt) s += g[i] * g[i];
  __shared__ float sb[8];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sb[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < 8 ? sb[threadIdx.x] : 0.f;
    s = warp_sum(s);
    if (threadIdx.x == 0) atomicAdd(&sumsq[base + blockIdx.y], (double)s);
  }
}

__global__ void __launch_bounds__(256) clip_scale_kernel(MTList L, const double* __restrict__ sumsq, int base,
                                                         float clip, float* __restrict__ norms) {
  float* g = (float*)L.a[blockIdx.y];
  const long long n = L.n[blockIdx.y];
  const float norm = (float)sqrt(sumsq[base + blockIdx.y]);
  if (blockIdx.x == 0 && threadIdx.x == 0 && norms) norms[base + blockIdx.y] = norm;
  const float coef = __fdiv_rn(clip, __fadd_rn(norm, 1e-6f));
  if (!(coef < 1.f)) return;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  const bool vec = (((uintptr_t)g) & 15) == 0;
  const long long n4 = vec ? n / 4 : 0;
  for (long long i = tid; i < n4; i += nt) {
    float4 a = reinterpret_cast<float4*>(g)[i];
    a.x *= coef; a.y *= coef; a.z *= coef; a.w *= coef;
    reinterpret_cast<float4*>(g)[i] = a;
  }
  for (long long i = n4 * 4 + tid; i < n; i += nt) g[i] *= coef;
}

}  // namespace

// teacher[i] = teacher[i] * m + student[i] * (1 - m), fp32, bit-exact with the reference's two ATen ops
ESVIT_API int esvit_ema_multi(void* const* teacher, const void* const* student, const long long* numel, int n,
                              double momentum, void* stream) {
  if (n < 0) return ESVIT_ERR_BAD_ARG;
  const float m = (float)momentum, om = (float)(1.0 - momentum);  // python double -> fp32 scalar, like ATen
  for (int base = 0; base < n; base += MT_MAX) {
    MTList L;
    const int cnt = n - base < MT_MAX ? n - base : MT_MAX;
    for (int i = 0; i < cnt; i++) { L.a[i] = teacher[base + i]; L.b[i] = student[base + i]; L.n[i] = numel[base + i]; }
    ema_kernel<<<dim3(64, cnt), 256, 0, (cudaStream_t)stream>>>(L, m, om);
  }
  ESVIT_LAUNCH_CHECK();
}

// sumsq_ws: double[n] workspace; norms: float[n] (pre-clip norms, may be null)
ESVIT_API int esvit_clip_multi(void* const* grads, const long long* numel, int n, float clip, double* sumsq_ws,
                               float* norms, void* stream) {
  if (n < 0) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(sumsq_ws, 0, sizeof(double) * (size_t)n, st);
  if (e != cudaSuccess) return (int)e;
  for (int pass = 0; pass < 2; pass++) {
    for (int base = 0; base < n; base += MT_MAX) {
      MTList L;
      const int cnt = n - base < MT_MAX ? n - base : MT_MAX;
      for (int i = 0; i < cnt; i++) { L.a[i] = grads[base + i]; L.b[i] = nullptr; L.n[i] = numel[base + i]; }
      if (pass == 0)
        sumsq_kernel<<<dim3(64, cnt), 256, 0, st>>>(L, sumsq_ws, base);
      else
        clip_scale_kernel<<<dim3(64, cnt), 256, 0, st>>>(L, sumsq_ws, base, clip, norms);
    }
  }
  ESVIT_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------------------------
// Fused optimiser pass: per-tensor gradient clip (utils.py:106-115) + AdamW (torch.optim.AdamW semantics,
// main_esvit.py:411) + teacher EMA (main_esvit.py:587-590) in ONE sweep over the parameters.
//
// All step-varying scalars are read from DEVICE memory so that a captured CUDA graph replays with fresh values:
//   hyper fp32[8]  = {lr, wd_group0, beta1, beta2, eps, ema_m, ema_1m, clip}
//   state fp32[n*2] per tensor: {step count (as float), flag}  flag bit0 = weight-decayed group, bit1 = skip
//                    (skip = the reference set p.grad = None: cancel_gradients_last_layer; AdamW then ignores the
//                    parameter entirely - no decay, no moment update, no step count - while the EMA still runs)
//   sumsq double[n] = per-tensor sum of squares of the RAW gradient (esvit_grad_sumsq_multi)
// AdamW per element (torch/optim/adamw.py, amsgrad=False, maximize=False):
//   p *= 1 - lr*wd ; m = lerp(m, g, 1-b1) ; v = b2*v + (1-b2) g^2 ;
//   p -= (lr / (1-b1^t)) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
// EMA: k = fl(fl(k*m) + fl(p_new*(1-m)))  - the two-rounding form of the reference loop, bit-exact.
namespace {

struct OptList {
  float* p[MT_MAX / 2];
  const float* g[MT_MAX / 2];
  float* m[MT_MAX / 2];
  float* v[MT_MAX / 2];
  float* k[MT_MAX / 2];
  bf16* sp[MT_MAX / 2];  // optional bf16 shadow of the updated parameter (GEMM operand of the next step)
  bf16* sk[MT_MAX / 2];  // optional bf16 shadow of the updated teacher parameter
  long long n[MT_MAX / 2];
};

struct OptScalars {
  float decay, b1, b2, eps, step_size, inv_sqrt_bc2, em, e1m, coef;
  bool skip;
};

__device__ __forceinline__ void opt_elem(float& pv, float gv, float& mv, float& vv, float& kv, bool has_k,
                                         const OptScalars& c) {
  if (!c.skip) {
    gv *= c.coef;
    pv *= c.decay;
    mv = mv + (gv - mv) * (1.f - c.b1);
    vv = vv * c.b2 + (1.f - c.b2) * gv * gv;
    const float denom = sqrtf(vv) * c.inv_sqrt_bc2 + c.eps;
    pv -= c.step_size * (mv / denom);
  }
  if (has_k) kv = __fadd_rn(__fmul_rn(kv, c.em), __fmul_rn(pv, c.e1m));
}

__global__ void __launch_bounds__(256) adamw_ema_kernel(OptList L, const float* __restrict__ hyper,
                                                        float* __restrict__ state, const double* __restrict__ sumsq,
                                                        int base) {
  const int ti = base + blockIdx.y;
  const long long n = L.n[blockIdx.y];
  float* p = L.p[blockIdx.y];
  const float* g = L.g[blockIdx.y];
  float* m = L.m[blockIdx.y];
  float* v = L.v[blockIdx.y];
  float* k = L.k[blockIdx.y];
  bf16* sp = L.sp[blockIdx.y];
  bf16* sk = L.sk[blockIdx.y];
  // 4 elements per thread only when every pointer allows 16-byte (shadows: 8-byte) accesses; gradient views into a flat
  // bucket at an odd offset take the scalar path, where a thread owns ONE element per grid stride
  const bool vec = ((((uintptr_t)p) | ((uintptr_t)g) | ((uintptr_t)m) | ((uintptr_t)v) | ((uintptr_t)k)) & 15) == 0 &&
                   ((((uintptr_t)sp) | ((uintptr_t)sk)) & 7) == 0;
  if ((long long)blockIdx.x * blockDim.x * (vec ? 4 : 1) >= n) return;  // big tensors get many CTAs, tiny ones one
  const float lr = hyper[0], wd0 = hyper[1], clip = hyper[7];
  const int flag = (int)state[2 * ti + 1];
  OptScalars c;
  c.b1 = hyper[2]; c.b2 = hyper[3]; c.eps = hyper[4]; c.em = hyper[5]; c.e1m = hyper[6];
  c.skip = (flag & 2) != 0;
  const float wd = (flag & 1) ? wd0 : 0.f;
  const float t = state[2 * ti] + 1.f;  // this step's count (bump_steps_kernel advances it after the sweep)
  c.coef = 1.f;
  if (clip > 0.f) {
    const float norm = (float)sqrt(sumsq[ti]);
    const float cc = __fdiv_rn(clip, __fadd_rn(norm, 1e-6f));
    if (cc < 1.f) c.coef = cc;
  }
  const float bc1 = 1.f - powf(c.b1, t), bc2 = 1.f - powf(c.b2, t);
  c.step_size = lr / bc1;
  c.inv_sqrt_bc2 = rsqrtf(bc2);
  c.decay = 1.f - lr * wd;
  const bool has_k = k != nullptr;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  const long long n4 = vec ? n / 4 : 0;
  for (long long i = tid; i < n4; i += nt) {
    float4 pv = reinterpret_cast<float4*>(p)[i], mv = make_float4(0, 0, 0, 0), vv = mv, gv = mv, kv = mv;
    if (!c.skip) {
      gv = reinterpret_cast<const float4*>(g)[i];
      mv = reinterpret_cast<float4*>(m)[i];
      vv = reinterpret_cast<float4*>(v)[i];
    }
    if (has_k) kv = reinterpret_cast<float4*>(k)[i];
    opt_elem(pv.x, gv.x, mv.x, vv.x, kv.x, has_k, c);
    opt_elem(pv.y, gv.y, mv.y, vv.y, kv.y, has_k, c);
    opt_elem(pv.z, gv.z, mv.z, vv.z, kv.z, has_k, c);
    opt_elem(pv.w, gv.w, mv.w, vv.w, kv.w, has_k, c);
    if (!c.skip) {
      reinterpret_cast<float4*>(p)[i] = pv;
      reinterpret_cast<float4*>(m)[i] = mv;
      reinterpret_cast<float4*>(v)[i] = vv;
      if (sp) {
        uint2 u; u.x = pack_bf162(pv.x, pv.y); u.y = pack_bf162(pv.z, pv.w);
        reinterpret_cast<uint2*>(sp)[i] = u;
      }
    }
    if (has_k) {
      reinterpret_cast<float4*>(k)[i] = kv;
      if (sk) {
        uint2 u; u.x = pack_bf162(kv.x, kv.y); u.y = pack_bf162(kv.z, kv.w);
        reinterpret_cast<uint2*>(sk)[i] = u;
      }
    }
  }
  for (long long i = n4 * 4 + tid; i < n; i += nt) {
    float pv = p[i], mv = 0.f, vv = 0.f, gv = 0.f, kv = 0.f;
    if (!c.skip) { gv = g[i]; mv = m[i]; vv = v[i]; }
    if (has_k) kv = k[i];
    opt_elem(pv, gv, mv, vv, kv, has_k, c);
    if (!c.skip) {
      p[i] = pv; m[i] = mv; v[i] = vv;
      if (sp) sp[i] = __float2bfloat16_rn(pv);
    }
    if (has_k) {
      k[i] = kv;
      if (sk) sk[i] = __float2bfloat16_rn(kv);
    }
  }
}

__global__ void bump_steps_kernel(float* __restrict__ state, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && (((int)state[2 * i + 1]) & 2) == 0) state[2 * i] += 1.f;
}

}  // namespace

// per-tensor sum of squares of fp32 gradients into sumsq double[n] (zeroed here)
ESVIT_API int esvit_grad_sumsq_multi(void* const* grads, const long long* numel, int n, double* sumsq, void* stream) {
  if (n < 0) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(sumsq, 0, sizeof(double) * (size_t)n, st);
  if (e != cudaSuccess) return (int)e;
  for (int base = 0; base < n; base += MT_MAX) {
    MTList L;
    const int cnt = n - base < MT_MAX ? n - base : MT_MAX;
    for (int i = 0; i < cnt; i++) { L.a[i] = grads[base + i]; L.b[i] = nullptr; L.n[i] = numel[base + i]; }
    sumsq_kernel<<<dim3(64, cnt), 256, 0, st>>>(L, sumsq, base);
  }
  ESVIT_LAUNCH_CHECK();
}

// teacher / param_bf16 / teacher_bf16 may be NULL (no EMA / no bf16 shadows; individual shadow entries may be NULL
// too); see the comment block above for hyper / state / sumsq
ESVIT_API int esvit_adamw_ema_multi(void* const* params, const void* const* grads, void* const* exp_avg,
                                    void* const* exp_avg_sq, void* const* teacher, void* const* param_bf16,
                                    void* const* teacher_bf16, const long long* numel, int n, const float* hyper,
                                    float* state, const double* sumsq, void* stream) {
  if (n < 0) return ESVIT_ERR_BAD_ARG;
  constexpr int CH = MT_MAX / 2;
  for (int base = 0; base < n; base += CH) {
    OptList L;
    const int cnt = n - base < CH ? n - base : CH;
    for (int i = 0; i < cnt; i++) {
      L.p[i] = (float*)params[base + i];
      L.g[i] = (const float*)grads[base + i];
      L.m[i] = (float*)exp_avg[base + i];
      L.v[i] = (float*)exp_avg_sq[base + i];
      L.k[i] = teacher ? (float*)teacher[base + i] : nullptr;
      L.sp[i] = param_bf16 ? (bf16*)param_bf16[base + i] : nullptr;
      L.sk[i] = (teacher && teacher_bf16) ? (bf16*)teacher_bf16[base + i] : nullptr;
      L.n[i] = numel[base + i];
    }
    adamw_ema_kernel<<<dim3(512, cnt), 256, 0, (cudaStream_t)stream>>>(L, hyper, state, sumsq, base);
  }
  if (n > 0) bump_steps_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(state, n);
  ESVIT_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------------------------
// Fused SGD-momentum / LARS pass: per-tensor clip (utils.py:106-115) + torch.optim.SGD(momentum=0.9) or utils.LARS
// (utils.py:519-557, main_esvit.py:412-415) + teacher EMA (main_esvit.py:587-590) in ONE sweep.
//
//   hyper fp32[8]  = {lr, wd_group0, momentum, eta, ema_m, ema_1m, clip, unused}
//   state fp32[n*2] per tensor: {steps taken (as float), flag}  flag bit0 = weight-decayed group, bit1 = skip,
//                    bit2 = LARS trust ratio applies (p.dim() != 1; never set for SGD).  The step count only records
//                    "has a momentum buffer" for state_dict: the update does not depend on it.
//   sums double[n] (SGD: sum g^2) or double[3n] (LARS, planar: sum g^2 | sum p^2 | sum g*p, esvit_lars_sums_multi)
// Per element, with c the clip coefficient and wd the tensor's decay (0 outside group 0):
//   d = c*g + wd*p ;  d *= q (bit2) ;  buf = momentum*buf + d ;  p -= lr*buf
// torch SGD clones d into the buffer on a tensor's first step; the buffer here starts at zero and 0.9*0 + d == d
// exactly, so the first step needs no special case.  LARS's mu starts at zeros in the reference too.
// LARS trust ratio q = eta*||p|| / ||d|| when both norms are > 0, else 1, with ||d|| expanded from the raw sums:
//   ||d||^2 = c^2 sum g^2 + 2 c wd sum g*p + wd^2 sum p^2     (double)
// The sums are double accumulators, so the expansion loses accuracy only when its terms cancel by ~1e10 (||d|| ~ 1e-5
// of ||c g|| + ||wd p||), which a training step does not produce; it saves a second pass over g and p.
namespace {

struct SgdList {
  float* p[MT_MAX / 2];
  const float* g[MT_MAX / 2];
  float* b[MT_MAX / 2];
  float* k[MT_MAX / 2];
  bf16* sp[MT_MAX / 2];
  bf16* sk[MT_MAX / 2];
  long long n[MT_MAX / 2];
};

struct SgdScalars {
  float lr, wd, mom, q, em, e1m, coef;
  bool skip;
};

__device__ __forceinline__ void sgd_elem(float& pv, float gv, float& bv, float& kv, bool has_k, const SgdScalars& c) {
  if (!c.skip) {
    float d = gv * c.coef;  // the clip, as the reference's g.mul_(coef) (coef == 1 when the tensor is not clipped)
    d = d + c.wd * pv;      // coupled L2: g.add(p, alpha=wd)
    d *= c.q;               // LARS trust ratio (1 otherwise)
    bv = bv * c.mom + d;
    pv = pv - c.lr * bv;
  }
  if (has_k) kv = __fadd_rn(__fmul_rn(kv, c.em), __fmul_rn(pv, c.e1m));
}

__global__ void __launch_bounds__(256) sgd_ema_kernel(SgdList L, const float* __restrict__ hyper,
                                                      const float* __restrict__ state, const double* __restrict__ sums,
                                                      int base, int ntot) {
  const int ti = base + blockIdx.y;
  const long long n = L.n[blockIdx.y];
  float* p = L.p[blockIdx.y];
  const float* g = L.g[blockIdx.y];
  float* b = L.b[blockIdx.y];
  float* k = L.k[blockIdx.y];
  bf16* sp = L.sp[blockIdx.y];
  bf16* sk = L.sk[blockIdx.y];
  const bool vec = ((((uintptr_t)p) | ((uintptr_t)g) | ((uintptr_t)b) | ((uintptr_t)k)) & 15) == 0 &&
                   ((((uintptr_t)sp) | ((uintptr_t)sk)) & 7) == 0;
  if ((long long)blockIdx.x * blockDim.x * (vec ? 4 : 1) >= n) return;
  const float clip = hyper[6];
  const int flag = (int)state[2 * ti + 1];
  SgdScalars c;
  c.lr = hyper[0]; c.mom = hyper[2]; c.em = hyper[4]; c.e1m = hyper[5];
  c.skip = (flag & 2) != 0;
  c.wd = (flag & 1) ? hyper[1] : 0.f;
  c.coef = 1.f;
  if (clip > 0.f) {  // the clip exactly as the AdamW sweep forms it
    const float norm = (float)sqrt(sums[ti]);
    const float cc = __fdiv_rn(clip, __fadd_rn(norm, 1e-6f));
    if (cc < 1.f) c.coef = cc;
  }
  c.q = 1.f;
  if ((flag & 4) && !c.skip) {
    const double cd = c.coef, wd = c.wd;
    const double pn = sqrt(sums[ntot + ti]);
    const double dd = cd * cd * sums[ti] + 2.0 * cd * wd * sums[2 * ntot + ti] + wd * wd * sums[ntot + ti];
    const double dn = sqrt(fmax(dd, 0.0));
    if (pn > 0.0 && dn > 0.0) c.q = (float)((double)hyper[3] * pn / dn);
  }
  const bool has_k = k != nullptr;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  const long long n4 = vec ? n / 4 : 0;
  for (long long i = tid; i < n4; i += nt) {
    float4 pv = reinterpret_cast<float4*>(p)[i], bv = make_float4(0, 0, 0, 0), gv = bv, kv = bv;
    if (!c.skip) {
      gv = reinterpret_cast<const float4*>(g)[i];
      bv = reinterpret_cast<float4*>(b)[i];
    }
    if (has_k) kv = reinterpret_cast<float4*>(k)[i];
    sgd_elem(pv.x, gv.x, bv.x, kv.x, has_k, c);
    sgd_elem(pv.y, gv.y, bv.y, kv.y, has_k, c);
    sgd_elem(pv.z, gv.z, bv.z, kv.z, has_k, c);
    sgd_elem(pv.w, gv.w, bv.w, kv.w, has_k, c);
    if (!c.skip) {
      reinterpret_cast<float4*>(p)[i] = pv;
      reinterpret_cast<float4*>(b)[i] = bv;
      if (sp) {
        uint2 u; u.x = pack_bf162(pv.x, pv.y); u.y = pack_bf162(pv.z, pv.w);
        reinterpret_cast<uint2*>(sp)[i] = u;
      }
    }
    if (has_k) {
      reinterpret_cast<float4*>(k)[i] = kv;
      if (sk) {
        uint2 u; u.x = pack_bf162(kv.x, kv.y); u.y = pack_bf162(kv.z, kv.w);
        reinterpret_cast<uint2*>(sk)[i] = u;
      }
    }
  }
  for (long long i = n4 * 4 + tid; i < n; i += nt) {
    float pv = p[i], bv = 0.f, gv = 0.f, kv = 0.f;
    if (!c.skip) { gv = g[i]; bv = b[i]; }
    if (has_k) kv = k[i];
    sgd_elem(pv, gv, bv, kv, has_k, c);
    if (!c.skip) {
      p[i] = pv; b[i] = bv;
      if (sp) sp[i] = __float2bfloat16_rn(pv);
    }
    if (has_k) {
      k[i] = kv;
      if (sk) sk[i] = __float2bfloat16_rn(kv);
    }
  }
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// L.a = gradient, L.b = parameter (NULL: only sum g^2 is needed for this tensor)
__global__ void __launch_bounds__(256) lars_sums_kernel(MTList L, double* __restrict__ sums, int base, int ntot) {
  const float* g = (const float*)L.a[blockIdx.y];
  const float* p = (const float*)L.b[blockIdx.y];
  const long long n = L.n[blockIdx.y];
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  if ((long long)blockIdx.x * blockDim.x >= n) return;
  const bool has_p = p != nullptr;
  const bool vec = ((((uintptr_t)g) | ((uintptr_t)p)) & 15) == 0;
  const long long n4 = vec ? n / 4 : 0;
  double sgg = 0.0, spp = 0.0, sgp = 0.0;
  for (long long i = tid; i < n4; i += nt) {
    const float4 a = reinterpret_cast<const float4*>(g)[i];
    sgg += (double)a.x * a.x + (double)a.y * a.y + (double)a.z * a.z + (double)a.w * a.w;
    if (has_p) {
      const float4 w = reinterpret_cast<const float4*>(p)[i];
      spp += (double)w.x * w.x + (double)w.y * w.y + (double)w.z * w.z + (double)w.w * w.w;
      sgp += (double)a.x * w.x + (double)a.y * w.y + (double)a.z * w.z + (double)a.w * w.w;
    }
  }
  for (long long i = n4 * 4 + tid; i < n; i += nt) {
    const double a = g[i];
    sgg += a * a;
    if (has_p) {
      const double w = p[i];
      spp += w * w;
      sgp += a * w;
    }
  }
  __shared__ double sb[3][8];
  sgg = warp_sum_d(sgg); spp = warp_sum_d(spp); sgp = warp_sum_d(sgp);
  if ((threadIdx.x & 31) == 0) {
    sb[0][threadIdx.x >> 5] = sgg; sb[1][threadIdx.x >> 5] = spp; sb[2][threadIdx.x >> 5] = sgp;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const bool in = threadIdx.x < 8;
    sgg = warp_sum_d(in ? sb[0][threadIdx.x] : 0.0);
    spp = warp_sum_d(in ? sb[1][threadIdx.x] : 0.0);
    sgp = warp_sum_d(in ? sb[2][threadIdx.x] : 0.0);
    if (threadIdx.x == 0) {
      const int ti = base + blockIdx.y;
      atomicAdd(&sums[ti], sgg);
      if (has_p) {
        atomicAdd(&sums[ntot + ti], spp);
        atomicAdd(&sums[2 * ntot + ti], sgp);
      }
    }
  }
}

}  // namespace

// sums double[3n] (zeroed here), planar: [0, n) sum g^2 (feeds the clip, like esvit_grad_sumsq_multi), [n, 2n) sum p^2,
// [2n, 3n) sum g*p; params[i] NULL (or params NULL) -> only sum g^2 of tensor i (its p is not read)
ESVIT_API int esvit_lars_sums_multi(const void* const* grads, const void* const* params, const long long* numel, int n,
                                    double* sums, void* stream) {
  if (n < 0) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(sums, 0, sizeof(double) * 3 * (size_t)n, st);
  if (e != cudaSuccess) return (int)e;
  for (int base = 0; base < n; base += MT_MAX) {
    MTList L;
    const int cnt = n - base < MT_MAX ? n - base : MT_MAX;
    for (int i = 0; i < cnt; i++) {
      L.a[i] = (void*)grads[base + i];
      L.b[i] = params ? params[base + i] : nullptr;
      L.n[i] = numel[base + i];
    }
    lars_sums_kernel<<<dim3(64, cnt), 256, 0, st>>>(L, sums, base, n);
  }
  ESVIT_LAUNCH_CHECK();
}

// teacher / param_bf16 / teacher_bf16 may be NULL as in esvit_adamw_ema_multi; see the comment block above
ESVIT_API int esvit_sgd_ema_multi(void* const* params, const void* const* grads, void* const* momentum_buf,
                                  void* const* teacher, void* const* param_bf16, void* const* teacher_bf16,
                                  const long long* numel, int n, const float* hyper, float* state, const double* sums,
                                  void* stream) {
  if (n < 0) return ESVIT_ERR_BAD_ARG;
  constexpr int CH = MT_MAX / 2;
  for (int base = 0; base < n; base += CH) {
    SgdList L;
    const int cnt = n - base < CH ? n - base : CH;
    for (int i = 0; i < cnt; i++) {
      L.p[i] = (float*)params[base + i];
      L.g[i] = (const float*)grads[base + i];
      L.b[i] = (float*)momentum_buf[base + i];
      L.k[i] = teacher ? (float*)teacher[base + i] : nullptr;
      L.sp[i] = param_bf16 ? (bf16*)param_bf16[base + i] : nullptr;
      L.sk[i] = (teacher && teacher_bf16) ? (bf16*)teacher_bf16[base + i] : nullptr;
      L.n[i] = numel[base + i];
    }
    sgd_ema_kernel<<<dim3(512, cnt), 256, 0, (cudaStream_t)stream>>>(L, hyper, state, sums, base, n);
  }
  if (n > 0) bump_steps_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(state, n);
  ESVIT_LAUNCH_CHECK();
}
