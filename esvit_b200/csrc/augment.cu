// Multi-crop augmentation (the reference's DataAugmentationDINO, datasets/build.py) on decoded uint8 images.
//
// Reference transforms, applied per crop with Pillow arithmetic (torchvision's PIL backend):
//   RandomResizedCrop(S, bicubic) -> RandomHorizontalFlip -> RandomApply(ColorJitter, 0.8) -> RandomGrayscale
//   -> utils.GaussianBlur (ImageFilter.GaussianBlur) -> [utils.Solarization] -> ToTensor -> Normalize
//
// Three kernels for all crops of a batch (DESIGN.md §4.7):
//   coeffs_kernel    Pillow's precompute_coeffs + normalize_coeffs_8bpc for both axes of every crop (bicubic a = -0.5,
//                    support scaled by the downscale factor, coefficients normalised in fp64 then rounded to 22-bit
//                    fixed point).  The tap count is unbounded: tables live in global memory.
//   resize_h_kernel  the horizontal pass over every row of the crop box into a uint8 intermediate [h, S, 3]; the flip
//                    is a mirrored output column.
//   color_kernel     one CTA per crop: the vertical pass into a planar uint8 crop in shared memory, the jitter ops in
//                    the sampled order (uint8 after each, as Pillow), grayscale, the 3+3 box-blur passes of Pillow's
//                    GaussianBlur, solarize, and ToTensor + Normalize in fp32 with streaming stores.
//
// The evaluation transforms (eval_linear.py / eval_knn.py: RandomResizedCrop(bilinear) + flip, Resize(256, bicubic) +
// CenterCrop) are one geometry per image: crop a box, resize it to (rh, rw), keep the S x S output window at (oy, ox),
// optionally flip.  Their kernels share the coefficient and horizontal-pass code above:
//   eval_coeffs_kernel    the window's tables of both axes, bilinear or bicubic per image;
//   eval_resize_h_kernel  the horizontal pass over the box rows the window's vertical taps touch;
//   eval_resize_v_kernel  the vertical pass, ToTensor + Normalize, coalesced fp32 stores of [B, 3, S, S].
//
// Every float/double expression that Pillow evaluates as a multiply followed by an add is written with _rn intrinsics
// so that no FMA contraction changes its rounding.
#include "common.cuh"

namespace aug {

// float64 parameter record of one crop (esvit_b200/augment.py PARAM_FIELDS)
enum { P_TOP, P_LEFT, P_H, P_W, P_FLIP, P_JITTER, P_PERM, P_BRIGHT = P_PERM + 4, P_CONTRAST, P_SAT, P_HUE, P_GRAY,
       P_BLUR, P_RADIUS, P_SOLAR, NPARAM };
// int64 per-crop geometry (esvit_b200/augment.py): source byte offset, source H, W, output S, intermediate byte
// offset, coefficient-table offset (int32 elements), horizontal / vertical tap counts, output address
enum { M_SRC, M_H, M_W, M_S, M_TMP, M_COEF, M_KH, M_KV, M_OUT, NMETA };

constexpr int PREC = 22;  // Pillow's PRECISION_BITS for 8-bit images

struct Bicubic {  // Pillow's bicubic_filter, a = -0.5
  static constexpr double support = 2.0;
  static __device__ __forceinline__ double filter(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(a + 2.0, x), a + 3.0), x), x), 1.0);
    if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), a);
    return 0.0;
  }
};

struct Bilinear {  // Pillow's bilinear_filter
  static constexpr double support = 1.0;
  static __device__ __forceinline__ double filter(double x) {
    if (x < 0.0) x = -x;
    return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
  }
};

// Entry i of the table of one axis of a resize in_size -> out_size whose outputs [o0, o0 + n) are kept, at tab:
// bounds [n][2] (first input index, tap count), then coefficients [n][ksize].  Pillow computes every output from its own
// taps, so a window's entries are those of the whole resize.
template <class Filter>
static __device__ void axis_coeffs(int in_size, int out_size, int o0, int n, int ksize, int i, int* tab) {
  const double scale = (double)in_size / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = __dmul_rn(Filter::support, filterscale);
  const double center = __dmul_rn((o0 + i) + 0.5, scale);
  const double ss = 1.0 / filterscale;
  int xmin = (int)__dadd_rn(__dsub_rn(center, support), 0.5);
  if (xmin < 0) xmin = 0;
  int xmax = (int)__dadd_rn(__dadd_rn(center, support), 0.5);
  if (xmax > in_size) xmax = in_size;
  xmax -= xmin;
  int* k = tab + 2 * n + (long long)i * ksize;
  double ww = 0.0;
  for (int x = 0; x < xmax; x++)
    ww = __dadd_rn(ww, Filter::filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss)));
  for (int x = 0; x < ksize; x++) {
    double w = 0.0;
    if (x < xmax) {
      w = Filter::filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss));
      if (ww != 0.0) w = __ddiv_rn(w, ww);
    }
    const double f = __dmul_rn(w, (double)(1 << PREC));
    k[x] = w < 0 ? (int)__dadd_rn(-0.5, f) : (int)__dadd_rn(0.5, f);
  }
  tab[2 * i] = xmin;
  tab[2 * i + 1] = xmax;
}

// grid (ceil(maxS / 128), 2, ncrops): one thread per (crop, axis, output index)
__global__ void __launch_bounds__(128) coeffs_kernel(const double* __restrict__ params, const long long* __restrict__ meta,
                                                     int* __restrict__ coef) {
  const long long* m = meta + (long long)blockIdx.z * NMETA;
  const double* p = params + (long long)blockIdx.z * NPARAM;
  const int S = (int)m[M_S], o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= S) return;
  const int kh = (int)m[M_KH], kv = (int)m[M_KV];
  int* tab = coef + m[M_COEF];
  if (blockIdx.y == 0) axis_coeffs<Bicubic>((int)p[P_W], S, 0, S, kh, o, tab);
  else axis_coeffs<Bicubic>((int)p[P_H], S, 0, S, kv, o, tab + (long long)S * (2 + kh));
}

static __device__ __forceinline__ uint8_t clip8(int ss) {  // Pillow's clip8 of a PRECISION_BITS accumulator
  const int v = ss >> PREC;
  return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v);
}

// out[y][flip ? S-1-ox : ox][c] = horizontal pass of source row top + y, for y in [0, rows); grid-stride over blockIdx.x
static __device__ __forceinline__ void resize_h_rows(const uint8_t* __restrict__ img, int W, int top, int left, int rows,
                                                     int S, const int* __restrict__ tab, int kh, bool flip,
                                                     uint8_t* __restrict__ out) {
  const long long n = (long long)rows * S;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(e / S), ox = (int)(e - (long long)y * S);
    const int xmin = tab[2 * ox], xn = tab[2 * ox + 1];
    const int* k = tab + 2 * S + (long long)ox * kh;
    const uint8_t* row = img + ((long long)(top + y) * W + left + xmin) * 3;
    int s0 = 1 << (PREC - 1), s1 = s0, s2 = s0;
    for (int x = 0; x < xn; x++) {
      const int w = __ldg(k + x);
      s0 += __ldg(row + 3 * x) * w;
      s1 += __ldg(row + 3 * x + 1) * w;
      s2 += __ldg(row + 3 * x + 2) * w;
    }
    uint8_t* o = out + ((long long)y * S + (flip ? S - 1 - ox : ox)) * 3;
    o[0] = clip8(s0);
    o[1] = clip8(s1);
    o[2] = clip8(s2);
  }
}

// grid (G, ncrops): tmp[y][flip ? S-1-ox : ox][c] = horizontal pass of box row y, for every row of the box
__global__ void __launch_bounds__(256) resize_h_kernel(const uint8_t* __restrict__ src, const double* __restrict__ params,
                                                       const long long* __restrict__ meta, const int* __restrict__ coef,
                                                       uint8_t* __restrict__ tmp) {
  const long long* m = meta + (long long)blockIdx.y * NMETA;
  const double* p = params + (long long)blockIdx.y * NPARAM;
  resize_h_rows(src + m[M_SRC], (int)m[M_W], (int)p[P_TOP], (int)p[P_LEFT], (int)p[P_H], (int)m[M_S],
                coef + m[M_COEF], (int)m[M_KH], p[P_FLIP] != 0.0, tmp + m[M_TMP]);
}

// ToTensor (u / 255) then Normalize ((x - mean) / std) in fp32, IEEE divisions in torchvision's order
static __device__ __forceinline__ float to_tensor_normalize(int u, float mu, float sd) {
  return __fdiv_rn(__fsub_rn(__fdiv_rn((float)u, 255.f), mu), sd);
}

// vertical pass of one output pixel: taps k[0, yn) down a column of a uint8 [rows, S, 3] intermediate, from col
static __device__ __forceinline__ void resize_v_px(const uint8_t* __restrict__ col, int S, const int* __restrict__ k,
                                                   int yn, uint8_t& r, uint8_t& g, uint8_t& b) {
  int s0 = 1 << (PREC - 1), s1 = s0, s2 = s0;
  for (int y = 0; y < yn; y++) {
    const int w = k[y];
    const uint8_t* px = col + (long long)y * S * 3;
    s0 += px[0] * w;
    s1 += px[1] * w;
    s2 += px[2] * w;
  }
  r = clip8(s0);
  g = clip8(s1);
  b = clip8(s2);
}

// Image.blend(a, b, f) on 8-bit bands: a + f * (b - a) in fp32, truncated, clipped
static __device__ __forceinline__ uint8_t blend(int a, int b, float f) {
  const float t = __fadd_rn((float)a, __fmul_rn(f, (float)(b - a)));
  return t <= 0.f ? 0 : t >= 255.f ? 255 : (uint8_t)(int)t;
}

static __device__ __forceinline__ int luma(int r, int g, int b) {  // convert('L')
  return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16;
}

static __device__ __forceinline__ uint8_t clip_int(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }

// Pillow's rgb2hsv_row (uint8 HSV), the hue shift of torchvision's adjust_hue, and Pillow's hsv2rgb
static __device__ void hue_shift(uint8_t& R, uint8_t& G, uint8_t& B, uint8_t dh) {
  const int r = R, g = G, b = B;
  const int maxc = max(r, max(g, b)), minc = min(r, min(g, b));
  int uh = 0, us = 0;
  const int uv = maxc;
  if (minc != maxc) {
    const float cr = (float)(maxc - minc);
    const float s = __fdiv_rn(cr, (float)maxc);
    const float rc = __fdiv_rn((float)(maxc - r), cr), gc = __fdiv_rn((float)(maxc - g), cr),
                bc = __fdiv_rn((float)(maxc - b), cr);
    float hf;
    if (r == maxc) hf = __fsub_rn(bc, gc);
    else if (g == maxc) hf = (float)__dsub_rn(__dadd_rn(2.0, (double)rc), (double)bc);
    else hf = (float)__dsub_rn(__dadd_rn(4.0, (double)gc), (double)rc);
    hf = (float)fmod(__dadd_rn(__ddiv_rn((double)hf, 6.0), 1.0), 1.0);
    uh = clip_int((int)__dmul_rn((double)hf, 255.0));
    us = clip_int((int)__dmul_rn((double)s, 255.0));
  }
  const int h = (uint8_t)(uh + dh), s = us, v = uv;
  if (s == 0) {
    R = G = B = (uint8_t)v;
    return;
  }
  const double h6 = __ddiv_rn(__dmul_rn((double)(float)h, 6.0), 255.0);
  const int i = (int)floor(h6);
  const float f = (float)__dsub_rn(h6, (double)(float)i);
  const float fs = (float)__ddiv_rn((double)(float)s, 255.0);
  const double vd = (double)(float)v;
  const uint8_t up = clip_int((int)round(__dmul_rn(vd, __dsub_rn(1.0, (double)fs))));
  const uint8_t uq = clip_int((int)round(__dmul_rn(vd, __dsub_rn(1.0, (double)__fmul_rn(fs, f)))));
  const uint8_t ut = clip_int((int)round(__dmul_rn(vd, __dsub_rn(1.0, __dmul_rn((double)fs, __dsub_rn(1.0, (double)f))))));
  const uint8_t uv8 = (uint8_t)v;
  switch (i % 6) {
    case 0: R = uv8; G = ut; B = up; break;
    case 1: R = uq; G = uv8; B = up; break;
    case 2: R = up; G = uv8; B = ut; break;
    case 3: R = up; G = uq; B = uv8; break;
    case 4: R = ut; G = up; B = uv8; break;
    default: R = uv8; G = up; B = uq; break;
  }
}

// _gaussian_blur_radius of Pillow's BoxBlur.c (3 passes): the box radius that approximates a Gaussian of `radius`
static __device__ float box_radius(float radius) {
  const float sigma2 = __fdiv_rn(__fmul_rn(radius, radius), 3.f);
  const float L = (float)sqrt(__dadd_rn(__dmul_rn(12.0, (double)sigma2), 1.0));
  const float l = (float)floor(__ddiv_rn(__dsub_rn((double)L, 1.0), 2.0));
  float a = __fmul_rn(__fadd_rn(__fmul_rn(2.f, l), 1.f), __fsub_rn(__fmul_rn(l, __fadd_rn(l, 1.f)), __fmul_rn(3.f, sigma2)));
  a = __fdiv_rn(a, __fmul_rn(6.f, __fsub_rn(sigma2, __fmul_rn(__fadd_rn(l, 1.f), __fadd_rn(l, 1.f)))));
  return __fadd_rn(l, a);
}

// One ImagingLineBoxBlur pass of a uint8 plane, along x (vertical = false) or y, edges clamped:
// out = (ww * sum(in[-r..r]) + fw * (in[-r-1] + in[r+1]) + 2^23) >> 24
static __device__ void box_pass(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int S, int r, uint32_t ww,
                                uint32_t fw, bool vertical) {
  for (int q = threadIdx.x; q < S * S; q += blockDim.x) {
    const int y = q / S, x = q - y * S;
    const int pos = vertical ? y : x;
    const uint8_t* line = vertical ? in + x : in + y * S;
    const int stride = vertical ? S : 1;
    uint32_t acc = 0;
    for (int t = -r; t <= r; t++) acc += line[min(max(pos + t, 0), S - 1) * stride];
    const uint32_t edge = line[max(pos - r - 1, 0) * stride] + line[min(pos + r + 1, S - 1) * stride];
    out[q] = (uint8_t)((acc * ww + edge * fw + (1u << 23)) >> 24);
  }
}

// one CTA per crop of output size S (crops [crop0, crop0 + gridDim.x)); dynamic smem 16 + 4 S^2 bytes
__global__ void __launch_bounds__(1024, 1) color_kernel(const double* __restrict__ params,
                                                        const long long* __restrict__ meta, const int* __restrict__ coef,
                                                        const uint8_t* __restrict__ tmp, const float* __restrict__ norm,
                                                        int crop0) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int c = crop0 + blockIdx.x;
  const long long* m = meta + (long long)c * NMETA;
  const double* p = params + (long long)c * NPARAM;
  const int S = (int)m[M_S], n = S * S, kh = (int)m[M_KH], kv = (int)m[M_KV];
  int* red = reinterpret_cast<int*>(smem);
  uint8_t* R = smem + 16;
  uint8_t* G = R + n;
  uint8_t* B = G + n;
  uint8_t* scr = B + n;

  // vertical pass of the uint8 intermediate (rows relative to the box top)
  const int* tab = coef + m[M_COEF] + (long long)S * (2 + kh);
  const uint8_t* t8 = tmp + m[M_TMP];
  for (int q = threadIdx.x; q < n; q += blockDim.x) {
    const int oy = q / S, ox = q - oy * S;
    const int ymin = tab[2 * oy];
    resize_v_px(t8 + ((long long)ymin * S + ox) * 3, S, tab + 2 * S + (long long)oy * kv, tab[2 * oy + 1], R[q], G[q],
                B[q]);
  }
  __syncthreads();

  if (p[P_JITTER] != 0.0) {
    for (int op = 0; op < 4; op++) {
      const int fn = (int)p[P_PERM + op];
      if (fn == 0) {  // brightness: blend with black
        const float f = (float)p[P_BRIGHT];
        for (int q = threadIdx.x; q < n; q += blockDim.x) {
          R[q] = blend(0, R[q], f);
          G[q] = blend(0, G[q], f);
          B[q] = blend(0, B[q], f);
        }
      } else if (fn == 1) {  // contrast: blend with int(mean(L) + 0.5) of the current crop
        if (threadIdx.x == 0) *red = 0;
        __syncthreads();
        int s = 0;
        for (int q = threadIdx.x; q < n; q += blockDim.x) s += luma(R[q], G[q], B[q]);
        s = __reduce_add_sync(0xffffffffu, s);
        if ((threadIdx.x & 31) == 0) atomicAdd(red, s);
        __syncthreads();
        const int mean = (int)__dadd_rn(__ddiv_rn((double)*red, (double)n), 0.5);
        const float f = (float)p[P_CONTRAST];
        for (int q = threadIdx.x; q < n; q += blockDim.x) {
          R[q] = blend(mean, R[q], f);
          G[q] = blend(mean, G[q], f);
          B[q] = blend(mean, B[q], f);
        }
      } else if (fn == 2) {  // saturation: blend with L
        const float f = (float)p[P_SAT];
        for (int q = threadIdx.x; q < n; q += blockDim.x) {
          const int l = luma(R[q], G[q], B[q]);
          R[q] = blend(l, R[q], f);
          G[q] = blend(l, G[q], f);
          B[q] = blend(l, B[q], f);
        }
      } else {  // hue: np.int32(hue * 255).astype(uint8) added to Pillow's uint8 H
        const uint8_t dh = (uint8_t)(int)__dmul_rn(p[P_HUE], 255.0);
        for (int q = threadIdx.x; q < n; q += blockDim.x) hue_shift(R[q], G[q], B[q], dh);
      }
      __syncthreads();
    }
  }
  if (p[P_GRAY] != 0.0) {
    for (int q = threadIdx.x; q < n; q += blockDim.x) R[q] = G[q] = B[q] = (uint8_t)luma(R[q], G[q], B[q]);
    __syncthreads();
  }
  if (p[P_BLUR] != 0.0) {  // ImagingGaussianBlur: 3 horizontal then 3 vertical box passes
    const float fr = box_radius((float)p[P_RADIUS]);
    const int r = (int)fr;
    const uint32_t ww = (uint32_t)__fdiv_rn(16777216.f, __fadd_rn(__fmul_rn(fr, 2.f), 1.f));
    const uint32_t fw = ((1u << 24) - (uint32_t)(r * 2 + 1) * ww) / 2;
    for (int ch = 0; ch < 3; ch++) {
      uint8_t* P = R + ch * n;
      for (int pass = 0; pass < 6; pass++) {
        const bool even = (pass & 1) == 0;
        box_pass(even ? P : scr, even ? scr : P, S, r, ww, fw, pass >= 3);
        __syncthreads();
      }
    }
  }
  // solarize, ToTensor + Normalize: fp32, streaming stores of [3, S, S]
  const bool solar = p[P_SOLAR] != 0.0;
  float* out = reinterpret_cast<float*>(m[M_OUT]);
  for (int ch = 0; ch < 3; ch++) {
    const uint8_t* P = R + ch * n;
    const float mu = norm[ch], sd = norm[3 + ch];
    for (int q = threadIdx.x; q < n; q += blockDim.x) {
      int u = P[q];
      if (solar && u >= 128) u = 255 - u;
      __stcs(out + (long long)ch * n + q, to_tensor_normalize(u, mu, sd));
    }
  }
}

// ---- evaluation transforms -------------------------------------------------------------------------------------------
// float64 record of one image (esvit_b200/augment.py EVAL_FIELDS): crop box, resized size, output window, flip, Pillow
// resample code (2 bilinear, 3 bicubic)
enum { R_TOP, R_LEFT, R_H, R_W, R_RH, R_RW, R_OY, R_OX, R_SIZE, R_FLIP, R_INTERP, NREC };
// int64 per-image geometry (esvit_b200/augment.py): source byte offset, source W, first box row of the window's vertical
// taps and their row count, intermediate byte offset, coefficient-table offset (int32 elements), horizontal / vertical
// tap counts
enum { E_SRC, E_W, E_Y0, E_ROWS, E_TMP, E_COEF, E_KH, E_KV, NEMETA };
constexpr int PIL_BICUBIC = 3;

template <class Filter>
static __device__ void eval_axis(const double* r, int axis, int S, int kh, int kv, int i, int* tab) {
  if (axis == 0) axis_coeffs<Filter>((int)r[R_W], (int)r[R_RW], (int)r[R_OX], S, kh, i, tab);
  else axis_coeffs<Filter>((int)r[R_H], (int)r[R_RH], (int)r[R_OY], S, kv, i, tab + (long long)S * (2 + kh));
}

// grid (ceil(S / 128), 2, nimg): one thread per (image, axis, window output)
__global__ void __launch_bounds__(128) eval_coeffs_kernel(const double* __restrict__ rec,
                                                          const long long* __restrict__ meta, int* __restrict__ coef,
                                                          int S) {
  const long long* m = meta + (long long)blockIdx.z * NEMETA;
  const double* r = rec + (long long)blockIdx.z * NREC;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S) return;
  const int kh = (int)m[E_KH], kv = (int)m[E_KV];
  int* tab = coef + m[E_COEF];
  if (r[R_INTERP] == PIL_BICUBIC) eval_axis<Bicubic>(r, blockIdx.y, S, kh, kv, i, tab);
  else eval_axis<Bilinear>(r, blockIdx.y, S, kh, kv, i, tab);
}

// grid (G, nimg): tmp[y][flip ? S-1-ox : ox][c] for box rows y0 + y, y in [0, rows)
__global__ void __launch_bounds__(256) eval_resize_h_kernel(const uint8_t* __restrict__ src,
                                                            const double* __restrict__ rec,
                                                            const long long* __restrict__ meta,
                                                            const int* __restrict__ coef, uint8_t* __restrict__ tmp,
                                                            int S) {
  const long long* m = meta + (long long)blockIdx.y * NEMETA;
  const double* r = rec + (long long)blockIdx.y * NREC;
  resize_h_rows(src + m[E_SRC], (int)m[E_W], (int)r[R_TOP] + (int)m[E_Y0], (int)r[R_LEFT], (int)m[E_ROWS], S,
                coef + m[E_COEF], (int)m[E_KH], r[R_FLIP] != 0.0, tmp + m[E_TMP]);
}

// grid (ceil(S^2 / 256), nimg): one thread per output pixel, consecutive threads on consecutive columns, so each
// channel plane of out [nimg, 3, S, S] is written with coalesced stores
__global__ void __launch_bounds__(256) eval_resize_v_kernel(const long long* __restrict__ meta,
                                                            const int* __restrict__ coef,
                                                            const uint8_t* __restrict__ tmp,
                                                            const float* __restrict__ norm, float* __restrict__ out,
                                                            int S) {
  const long long* m = meta + (long long)blockIdx.y * NEMETA;
  const int n = S * S, q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const int oy = q / S, ox = q - oy * S;
  const int* tab = coef + m[E_COEF] + (long long)S * (2 + (int)m[E_KH]);
  const int ymin = tab[2 * oy] - (int)m[E_Y0];
  uint8_t u[3];
  resize_v_px(tmp + m[E_TMP] + ((long long)ymin * S + ox) * 3, S, tab + 2 * S + (long long)oy * (int)m[E_KV],
              tab[2 * oy + 1], u[0], u[1], u[2]);
  float* o = out + (long long)blockIdx.y * 3 * n + q;
#pragma unroll
  for (int ch = 0; ch < 3; ch++) __stcs(o + (long long)ch * n, to_tensor_normalize(u[ch], norm[ch], norm[3 + ch]));
}

}  // namespace aug

using namespace aug;

ESVIT_API int esvit_augment_coeffs(const double* params, const long long* meta, int* coef, int ncrops, int max_S,
                                   void* stream) {
  if (ncrops <= 0 || max_S <= 0 || ncrops > 65535) return ESVIT_ERR_BAD_ARG;
  coeffs_kernel<<<dim3((max_S + 127) / 128, 2, ncrops), 128, 0, (cudaStream_t)stream>>>(params, meta, coef);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_augment_resize_h(const uint8_t* src, const double* params, const long long* meta, const int* coef,
                                     uint8_t* tmp, int ncrops, long long max_pixels, void* stream) {
  if (ncrops <= 0 || ncrops > 65535 || max_pixels <= 0) return ESVIT_ERR_BAD_ARG;
  const long long blocks = (max_pixels + 255) / 256;
  const int gx = (int)(blocks < 64 ? blocks : 64);
  resize_h_kernel<<<dim3(gx, ncrops), 256, 0, (cudaStream_t)stream>>>(src, params, meta, coef, tmp);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_augment_color(const double* params, const long long* meta, const int* coef, const uint8_t* tmp,
                                  const float* norm, int crop0, int ncrops, int S, void* stream) {
  const int smem = 16 + 4 * S * S;
  if (ncrops <= 0 || crop0 < 0 || S <= 0 || smem > 227 * 1024) return ESVIT_ERR_BAD_ARG;
  cudaError_t e = cudaFuncSetAttribute(color_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return (int)e;
  color_kernel<<<ncrops, 1024, smem, (cudaStream_t)stream>>>(params, meta, coef, tmp, norm, crop0);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_augment_eval_coeffs(const double* rec, const long long* meta, int* coef, int nimg, int S,
                                        void* stream) {
  if (nimg <= 0 || nimg > 65535 || S <= 0) return ESVIT_ERR_BAD_ARG;
  eval_coeffs_kernel<<<dim3((S + 127) / 128, 2, nimg), 128, 0, (cudaStream_t)stream>>>(rec, meta, coef, S);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_augment_eval_resize_h(const uint8_t* src, const double* rec, const long long* meta, const int* coef,
                                          uint8_t* tmp, int nimg, int S, long long max_pixels, void* stream) {
  if (nimg <= 0 || nimg > 65535 || S <= 0 || max_pixels <= 0) return ESVIT_ERR_BAD_ARG;
  const long long blocks = (max_pixels + 255) / 256;
  const int gx = (int)(blocks < 64 ? blocks : 64);
  eval_resize_h_kernel<<<dim3(gx, nimg), 256, 0, (cudaStream_t)stream>>>(src, rec, meta, coef, tmp, S);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_augment_eval_resize_v(const long long* meta, const int* coef, const uint8_t* tmp, const float* norm,
                                          float* out, int nimg, int S, void* stream) {
  if (nimg <= 0 || nimg > 65535 || S <= 0 || (long long)S * S > 0x7fffffffLL) return ESVIT_ERR_BAD_ARG;
  const int gx = (int)(((long long)S * S + 255) / 256);
  eval_resize_v_kernel<<<dim3(gx, nimg), 256, 0, (cudaStream_t)stream>>>(meta, coef, tmp, norm, out, S);
  ESVIT_LAUNCH_CHECK();
}
