// kernels_simt.cu - SIMT kernels of the stage forward pass (sm_90a).
//
// These are the non-contraction ops of the reference's `model.predict` (src/node.py:105-106):
// max-pool, global-average-pool, dense (HBM-bound GEMV at batch 1), softmax, standalone
// BN/ReLU/Add/ZeroPad for arbitrary cut points, format encode/decode, and the device-side flag
// kernels of the hop.  It also holds the exact-fp32 FFMA implicit-GEMM convolution that (a) serves
// shapes the wgmma kernel does not take (C_in = 3 stem) and (b) is the in-library cross-check of
// the tensor-core path.
#include <stdlib.h>

#include "common.cuh"

namespace defer {

// =============================================================================================
// conv: implicit GEMM, fp32 FFMA.  M = n*ho*wo pixels, N = cout, K = kh*kw*cin.
// 64x64 tile, BK = 16, 256 threads, 4x4 register tile per thread, register-prefetched.
// =============================================================================================
constexpr int CBM = 64, CBN = 64, CBK = 16;

template <int FIN, int FOUT, bool VEC4>
__global__ void __launch_bounds__(256) conv_simt_kernel(const ConvParams p) {
  __shared__ __align__(16) float As[CBK][CBM + 4];
  __shared__ __align__(16) float Bs[CBK][CBN + 4];

  const int t = threadIdx.x;
  const int M = p.n * p.ho * p.wo;
  const int K = p.kh * p.kw * p.cin;
  const int m0 = blockIdx.x * CBM;
  const int n0 = blockIdx.y * CBN;
  const size_t plane_in = (size_t)p.n * p.h * p.w_in * p.cin;
  const size_t plane_out = (size_t)M * p.cout;

  // A-load role: one pixel row, 4 consecutive k
  const int ar = t >> 2;
  const int akq = (t & 3) * 4;
  const int am = m0 + ar;
  const bool a_valid = am < M;
  int a_nb = 0, a_ih0 = 0, a_iw0 = 0;
  if (a_valid) {
    int ow = am % p.wo;
    int tmp = am / p.wo;
    int oh = tmp % p.ho;
    a_nb = tmp / p.ho;
    a_ih0 = oh * p.sh - p.pad_t;
    a_iw0 = ow * p.sw - p.pad_l;
  }
  // B-load role: one k row, 4 consecutive couts
  const int bk = t >> 4;
  const int bnq = (t & 15) * 4;
  const bool b_vec = (p.cout % 4 == 0) && (n0 + bnq + 3 < p.cout);

  const int ty = t >> 4, tx = t & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  float a_reg[4];
  float b_reg[4];

  auto load_tile = [&](int k0) {
    // ---- A
    if constexpr (VEC4) {
      int k = k0 + akq;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (a_valid && k < K) {
        int tap = k / p.cin;
        int ci = k - tap * p.cin;
        int khi = tap / p.kw;
        int kwi = tap - khi * p.kw;
        int ih = a_ih0 + khi, iw = a_iw0 + kwi;
        if (ih >= 0 && ih < p.h && iw >= 0 && iw < p.w_in) {
          size_t idx = (((size_t)a_nb * p.h + ih) * p.w_in + iw) * p.cin + ci;
          v = act_load4<FIN>(p.x, plane_in, idx);
        }
      }
      a_reg[0] = v.x; a_reg[1] = v.y; a_reg[2] = v.z; a_reg[3] = v.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int k = k0 + akq + j;
        float v = 0.f;
        if (a_valid && k < K) {
          int tap = k / p.cin;
          int ci = k - tap * p.cin;
          int khi = tap / p.kw;
          int kwi = tap - khi * p.kw;
          int ih = a_ih0 + khi, iw = a_iw0 + kwi;
          if (ih >= 0 && ih < p.h && iw >= 0 && iw < p.w_in) {
            size_t idx = (((size_t)a_nb * p.h + ih) * p.w_in + iw) * p.cin + ci;
            v = act_load<FIN>(p.x, plane_in, idx);
          }
        }
        a_reg[j] = v;
      }
    }
    // ---- B
    int k = k0 + bk;
    if (k < K) {
      const float* wp = p.w + (size_t)k * p.cout + n0 + bnq;
      if (b_vec) {
        float4 v = __ldg(reinterpret_cast<const float4*>(wp));
        b_reg[0] = v.x; b_reg[1] = v.y; b_reg[2] = v.z; b_reg[3] = v.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) b_reg[j] = (n0 + bnq + j < p.cout) ? __ldg(wp + j) : 0.f;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) b_reg[j] = 0.f;
    }
  };

  load_tile(0);
  for (int k0 = 0; k0 < K; k0 += CBK) {
#pragma unroll
    for (int j = 0; j < 4; ++j) As[akq + j][ar] = a_reg[j];
    *reinterpret_cast<float4*>(&Bs[bk][bnq]) = make_float4(b_reg[0], b_reg[1], b_reg[2], b_reg[3]);
    __syncthreads();
    if (k0 + CBK < K) load_tile(k0 + CBK);
#pragma unroll
    for (int k = 0; k < CBK; ++k) {
      float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      float av[4] = {a.x, a.y, a.z, a.w};
      float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }

  // ---- epilogue: scale/shift (bias + BN folded), residual, relu, store in the stage format
  const int c0 = n0 + tx * 4;
  if (c0 >= p.cout) return;
  const bool vec_out = (p.cout % 4 == 0) && (c0 + 3 < p.cout);
  float sc[4], sf[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int c = c0 + j;
    sc[j] = (p.scale && c < p.cout) ? __ldg(p.scale + c) : 1.f;
    sf[j] = (p.shift && c < p.cout) ? __ldg(p.shift + c) : 0.f;
  }
  const bool relu = p.flags & DEFER_FLAG_RELU;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int m = m0 + ty * 4 + i;
    if (m >= M) continue;
    size_t o = (size_t)m * p.cout + c0;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = fmaf(acc[i][j], sc[j], sf[j]);
    if (vec_out) {
      if (p.res) {
        float4 r = act_load4<FOUT>(p.res, plane_out, o);
        v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
      }
      if (relu) {
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = fmaxf(v[j], 0.f);
      }
      act_store4<FOUT>(p.y, plane_out, o, make_float4(v[0], v[1], v[2], v[3]));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (c0 + j < p.cout) {
          float u = v[j];
          if (p.res) u += act_load<FOUT>(p.res, plane_out, o + j);
          if (relu) u = fmaxf(u, 0.f);
          act_store<FOUT>(p.y, plane_out, o + j, u);
        }
      }
    }
  }
}

// =============================================================================================
// RGB stem: 7x7 / stride 2, C_in = 3, C_out = 64 (+ bias/BN scale-shift + ReLU).  K = 147 is hostile to
// TMA / UMMA (C_in = 3), so this is a direct fp32 convolution: one CTA = 8x8 output pixels x 64 channels,
// the 21x21x3 input patch and the whole 7x7x3x64 filter bank live in shared memory, each thread owns
// 4 consecutive pixels x 8 channels (32 fp32 accumulators) and per (kh, ci) reuses a 13-value input
// window across the 7 kw taps (27 shared loads : 224 FFMA).
// =============================================================================================
constexpr int STEM_T = 8;                   // output tile edge
constexpr int STEM_P = STEM_T * 2 + 5;      // input patch edge (21)

template <int FOUT>
__global__ void __launch_bounds__(128) stem7x7s2_kernel(const ConvParams p) {
  __shared__ __align__(16) float s_in[STEM_P * STEM_P * 3];
  __shared__ __align__(16) float s_w[147 * 64];
  const int t = threadIdx.x;
  const int tiles_w = (p.wo + STEM_T - 1) / STEM_T;
  const int tiles_h = (p.ho + STEM_T - 1) / STEM_T;
  int bid = blockIdx.x;
  const int tw = bid % tiles_w;
  bid /= tiles_w;
  const int th = bid % tiles_h;
  const int nb = bid / tiles_h;
  const int oh0 = th * STEM_T, ow0 = tw * STEM_T;
  const int ih0 = oh0 * 2 - p.pad_t, iw0 = ow0 * 2 - p.pad_l;

  // filter bank [kh][kw][ci][co] is already the HWIO order of the shipped weights: straight copy
  for (int i = t; i < 147 * 64 / 4; i += 128)
    reinterpret_cast<float4*>(s_w)[i] = __ldg(reinterpret_cast<const float4*>(p.w) + i);
  const float* xin = reinterpret_cast<const float*>(p.x) + (size_t)nb * p.h * p.w_in * 3;
  for (int i = t; i < STEM_P * STEM_P * 3; i += 128) {
    int ci = i % 3;
    int pc = (i / 3) % STEM_P;
    int pr = i / (3 * STEM_P);
    int ih = ih0 + pr, iw = iw0 + pc;
    float v = 0.f;
    if (ih >= 0 && ih < p.h && iw >= 0 && iw < p.w_in) v = __ldg(xin + ((size_t)ih * p.w_in + iw) * 3 + ci);
    s_in[i] = v;
  }
  __syncthreads();

  const int cg = t >> 4;           // channel group: channels cg*8 .. cg*8+7
  const int pg = t & 15;
  const int prow = pg >> 1;        // output row in the tile
  const int pc0 = (pg & 1) * 4;    // first of 4 consecutive output columns
  float acc[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  for (int kh = 0; kh < 7; ++kh) {
    const float* rowp = s_in + ((prow * 2 + kh) * STEM_P + pc0 * 2) * 3;
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
      float win[13];
#pragma unroll
      for (int j = 0; j < 13; ++j) win[j] = rowp[j * 3 + ci];
#pragma unroll
      for (int kw = 0; kw < 7; ++kw) {
        const float4* wp = reinterpret_cast<const float4*>(s_w + ((kh * 7 + kw) * 3 + ci) * 64 + cg * 8);
        const float4 w0 = wp[0], w1 = wp[1];
        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float xv = win[2 * i + kw];
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(xv, wv[j], acc[i][j]);
        }
      }
    }
  }

  const size_t plane_out = (size_t)p.n * p.ho * p.wo * 64;
  float sc[8], sf[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    sc[j] = p.scale ? __ldg(p.scale + cg * 8 + j) : 1.f;
    sf[j] = p.shift ? __ldg(p.shift + cg * 8 + j) : 0.f;
  }
  const bool relu = p.flags & DEFER_FLAG_RELU;
  const int oh = oh0 + prow;
  if (oh >= p.ho) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int ow = ow0 + pc0 + i;
    if (ow >= p.wo) continue;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[j] = fmaf(acc[i][j], sc[j], sf[j]);
      if (relu) v[j] = fmaxf(v[j], 0.f);
    }
    const size_t o = (((size_t)nb * p.ho + oh) * p.wo + ow) * 64 + cg * 8;
    act_store4<FOUT>(p.y, plane_out, o, make_float4(v[0], v[1], v[2], v[3]));
    act_store4<FOUT>(p.y, plane_out, o + 4, make_float4(v[4], v[5], v[6], v[7]));
  }
}

static bool stem_eligible(const ConvParams& p, bool x_is_f32) {
  return x_is_f32 && p.kh == 7 && p.kw == 7 && p.sh == 2 && p.sw == 2 && p.cin == 3 && p.cout == 64 && p.res == nullptr &&
         getenv("DEFER_NO_STEM_KERNEL") == nullptr;
}

template <int FOUT>
static int launch_stem_t(const ConvParams& p, cudaStream_t st) {
  const int tiles = ((p.wo + STEM_T - 1) / STEM_T) * ((p.ho + STEM_T - 1) / STEM_T) * p.n;
  prefer_max_smem(stem7x7s2_kernel<FOUT>);
  stem7x7s2_kernel<FOUT><<<tiles, 128, 0, st>>>(p);
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

template <int FIN, int FOUT>
static int launch_conv_simt_t(const ConvParams& p, cudaStream_t st) {
  int M = p.n * p.ho * p.wo;
  dim3 grid((M + CBM - 1) / CBM, (p.cout + CBN - 1) / CBN);
  if (p.cin % 4 == 0) {
    prefer_max_smem(conv_simt_kernel<FIN, FOUT, true>);
    conv_simt_kernel<FIN, FOUT, true><<<grid, 256, 0, st>>>(p);
  } else {
    prefer_max_smem(conv_simt_kernel<FIN, FOUT, false>);
    conv_simt_kernel<FIN, FOUT, false><<<grid, 256, 0, st>>>(p);
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

int launch_conv_simt(int fmt, bool x_is_f32, const ConvParams& p, cudaStream_t st) {
  if (stem_eligible(p, x_is_f32)) {
    switch (fmt) {
      case FMT_F32: return launch_stem_t<FMT_F32>(p, st);
      case FMT_BF16X2: return launch_stem_t<FMT_BF16X2>(p, st);
      case FMT_BF16: return launch_stem_t<FMT_BF16>(p, st);
    }
  }
  switch (fmt) {
    case FMT_F32: return launch_conv_simt_t<FMT_F32, FMT_F32>(p, st);
    case FMT_BF16X2:
      return x_is_f32 ? launch_conv_simt_t<FMT_F32, FMT_BF16X2>(p, st) : launch_conv_simt_t<FMT_BF16X2, FMT_BF16X2>(p, st);
    case FMT_BF16:
      return x_is_f32 ? launch_conv_simt_t<FMT_F32, FMT_BF16>(p, st) : launch_conv_simt_t<FMT_BF16, FMT_BF16>(p, st);
  }
  set_error("launch_conv_simt: bad fmt %d", fmt);
  return DEFER_ERR_INVALID;
}

// =============================================================================================
// Tensor-core stem, step 1: im2col of the fp32 RGB image into the stage's activation format.
// Row m = output pixel, column k = (kh * KW + kw) * C_in + ci  (the HWIO order of the shipped filter, so the
// filter bank IS the [K, C_out] GEMM operand), zero for taps in the padding and for k >= K up to K_pad (a
// multiple of 64).  The result feeds the wgmma conv kernel as a 1x1 convolution over K_pad channels.
// One thread = 8 consecutive k of one pixel: a 16-byte store per bf16 plane.
// =============================================================================================
// One CTA = one output row of one image.  The kh input rows that row needs are staged in shared memory with coalesced
// 16-byte loads (rows in the zero padding are stored as zeros); a patch is then kh runs of kw*cin CONTIGUOUS floats
// (NHWC), so k -> (kernel row a, offset jj) and one range check on the flat column index covers the left / right
// padding.  One work item = 8 consecutive k of one pixel = a 16-byte store per bf16 plane; consecutive items are
// consecutive addresses, so the patch matrix is written fully coalesced.
template <int FMT>
__global__ void __launch_bounds__(256) stem_im2col_kernel(const float* __restrict__ x, void* __restrict__ out, int n, int h,
                                                          int w, int cin, int kh, int kw, int sh, int sw, int pad_t,
                                                          int pad_l, int ho, int wo, int K, int K_pad) {
  extern __shared__ float rows[];                 // [kh][w * cin]
  const int oh = blockIdx.x % ho;
  const int nb = blockIdx.x / ho;
  const int row_len = w * cin;
  const int run = kw * cin;                       // contiguous floats per kernel row of a patch
  const float* xin = x + (size_t)nb * h * row_len;
  for (int a = 0; a < kh; ++a) {
    const int ih = oh * sh - pad_t + a;
    float* dst = rows + a * row_len;
    if (ih >= 0 && ih < h) {
      const float* src = xin + (size_t)ih * row_len;
      if ((row_len & 3) == 0) {
        const float4* s4 = reinterpret_cast<const float4*>(src);
        for (int i = threadIdx.x; i < (row_len >> 2); i += blockDim.x) reinterpret_cast<float4*>(dst)[i] = __ldg(s4 + i);
      } else {
        for (int i = threadIdx.x; i < row_len; i += blockDim.x) dst[i] = __ldg(src + i);
      }
    } else {
      for (int i = threadIdx.x; i < row_len; i += blockDim.x) dst[i] = 0.f;
    }
  }
  __syncthreads();
  const int groups = K_pad >> 3;
  const int items = wo * groups;
  const size_t plane = (size_t)n * ho * wo * K_pad;
  const size_t row_base = ((size_t)nb * ho + oh) * wo;
  for (int it = threadIdx.x; it < items; it += blockDim.x) {
    const int ow = it / groups;
    const int g = it - ow * groups;
    const int col0 = (ow * sw - pad_l) * cin;     // flat column of the patch's first element inside an input row
    int k = g * 8;
    int a = k / run, jj = k - a * run;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j, ++k) {
      float val = 0.f;
      if (k < K) {
        const int col = col0 + jj;
        if (col >= 0 && col < row_len) val = rows[a * row_len + col];
      }
      v[j] = val;
      if (++jj == run) { jj = 0; ++a; }
    }
    const size_t o = (row_base + ow) * K_pad + (size_t)g * 8;
    if constexpr (FMT == FMT_BF16X2) {
      uint4 hv, lv;
      split_bf16x2(v[0], v[1], hv.x, lv.x);
      split_bf16x2(v[2], v[3], hv.y, lv.y);
      split_bf16x2(v[4], v[5], hv.z, lv.z);
      split_bf16x2(v[6], v[7], hv.w, lv.w);
      __nv_bfloat16* pb = reinterpret_cast<__nv_bfloat16*>(out);
      *reinterpret_cast<uint4*>(pb + o) = hv;
      *reinterpret_cast<uint4*>(pb + plane + o) = lv;
    } else {
      uint4 hv;
      hv.x = pack_bf16x2(v[0], v[1]);
      hv.y = pack_bf16x2(v[2], v[3]);
      hv.z = pack_bf16x2(v[4], v[5]);
      hv.w = pack_bf16x2(v[6], v[7]);
      *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(out) + o) = hv;
    }
  }
}

int launch_stem_im2col(int fmt, const float* x, void* out, int n, int h, int w, int cin, int kh, int kw, int sh, int sw,
                       int pad_t, int pad_l, int ho, int wo, int K_pad, cudaStream_t st) {
  const int K = kh * kw * cin;
  if (K_pad % 64 != 0 || K_pad < K) {
    set_error("stem im2col: bad K_pad %d for K %d", K_pad, K);
    return DEFER_ERR_INVALID;
  }
  const size_t smem = (size_t)kh * w * cin * sizeof(float);
  if (smem > 160 * 1024) {
    set_error("stem im2col: %d input rows of %d floats do not fit in shared memory", kh, w * cin);
    return DEFER_ERR_INVALID;
  }
  const unsigned grid = (unsigned)((size_t)n * ho);
  auto go = [&](auto kernel) -> int {
    // the two instantiations have the same type, so this lambda (and its static) is shared: one flag per format
    static bool attr_set[3][64] = {};
    int dev = 0;
    DEFER_CUDA(cudaGetDevice(&dev));
    if (dev < 64 && !attr_set[fmt][dev]) {
      DEFER_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
      prefer_max_smem(kernel);
      attr_set[fmt][dev] = true;
    }
    kernel<<<grid, 256, smem, st>>>(x, out, n, h, w, cin, kh, kw, sh, sw, pad_t, pad_l, ho, wo, K, K_pad);
    DEFER_CUDA(cudaGetLastError());
    return DEFER_OK;
  };
  switch (fmt) {
    case FMT_BF16X2: return go(stem_im2col_kernel<FMT_BF16X2>);
    case FMT_BF16: return go(stem_im2col_kernel<FMT_BF16>);
    default: set_error("stem im2col: format %d has no tensor-core path", fmt); return DEFER_ERR_INVALID;
  }
}

// =============================================================================================
// max-pool with fused ZeroPadding2D (taps outside the tensor read 0.0, as Keras' explicit pad does)
// one thread per (pixel, 4 channels)
// =============================================================================================
template <int FMT>
__global__ void __launch_bounds__(256) maxpool_kernel(const void* __restrict__ x, void* __restrict__ y, int n, int h,
                                                      int w, int c, int ph, int pw, int sh, int sw, int pad_t,
                                                      int pad_l, int ho, int wo) {
  const int c4 = c >> 2;
  size_t total = (size_t)n * ho * wo * c4;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int cg = (int)(i % c4);
  size_t pix = i / c4;
  int ow = (int)(pix % wo);
  size_t t2 = pix / wo;
  int oh = (int)(t2 % ho);
  int nb = (int)(t2 / ho);
  const size_t plane_in = (size_t)n * h * w * c, plane_out = (size_t)n * ho * wo * c;
  float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  for (int a = 0; a < ph; ++a) {
    int ih = oh * sh - pad_t + a;
    for (int b = 0; b < pw; ++b) {
      int iw = ow * sw - pad_l + b;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ih >= 0 && ih < h && iw >= 0 && iw < w)
        v = act_load4<FMT>(x, plane_in, (((size_t)nb * h + ih) * w + iw) * c + cg * 4);
      m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
    }
  }
  act_store4<FMT>(y, plane_out, pix * c + cg * 4, m);
}

// 8 channels per thread, 16-byte loads / stores per bf16 plane (the pool is a pure HBM stream: wide accesses halve the
// instruction count of the 4-channel version).  max() is exact on bf16 values, so it is taken plane-wise on the decoded sums
// exactly like the 4-channel kernel: decode hi + lo -> fp32, max, re-split.
template <int FMT>
__global__ void __launch_bounds__(256) maxpool8_kernel(const void* __restrict__ x, void* __restrict__ y, int n, int h, int w,
                                                       int c, int ph, int pw, int sh, int sw, int pad_t, int pad_l, int ho,
                                                       int wo) {
  const int c8 = c >> 3;
  const size_t total = (size_t)n * ho * wo * c8;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int cg = (int)(i % c8);
  const size_t pix = i / c8;
  const int ow = (int)(pix % wo);
  const size_t t2 = pix / wo;
  const int oh = (int)(t2 % ho);
  const int nb = (int)(t2 / ho);
  const size_t plane_in = (size_t)n * h * w * c, plane_out = (size_t)n * ho * wo * c;
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
  float m[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
  for (int a = 0; a < ph; ++a) {
    const int ih = oh * sh - pad_t + a;
    for (int b = 0; b < pw; ++b) {
      const int iw = ow * sw - pad_l + b;
      float v[8];
      if (ih >= 0 && ih < h && iw >= 0 && iw < w) {
        const size_t o = (((size_t)nb * h + ih) * w + iw) * c + (size_t)cg * 8;
        const uint4 hv = __ldg(reinterpret_cast<const uint4*>(xp + o));
        const uint32_t* hw = reinterpret_cast<const uint32_t*>(&hv);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          v[2 * t] = __uint_as_float(hw[t] << 16);
          v[2 * t + 1] = __uint_as_float(hw[t] & 0xffff0000u);
        }
        if constexpr (FMT == FMT_BF16X2) {
          const uint4 lv = __ldg(reinterpret_cast<const uint4*>(xp + plane_in + o));
          const uint32_t* lw = reinterpret_cast<const uint32_t*>(&lv);
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            v[2 * t] += __uint_as_float(lw[t] << 16);
            v[2 * t + 1] += __uint_as_float(lw[t] & 0xffff0000u);
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;      // Keras' explicit ZeroPadding2D: padded taps read 0.0
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], v[j]);
    }
  }
  __nv_bfloat16* yp = reinterpret_cast<__nv_bfloat16*>(y);
  const size_t o = pix * c + (size_t)cg * 8;
  uint4 hv, lv;
  if constexpr (FMT == FMT_BF16X2) {
    split_bf16x2(m[0], m[1], hv.x, lv.x);
    split_bf16x2(m[2], m[3], hv.y, lv.y);
    split_bf16x2(m[4], m[5], hv.z, lv.z);
    split_bf16x2(m[6], m[7], hv.w, lv.w);
    *reinterpret_cast<uint4*>(yp + o) = hv;
    *reinterpret_cast<uint4*>(yp + plane_out + o) = lv;
  } else {
    hv.x = pack_bf16x2(m[0], m[1]);
    hv.y = pack_bf16x2(m[2], m[3]);
    hv.z = pack_bf16x2(m[4], m[5]);
    hv.w = pack_bf16x2(m[6], m[7]);
    *reinterpret_cast<uint4*>(yp + o) = hv;
  }
}

int launch_maxpool(int fmt, const void* x, void* y, int n, int h, int w, int c, int ph, int pw, int sh, int sw,
                   int pad_t, int pad_l, int ho, int wo, cudaStream_t st) {
  if (c % 4 != 0) {
    set_error("maxpool: channels %d not a multiple of 4", c);
    return DEFER_ERR_INVALID;
  }
  static const bool wide = getenv("DEFER_MAXPOOL8") == nullptr || atoi(getenv("DEFER_MAXPOOL8")) != 0;
  if (wide && c % 8 == 0 && (fmt == FMT_BF16X2 || fmt == FMT_BF16)) {
    const size_t total8 = (size_t)n * ho * wo * (c / 8);
    const unsigned grid8 = (unsigned)((total8 + 255) / 256);
    if (fmt == FMT_BF16X2) {
      prefer_max_smem(maxpool8_kernel<FMT_BF16X2>);
      maxpool8_kernel<FMT_BF16X2><<<grid8, 256, 0, st>>>(x, y, n, h, w, c, ph, pw, sh, sw, pad_t, pad_l, ho, wo);
    } else {
      prefer_max_smem(maxpool8_kernel<FMT_BF16>);
      maxpool8_kernel<FMT_BF16><<<grid8, 256, 0, st>>>(x, y, n, h, w, c, ph, pw, sh, sw, pad_t, pad_l, ho, wo);
    }
    DEFER_CUDA(cudaGetLastError());
    return DEFER_OK;
  }
  size_t total = (size_t)n * ho * wo * (c / 4);
  unsigned grid = (unsigned)((total + 255) / 256);
  switch (fmt) {
    case FMT_F32: prefer_max_smem(maxpool_kernel<FMT_F32>); maxpool_kernel<FMT_F32><<<grid, 256, 0, st>>>(x, y, n, h, w, c, ph, pw, sh, sw, pad_t, pad_l, ho, wo); break;
    case FMT_BF16X2: prefer_max_smem(maxpool_kernel<FMT_BF16X2>); maxpool_kernel<FMT_BF16X2><<<grid, 256, 0, st>>>(x, y, n, h, w, c, ph, pw, sh, sw, pad_t, pad_l, ho, wo); break;
    case FMT_BF16: prefer_max_smem(maxpool_kernel<FMT_BF16>); maxpool_kernel<FMT_BF16><<<grid, 256, 0, st>>>(x, y, n, h, w, c, ph, pw, sh, sw, pad_t, pad_l, ho, wo); break;
    default: set_error("maxpool: bad fmt"); return DEFER_ERR_INVALID;
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

// =============================================================================================
// global average pool: (n, h*w, c) -> (n, c).  One warp-row of channels per block slice; threads
// stride over channels (coalesced), loop over pixels; pixel range split over threadIdx.y and
// combined through shared memory.
// =============================================================================================
template <int FMT>
__global__ void __launch_bounds__(256) gap_kernel(const void* __restrict__ x, void* __restrict__ y, int hw, int c) {
  __shared__ float red[8][32];
  const int nb = blockIdx.y;
  const int ch = blockIdx.x * 32 + threadIdx.x;
  const size_t plane_in = (size_t)gridDim.y * hw * c, plane_out = (size_t)gridDim.y * c;
  float s = 0.f;
  if (ch < c) {
    for (int p = threadIdx.y; p < hw; p += 8) s += act_load<FMT>(x, plane_in, ((size_t)nb * hw + p) * c + ch);
  }
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && ch < c) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x];
    act_store<FMT>(y, plane_out, (size_t)nb * c + ch, t / (float)hw);
  }
}

int launch_gap(int fmt, const void* x, void* y, int n, int h, int w, int c, cudaStream_t st) {
  dim3 grid((c + 31) / 32, n), block(32, 8);
  switch (fmt) {
    case FMT_F32: prefer_max_smem(gap_kernel<FMT_F32>); gap_kernel<FMT_F32><<<grid, block, 0, st>>>(x, y, h * w, c); break;
    case FMT_BF16X2: prefer_max_smem(gap_kernel<FMT_BF16X2>); gap_kernel<FMT_BF16X2><<<grid, block, 0, st>>>(x, y, h * w, c); break;
    case FMT_BF16: prefer_max_smem(gap_kernel<FMT_BF16>); gap_kernel<FMT_BF16><<<grid, block, 0, st>>>(x, y, h * w, c); break;
    default: set_error("gap: bad fmt"); return DEFER_ERR_INVALID;
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

// =============================================================================================
// dense: y[b][u] = sum_f x[b][f] * W[f][u] + bias[u].  HBM-bound weight stream at batch 1:
// thread = output unit (coalesced over u), F split across blockIdx.y for parallelism, partials
// reduced in a fixed order by a second kernel (deterministic, no atomics).
// =============================================================================================
constexpr int DENSE_TB = 128;     // units per block
constexpr int DENSE_MAXB = 8;     // batch chunk held in registers

// split counts aim at ~2 waves of the 132 SMs of an H100 SXM; a fixed number (not the device's) keeps the summation
// order, and so the bits of the result, the same on every GPU
constexpr int DENSE_WAVE_SMS = 132;

int dense_splits(int n, int in_features, int units) {
  int col_blocks = (units + DENSE_TB - 1) / DENSE_TB;
  int want = (2 * DENSE_WAVE_SMS + col_blocks - 1) / col_blocks;
  int max_split = (in_features + 31) / 32;              // at least 32 rows per split
  int s = want < max_split ? want : max_split;
  int min_split = (in_features + 1023) / 1024;          // keep the x slice of a split small in smem
  if (s < min_split) s = min_split;
  return s < 1 ? 1 : s;
}

template <int FMT, typename WT>
__global__ void __launch_bounds__(DENSE_TB) dense_partial_kernel(const void* __restrict__ x, const WT* __restrict__ w,
                                                                 float* __restrict__ partial, int n, int F, int U,
                                                                 int rows_per_split) {
  extern __shared__ float xs[];  // [nb_chunk][rows]
  const int u = blockIdx.x * DENSE_TB + threadIdx.x;
  const int f0 = blockIdx.y * rows_per_split;
  const int f1 = min(F, f0 + rows_per_split);
  const int rows = f1 - f0;
  const size_t plane = (size_t)n * F;
  for (int b0 = 0; b0 < n; b0 += DENSE_MAXB) {
    const int nb = min(DENSE_MAXB, n - b0);
    __syncthreads();
    for (int i = threadIdx.x; i < nb * rows; i += DENSE_TB) {
      int b = i / rows, f = i - b * rows;
      xs[b * rows_per_split + f] = act_load<FMT>(x, plane, (size_t)(b0 + b) * F + f0 + f);
    }
    __syncthreads();
    float acc[DENSE_MAXB];
#pragma unroll
    for (int b = 0; b < DENSE_MAXB; ++b) acc[b] = 0.f;
    if (u < U) {
      const WT* wp = w + (size_t)f0 * U + u;
#pragma unroll 8
      for (int f = 0; f < rows; ++f) {
        float wv;
        if constexpr (sizeof(WT) == 2) wv = __bfloat162float(wp[(size_t)f * U]);
        else wv = __ldg(reinterpret_cast<const float*>(wp) + (size_t)f * U);
#pragma unroll
        for (int b = 0; b < DENSE_MAXB; ++b)
          if (b < nb) acc[b] = fmaf(xs[b * rows_per_split + f], wv, acc[b]);
      }
#pragma unroll
      for (int b = 0; b < DENSE_MAXB; ++b)
        if (b < nb) partial[((size_t)blockIdx.y * n + b0 + b) * U + u] = acc[b];
    }
  }
}

template <int FOUT>
__global__ void __launch_bounds__(256) dense_reduce_kernel(const float* __restrict__ partial,
                                                           const float* __restrict__ bias, void* __restrict__ y,
                                                           int n, int U, int splits, uint32_t flags) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t total = (size_t)n * U;
  if (i >= total) return;
  int u = (int)(i % U);
  float s = 0.f;
  for (int k = 0; k < splits; ++k) s += partial[(size_t)k * total + i];
  if (bias) s += __ldg(bias + u);
  if (flags & DEFER_FLAG_RELU) s = fmaxf(s, 0.f);
  act_store<FOUT>(y, total, i, s);
}

// ---------------------------------------------------------------------------------------------
// Fused dense (default when units % 4 == 0): ONE launch does the weight stream, the split reduction and the
// bias / ReLU epilogue.  CTA = 8 warps x (32 lanes x 4 units): every warp takes every 8th row of the CTA's
// K slice, so a thread has 8 independent 16-byte weight loads in flight per round trip; the 8 warps are
// summed in warp order through shared memory, the per-split partial goes to global memory, and the LAST CTA
// to arrive at a column block (arrival counter, self re-arming) adds the splits in split order - the result
// does not depend on arrival order, no float atomics.
// ---------------------------------------------------------------------------------------------
constexpr int DF_THREADS = 256;
constexpr int DF_WARPS = 8;
constexpr int DF_COLS = 128;

constexpr size_t DF_HEADER = 4096;   // arrival counters (one per 128-unit column block) live at the start of the workspace

size_t dense_workspace_bytes(int n, int in_features, int units) {
  return DF_HEADER + (size_t)dense_splits(n, in_features, units) * n * units * sizeof(float);
}

static int dense_fused_splits(int n, int F, int U) {
  const int col_blocks = (U + DF_COLS - 1) / DF_COLS;
  int want = (2 * DENSE_WAVE_SMS + col_blocks - 1) / col_blocks;
  int max_split = F / 64;                   // >= 8 rows per warp
  if (max_split < 1) max_split = 1;
  int s = want < max_split ? want : max_split;
  const int cap = dense_splits(n, F, U);    // the workspace is sized for dense_splits()
  if (s > cap) s = cap;
  int min_split = (F + 1023) / 1024;
  if (s < min_split) s = min_split;
  return s < 1 ? 1 : s;
}

template <int FMT, typename WT, int FOUT>
__global__ void __launch_bounds__(DF_THREADS) dense_fused_kernel(const void* __restrict__ x, const WT* __restrict__ w,
                                                                 const float* __restrict__ bias, void* __restrict__ y,
                                                                 float* __restrict__ partial, unsigned int* __restrict__ counters,
                                                                 int n, int F, int U, int rows_per_split, int splits,
                                                                 uint32_t flags) {
  extern __shared__ float dsm[];
  __shared__ int s_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nbc = n < DENSE_MAXB ? n : DENSE_MAXB;
  float* xs = dsm;                                       // [nbc][rows_per_split]
  float* red = dsm + (((size_t)nbc * rows_per_split + 3) & ~(size_t)3);   // [DF_WARPS][nbc][DF_COLS], 16-byte aligned
  const int ub = blockIdx.x * DF_COLS;
  const int u0 = ub + lane * 4;
  const int f0 = blockIdx.y * rows_per_split;
  const int f1 = min(F, f0 + rows_per_split);
  const int rows = f1 - f0;
  const size_t plane = (size_t)n * F;
  for (int b0 = 0; b0 < n; b0 += DENSE_MAXB) {
    const int nb = min(DENSE_MAXB, n - b0);
    __syncthreads();
    for (int i = tid; i < nb * rows; i += DF_THREADS) {
      int b = i / rows, f = i - b * rows;
      xs[b * rows_per_split + f] = act_load<FMT>(x, plane, (size_t)(b0 + b) * F + f0 + f);
    }
    __syncthreads();
    float acc[DENSE_MAXB][4];
#pragma unroll
    for (int b = 0; b < DENSE_MAXB; ++b) acc[b][0] = acc[b][1] = acc[b][2] = acc[b][3] = 0.f;
    if (u0 < U) {
      const WT* wp = w + (size_t)f0 * U + u0;
#pragma unroll 8
      for (int f = warp; f < rows; f += DF_WARPS) {
        float4 wv;
        if constexpr (sizeof(WT) == 2) {
          const uint2 r = __ldg(reinterpret_cast<const uint2*>(wp + (size_t)f * U));
          wv = make_float4(__uint_as_float(r.x << 16), __uint_as_float(r.x & 0xffff0000u), __uint_as_float(r.y << 16),
                           __uint_as_float(r.y & 0xffff0000u));
        } else {
          wv = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(wp) + (size_t)f * U));
        }
#pragma unroll
        for (int b = 0; b < DENSE_MAXB; ++b)
          if (b < nb) {
            const float xv = xs[b * rows_per_split + f];
            acc[b][0] = fmaf(xv, wv.x, acc[b][0]);
            acc[b][1] = fmaf(xv, wv.y, acc[b][1]);
            acc[b][2] = fmaf(xv, wv.z, acc[b][2]);
            acc[b][3] = fmaf(xv, wv.w, acc[b][3]);
          }
      }
    }
#pragma unroll
    for (int b = 0; b < DENSE_MAXB; ++b)
      if (b < nb)
        *reinterpret_cast<float4*>(red + ((size_t)warp * nbc + b) * DF_COLS + lane * 4) =
            make_float4(acc[b][0], acc[b][1], acc[b][2], acc[b][3]);
    __syncthreads();
    for (int i = tid; i < nb * DF_COLS; i += DF_THREADS) {
      const int b = i / DF_COLS, c = i - b * DF_COLS;
      if (ub + c < U) {
        float sum = 0.f;
#pragma unroll
        for (int wq = 0; wq < DF_WARPS; ++wq) sum += red[((size_t)wq * nbc + b) * DF_COLS + c];
        __stcg(partial + ((size_t)blockIdx.y * n + b0 + b) * U + ub + c, sum);
      }
    }
  }
  // ---- arrival: the last CTA of this column block folds the splits (fixed order) and finishes the layer
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned prev = atomicAdd(counters + blockIdx.x, 1u);
    const int last = prev == (unsigned)(splits - 1);
    if (last) counters[blockIdx.x] = 0;   // re-arm for the next launch on this lane
    s_last = last;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const size_t total = (size_t)n * U;
  for (int i = tid; i < n * DF_COLS; i += DF_THREADS) {
    const int b = i / DF_COLS, c = i - b * DF_COLS;
    const int u = ub + c;
    if (u >= U) continue;
    float sum = 0.f;
    for (int k = 0; k < splits; ++k) sum += __ldcg(partial + ((size_t)k * n + b) * U + u);
    if (bias) sum += __ldg(bias + u);
    if (flags & DEFER_FLAG_RELU) sum = fmaxf(sum, 0.f);
    act_store<FOUT>(y, total, (size_t)b * U + u, sum);
  }
}

template <int FMT, typename WT, int FOUT>
static int launch_dense_fused_t(const void* x, const void* w, const float* bias, void* y, float* partial, unsigned int* counters,
                                int n, int F, int U, uint32_t flags, cudaStream_t st) {
  int splits = dense_fused_splits(n, F, U);
  int rows = (F + splits - 1) / splits;
  splits = (F + rows - 1) / rows;
  const int nbc = n < DENSE_MAXB ? n : DENSE_MAXB;
  const size_t smem = ((((size_t)nbc * rows + 3) & ~(size_t)3) + (size_t)DF_WARPS * nbc * DF_COLS) * sizeof(float);
  if (smem > 96 * 1024) {
    set_error("dense: smem %zu too large", smem);
    return DEFER_ERR_INVALID;
  }
  static bool attr_set[64] = {false};
  int dev = 0;
  DEFER_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && !attr_set[dev]) {
    DEFER_CUDA(cudaFuncSetAttribute(dense_fused_kernel<FMT, WT, FOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    prefer_max_smem(dense_fused_kernel<FMT, WT, FOUT>);
    attr_set[dev] = true;
  }
  dim3 grid((U + DF_COLS - 1) / DF_COLS, splits);
  dense_fused_kernel<FMT, WT, FOUT><<<grid, DF_THREADS, smem, st>>>(x, (const WT*)w, bias, y, partial, counters, n, F, U, rows,
                                                                   splits, flags);
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

template <int FMT, typename WT>
static int launch_dense_fused_f(int fout, const void* x, const void* w, const float* bias, void* y, float* partial,
                                unsigned int* counters, int n, int F, int U, uint32_t flags, cudaStream_t st) {
  switch (fout) {
    case FMT_F32: return launch_dense_fused_t<FMT, WT, FMT_F32>(x, w, bias, y, partial, counters, n, F, U, flags, st);
    case FMT_BF16X2: return launch_dense_fused_t<FMT, WT, FMT_BF16X2>(x, w, bias, y, partial, counters, n, F, U, flags, st);
    case FMT_BF16: return launch_dense_fused_t<FMT, WT, FMT_BF16>(x, w, bias, y, partial, counters, n, F, U, flags, st);
  }
  set_error("dense: bad output fmt %d", fout);
  return DEFER_ERR_INVALID;
}

int launch_dense(int fmt, const void* x, const void* w, bool w_is_bf16, const float* bias, void* y, bool y_is_f32,
                 float* partial, int n, int F, int U, uint32_t flags, cudaStream_t st) {
  static const bool fused_on = getenv("DEFER_DENSE_FUSED") == nullptr || atoi(getenv("DEFER_DENSE_FUSED")) != 0;
  // workspace layout (dense_workspace_bytes): [arrival counters, 4 KB, zeroed once | split partials]
  unsigned int* counters = reinterpret_cast<unsigned int*>(partial);
  partial = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(partial) + DF_HEADER);
  if (fused_on && U % 4 == 0 && (size_t)((U + DF_COLS - 1) / DF_COLS) * sizeof(unsigned int) <= DF_HEADER) {
    const int fout = y_is_f32 ? FMT_F32 : fmt;
    switch (fmt) {
      case FMT_F32:
        return w_is_bf16 ? launch_dense_fused_f<FMT_F32, __nv_bfloat16>(fout, x, w, bias, y, partial, counters, n, F, U, flags, st)
                         : launch_dense_fused_f<FMT_F32, float>(fout, x, w, bias, y, partial, counters, n, F, U, flags, st);
      case FMT_BF16X2:
        return w_is_bf16 ? launch_dense_fused_f<FMT_BF16X2, __nv_bfloat16>(fout, x, w, bias, y, partial, counters, n, F, U, flags, st)
                         : launch_dense_fused_f<FMT_BF16X2, float>(fout, x, w, bias, y, partial, counters, n, F, U, flags, st);
      case FMT_BF16:
        return w_is_bf16 ? launch_dense_fused_f<FMT_BF16, __nv_bfloat16>(fout, x, w, bias, y, partial, counters, n, F, U, flags, st)
                         : launch_dense_fused_f<FMT_BF16, float>(fout, x, w, bias, y, partial, counters, n, F, U, flags, st);
      default: set_error("dense: bad fmt"); return DEFER_ERR_INVALID;
    }
  }
  int splits = dense_splits(n, F, U);
  int rows = (F + splits - 1) / splits;
  splits = (F + rows - 1) / rows;
  dim3 grid((U + DENSE_TB - 1) / DENSE_TB, splits);
  int nbc = n < DENSE_MAXB ? n : DENSE_MAXB;
  size_t smem = (size_t)nbc * rows * sizeof(float);
  if (smem > 48 * 1024) {
    set_error("dense: smem %zu too large", smem);
    return DEFER_ERR_INVALID;
  }
#define DENSE_LAUNCH(FM)                                                                                           \
  if (w_is_bf16) {                                                                                                 \
    prefer_max_smem(dense_partial_kernel<FM, __nv_bfloat16>);                                                      \
    dense_partial_kernel<FM, __nv_bfloat16><<<grid, DENSE_TB, smem, st>>>(x, (const __nv_bfloat16*)w, partial, n, F, U, rows); \
  } else {                                                                                                         \
    prefer_max_smem(dense_partial_kernel<FM, float>);                                                              \
    dense_partial_kernel<FM, float><<<grid, DENSE_TB, smem, st>>>(x, (const float*)w, partial, n, F, U, rows);     \
  }
  switch (fmt) {
    case FMT_F32: DENSE_LAUNCH(FMT_F32); break;
    case FMT_BF16X2: DENSE_LAUNCH(FMT_BF16X2); break;
    case FMT_BF16: DENSE_LAUNCH(FMT_BF16); break;
    default: set_error("dense: bad fmt"); return DEFER_ERR_INVALID;
  }
#undef DENSE_LAUNCH
  DEFER_CUDA(cudaGetLastError());
  size_t total = (size_t)n * U;
  unsigned g2 = (unsigned)((total + 255) / 256);
  int fout = y_is_f32 ? FMT_F32 : fmt;
  switch (fout) {
    case FMT_F32: prefer_max_smem(dense_reduce_kernel<FMT_F32>); dense_reduce_kernel<FMT_F32><<<g2, 256, 0, st>>>(partial, bias, y, n, U, splits, flags); break;
    case FMT_BF16X2: prefer_max_smem(dense_reduce_kernel<FMT_BF16X2>); dense_reduce_kernel<FMT_BF16X2><<<g2, 256, 0, st>>>(partial, bias, y, n, U, splits, flags); break;
    case FMT_BF16: prefer_max_smem(dense_reduce_kernel<FMT_BF16>); dense_reduce_kernel<FMT_BF16><<<g2, 256, 0, st>>>(partial, bias, y, n, U, splits, flags); break;
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

// =============================================================================================
// softmax over the last axis, one block per row, warp-shuffle max / sum reductions
// =============================================================================================
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(256) softmax_kernel(const float* __restrict__ x, float* __restrict__ y, int c) {
  __shared__ float red[8];
  __shared__ float bcast;
  const float* xr = x + (size_t)blockIdx.x * c;
  float* yr = y + (size_t)blockIdx.x * c;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < c; i += 256) m = fmaxf(m, xr[i]);
  m = warp_max(m);
  if (lane == 0) red[wid] = m;
  __syncthreads();
  if (wid == 0) {
    float v = lane < 8 ? red[lane] : -INFINITY;
    v = warp_max(v);
    if (lane == 0) bcast = v;
  }
  __syncthreads();
  m = bcast;
  float s = 0.f;
  for (int i = threadIdx.x; i < c; i += 256) s += expf(xr[i] - m);
  s = warp_sum(s);
  __syncthreads();
  if (lane == 0) red[wid] = s;
  __syncthreads();
  if (wid == 0) {
    float v = lane < 8 ? red[lane] : 0.f;
    v = warp_sum(v);
    if (lane == 0) bcast = v;
  }
  __syncthreads();
  const float inv = 1.f / bcast;
  for (int i = threadIdx.x; i < c; i += 256) yr[i] = expf(xr[i] - m) * inv;
}

int launch_softmax(const float* x, float* y, int n, int c, cudaStream_t st) {
  prefer_max_smem(softmax_kernel); softmax_kernel<<<n, 256, 0, st>>>(x, y, c);
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

// =============================================================================================
// standalone elementwise ops (arbitrary cut points): AFFINE (BN), RELU, ADD; 4 channels / thread
// =============================================================================================
template <int FMT, int KIND>
__global__ void __launch_bounds__(256) eltwise_kernel(const void* __restrict__ a, const void* __restrict__ b,
                                                      const float* __restrict__ scale, const float* __restrict__ shift,
                                                      void* __restrict__ y, size_t n_elems, int c, uint32_t flags) {
  size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= n_elems) return;
  float4 v = act_load4<FMT>(a, n_elems, i);
  if constexpr (KIND == DEFER_OP_AFFINE) {
    int ch = (int)(i % c);
    float4 s = scale ? __ldg(reinterpret_cast<const float4*>(scale + ch)) : make_float4(1.f, 1.f, 1.f, 1.f);
    float4 t = shift ? __ldg(reinterpret_cast<const float4*>(shift + ch)) : make_float4(0.f, 0.f, 0.f, 0.f);
    v.x = fmaf(v.x, s.x, t.x); v.y = fmaf(v.y, s.y, t.y); v.z = fmaf(v.z, s.z, t.z); v.w = fmaf(v.w, s.w, t.w);
  } else if constexpr (KIND == DEFER_OP_ADD) {
    float4 u = act_load4<FMT>(b, n_elems, i);
    v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
  }
  if (KIND == DEFER_OP_RELU || (flags & DEFER_FLAG_RELU)) {
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
  }
  act_store4<FMT>(y, n_elems, i, v);
}

// ReLU on the BF16X2 format works on the planes directly: an element either passes through with its
// (hi, lo) pair untouched or becomes (0, 0).  Re-splitting hi+lo could pick the other representation of
// the same value at rounding ties, which would make results depend on where the model is cut.
__global__ void __launch_bounds__(256) relu_planes_kernel(const uint32_t* __restrict__ x, uint32_t* __restrict__ y,
                                                          size_t n_pairs) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;   // one bf16 pair of the hi plane (and of the lo plane)
  if (i >= n_pairs) return;
  uint32_t h = x[i], l = x[n_pairs + i];
  // keep an element iff hi > 0 (sign bit clear and non-zero); |lo| <= ulp(hi)/2 never flips the sign
  uint32_t keep_lo = ((h & 0x8000u) == 0 && (h & 0x7fffu) != 0) ? 0x0000ffffu : 0u;
  uint32_t keep_hi = ((h & 0x80000000u) == 0 && (h & 0x7fff0000u) != 0) ? 0xffff0000u : 0u;
  uint32_t m = keep_lo | keep_hi;
  y[i] = h & m;
  y[n_pairs + i] = l & m;
}

template <int FMT>
static int launch_eltwise_t(int kind, const void* a, const void* b, const float* scale, const float* shift, void* y,
                            size_t n_elems, int c, uint32_t flags, cudaStream_t st) {
  unsigned grid = (unsigned)((n_elems / 4 + 255) / 256);
  switch (kind) {
    case DEFER_OP_AFFINE: prefer_max_smem(eltwise_kernel<FMT, DEFER_OP_AFFINE>); eltwise_kernel<FMT, DEFER_OP_AFFINE><<<grid, 256, 0, st>>>(a, b, scale, shift, y, n_elems, c, flags); break;
    case DEFER_OP_RELU: prefer_max_smem(eltwise_kernel<FMT, DEFER_OP_RELU>); eltwise_kernel<FMT, DEFER_OP_RELU><<<grid, 256, 0, st>>>(a, b, scale, shift, y, n_elems, c, flags); break;
    case DEFER_OP_ADD: prefer_max_smem(eltwise_kernel<FMT, DEFER_OP_ADD>); eltwise_kernel<FMT, DEFER_OP_ADD><<<grid, 256, 0, st>>>(a, b, scale, shift, y, n_elems, c, flags); break;
    default: set_error("eltwise: bad kind %d", kind); return DEFER_ERR_INVALID;
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

int launch_eltwise(int fmt, int kind, const void* a, const void* b, const float* scale, const float* shift, void* y,
                   size_t n_pix, int c, uint32_t flags, cudaStream_t st) {
  if (c % 4 != 0) {
    set_error("eltwise: channels %d not a multiple of 4", c);
    return DEFER_ERR_INVALID;
  }
  size_t n_elems = n_pix * (size_t)c;
  if (fmt == FMT_BF16X2 && kind == DEFER_OP_RELU) {
    size_t n_pairs = n_elems / 2;
    prefer_max_smem(relu_planes_kernel); relu_planes_kernel<<<(unsigned)((n_pairs + 255) / 256), 256, 0, st>>>((const uint32_t*)a, (uint32_t*)y, n_pairs);
    DEFER_CUDA(cudaGetLastError());
    return DEFER_OK;
  }
  switch (fmt) {
    case FMT_F32: return launch_eltwise_t<FMT_F32>(kind, a, b, scale, shift, y, n_elems, c, flags, st);
    case FMT_BF16X2: return launch_eltwise_t<FMT_BF16X2>(kind, a, b, scale, shift, y, n_elems, c, flags, st);
    case FMT_BF16: return launch_eltwise_t<FMT_BF16>(kind, a, b, scale, shift, y, n_elems, c, flags, st);
  }
  set_error("eltwise: bad fmt");
  return DEFER_ERR_INVALID;
}

// standalone ZeroPadding2D (scalar; only reached for exotic cut points)
template <int FMT>
__global__ void __launch_bounds__(256) pad_kernel(const void* __restrict__ x, void* __restrict__ y, int n, int h, int w,
                                                  int c, int pad_t, int pad_l, int ho, int wo) {
  size_t total = (size_t)n * ho * wo * c;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int ch = (int)(i % c);
  size_t pix = i / c;
  int ow = (int)(pix % wo);
  size_t t2 = pix / wo;
  int oh = (int)(t2 % ho);
  int nb = (int)(t2 / ho);
  int ih = oh - pad_t, iw = ow - pad_l;
  float v = 0.f;
  if (ih >= 0 && ih < h && iw >= 0 && iw < w)
    v = act_load<FMT>(x, (size_t)n * h * w * c, (((size_t)nb * h + ih) * w + iw) * c + ch);
  act_store<FMT>(y, total, i, v);
}

int launch_pad(int fmt, const void* x, void* y, int n, int h, int w, int c, int pad_t, int pad_l, int ho, int wo,
               cudaStream_t st) {
  size_t total = (size_t)n * ho * wo * c;
  unsigned grid = (unsigned)((total + 255) / 256);
  switch (fmt) {
    case FMT_F32: prefer_max_smem(pad_kernel<FMT_F32>); pad_kernel<FMT_F32><<<grid, 256, 0, st>>>(x, y, n, h, w, c, pad_t, pad_l, ho, wo); break;
    case FMT_BF16X2: prefer_max_smem(pad_kernel<FMT_BF16X2>); pad_kernel<FMT_BF16X2><<<grid, 256, 0, st>>>(x, y, n, h, w, c, pad_t, pad_l, ho, wo); break;
    case FMT_BF16: prefer_max_smem(pad_kernel<FMT_BF16>); pad_kernel<FMT_BF16><<<grid, 256, 0, st>>>(x, y, n, h, w, c, pad_t, pad_l, ho, wo); break;
    default: set_error("pad: bad fmt"); return DEFER_ERR_INVALID;
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

// =============================================================================================
// format conversion
// =============================================================================================
template <int FMT>
__global__ void __launch_bounds__(256) encode_kernel(const float* __restrict__ x, void* __restrict__ y, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) act_store<FMT>(y, n, i, x[i]);
}
template <int FMT>
__global__ void __launch_bounds__(256) decode_kernel(const void* __restrict__ x, float* __restrict__ y, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = act_load<FMT>(x, n, i);
}
int launch_encode(int fmt, const float* x, void* y, size_t n, cudaStream_t st) {
  unsigned grid = (unsigned)((n + 255) / 256);
  switch (fmt) {
    case FMT_F32: prefer_max_smem(encode_kernel<FMT_F32>); encode_kernel<FMT_F32><<<grid, 256, 0, st>>>(x, y, n); break;
    case FMT_BF16X2: prefer_max_smem(encode_kernel<FMT_BF16X2>); encode_kernel<FMT_BF16X2><<<grid, 256, 0, st>>>(x, y, n); break;
    case FMT_BF16: prefer_max_smem(encode_kernel<FMT_BF16>); encode_kernel<FMT_BF16><<<grid, 256, 0, st>>>(x, y, n); break;
    default: set_error("encode: bad fmt"); return DEFER_ERR_INVALID;
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}
int launch_decode(int fmt, const void* x, float* y, size_t n, cudaStream_t st) {
  unsigned grid = (unsigned)((n + 255) / 256);
  switch (fmt) {
    case FMT_F32: prefer_max_smem(decode_kernel<FMT_F32>); decode_kernel<FMT_F32><<<grid, 256, 0, st>>>(x, y, n); break;
    case FMT_BF16X2: prefer_max_smem(decode_kernel<FMT_BF16X2>); decode_kernel<FMT_BF16X2><<<grid, 256, 0, st>>>(x, y, n); break;
    case FMT_BF16: prefer_max_smem(decode_kernel<FMT_BF16>); decode_kernel<FMT_BF16><<<grid, 256, 0, st>>>(x, y, n); break;
    default: set_error("decode: bad fmt"); return DEFER_ERR_INVALID;
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}
int launch_copy_act(int fmt, const void* x, void* y, size_t n, cudaStream_t st) {
  // planes are contiguous ([hi | lo]): a byte copy keeps every (hi, lo) pair exactly as stored
  DEFER_CUDA(cudaMemcpyAsync(y, x, n * fmt_bytes_per_elem(fmt), cudaMemcpyDeviceToDevice, st));
  return DEFER_OK;
}

// Keras preprocess_input on a uint8 RGB image.  Caffe mode (TF false): y[p, c] = float(x[p, 2 - c]) + shift[c], one
// exactly rounded fp32 add per element (shift = -mean, so this is the host's float32(x) - mean bit for bit).  Tf mode
// (TF true, shift unused): y[p, c] = keras_tf_preprocess(float(x[p, c])), the host's float32(x) / 127.5 - 1 bit for bit.
// VEC: a thread reads four pixels as three 32-bit words and writes them as three float4; the last n_pix % 4 pixels go
// one per thread.
template <bool VEC, bool TF>
__device__ __forceinline__ void preprocess_body(const uint8_t* __restrict__ x, const float* __restrict__ shift,
                                                float* __restrict__ y, size_t n_pix) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  if constexpr (!TF) {
    s0 = __ldg(shift); s1 = __ldg(shift + 1); s2 = __ldg(shift + 2);
  }
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (VEC) {
    const size_t groups = n_pix / 4;
    if (i < groups) {
      const uint32_t* xv = reinterpret_cast<const uint32_t*>(x) + 3 * i;
      const uint32_t wd[3] = {__ldg(xv), __ldg(xv + 1), __ldg(xv + 2)};
      float b[12], o[12];
#pragma unroll
      for (int j = 0; j < 12; ++j) b[j] = (float)((wd[j >> 2] >> (8 * (j & 3))) & 0xffu);
      if constexpr (TF) {
#pragma unroll
        for (int j = 0; j < 12; ++j) o[j] = keras_tf_preprocess(b[j]);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          o[3 * q] = __fadd_rn(b[3 * q + 2], s0);
          o[3 * q + 1] = __fadd_rn(b[3 * q + 1], s1);
          o[3 * q + 2] = __fadd_rn(b[3 * q], s2);
        }
      }
      float4* yv = reinterpret_cast<float4*>(y) + 3 * i;
      yv[0] = make_float4(o[0], o[1], o[2], o[3]);
      yv[1] = make_float4(o[4], o[5], o[6], o[7]);
      yv[2] = make_float4(o[8], o[9], o[10], o[11]);
      return;
    }
    i = groups * 4 + (i - groups);
  }
  if (i >= n_pix) return;
  const uint8_t* px = x + 3 * i;
  float* py = y + 3 * i;
  if constexpr (TF) {
    py[0] = keras_tf_preprocess((float)px[0]);
    py[1] = keras_tf_preprocess((float)px[1]);
    py[2] = keras_tf_preprocess((float)px[2]);
  } else {
    py[0] = __fadd_rn((float)px[2], s0);
    py[1] = __fadd_rn((float)px[1], s1);
    py[2] = __fadd_rn((float)px[0], s2);
  }
}
template <bool VEC>
__global__ void __launch_bounds__(256) preprocess_kernel(const uint8_t* __restrict__ x, const float* __restrict__ shift,
                                                         float* __restrict__ y, size_t n_pix) {
  preprocess_body<VEC, false>(x, shift, y, n_pix);
}
template <bool VEC>
__global__ void __launch_bounds__(256) preprocess_tf_kernel(const uint8_t* __restrict__ x, float* __restrict__ y,
                                                            size_t n_pix) {
  preprocess_body<VEC, true>(x, nullptr, y, n_pix);
}
int launch_preprocess(const uint8_t* x, const float* shift, float* y, size_t n_pix, cudaStream_t st) {
  if (n_pix == 0) return DEFER_OK;
  const bool vec = reinterpret_cast<uintptr_t>(x) % 4 == 0 && reinterpret_cast<uintptr_t>(y) % 16 == 0;
  const size_t threads = vec ? n_pix / 4 + n_pix % 4 : n_pix;
  const unsigned grid = (unsigned)((threads + 255) / 256);
  if (vec) {
    prefer_max_smem(preprocess_kernel<true>);
    preprocess_kernel<true><<<grid, 256, 0, st>>>(x, shift, y, n_pix);
  } else {
    prefer_max_smem(preprocess_kernel<false>);
    preprocess_kernel<false><<<grid, 256, 0, st>>>(x, shift, y, n_pix);
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}
int launch_preprocess_tf(const uint8_t* x, float* y, size_t n_pix, cudaStream_t st) {
  if (n_pix == 0) return DEFER_OK;
  const bool vec = reinterpret_cast<uintptr_t>(x) % 4 == 0 && reinterpret_cast<uintptr_t>(y) % 16 == 0;
  const size_t threads = vec ? n_pix / 4 + n_pix % 4 : n_pix;
  const unsigned grid = (unsigned)((threads + 255) / 256);
  if (vec) {
    prefer_max_smem(preprocess_tf_kernel<true>);
    preprocess_tf_kernel<true><<<grid, 256, 0, st>>>(x, y, n_pix);
  } else {
    prefer_max_smem(preprocess_tf_kernel<false>);
    preprocess_tf_kernel<false><<<grid, 256, 0, st>>>(x, y, n_pix);
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

// Keras load_img resize (DEFER_OP_RESIZE): one axis of Pillow's 8-bit separable resampling over a uint8 RGB image.
// Output i of the axis reads source [first, first + count) with int32 taps of 22 fractional bits:
// y = clamp((2^21 + sum x * tap) >> 22, 0, 255), the same integer arithmetic as Pillow, so the result is exact.
// HORIZ: one thread per output pixel, reading `count` consecutive source pixels of its row (3 bytes each).
// Vertical: one thread per output byte, reading `count` rows at a stride of w * 3 bytes - consecutive threads read
// consecutive bytes of a row.  Tables go through the read-only path; rows are independent of the batch index.
__device__ __forceinline__ uint8_t resize_clip8(int acc) { return (uint8_t)min(max(acc >> 22, 0), 255); }

// The integer arithmetic of every resize kernel, in one place so the fixed-size and the per-sample paths cannot drift:
// dst[c] = clamp((2^21 + sum_{k < count} src[k * step + c] * taps[k]) >> 22, 0, 255) for c < C.
template <int C>
__device__ __forceinline__ void resize_accumulate(const uint8_t* __restrict__ src, size_t step,
                                                  const int32_t* __restrict__ taps, int count, uint8_t* __restrict__ dst) {
  int a[C];
#pragma unroll
  for (int c = 0; c < C; ++c) a[c] = 1 << 21;
  for (int k = 0; k < count; ++k) {
    const int t = __ldg(taps + k);
    const uint8_t* p = src + k * step;
#pragma unroll
    for (int c = 0; c < C; ++c) a[c] += (int)__ldg(p + c) * t;
  }
#pragma unroll
  for (int c = 0; c < C; ++c) dst[c] = resize_clip8(a[c]);
}

template <bool HORIZ>
__global__ void __launch_bounds__(256) resize_u8_kernel(const uint8_t* __restrict__ x, uint8_t* __restrict__ y,
                                                        const int32_t* __restrict__ bounds, const int32_t* __restrict__ taps,
                                                        int ksize, int h_in, int w_in, int h_out, int w_out, size_t n_out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_out) return;
  if constexpr (HORIZ) {                         // i = output pixel; rows of input and output correspond 1:1
    const int xo = (int)(i % w_out);
    const size_t row = i / w_out;
    const int first = __ldg(bounds + 2 * xo), count = __ldg(bounds + 2 * xo + 1);
    resize_accumulate<3>(x + (row * w_in + first) * 3, 3, taps + (size_t)xo * ksize, count, y + i * 3);
  } else {                                       // i = output byte; columns (x, c) of input and output correspond 1:1
    const size_t row_bytes = (size_t)w_out * 3;
    const size_t col = i % row_bytes, r = i / row_bytes;
    const int yo = (int)(r % h_out);
    const size_t img = r / h_out;
    const int first = __ldg(bounds + 2 * yo), count = __ldg(bounds + 2 * yo + 1);
    resize_accumulate<1>(x + (img * h_in + first) * row_bytes + col, row_bytes, taps + (size_t)yo * ksize, count, y + i);
  }
}
int launch_resize(const uint8_t* x, uint8_t* y, const int32_t* bounds, const int32_t* taps, int ksize, int n, int h_in,
                  int w_in, int h_out, int w_out, bool horiz, cudaStream_t st) {
  const size_t n_out = (size_t)n * h_out * w_out * (horiz ? 1 : 3);
  if (n_out == 0) return DEFER_OK;
  const unsigned grid = (unsigned)((n_out + 255) / 256);
  if (horiz) {
    prefer_max_smem(resize_u8_kernel<true>);
    resize_u8_kernel<true><<<grid, 256, 0, st>>>(x, y, bounds, taps, ksize, h_in, w_in, h_out, w_out, n_out);
  } else {
    prefer_max_smem(resize_u8_kernel<false>);
    resize_u8_kernel<false><<<grid, 256, 0, st>>>(x, y, bounds, taps, ksize, h_in, w_in, h_out, w_out, n_out);
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

// Keras load_img resize of images of mixed sizes (DEFER_OP_RESIZE, modes DEFER_RESIZE_SAMPLE_W / _H).  Sample s of the
// microbatch reads its geometry and tables from its own int32 block (layout in include/defer_b200.h), so one launch - and
// one lane graph - serves any mix of sizes up to the slot's (H, W).  blockIdx.y = sample.
// SAMPLE_W: x = the input slots (n, H, W, 3), image s packed at the start of its slot as (h_in, w_in, 3);
//           y = (n, H, W_out, 3), rows [0, h_in) written, one thread per output pixel.
// SAMPLE_H: x = that (n, H, W_out, 3) buffer, rows [0, h_in) read; y = (n, H_out, W_out, 3), one thread per output byte.
// Memory safety does not depend on the block: h_in / w_in are clamped into [1, H] / [1, W], first into [0, in_len) and
// count into [0, min(kcap, in_len - first)], so a stale, zero or corrupt block gives wrong bytes, never a read outside
// the sample's slot.  A zero block (a never-written sample of a partial group) gives zero bytes.
template <bool HORIZ>
__global__ void __launch_bounds__(256) resize_frames_u8_kernel(const uint8_t* __restrict__ x, uint8_t* __restrict__ y,
                                                               const int32_t* __restrict__ tables, int block_ints, int H,
                                                               int W, int H_out, int W_out, int kw_w, int kw_h) {
  const int s = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int32_t* blk = tables + (size_t)s * block_ints;
  const int h_in = min(max(__ldg(blk), 1), H);
  if constexpr (HORIZ) {
    if (i >= h_in * W_out) return;               // rows past this sample's height
    const int w_in = min(max(__ldg(blk + 1), 1), W);
    const int xo = i % W_out, row = i / W_out;
    const int32_t* bounds = blk + 2;
    const int first = min(max(__ldg(bounds + 2 * xo), 0), w_in - 1);
    const int count = min(max(__ldg(bounds + 2 * xo + 1), 0), min(kw_w, w_in - first));
    resize_accumulate<3>(x + (size_t)s * H * W * 3 + ((size_t)row * w_in + first) * 3, 3,
                         bounds + 2 * W_out + (size_t)xo * kw_w, count, y + ((size_t)s * H * W_out + i) * 3);
  } else {
    const int row_bytes = W_out * 3;
    if (i >= H_out * row_bytes) return;
    const int col = i % row_bytes, yo = i / row_bytes;
    const int32_t* bounds = blk + 2 + W_out * (2 + kw_w);
    const int first = min(max(__ldg(bounds + 2 * yo), 0), h_in - 1);
    const int count = min(max(__ldg(bounds + 2 * yo + 1), 0), min(kw_h, h_in - first));
    resize_accumulate<1>(x + ((size_t)s * H + first) * row_bytes + col, (size_t)row_bytes,
                         bounds + 2 * H_out + (size_t)yo * kw_h, count, y + (size_t)s * H_out * row_bytes + i);
  }
}
int launch_resize_frames(int pass, const uint8_t* x, uint8_t* y, const int32_t* tables, int n, int H, int W, int H_out,
                         int W_out, int kw_w, int kw_h, cudaStream_t st) {
  const int block_ints = 2 + W_out * (2 + kw_w) + H_out * (2 + kw_h);
  const bool horiz = pass == DEFER_RESIZE_SAMPLE_W;
  const size_t per_sample = horiz ? (size_t)H * W_out : (size_t)H_out * W_out * 3;
  const dim3 grid((unsigned)((per_sample + 255) / 256), (unsigned)n);
  if (horiz) {
    prefer_max_smem(resize_frames_u8_kernel<true>);
    resize_frames_u8_kernel<true><<<grid, 256, 0, st>>>(x, y, tables, block_ints, H, W, H_out, W_out, kw_w, kw_h);
  } else {
    prefer_max_smem(resize_frames_u8_kernel<false>);
    resize_frames_u8_kernel<false><<<grid, 256, 0, st>>>(x, y, tables, block_ints, H, W, H_out, W_out, kw_w, kw_h);
  }
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

__global__ void __launch_bounds__(256) f32_to_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = __float2bfloat16_rn(x[i]);
}
int launch_f32_to_bf16(const float* x, void* y, size_t n, cudaStream_t st) {
  unsigned grid = (unsigned)((n + 255) / 256);
  prefer_max_smem(f32_to_bf16_kernel); f32_to_bf16_kernel<<<grid, 256, 0, st>>>(x, (__nv_bfloat16*)y, n);
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

// =============================================================================================
// hop flags.  Each slot is used strictly in sequence, so the k-th use waits for / publishes the
// value k; the running count lives in device memory so the kernels are CUDA-graph friendly.
//   wait:   want = ++(*counter) - minus;  spin until *flag >= want   (acquire, system scope)
//   signal: v = ++(*counter);  fence.sys;  *remote_flag = v          (release, system scope)
// A wait that exceeds its budget records DEFER_ERR_TIMEOUT in *status and returns (never hangs).
// =============================================================================================
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Flag protocol of the hop.  A flag holds the number of microbatches signalled so far on that slot (bits 0..30);
// bit 31 is POISON: a stage whose sticky status is non-zero (its own wait timed out, or it saw poison) signals
// `count | POISON`, so the failure travels down the chain with the ready flags (and up with the free flags) and the
// last stage's result call reports it - a stalled peer can never turn into silently wrong results.
constexpr uint32_t FLAG_POISON = 0x80000000u;

__global__ void wait_flag_kernel(const uint32_t* flag, uint32_t* counter, int minus, int* status,
                                 unsigned long long timeout_ns) {
  if (threadIdx.x != 0) return;
  uint32_t want = ++(*counter) - (uint32_t)minus;
  if (want == 0) return;
  if (*reinterpret_cast<volatile int*>(status) != 0) return;  // pipeline already failed: do not spin again
  unsigned long long t0 = globaltimer_ns();
  unsigned spins = 0;
  for (;;) {
    const uint32_t f = ld_acquire_sys(flag);
    if (f & FLAG_POISON) {                       // the neighbour failed: inherit the failure
      atomicExch(status, (int)DEFER_ERR_TIMEOUT);
      break;
    }
    if (f >= want) break;
    if ((++spins & 0x3ff) == 0) {
      if (globaltimer_ns() - t0 > timeout_ns) {
        atomicExch(status, (int)DEFER_ERR_TIMEOUT);
        break;
      }
    }
    __nanosleep(64);
  }
}

__global__ void signal_flag_kernel(uint32_t* remote_flag, uint32_t* counter, const int* status) {
  if (threadIdx.x != 0) return;
  uint32_t v = ++(*counter);
  if (*reinterpret_cast<const volatile int*>(status) != 0) v |= FLAG_POISON;
  __threadfence_system();
  st_release_sys(remote_flag, v);
}

int launch_wait_flag(const uint32_t* flag, uint32_t* counter, int minus, int* status, unsigned long long timeout_ns,
                     cudaStream_t st) {
  prefer_max_smem(wait_flag_kernel); wait_flag_kernel<<<1, 32, 0, st>>>(flag, counter, minus, status, timeout_ns);
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}
int launch_signal_flag(uint32_t* remote_flag, uint32_t* counter, const int* status, cudaStream_t st) {
  prefer_max_smem(signal_flag_kernel); signal_flag_kernel<<<1, 32, 0, st>>>(remote_flag, counter, status);
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

}  // namespace defer
