// common.cuh - shared helpers for libdefer_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/defer_b200.h"

namespace defer {

// ---------------------------------------------------------------------------------------------
// error plumbing: CUDA errors are translated into defer_status + a thread-local message, never thrown
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
const char* get_error();

#define DEFER_CUDA(expr)                                                                  \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      ::defer::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return DEFER_ERR_CUDA;                                                              \
    }                                                                                     \
  } while (0)

#define DEFER_CHECK(cond, ...)                                                            \
  do {                                                                                    \
    if (!(cond)) {                                                                        \
      ::defer::set_error(__VA_ARGS__);                                                    \
      return DEFER_ERR_INVALID;                                                           \
    }                                                                                     \
  } while (0)

#define DEFER_TRY(expr)                                                                   \
  do {                                                                                    \
    int _s = (expr);                                                                      \
    if (_s != DEFER_OK) return _s;                                                        \
  } while (0)

// ---------------------------------------------------------------------------------------------
// Every kernel of the library asks for the same (maximum) shared-memory carve-out.  Lanes run
// concurrently on one GPU; CTAs of kernels that want different L1/shared splits cannot share an SM, and
// switching the split drains it.  One uniform configuration lets tiny SIMT kernels and 200 KB wgmma
// tiles co-reside.  Called once per (kernel, device).
// ---------------------------------------------------------------------------------------------
void prefer_max_smem_impl(const void* func);
template <class K>
inline void prefer_max_smem(K kernel) { prefer_max_smem_impl(reinterpret_cast<const void*>(kernel)); }

// ---------------------------------------------------------------------------------------------
// activation formats (defer_fmt).  BF16X2 stores v as hi = bf16(v), lo = bf16(v - hi) in two planes:
// hi plane at element offset 0, lo plane at element offset `plane` (= total elements of the tensor).
// ---------------------------------------------------------------------------------------------
constexpr int FMT_F32 = DEFER_FMT_F32;
constexpr int FMT_BF16X2 = DEFER_FMT_BF16X2;
constexpr int FMT_BF16 = DEFER_FMT_BF16;

__host__ __device__ inline size_t fmt_bytes_per_elem(int fmt) { return fmt == FMT_BF16 ? 2 : 4; }

template <int FMT>
__device__ __forceinline__ float act_load(const void* __restrict__ base, size_t plane, size_t i) {
  if constexpr (FMT == FMT_F32) {
    return __ldg(reinterpret_cast<const float*>(base) + i);
  } else if constexpr (FMT == FMT_BF16) {
    return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[i]);
  } else {
    const __nv_bfloat16* p = reinterpret_cast<const __nv_bfloat16*>(base);
    return __bfloat162float(p[i]) + __bfloat162float(p[plane + i]);
  }
}

template <int FMT>
__device__ __forceinline__ void act_store(void* __restrict__ base, size_t plane, size_t i, float v) {
  if constexpr (FMT == FMT_F32) {
    reinterpret_cast<float*>(base)[i] = v;
  } else if constexpr (FMT == FMT_BF16) {
    reinterpret_cast<__nv_bfloat16*>(base)[i] = __float2bfloat16_rn(v);
  } else {
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base);
    __nv_bfloat16 hi = __float2bfloat16_rn(v);
    p[i] = hi;
    p[plane + i] = __float2bfloat16_rn(v - __bfloat162float(hi));
  }
}

// 4 consecutive elements (i % 4 == 0, 16-byte / 8-byte aligned as the format requires)
template <int FMT>
__device__ __forceinline__ float4 act_load4(const void* __restrict__ base, size_t plane, size_t i) {
  if constexpr (FMT == FMT_F32) {
    return __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + i));
  } else if constexpr (FMT == FMT_BF16) {
    uint2 r = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(base) + i);
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&r.x);
    __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&r.y);
    return make_float4(__low2float(a), __high2float(a), __low2float(b), __high2float(b));
  } else {
    const __nv_bfloat16* p = reinterpret_cast<const __nv_bfloat16*>(base);
    uint2 rh = *reinterpret_cast<const uint2*>(p + i);
    uint2 rl = *reinterpret_cast<const uint2*>(p + plane + i);
    __nv_bfloat162 ha = *reinterpret_cast<__nv_bfloat162*>(&rh.x), hb = *reinterpret_cast<__nv_bfloat162*>(&rh.y);
    __nv_bfloat162 la = *reinterpret_cast<__nv_bfloat162*>(&rl.x), lb = *reinterpret_cast<__nv_bfloat162*>(&rl.y);
    return make_float4(__low2float(ha) + __low2float(la), __high2float(ha) + __high2float(la),
                       __low2float(hb) + __low2float(lb), __high2float(hb) + __high2float(lb));
  }
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// split v into (hi, lo) bf16 pairs for two values
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = pack_bf16x2(a, b);   // one packed F2FP (round-to-nearest-even), not two scalar F2F on the slow conversion pipe
  lo = pack_bf16x2(a - __uint_as_float(hi << 16), b - __uint_as_float(hi & 0xffff0000u));
}

// Keras 'tf'-mode preprocess_input of one byte value b (0..255, exact in fp32): fl32(fl32(b / 127.5) - 1), bit for bit,
// without a division (__fdiv_rn carries a called slow path, which the wgmma kernels must not contain).  q = b * r with
// r = fl32(1 / 127.5) is off by one ulp for 111 of the 256 bytes; one exact remainder e = b - q * 127.5 (a single FMA)
// and one correction q + e * r give the correctly rounded quotient for all 256.  Every step is an explicit _rn
// intrinsic, so nvcc cannot contract or reorder it: FMUL, FFMA, FFMA, FADD.
__device__ __forceinline__ float keras_tf_preprocess(float b) {
  const float r = __uint_as_float(0x3C008081u);   // fl32(1 / 127.5)
  float q = __fmul_rn(b, r);
  const float e = __fmaf_rn(-q, 127.5f, b);
  q = __fmaf_rn(e, r, q);
  return __fsub_rn(q, 1.0f);
}

template <int FMT>
__device__ __forceinline__ void act_store4(void* __restrict__ base, size_t plane, size_t i, float4 v) {
  if constexpr (FMT == FMT_F32) {
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + i) = v;
  } else if constexpr (FMT == FMT_BF16) {
    uint2 r;
    r.x = pack_bf16x2(v.x, v.y);
    r.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(base) + i) = r;
  } else {
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base);
    uint2 h, l;
    split_bf16x2(v.x, v.y, h.x, l.x);
    split_bf16x2(v.z, v.w, h.y, l.y);
    *reinterpret_cast<uint2*>(p + i) = h;
    *reinterpret_cast<uint2*>(p + plane + i) = l;
  }
}

// ---------------------------------------------------------------------------------------------
// kernel-launch parameter blocks shared between the stage runtime and the per-kernel entry points
// ---------------------------------------------------------------------------------------------
struct ConvParams {
  const void* x;        // input activations (fmt or f32)
  const float* w;       // fp32 HWIO ([kh][kw][cin][cout]) - SIMT path
  const float* scale;   // per-cout (may be null => 1)
  const float* shift;   // per-cout (may be null => 0)
  const void* res;      // residual in act fmt (may be null)
  void* y;              // output, act fmt
  int n, h, w_in, cin;  // input dims
  int ho, wo, cout;
  int kh, kw, sh, sw, pad_t, pad_l;
  uint32_t flags;
};

int launch_conv_simt(int fmt, bool x_is_f32, const ConvParams& p, cudaStream_t st);
// tensor-core stem: fp32 image -> [pixels, K_pad] patch matrix in the stage format (then a 1x1 wgmma conv)
int launch_stem_im2col(int fmt, const float* x, void* out, int n, int h, int w, int cin, int kh, int kw, int sh, int sw,
                       int pad_t, int pad_l, int ho, int wo, int K_pad, cudaStream_t st);
int launch_maxpool(int fmt, const void* x, void* y, int n, int h, int w, int c, int ph, int pw, int sh, int sw,
                   int pad_t, int pad_l, int ho, int wo, cudaStream_t st);
int launch_gap(int fmt, const void* x, void* y, int n, int h, int w, int c, cudaStream_t st);
// dense: `partial` is a workspace of dense_workspace_bytes(...) bytes, zeroed once (arrival counters)
int dense_splits(int n, int in_features, int units);
// dense workspace: split partials + arrival counters of the fused kernel; must be zero-initialised once
size_t dense_workspace_bytes(int n, int in_features, int units);
int launch_dense(int fmt, const void* x, const void* w, bool w_is_bf16, const float* bias, void* y, bool y_is_f32,
                 float* partial, int n, int in_features, int units, uint32_t flags, cudaStream_t st);
int launch_softmax(const float* x, float* y, int n, int c, cudaStream_t st);
int launch_eltwise(int fmt, int kind, const void* a, const void* b, const float* scale, const float* shift, void* y,
                   size_t n_pix, int c, uint32_t flags, cudaStream_t st);
int launch_pad(int fmt, const void* x, void* y, int n, int h, int w, int c, int pad_t, int pad_l, int ho, int wo,
               cudaStream_t st);
int launch_encode(int fmt, const float* x, void* y, size_t n_elems, cudaStream_t st);
int launch_decode(int fmt, const void* x, float* y, size_t n_elems, cudaStream_t st);
int launch_copy_act(int fmt, const void* x, void* y, size_t n_elems, cudaStream_t st);
int launch_f32_to_bf16(const float* x, void* y, size_t n, cudaStream_t st);
// Keras caffe preprocess_input: uint8 RGB (n_pix pixels x 3) -> fp32 BGR + shift (DEFER_OP_PREPROCESS)
int launch_preprocess(const uint8_t* x, const float* shift, float* y, size_t n_pix, cudaStream_t st);
// Keras tf preprocess_input: uint8 RGB (n_pix pixels x 3) -> fp32 b / 127.5 - 1, channels kept (DEFER_PRE_TF)
int launch_preprocess_tf(const uint8_t* x, float* y, size_t n_pix, cudaStream_t st);
// Keras load_img resize, one axis (DEFER_OP_RESIZE): uint8 RGB (n, h_in, w_in, 3) -> (n, h_out, w_out, 3), resampling
// the width (horiz) or the height; the other axis keeps its length.  bounds [out, 2] (first, count), taps [out, ksize].
int launch_resize(const uint8_t* x, uint8_t* y, const int32_t* bounds, const int32_t* taps, int ksize, int n, int h_in,
                  int w_in, int h_out, int w_out, bool horiz, cudaStream_t st);
// Keras load_img resize of mixed sizes, one pass (DEFER_OP_RESIZE, pass = DEFER_RESIZE_SAMPLE_W | _H): each of the n
// samples reads its size and tables from its int32 block in `tables` (layout: include/defer_b200.h).
int launch_resize_frames(int pass, const uint8_t* x, uint8_t* y, const int32_t* tables, int n, int H, int W, int H_out,
                         int W_out, int kw_w, int kw_h, cudaStream_t st);
// Where one decode launch finds sample s: its file at files + s * file, its block at blocks + s * block_ints, its
// workspace at workspace + s * ws; and which samples it decodes (decode_takes).  The single-format ops pass nullptr and
// derive them from (H, W); DEFER_OP_IMAGE_DECODE passes the image slot's, and one format per launch.
struct DecodeStrides {
  size_t file, ws;
  int block_ints;
  int take;   // 0: every sample; DEFER_IMAGE_JPEG: those tagged JPEG; DEFER_IMAGE_PNG: every sample not tagged JPEG
};
__device__ __forceinline__ bool decode_takes(const int32_t* blk, int take) {
  return take == 0 || (blk[DEFER_IMAGE_TAG] == DEFER_IMAGE_JPEG) == (take == DEFER_IMAGE_JPEG);
}
// DEFER_OP_JPEG_DECODE (jpeg.cu): n JPEG files in H * W * 3-byte slots, with their blocks -> n U8 (H, W, 3) images, through a
// workspace of jpeg_workspace_bytes(H, W, n) (256-byte aligned)
size_t jpeg_workspace_bytes(int H, int W, int n);
// one sample's workspace bytes (a multiple of 256), and where its coefficients and planes start
size_t jpeg_ws_stride(int H, int W, size_t* coef_off, size_t* plane_off);
// the bounds (H, W) the decode takes: H * W * 24 + DEFER_JPEG_SUBSEQ_BITS < 2^31
bool jpeg_bound_ok(int H, int W);
int launch_jpeg_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace, uint8_t* y,
                       cudaStream_t st, const DecodeStrides* strides = nullptr);
// DEFER_OP_PNG_DECODE (png.cu): n PNG files in DEFER_PNG_SLOT_BYTES(H, W)-byte slots, with their blocks -> n U8 (H, W, 3)
// images, through a workspace of png_workspace_bytes(H, W, n) (256-byte aligned)
size_t png_workspace_bytes(int H, int W, int n);
// one sample's workspace bytes (a multiple of 256), and where its scanlines start
size_t png_ws_stride(int H, int W, size_t* raw_off);
// the bounds (H, W) the decode takes: the slot fits the blocks' int32 offsets
bool png_bound_ok(int H, int W);
int launch_png_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace, uint8_t* y,
                      cudaStream_t st, const DecodeStrides* strides = nullptr);
// DEFER_OP_IMAGE_DECODE (image.cu): n JPEG or PNG files in DEFER_PNG_SLOT_BYTES(H, W)-byte slots, with their tagged
// blocks -> n U8 (H, W, 3) images, through a workspace of image_workspace_bytes(H, W, n) (256-byte aligned)
size_t image_workspace_bytes(int H, int W, int n);
// the bounds (H, W) both decodes take
bool image_bound_ok(int H, int W);
int launch_image_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace, uint8_t* y,
                        cudaStream_t st);

// flag protocol kernels (see stage.cu)
int launch_wait_flag(const uint32_t* flag, uint32_t* counter, int minus, int* status, unsigned long long timeout_ns,
                     cudaStream_t st);
int launch_signal_flag(uint32_t* remote_flag, uint32_t* counter, const int* status, cudaStream_t st);

}  // namespace defer
