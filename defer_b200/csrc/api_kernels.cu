// api_kernels.cu - per-kernel C-ABI entry points (raw device pointers) for parity tests and ncu.
#include <vector>

#include "common.cuh"
#include "conv_umma.cuh"

using namespace defer;

extern "C" {

int defer_k_conv(int fmt, int backend, const void* x, int x_is_f32, const float* w_hwio, const float* scale,
                 const float* shift, const void* residual, void* y, int n, int h, int w, int cin, int cout, int kh, int kw,
                 int sh, int sw, int pad_t, int pad_l, int pad_b, int pad_r, uint32_t flags, void* stream) {
  DEFER_CHECK(x && w_hwio && y, "k_conv: null pointer");
  DEFER_CHECK(fmt >= 0 && fmt <= 2, "k_conv: bad fmt");
  cudaStream_t st = (cudaStream_t)stream;
  int ho = (h + pad_t + pad_b - kh) / sh + 1, wo = (w + pad_l + pad_r - kw) / sw + 1;
  DEFER_CHECK(ho >= 1 && wo >= 1, "k_conv: empty output");
  if (residual) flags |= DEFER_FLAG_RESIDUAL;
  if (backend >= 2 && backend <= 7) {
    // 2: one tile per CTA (conv_umma_kernel) | 3: persistent grid, 64-wide N tiles | 4 / 5: streaming persistent kernel
    // with 64- / 128-wide N tiles | 6 / 7: the same, planned for an output in a peer GPU's slot
    DEFER_CHECK(fmt != DEFER_FMT_F32 && !x_is_f32, "k_conv: wgmma backend needs BF16X2/BF16 activations");
    DEFER_CHECK(umma_conv_supported(fmt, n, h, w, cin, ho, wo, cout, kh, kw, sh, sw, pad_t, pad_l),
                "k_conv: shape not supported by the wgmma kernel");
    UmmaConvPlan plan;
    UmmaConvLaneArgs args;
    void* dev_op = nullptr;
    const int stream_bn = backend >= 4 ? ((backend & 1) ? 128 : 64) : 0;
    int rc = umma_conv_prepare(&plan, fmt, n, h, w, cin, ho, wo, cout, kh, kw, sh, sw, pad_t, pad_l, flags, w_hwio, scale, shift,
                               /*mega=*/backend == 3, stream_bn);
    args.direct_out = backend >= 6;
    if (rc == DEFER_OK) rc = umma_conv_bind(plan, &args, x, residual, y);
    const int n_tiles = plan.m_tiles * (cout / plan.bn);
    if (backend == 2) {
      if (rc == DEFER_OK) rc = launch_conv_umma(plan, args, st);
    } else {
      std::vector<unsigned char> host(umma_mega_op_bytes());
      if (rc == DEFER_OK) rc = umma_mega_fill(host.data(), plan, args);
      if (rc == DEFER_OK && cudaMalloc(&dev_op, host.size()) != cudaSuccess) rc = DEFER_ERR_CUDA;
      if (rc == DEFER_OK) cudaMemcpy(dev_op, host.data(), host.size(), cudaMemcpyHostToDevice);
      if (rc == DEFER_OK)
        rc = backend == 3 ? launch_conv_persistent(plan.nplanes, dev_op, n_tiles, false, st)
                          : launch_conv_stream(plan.nplanes, plan.bn, dev_op, n_tiles, plan.k_blocks, false, st);
    }
    cudaError_t e = cudaStreamSynchronize(st);
    if (dev_op) cudaFree(dev_op);
    umma_conv_unbind(&args);
    umma_conv_release(plan);
    if (rc != DEFER_OK) return rc;
    DEFER_CUDA(e);
    return DEFER_OK;
  }
  ConvParams p;
  p.x = x; p.w = w_hwio; p.scale = scale; p.shift = shift; p.res = residual; p.y = y;
  p.n = n; p.h = h; p.w_in = w; p.cin = cin; p.ho = ho; p.wo = wo; p.cout = cout;
  p.kh = kh; p.kw = kw; p.sh = sh; p.sw = sw; p.pad_t = pad_t; p.pad_l = pad_l; p.flags = flags;
  return launch_conv_simt(fmt, x_is_f32 != 0, p, st);
}

int defer_k_maxpool(int fmt, const void* x, void* y, int n, int h, int w, int c, int ph, int pw, int sh, int sw, int pad_t,
                    int pad_l, int pad_b, int pad_r, void* stream) {
  DEFER_CHECK(x && y, "k_maxpool: null pointer");
  int ho = (h + pad_t + pad_b - ph) / sh + 1, wo = (w + pad_l + pad_r - pw) / sw + 1;
  return launch_maxpool(fmt, x, y, n, h, w, c, ph, pw, sh, sw, pad_t, pad_l, ho, wo, (cudaStream_t)stream);
}

int defer_k_gap(int fmt, const void* x, void* y, int n, int h, int w, int c, void* stream) {
  DEFER_CHECK(x && y, "k_gap: null pointer");
  return launch_gap(fmt, x, y, n, h, w, c, (cudaStream_t)stream);
}

int defer_k_dense(int fmt, const void* x, const float* w_io, const float* bias, void* y, int y_is_f32, int n,
                  int in_features, int units, uint32_t flags, void* stream) {
  DEFER_CHECK(x && w_io && y, "k_dense: null pointer");
  float* partial = nullptr;
  size_t bytes = dense_workspace_bytes(n, in_features, units);
  DEFER_CUDA(cudaMalloc((void**)&partial, bytes));
  DEFER_CUDA(cudaMemsetAsync(partial, 0, bytes, (cudaStream_t)stream));
  int rc = launch_dense(fmt, x, w_io, false, bias, y, y_is_f32 != 0, partial, n, in_features, units, flags, (cudaStream_t)stream);
  cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
  cudaFree(partial);
  if (rc != DEFER_OK) return rc;
  DEFER_CUDA(e);
  return DEFER_OK;
}

int defer_k_softmax(const float* x, float* y, int n, int c, void* stream) {
  DEFER_CHECK(x && y, "k_softmax: null pointer");
  return launch_softmax(x, y, n, c, (cudaStream_t)stream);
}

int defer_k_eltwise(int fmt, int kind, const void* a, const void* b, const float* scale, const float* shift, void* y, int n,
                    int h, int w, int c, uint32_t flags, void* stream) {
  DEFER_CHECK(a && y, "k_eltwise: null pointer");
  DEFER_CHECK(kind != DEFER_OP_ADD || b, "k_eltwise: ADD needs b");
  return launch_eltwise(fmt, kind, a, b, scale, shift, y, (size_t)n * h * w, c, flags, (cudaStream_t)stream);
}

int defer_k_encode(int fmt, const float* x_f32, void* y_act, uint64_t n_elems, void* stream) {
  DEFER_CHECK(x_f32 && y_act, "k_encode: null pointer");
  return launch_encode(fmt, x_f32, y_act, n_elems, (cudaStream_t)stream);
}

int defer_k_decode(int fmt, const void* x_act, float* y_f32, uint64_t n_elems, void* stream) {
  DEFER_CHECK(x_act && y_f32, "k_decode: null pointer");
  return launch_decode(fmt, x_act, y_f32, n_elems, (cudaStream_t)stream);
}

int defer_k_preprocess(const uint8_t* x, const float* shift, float* y, int n, int h, int w, int c, void* stream) {
  DEFER_CHECK(x && shift && y, "k_preprocess: null pointer");
  DEFER_CHECK(n >= 1 && h >= 1 && w >= 1, "k_preprocess: empty image (%d,%d,%d)", n, h, w);
  DEFER_CHECK(c == 3, "k_preprocess: caffe preprocessing needs 3 channels (RGB), got %d", c);
  return launch_preprocess(x, shift, y, (size_t)n * h * w, (cudaStream_t)stream);
}

int defer_k_preprocess_tf(const uint8_t* x, float* y, int n, int h, int w, int c, void* stream) {
  DEFER_CHECK(x && y, "k_preprocess_tf: null pointer");
  DEFER_CHECK(n >= 1 && h >= 1 && w >= 1, "k_preprocess_tf: empty image (%d,%d,%d)", n, h, w);
  DEFER_CHECK(c == 3, "k_preprocess_tf: preprocessing needs 3 channels (RGB), got %d", c);
  return launch_preprocess_tf(x, y, (size_t)n * h * w, (cudaStream_t)stream);
}

int defer_k_resize(const uint8_t* x, uint8_t* y, const int32_t* bounds, const int32_t* taps, int ksize, int n, int h_in,
                   int w_in, int h_out, int w_out, int c, void* stream) {
  DEFER_CHECK(x && y && bounds && taps, "k_resize: null pointer");
  DEFER_CHECK(n >= 1 && h_in >= 1 && w_in >= 1 && h_out >= 1 && w_out >= 1 && ksize >= 1,
              "k_resize: bad sizes (n %d, %dx%d -> %dx%d, ksize %d)", n, h_in, w_in, h_out, w_out, ksize);
  DEFER_CHECK(c == 3, "k_resize: the resize takes RGB images (3 channels), got %d", c);
  DEFER_CHECK((h_in != h_out) != (w_in != w_out), "k_resize: exactly one axis must change (%dx%d -> %dx%d)", h_in, w_in,
              h_out, w_out);
  return launch_resize(x, y, bounds, taps, ksize, n, h_in, w_in, h_out, w_out, w_in != w_out, (cudaStream_t)stream);
}

int defer_k_resize_frames(int pass, const uint8_t* x, uint8_t* y, const int32_t* tables, int n, int H, int W, int H_out,
                          int W_out, int kw_w, int kw_h, int c, void* stream) {
  DEFER_CHECK(x && y && tables, "k_resize_frames: null pointer");
  DEFER_CHECK(pass == DEFER_RESIZE_SAMPLE_W || pass == DEFER_RESIZE_SAMPLE_H, "k_resize_frames: pass %d is not %d (width) or %d "
              "(height)", pass, DEFER_RESIZE_SAMPLE_W, DEFER_RESIZE_SAMPLE_H);
  DEFER_CHECK(n >= 1 && n <= 65535 && H >= 1 && W >= 1 && H_out >= 1 && W_out >= 1 && kw_w >= 1 && kw_h >= 1,
              "k_resize_frames: bad sizes (n %d, %dx%d -> %dx%d, kw %d/%d)", n, H, W, H_out, W_out, kw_w, kw_h);
  DEFER_CHECK(c == 3, "k_resize_frames: the resize takes RGB images (3 channels), got %d", c);
  DEFER_CHECK(((uintptr_t)tables & 3) == 0, "k_resize_frames: tables must be 4-byte aligned");
  return launch_resize_frames(pass, x, y, tables, n, H, W, H_out, W_out, kw_w, kw_h, (cudaStream_t)stream);
}

}  // extern "C"
