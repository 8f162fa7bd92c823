// conv_umma.cuh - interface of the wgmma implicit-GEMM convolution (conv_umma.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace defer {

// Shape-level plan: tiling, transformed weights (bf16 [tap][cout][cin], hi/lo planes), tensor map
// for the weights.  Built once per op.
struct UmmaConvPlan {
  int fmt = 0, nplanes = 1;
  int n = 0, h = 0, w = 0, cin = 0, ho = 0, wo = 0, cout = 0;
  int kh = 1, kw = 1, sh = 1, sw = 1, pad_t = 0, pad_l = 0;
  uint32_t flags = 0;
  // M tile t = the 128 consecutive output pixels [128 t, 128 t + 128) in (n, ho, wo) order
  int m_tiles = 0;         // ceil(n * ho * wo / 128)
  int im2col = 0;          // A tile: 1 = TMA im2col load of the NHWC input; 0 = tiled load of the [M, C] view (1x1, stride 1)
  int bn = 64;             // N tile (cout per CTA)
  int k_blocks = 0;        // taps * cin / 64
  int splits = 1;          // split-K factor (grid.z)
  int cluster = 0;         // 1: the splits of a tile are one thread-block cluster, reduced through DSMEM
  int stages = 4;          // smem ring depth of the one-tile-per-CTA kernel (fewer stages -> more CTAs per SM)
  int stream = 0;          // 1: plan of the streaming persistent kernel (conv_stream_kernel), N tile = bn
  void* w_dev = nullptr;   // transformed weights
  const float* scale = nullptr;
  const float* shift = nullptr;
  // a standalone affine op folded into the epilogue (set by the caller after umma_conv_prepare): y2 = [relu](fmaf(stored, scale2, shift2))
  bool aff = false;
  const float* scale2 = nullptr;
  const float* shift2 = nullptr;
  int relu2 = 0;
  int store_first = 1;     // 0: the conv's own output is not written (only the affine op's)
  CUtensorMap tmap_w[2];   // hi, lo
  bool ready = false;
};

// Per-lane binding: tensor maps of the input activation planes + raw pointers for the epilogue.
struct UmmaConvLaneArgs {
  CUtensorMap tmap_x[2];
  bool direct_out = false;           // output lives in a peer GPU's slot (the epilogue's plain stores reach it)
  const void* res = nullptr;
  void* y = nullptr;
  void* y2 = nullptr;                // output of the folded affine op (UmmaConvPlan::aff)
  float* partial = nullptr;          // split-K partial tiles (per lane: lanes run concurrently)
  unsigned int* counters = nullptr;  // split-K arrival counters, one per output tile
};

// false also when the corners of the shape's im2col bounding box are outside what TMA encodes for a rank-4 tensor
bool umma_conv_supported(int fmt, int n, int h, int w, int cin, int ho, int wo, int cout, int kh, int kw, int sh, int sw,
                         int pad_t, int pad_l);
int umma_conv_prepare(UmmaConvPlan* plan, int fmt, int n, int h, int w, int cin, int ho, int wo, int cout, int kh, int kw,
                      int sh, int sw, int pad_t, int pad_l, uint32_t flags, const float* w_hwio_dev, const float* scale_dev,
                      const float* shift_dev, bool mega = false, int stream_bn = 0);
int umma_conv_bind(const UmmaConvPlan& plan, UmmaConvLaneArgs* args, const void* x, const void* res, void* y);
void umma_conv_unbind(UmmaConvLaneArgs* args);
int launch_conv_umma(const UmmaConvPlan& plan, const UmmaConvLaneArgs& args, cudaStream_t st);
void umma_conv_release(UmmaConvPlan& plan);

// Stage megakernel: a run of consecutive convs in ONE cluster launch (conv_umma.cu, conv_mega_kernel).
size_t umma_mega_op_bytes();
int umma_mega_fill(void* host_dst, const UmmaConvPlan& plan, const UmmaConvLaneArgs& args);   // one op descriptor
int umma_mega_cluster_size();
int launch_conv_mega(int nplanes, const void* dev_ops, int n_ops, cudaStream_t st);
// one op on the streaming persistent kernel (deep operand ring, epilogue staged outside it)
int launch_conv_stream(int nplanes, int bn, const void* dev_op, int n_tiles, int k_blocks, bool aff, cudaStream_t st);
// fused stem: conv over a few-channel fp32 image with the im2col done inside the persistent kernel, from an image window
// per output tile staged in shared memory.  Fusable when that window fits the kernel's window buffer.
bool umma_stem_fusable(int fmt, int cin, int ho, int wo, int cout, int kh, int kw, int sh, int sw, uint32_t flags);
// turns a persistent-kernel op descriptor (umma_mega_fill of the 1x1 plan over the patch matrix) into the fused stem's:
// sets the image and the 2-D output tiling; returns the number of tiles to launch
int umma_mega_set_stem(void* host_op, const float* x, int h, int w, int cin, int kh, int kw, int sh, int sw, int pad_t, int pad_l);
// ... reading a uint8 RGB image instead, preprocessed on the fly (after umma_mega_set_stem): channel c of the conv input
// is float(image[.., 2 - c]) + shift[c] (Keras caffe mode), or with tf float(image[.., c]) / 127.5 - 1 (Keras tf mode,
// shift unused)
void umma_mega_set_stem_u8(void* host_op, const uint8_t* x, const float shift[3]);
int launch_conv_stem(int nplanes, const void* dev_op, int n_tiles, bool u8, bool tf, cudaStream_t st);
// one op on a persistent grid (64-wide N tiles): for ops with many tiles
int launch_conv_persistent(int nplanes, const void* dev_op, int n_tiles, bool aff, cudaStream_t st);

}  // namespace defer
