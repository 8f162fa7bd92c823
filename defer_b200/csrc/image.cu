// image.cu - DEFER_OP_IMAGE_DECODE: a microbatch whose samples are JPEG or PNG files, each told by the tag of its block.
// The three JPEG kernels (jpeg.cu) run on the samples tagged DEFER_IMAGE_JPEG, then the three PNG kernels (png.cu) on
// every other sample, on the same stream.  Both read their samples at the image slot's strides: the file slot of
// DEFER_PNG_SLOT_BYTES(H, W), the block of DEFER_IMAGE_BLOCK_INTS and the workspace of the larger of the two formats'
// per-sample strides (a sample is one format at a time).  Each CTA of the other format's samples reads one block int
// and exits, as the pixel kernels' CTAs past a sample's own size do.
#include <algorithm>

#include "common.cuh"

namespace defer {

static size_t image_ws_stride(int H, int W) {
  return std::max(jpeg_ws_stride(H, W, nullptr, nullptr), png_ws_stride(H, W, nullptr));   // both multiples of 256
}

size_t image_workspace_bytes(int H, int W, int n) { return image_ws_stride(H, W) * (size_t)n; }

bool image_bound_ok(int H, int W) { return jpeg_bound_ok(H, W) && png_bound_ok(H, W); }

int launch_image_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace, uint8_t* y,
                        cudaStream_t st) {
  DecodeStrides d;
  d.file = DEFER_PNG_SLOT_BYTES((size_t)H, (size_t)W);
  d.ws = image_ws_stride(H, W);
  d.block_ints = DEFER_IMAGE_BLOCK_INTS;
  d.take = DEFER_IMAGE_JPEG;
  DEFER_TRY(launch_jpeg_decode(files, blocks, n, H, W, workspace, y, st, &d));
  d.take = DEFER_IMAGE_PNG;
  return launch_png_decode(files, blocks, n, H, W, workspace, y, st, &d);
}

}  // namespace defer

using namespace defer;

extern "C" {

int defer_k_image_workspace(int H, int W, int n, uint64_t* bytes, uint64_t* sample_stride, uint64_t* coef_off,
                            uint64_t* plane_off, uint64_t* raw_off) {
  DEFER_CHECK(H >= 1 && W >= 1 && n >= 1 && image_bound_ok(H, W), "k_image_workspace: bad bound %dx%d (n %d)", H, W, n);
  size_t coef = 0, planes = 0, raw = 0;
  jpeg_ws_stride(H, W, &coef, &planes);
  png_ws_stride(H, W, &raw);
  const size_t stride = image_ws_stride(H, W);
  if (bytes) *bytes = stride * (uint64_t)n;
  if (sample_stride) *sample_stride = stride;
  if (coef_off) *coef_off = coef;
  if (plane_off) *plane_off = planes;
  if (raw_off) *raw_off = raw;
  return DEFER_OK;
}

int defer_k_image_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace, uint8_t* y,
                         void* stream) {
  DEFER_CHECK(files && blocks && workspace && y, "k_image_decode: null pointer");
  DEFER_CHECK(n >= 1 && n <= 65535 && H >= 1 && W >= 1 && image_bound_ok(H, W),
              "k_image_decode: bad sizes (n %d, bound %dx%d)", n, H, W);
  DEFER_CHECK(((uintptr_t)blocks & 3) == 0 && ((uintptr_t)workspace & 255) == 0,
              "k_image_decode: blocks must be 4-byte and the workspace 256-byte aligned");
  return launch_image_decode(files, blocks, n, H, W, workspace, y, (cudaStream_t)stream);
}

}  // extern "C"
