// conv_umma.cu - wgmma implicit-GEMM convolution for sm_90a (Hopper).
//
// The contraction of every Conv2D whose C_in is a multiple of 64 (all ResNet / VGG convs but the
// RGB stem).  GEMM view: M = output pixels, N = C_out, K = taps x C_in.
//
//   * A (activations, NHWC bf16 planes) is never im2col'ed in memory: TMA does it.  M tile t is the 128
//     consecutive output pixels [128 t, 128 t + 128) in (n, ho, wo) order, across rows and images.  For tap
//     (kh, kw) and a 64-channel block its A tile is one im2col load: the pixel walk starts at the input corner of
//     the tile's first output pixel and steps by the conv stride through a bounding box whose corners are the
//     padding, and each pixel is read at the tap offset (kw, kh) from its corner.  TMA zero-fills out-of-bounds
//     pixels, which IS the 'same' / ZeroPadding2D border and the rows past the batch.  1x1/stride-1 convs load
//     the flat [M, C] view with a tiled load instead.
//   * B (weights) is pre-arranged once as [tap][C_out][C_in] bf16 (K-major), a 3-D TMA box.
//   * Both land in 128B-swizzled shared memory (a ring of stages guarded by mbarriers) and feed
//     wgmma.mma_async m64nBNk16 issued by two consumer warpgroups (rows 0-63 and 64-127 of the tile);
//     the fp32 accumulator lives in their registers.
//   * BF16X2 format (fp32 parity path): activations and weights are (hi, lo) bf16 planes and each
//     K = 16 step issues hi*hi + lo*hi + hi*lo (bf16x3, ~2^-16 relative) into the same accumulator.
//   * Epilogue (the consumer warpgroups): the accumulator tile goes through a 32 KB shared-memory staging tile
//     (after the operand ring) into whole rows; per-channel scale/shift (bias + BN) -> + residual -> relu ->
//     re-split to bf16 planes -> 16-byte st.global (plain stores, so the output may be a peer GPU's input slot:
//     the hop is fused into the kernel).
//   * Split-K for weight-heavy small-M layers (7x7, 14x14 maps at batch 1): either partial tiles in an
//     fp32 workspace reduced by the last-arriving CTA, or (DEFER_UMMA_CLUSTER=1) the splits of a tile as
//     one thread-block cluster reducing through distributed shared memory.  Both sum in a fixed order.
//
// Warp roles (384 threads): warpgroups 0-1 consume (wgmma + epilogue), warpgroup 2 produces (one thread
// issues the TMA loads).  The same body runs one tile per CTA (conv_umma_kernel) or walks a tile list
// (conv_stream_kernel: persistent grid, or one cluster walking a run of ops separated by cluster barriers).
// The fused RGB stem (conv_stem_kernel and its uint8 variants) has a body of its own: all 128 producer threads
// build the A operand from an image window they stage in shared memory.
#include <cuda.h>
#include <string.h>

#include <type_traits>

#include <vector>

#include "common.cuh"
#include "conv_umma.cuh"

namespace defer {

static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

namespace {

constexpr int BM = 128;          // M tile: two wgmma m64 halves
constexpr int BK = 64;           // K elements per stage (128 B of bf16 = one swizzle atom row)
constexpr int CONS_THREADS = 256;
constexpr int NUM_THREADS = CONS_THREADS + 128;
constexpr int SMEM_CAP = 227 * 1024 - 256;   // opt-in shared memory per block on H100 (227 KB), less static smem
constexpr int CTL_BYTES = 256;         // mbarriers
constexpr int MAX_STAGES = 8;
constexpr int MEGA_BN = 64;
constexpr int STG_COLS = 64;                    // epilogue staging tile: BM rows x 64 fp32 columns (a BN = 128 tile takes two passes)
constexpr int STG_BYTES = BM * STG_COLS * 4;   // 32 KB, after the operand ring

struct KParams {
  // geometry
  int n, ho, wo, cout;
  int tile_h, tile_w, tiles_h, tiles_w;           // fused stem: M tile = tile_h x tile_w pixels of one image
  int im2col;                                     // A tile: 1 = im2col load, 0 = tiled load of the [M, C] view
  int m_total;                                    // n*ho*wo
  int kh, kw, sh, sw, pad_t, pad_l;
  int cblocks;                                    // cin / 64
  int k_blocks;                                   // taps * cblocks
  int splits;
  int cluster;                                    // 1: the `splits` CTAs of a tile form one thread-block cluster (DSMEM reduction)
  uint32_t flags;
  const float* scale;
  const float* shift;
  const void* res;
  void* y;
  float* partial;
  unsigned int* counters;
  size_t plane_out;                               // n*ho*wo*cout (elements) - offset of the lo plane
};

// One op as the kernels read it (kernel parameter or device memory).
struct alignas(128) MegaOp {
  CUtensorMap tmx[2];
  CUtensorMap tmw[2];
  KParams p;
  int m_tiles, n_tiles;     // tiles of this op: m fastest
  // fused stem: the fp32 NHWC image the patch rows are built from, the real conv geometry and the image window of one
  // M tile (stem_win_rows x stem_win_cols values, see stem_body)
  const float* stem_x;
  int stem_h, stem_w, stem_cin, stem_kh, stem_kw, stem_sh, stem_sw, stem_pad_t, stem_pad_l, stem_K;
  int stem_win_rows, stem_win_cols;
  // fused stem over a uint8 RGB image instead (conv_stem_u8_kernel): Keras caffe preprocessing on the fly,
  // value[c] = float(image[2 - c]) + stem_shift[c]; or Keras tf preprocessing (conv_stem_u8tf_kernel, stem_shift unused),
  // value[c] = float(image[c]) / 127.5 - 1
  const uint8_t* stem_u8;
  float stem_shift[3];
  // second epilogue output (conv_umma_aff_kernel / conv_stream_aff_kernel): a standalone per-channel affine(+ReLU) of
  // the stored result, y2 = [relu](fmaf(stored, scale2[c], shift2[c])).
  const float* scale2;
  const float* shift2;
  void* y2;
  int relu2;
  int store_first;           // 0: only y2 is written (nothing else reads the conv's own output)
};

template <int NPLANES, int BN>
struct Smem {
  static constexpr int A_PLANE = BM * 128;   // bytes
  static constexpr int B_PLANE = BN * 128;
  static constexpr int STAGE = NPLANES * (A_PLANE + B_PLANE);
  static constexpr int RED = BM * BN * 4;    // fp32 partial tile of the cluster split-K reduction
  __host__ __device__ static constexpr int ring(int stages, bool red) {
    return (red && stages * STAGE < RED) ? RED : stages * STAGE;
  }
  // ring | epilogue staging tile | mbarriers, + slack for the manual 1024-B alignment of the dynamic smem base
  __host__ __device__ static constexpr int total(int stages, bool red) {
    return ring(stages, red) + STG_BYTES + CTL_BYTES + 1024;
  }
  __host__ __device__ static constexpr int max_stages() {
    return (SMEM_CAP - STG_BYTES - CTL_BYTES - 1024) / STAGE > MAX_STAGES ? MAX_STAGES
                                                                          : (SMEM_CAP - STG_BYTES - CTL_BYTES - 1024) / STAGE;
  }
};
static_assert(Smem<2, 128>::max_stages() == 3 && Smem<2, 64>::max_stages() == 4, "BF16X2 ring depths");
static_assert(Smem<1, 64>::max_stages() == 8 && Smem<1, 128>::max_stages() == 6, "BF16 ring depths");

// ---------------------------------------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n.reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a protocol bug must surface as an error, never as a hung GPU.  No function call on this path (a call
// inside the main loop would make ptxas serialize every wgmma), so the timeout only records its tag before trapping.
__device__ int g_conv_wait_timeout_tag;
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int tag) {
  if (mbar_try_wait(bar, parity)) return;
  unsigned long long t0 = gtimer();
  unsigned spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0xfff) == 0 && gtimer() - t0 > 2000000000ull) {
      g_conv_wait_timeout_tag = tag;
      asm volatile("trap;");
    }
  }
}

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// im2col load: (c0, w, h, n) is the input corner of the first pixel of the walk, (ow, oh) the tap offset of every pixel
__device__ __forceinline__ void tma_load_im2col_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int w, int h,
                                                   int n, uint16_t ow, uint16_t oh) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2], {%7, %8};"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(w), "r"(h), "r"(n), "h"(ow), "h"(oh)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ---- thread-block cluster / distributed shared memory
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
// address of the same shared-memory offset in CTA `rank` of this cluster
__device__ __forceinline__ uint32_t dsmem_map(uint32_t local_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ float4 dsmem_ld4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void cons_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void prod_bar_sync() { asm volatile("bar.sync 2, 128;" ::: "memory"); }

// ---- wgmma
// SWIZZLE_128B, K-major shared-memory matrix descriptor (sm_90 GMMA): start>>4 | LBO(=16 B, unused for swizzled
// K-major)>>4 << 16 | SBO(=1024 B: one 8-row swizzle atom)>>4 << 32 | layout SWIZZLE_128B (1) << 62.  The K = 16
// slices of a 64-wide row start 32 B apart inside the swizzle atom.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from touching accumulator registers across an outstanding wgmma
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x BN] (+)= A[64 x 16] * B[BN x 16]^T, bf16 in, fp32 accumulate, both operands K-major in shared memory
template <int BN>
__device__ __forceinline__ void wgmma_bf16(float (&d)[BN / 2], uint64_t a, uint64_t b);

template <>
__device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
      "%23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(1));
}

template <>
__device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
      "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, "
      "%45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, "
      "1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(1));
}

// accumulator row r of the tile at (n0, h0, w0) -> output pixel (linear NHW index) and whether it exists.  A conv tile
// starts at pixel w0; a fused stem tile (STEM) is tile_h x tile_w pixels of image n0.
template <bool STEM>
__device__ __forceinline__ void row_to_pixel(const KParams& p, int r, int n0, int h0, int w0, bool& valid, size_t& pix) {
  if (!STEM) {
    const int m = w0 + r;
    valid = m < p.m_total;
    pix = (size_t)m;
  } else {
    const int th = r / p.tile_w;
    const int oh = h0 + th, ow = w0 + r % p.tile_w;
    valid = th < p.tile_h && oh < p.ho && ow < p.wo;
    pix = ((size_t)n0 * p.ho + oh) * p.wo + ow;
  }
}

// ---- the epilogue: per-channel scale/shift (bias + BN) -> + residual -> ReLU -> split to the bf16 planes -> st.global
// The operands it needs, read from the op once per tile.  MODE 1 / 2 read their op from device memory; a field read inside
// the store loop would be re-read after every store (a generic store may alias the op), and each residual load would wait
// for that re-read.
struct EpiArgs {
  const float* scale;
  const float* shift;
  const __nv_bfloat16* res;
  __nv_bfloat16* y;
  size_t plane;          // element offset of the lo plane (output and residual have the same shape)
  int cout;
  bool relu;
  bool store_first;      // AFF: 0 = only y2 is written
  bool relu2;
  const float* scale2;   // AFF: folded affine op
  const float* shift2;
  __nv_bfloat16* y2;
};

__device__ __forceinline__ EpiArgs epi_args(const MegaOp& op) {
  const KParams& p = op.p;
  EpiArgs e;
  e.scale = p.scale;
  e.shift = p.shift;
  e.res = reinterpret_cast<const __nv_bfloat16*>(p.res);
  e.y = reinterpret_cast<__nv_bfloat16*>(p.y);
  e.plane = p.plane_out;
  e.cout = p.cout;
  e.relu = (p.flags & DEFER_FLAG_RELU) != 0;
  e.store_first = op.store_first != 0;
  e.relu2 = op.relu2 != 0;
  e.scale2 = op.scale2;
  e.shift2 = op.shift2;
  e.y2 = reinterpret_cast<__nv_bfloat16*>(op.y2);
  return e;
}

// fp32 staging tile, 128 rows x 64 columns (256 B per row).  The 16-B chunk j of row r sits at chunk j ^ 2 (r & 7): the
// fragment writes (a half-warp writes 4 rows x 8 columns, one float2 per lane) and the row reads (a quarter-warp reads
// 8 chunks of one row, one float4 per lane) are then free of bank conflicts.
__device__ __forceinline__ uint32_t stg_off(int r, int c) {
  return (uint32_t)(r * STG_COLS + (((c >> 2) ^ ((r & 7) << 1)) << 2) + (c & 3)) * 4u;
}
__device__ __forceinline__ void sts2(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b));
}
__device__ __forceinline__ float4 lds4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
// plain st.global (no cache hint, no TMA): the output may be a peer GPU's input slot (DEFER_HOP=direct|tma)
__device__ __forceinline__ void stg4(void* p, uint4 v) {
  asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));
}

__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

// The epilogue of one output tile, staged through shared memory in passes of 64 columns.
//   phase 1: the consumers write their accumulator fragments into the staging tile;
//   phase 2: thread t owns the 8 channels 8 (t % 8) .. + 7 of rows t / 8 + 32 k (k = 0..3).  It issues all of its residual
//   loads (16 B per plane per row) before the barrier and uses them after it, and stores 16 B per plane per row, so a warp
//   writes four whole 128-B row segments per plane.
// Per element the arithmetic and its order are those of the conv's definition: fmaf(acc, scale, shift), + res_hi, + res_lo,
// ReLU, split.  AFF then applies the folded affine op to the value as stored - hi + lo (BF16X2) or the bf16 (BF16), exactly
// what eltwise_kernel<FMT, DEFER_OP_AFFINE> reads back - with the same fmaf, ReLU and split, into y2.  The folded result is
// therefore bit-identical to the conv followed by the standalone affine op.
// qmask: the 8-column groups q (acc[4q .. 4q + 3]) this CTA stores (cluster split-K: those it reduced; otherwise all).
template <int NPLANES, int BN, bool AFF, bool STEM = false>
__device__ __forceinline__ void epi_tile(const KParams& p, const EpiArgs& e, uint32_t stg, const float (&acc)[BN / 2],
                                         uint32_t qmask, int c_base, int n0, int h0, int w0) {
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int row0 = (tid >> 7) * 64 + ((tid >> 5) & 3) * 16 + (lane >> 2);   // fragment rows row0, row0 + 8
  const int col_l = 2 * (lane & 3);
  const int jg = tid & 7;                                                   // phase-2 channel group
  const int rb = tid >> 3;                                                  // phase-2 rows rb + 32 k
  // the two chunks of a channel group, read in the order that spreads a quarter-warp over all 32 banks
  const int ca = 2 * jg + ((jg >> 2) & 1), cb = ca ^ 1;
  const bool swap = (jg >> 2) & 1;
  size_t orow[4];
  uint32_t vmask = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    bool v;
    size_t pix;
    row_to_pixel<STEM>(p, rb + 32 * k, n0, h0, w0, v, pix);
    orow[k] = pix * (size_t)e.cout;
    vmask |= (uint32_t)v << k;
  }
#pragma unroll
  for (int P = 0; P < BN / STG_COLS; ++P) {
    const bool mine = (qmask >> (8 * P + jg)) & 1u;
    const int c = c_base + STG_COLS * P + 8 * jg;
    cons_bar_sync();   // every consumer is done reading the staging tile (previous pass or previous tile)
#pragma unroll
    for (int qq = 0; qq < 8; ++qq) {
      const int q = 8 * P + qq;
      if (!((qmask >> q) & 1u)) continue;
      sts2(stg + stg_off(row0, 8 * qq + col_l), acc[4 * q], acc[4 * q + 1]);
      sts2(stg + stg_off(row0 + 8, 8 * qq + col_l), acc[4 * q + 2], acc[4 * q + 3]);
    }
    // the residual and the per-channel operands: all loads of the pass are in flight across the barrier, before any is
    // used (issued after the fragment writes, whose registers are free by then)
    uint4 rh[4], rl[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      rh[k] = rl[k] = make_uint4(0u, 0u, 0u, 0u);
      if (e.res && mine && ((vmask >> k) & 1u)) {
        rh[k] = __ldcg(reinterpret_cast<const uint4*>(e.res + orow[k] + c));
        if (NPLANES == 2) rl[k] = __ldcg(reinterpret_cast<const uint4*>(e.res + e.plane + orow[k] + c));
      }
    }
    float sc[8], sf[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { sc[i] = 1.f; sf[i] = 0.f; }
    if (mine) {
      if (e.scale) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(e.scale + c));
        const float4 b = __ldg(reinterpret_cast<const float4*>(e.scale + c + 4));
        sc[0] = a.x; sc[1] = a.y; sc[2] = a.z; sc[3] = a.w; sc[4] = b.x; sc[5] = b.y; sc[6] = b.z; sc[7] = b.w;
      }
      if (e.shift) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(e.shift + c));
        const float4 b = __ldg(reinterpret_cast<const float4*>(e.shift + c + 4));
        sf[0] = a.x; sf[1] = a.y; sf[2] = a.z; sf[3] = a.w; sf[4] = b.x; sf[5] = b.y; sf[6] = b.z; sf[7] = b.w;
      }
    }
    cons_bar_sync();
    if (!mine) continue;

#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (!((vmask >> k) & 1u)) continue;
      const int r = rb + 32 * k;
      const float4 xa = lds4(stg + stg_off(r, 4 * ca));
      const float4 xb = lds4(stg + stg_off(r, 4 * cb));
      const float4 x0 = swap ? xb : xa, x1 = swap ? xa : xb;
      float v[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
      const uint32_t hw[4] = {rh[k].x, rh[k].y, rh[k].z, rh[k].w};
      const uint32_t lw[4] = {rl[k].x, rl[k].y, rl[k].z, rl[k].w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        v[i] = fmaf(v[i], sc[i], sf[i]);
        if (e.res) {
          v[i] += (i & 1) ? bf_hi(hw[i >> 1]) : bf_lo(hw[i >> 1]);
          if (NPLANES == 2) v[i] += (i & 1) ? bf_hi(lw[i >> 1]) : bf_lo(lw[i >> 1]);
        }
        if (e.relu) v[i] = fmaxf(v[i], 0.f);
      }
      uint4 hi, lo = make_uint4(0u, 0u, 0u, 0u);
      if (NPLANES == 2) {
        split_bf16x2(v[0], v[1], hi.x, lo.x);
        split_bf16x2(v[2], v[3], hi.y, lo.y);
        split_bf16x2(v[4], v[5], hi.z, lo.z);
        split_bf16x2(v[6], v[7], hi.w, lo.w);
      } else {
        hi = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
      }
      const size_t o = orow[k] + c;
      if (!AFF || e.store_first) {
        stg4(e.y + o, hi);
        if (NPLANES == 2) stg4(e.y + e.plane + o, lo);
      }
      if constexpr (AFF) {
        float s2[8], t2[8];
        {
          const float4 a = __ldg(reinterpret_cast<const float4*>(e.scale2 + c));
          const float4 b = __ldg(reinterpret_cast<const float4*>(e.scale2 + c + 4));
          const float4 d = __ldg(reinterpret_cast<const float4*>(e.shift2 + c));
          const float4 f = __ldg(reinterpret_cast<const float4*>(e.shift2 + c + 4));
          s2[0] = a.x; s2[1] = a.y; s2[2] = a.z; s2[3] = a.w; s2[4] = b.x; s2[5] = b.y; s2[6] = b.z; s2[7] = b.w;
          t2[0] = d.x; t2[1] = d.y; t2[2] = d.z; t2[3] = d.w; t2[4] = f.x; t2[5] = f.y; t2[6] = f.z; t2[7] = f.w;
        }
        const uint32_t sh[4] = {hi.x, hi.y, hi.z, hi.w};
        const uint32_t sl[4] = {lo.x, lo.y, lo.z, lo.w};
        float u[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          u[i] = (i & 1) ? bf_hi(sh[i >> 1]) : bf_lo(sh[i >> 1]);
          if (NPLANES == 2) u[i] = u[i] + ((i & 1) ? bf_hi(sl[i >> 1]) : bf_lo(sl[i >> 1]));
          u[i] = fmaf(u[i], s2[i], t2[i]);
          if (e.relu2) u[i] = fmaxf(u[i], 0.f);
        }
        uint4 h2, l2;
        if (NPLANES == 2) {
          split_bf16x2(u[0], u[1], h2.x, l2.x);
          split_bf16x2(u[2], u[3], h2.y, l2.y);
          split_bf16x2(u[4], u[5], h2.z, l2.z);
          split_bf16x2(u[6], u[7], h2.w, l2.w);
          stg4(e.y2 + o, h2);
          stg4(e.y2 + e.plane + o, l2);
        } else {
          h2 = make_uint4(pack_bf16x2(u[0], u[1]), pack_bf16x2(u[2], u[3]), pack_bf16x2(u[4], u[5]), pack_bf16x2(u[6], u[7]));
          stg4(e.y2 + o, h2);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- the kernel body
// MODE 0: one (tile, split) per CTA: tile = (blockIdx.x, blockIdx.y), split = blockIdx.z (grid split-K or cluster split-K)
// MODE 1: persistent grid: CTA b walks tiles b, b + gridDim.x, ... of one op
// MODE 2: one cluster walks a run of ops; tiles are dealt round-robin to its CTAs, a cluster barrier separates ops
template <int NPLANES, int BN, int MODE, bool AFF = false>
__device__ __forceinline__ void conv_body(const MegaOp* ops, int n_ops, int stages, int pdl) {
  using L = Smem<NPLANES, BN>;
  constexpr int R = BN / 2;   // accumulator registers per consumer thread
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t ring = smem_u32(smem);
  const bool red = MODE == 0 && ops[0].p.cluster;
  const uint32_t stg = ring + L::ring(stages, red);   // epilogue staging tile, outside the ring
  const uint32_t bar_base = stg + STG_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (stages + s); };
  __shared__ int s_is_last;

  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), CONS_THREADS / 32);   // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (pdl) {
    // programmatic dependent launch: the set-up above overlapped the previous kernel of this lane; its outputs are
    // visible only after this wait.  Our own dependents may start their prologue right away.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  }

  uint32_t it = 0;   // k-blocks through the ring so far (same sequence in every role)
  for (int o = 0; o < n_ops; ++o) {
    const MegaOp& op = ops[o];
    const KParams& p = op.p;
    const int total = op.m_tiles * op.n_tiles;
    int t_first, t_step;
    if (MODE == 0) {
      t_first = blockIdx.y * op.m_tiles + blockIdx.x;
      t_step = total;
    } else if (MODE == 1) {
      t_first = blockIdx.x;
      t_step = gridDim.x;
    } else {
      t_first = (int)cluster_ctarank();
      t_step = (int)cluster_nctarank();
    }
    const int split = MODE == 0 ? (int)blockIdx.z : 0;
    const int kb_begin = (split * p.k_blocks) / p.splits;   // balanced ranges; host guarantees k_blocks >= splits
    const int kb_end = ((split + 1) * p.k_blocks) / p.splits;

    for (int t = t_first; t < total; t += t_step) {
      const int m0 = (t % op.m_tiles) * BM;   // first output pixel of the tile
      const int c_base = (t / op.m_tiles) * BN;

      if (tid >= CONS_THREADS) {
        // =================================================================== producer
        if (tid == CONS_THREADS) {
          // im2col: input corner of pixel m0 = (n, oh, ow), the start of the tile's pixel walk
          const int ow = m0 % p.wo;
          const int oh = (m0 / p.wo) % p.ho;
          const int cw = ow * p.sw - p.pad_l, ch = oh * p.sh - p.pad_t, cn = m0 / (p.wo * p.ho);
          uint32_t i2 = it;
          for (int kb = kb_begin; kb < kb_end; ++kb, ++i2) {
            const int stage = (int)(i2 % (uint32_t)stages);
            const uint32_t phase = (i2 / (uint32_t)stages) & 1u;
            mbar_wait(empty_bar(stage), phase ^ 1u, 1);
            const uint32_t a_dst = ring + stage * L::STAGE;
            const uint32_t b_dst = a_dst + NPLANES * L::A_PLANE;
            const int tap = kb / p.cblocks;
            const int cb = kb - tap * p.cblocks;
            const uint16_t khi = (uint16_t)(tap / p.kw);
            const uint16_t kwi = (uint16_t)(tap - khi * p.kw);
            // every A load fills all 128 rows (zeros past the batch), so the byte count is the same for every tile
            mbar_arrive_expect_tx(full_bar(stage), NPLANES * (uint32_t)(L::A_PLANE + L::B_PLANE));
#pragma unroll
            for (int pl = 0; pl < NPLANES; ++pl) {
              if (p.im2col)
                tma_load_im2col_4d(a_dst + pl * L::A_PLANE, &op.tmx[pl], full_bar(stage), cb * BK, cw, ch, cn, kwi, khi);
              else
                tma_load_4d(a_dst + pl * L::A_PLANE, &op.tmx[pl], full_bar(stage), cb * BK, m0, 0, 0);
              tma_load_3d(b_dst + pl * L::B_PLANE, &op.tmw[pl], full_bar(stage), cb * BK, c_base, tap);
            }
          }
        }
        it += (uint32_t)(kb_end - kb_begin);
        continue;
      }

      // ===================================================================== consumers: main loop
      const int wg = tid >> 7;
      const int lane = tid & 31;
      float acc[R];
#pragma unroll
      for (int i = 0; i < R; ++i) acc[i] = 0.f;
      int prev_stage = -1;
      for (int kb = kb_begin; kb < kb_end; ++kb, ++it) {
        const int stage = (int)(it % (uint32_t)stages);
        mbar_wait(full_bar(stage), (it / (uint32_t)stages) & 1u, 2);
        const uint32_t a_addr = ring + stage * L::STAGE + wg * (64 * 128);
        const uint32_t b_addr = ring + stage * L::STAGE + NPLANES * L::A_PLANE;
        wg_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t a_hi = make_sw128_desc(a_addr + k * 32);
          const uint64_t b_hi = make_sw128_desc(b_addr + k * 32);
          wgmma_bf16<BN>(acc, a_hi, b_hi);
          if (NPLANES == 2) {
            wgmma_bf16<BN>(acc, make_sw128_desc(a_addr + L::A_PLANE + k * 32), b_hi);
            wgmma_bf16<BN>(acc, a_hi, make_sw128_desc(b_addr + L::B_PLANE + k * 32));
          }
        }
        wg_commit();
        wg_wait<1>();   // the previous k-block's wgmmas are done: its stage may be refilled
        acc_fence(acc);
        if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar(prev_stage));
        prev_stage = stage;
      }
      wg_wait<0>();
      acc_fence(acc);
      if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar(prev_stage));

      // ===================================================================== consumers: epilogue
      // wgmma m64nN accumulator layout: register i of thread (warp w, lane l) of warpgroup g holds row
      // 64g + 16w + l/4 + 8*((i/2)&1), column 8*(i/4) + 2*(l%4) + (i&1)

      if (MODE == 0 && p.cluster) {
        // ---- cluster split-K: the S CTAs of the cluster hold the S partial tiles of ONE output tile.  Each parks its
        // partial in its own shared memory; after a cluster barrier CTA j reduces the column groups q = j, j + S, ...
        // in rank order (deterministic) straight out of its peers' shared memory (DSMEM) and runs their epilogue.
        cons_bar_sync();   // both warpgroups are done reading the ring
        float4* red_buf = reinterpret_cast<float4*>(smem);
#pragma unroll
        for (int q = 0; q < R / 4; ++q)
          red_buf[q * CONS_THREADS + tid] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
        break;   // to the cluster reduction below (MODE 0 has exactly one tile)
      }
      if (MODE == 0 && p.splits > 1) {
        // ---- grid split-K: publish the raw partial tile; the last CTA of this (tile, n-block) reduces them
        const size_t tile_lin = (size_t)t;
        float4* mine = reinterpret_cast<float4*>(p.partial) + (tile_lin * p.splits + split) * (R / 4) * CONS_THREADS;
#pragma unroll
        for (int q = 0; q < R / 4; ++q)
          __stcg(mine + q * CONS_THREADS + tid, make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]));
        __threadfence();
        cons_bar_sync();
        if (tid == 0) {
          const unsigned prev = atomicAdd(p.counters + tile_lin, 1u);
          const int last = prev == (unsigned)(p.splits - 1);
          if (last) p.counters[tile_lin] = 0;   // re-arm for the next launch
          s_is_last = last;
        }
        cons_bar_sync();
        if (!s_is_last) continue;
        __threadfence();
#pragma unroll
        for (int i = 0; i < R; ++i) acc[i] = 0.f;
        for (int s = 0; s < p.splits; ++s) {
          const float4* src = reinterpret_cast<const float4*>(p.partial) + (tile_lin * p.splits + s) * (R / 4) * CONS_THREADS;
#pragma unroll
          for (int q = 0; q < R / 4; ++q) {
            const float4 v = __ldcg(src + q * CONS_THREADS + tid);
            acc[4 * q] += v.x; acc[4 * q + 1] += v.y; acc[4 * q + 2] += v.z; acc[4 * q + 3] += v.w;
          }
        }
      }
      epi_tile<NPLANES, BN, AFF>(p, epi_args(op), stg, acc, 0xffffu, c_base, 0, 0, m0);
    }

    if (MODE == 0 && p.cluster) {
      cluster_sync_all();
      if (tid < CONS_THREADS) {
        // this CTA reduces and stores the column groups q = rank, rank + S, ...; the partials it reads over DSMEM sit at
        // the start of each peer's ring, the staging tile after it, so peers may still be reading while this CTA stages
        const int S = p.splits;
        const int rank = (int)cluster_ctarank();
        const uint32_t mine = ring + (uint32_t)tid * 16u;
        float acc[R];
        uint32_t qmask = 0;
#pragma unroll
        for (int q = 0; q < R / 4; ++q) {
          acc[4 * q] = acc[4 * q + 1] = acc[4 * q + 2] = acc[4 * q + 3] = 0.f;
          if (q % S != rank) continue;
          qmask |= 1u << q;
          const uint32_t addr = mine + (uint32_t)(q * CONS_THREADS) * 16u;
          float4 a = dsmem_ld4(dsmem_map(addr, 0));
          for (int s = 1; s < S; ++s) {
            const float4 v = dsmem_ld4(dsmem_map(addr, (uint32_t)s));
            a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
          }
          acc[4 * q] = a.x; acc[4 * q + 1] = a.y; acc[4 * q + 2] = a.z; acc[4 * q + 3] = a.w;
        }
        epi_tile<NPLANES, BN, AFF>(p, epi_args(op), stg, acc, qmask, (int)blockIdx.y * BN, 0, 0, (int)blockIdx.x * BM);
      }
      cluster_sync_all();   // no CTA may leave (and free its shared memory) while a peer still reads it
    }
    if (MODE == 2 && o + 1 < n_ops) {
      // the next op reads this op's output through TMA (async proxy): order the generic-proxy stores before it
      asm volatile("fence.proxy.async.global;" ::: "memory");
      cluster_sync_all();
    }
  }
}

template <int NPLANES, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_umma_kernel(const __grid_constant__ MegaOp op, int stages, int pdl) {
  conv_body<NPLANES, BN, 0>(&op, 1, stages, pdl);
}

template <int NPLANES, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_stream_kernel(const MegaOp* __restrict__ ops, int stages, int pdl) {
  conv_body<NPLANES, BN, 1>(ops, 1, stages, pdl);
}

// the same two executors with a folded affine op as a second epilogue output (MegaOp::y2)
template <int NPLANES, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_umma_aff_kernel(const __grid_constant__ MegaOp op, int stages, int pdl) {
  conv_body<NPLANES, BN, 0, true>(&op, 1, stages, pdl);
}

template <int NPLANES, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_stream_aff_kernel(const MegaOp* __restrict__ ops, int stages, int pdl) {
  conv_body<NPLANES, BN, 1, true>(ops, 1, stages, pdl);
}

template <int NPLANES>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_mega_kernel(const MegaOp* __restrict__ ops, int n_ops, int stages) {
  conv_body<NPLANES, MEGA_BN, 2>(ops, n_ops, stages, 0);
}

// ---------------------------------------------------------------------------------------------- the fused RGB stem
// conv_stem_kernel, conv_stem_u8_kernel, conv_stem_u8tf_kernel: a persistent grid over the tiles of a conv whose input has
// a few channels (K = kh * kw * cin <= 256, zero-padded to whole k-blocks; C_out = 64), with no patch matrix in memory.
// The M tile is tile_h x tile_w output pixels of one image, so its input footprint is a window of
//   stem_win_rows = (tile_h - 1) * sh + kh rows  x  stem_win_cols = ((tile_w - 1) * sw + kw) * cin values.
// For each tile the producer warpgroup fills that window in shared memory with the conv input's fp32 values: the fp32 image
// itself, or the uint8 image preprocessed (Keras caffe: channel c <- float(image[2 - c]) + stem_shift[c]; Keras tf:
// keras_tf_preprocess(float(image[c])) - bit for bit what preprocess_kernel / preprocess_tf_kernel write), and zeros
// outside the image, since the padding belongs to the preprocessed tensor.  Consecutive threads load consecutive values of
// a window row, and every load of a window is issued before any is converted.  The window is double-buffered: the loads of
// the next tile are in flight while the k-blocks of this one are built.
// The builder writes patch row r (pixel th = r / tile_w, tw = r % tile_w of the tile) of k-block kb in the SWIZZLE_128B
// layout TMA would have produced: k = a * kw * cin + jj is window value (th * sh + a) * stem_win_cols + tw * sw * cin + jj
// for k < K, and 0 beyond.  Same values, same split and same K order as the patch matrix of stem_im2col_kernel, so the
// fused stem and the im2col path agree bitwise.
enum StemIn { STEM_F32, STEM_U8_CAFFE, STEM_U8_TF };
constexpr int PROD_THREADS = NUM_THREADS - CONS_THREADS;
constexpr int STEM_WIN_BYTES = 24 * 1024;                         // one window buffer; two are resident
constexpr int STEM_WIN_VALS = STEM_WIN_BYTES / 4;
constexpr int STEM_FILL = STEM_WIN_VALS / PROD_THREADS;           // window values per producer thread, held in registers
constexpr int STEM_TILE_W = 16;                                   // 8 x 16 output pixels per M tile (fewer columns on a narrow map)

template <int NPLANES>
struct StemSmem {
  static constexpr int STAGE = Smem<NPLANES, 64>::STAGE;
  // ring | epilogue staging tile | two window buffers | mbarriers, + slack for the 1024-B alignment of the base
  __host__ __device__ static constexpr int total(int stages) {
    return stages * STAGE + STG_BYTES + 2 * STEM_WIN_BYTES + CTL_BYTES + 1024;
  }
  __host__ __device__ static constexpr int max_stages() {
    return (SMEM_CAP - STG_BYTES - 2 * STEM_WIN_BYTES - CTL_BYTES - 1024) / STAGE > MAX_STAGES
               ? MAX_STAGES
               : (SMEM_CAP - STG_BYTES - 2 * STEM_WIN_BYTES - CTL_BYTES - 1024) / STAGE;
  }
};
// BF16X2: 3 stages of 48 KB hold the whole K loop of a tile (K <= 256: at most 4 k-blocks) next to the two windows
static_assert(StemSmem<2>::max_stages() == 3 && StemSmem<1>::max_stages() == 6, "stem ring depths with two image windows");
static_assert(STEM_FILL * PROD_THREADS == STEM_WIN_VALS, "the producer threads cover a whole window");

// the stem's operands, read from the op once per kernel (a field read after a shared-memory store would be re-read)
struct StemGeo {
  const float* x;
  const uint8_t* u8;
  float s0, s1, s2;
  int H, rowlen;        // image rows, values per image row (w * cin)
  int cin, sh, sw, pad_t, pad_l;
  int wcols, nwin;      // window: values per row, values in all
  int run, K;           // kw * cin, kh * kw * cin
};

__device__ __forceinline__ StemGeo stem_geo(const MegaOp& op) {
  StemGeo g;
  g.x = op.stem_x;
  g.u8 = op.stem_u8;
  g.s0 = op.stem_shift[0]; g.s1 = op.stem_shift[1]; g.s2 = op.stem_shift[2];
  g.H = op.stem_h;
  g.rowlen = op.stem_w * op.stem_cin;
  g.cin = op.stem_cin; g.sh = op.stem_sh; g.sw = op.stem_sw; g.pad_t = op.stem_pad_t; g.pad_l = op.stem_pad_l;
  g.wcols = op.stem_win_cols;
  g.nwin = op.stem_win_rows * op.stem_win_cols;
  g.run = op.stem_kw * op.stem_cin;
  g.K = op.stem_K;
  return g;
}

// output pixel of row 0 of stem tile m_tile (a stem tile never spans two images)
__device__ __forceinline__ void stem_tile_origin(const KParams& p, int m_tile, int& n0, int& h0, int& w0) {
  const int t2 = m_tile / p.tiles_w;
  n0 = t2 / p.tiles_h;
  h0 = (t2 - n0 * p.tiles_h) * p.tile_h;
  w0 = (m_tile - t2 * p.tiles_w) * p.tile_w;
}

// This thread's values of the window of the tile at (n0, h0, w0): value e = ptid + 128 j (row e / wcols, column e % wcols).
// Out-of-image values are marked: 0 (fp32: +0.f) or 0x100 (uint8).
template <int IN>
__device__ __forceinline__ void stem_fill_load(const StemGeo& g, int ptid, int n0, int h0, int w0, uint32_t (&raw)[STEM_FILL]) {
  const int ih0 = h0 * g.sh - g.pad_t, col0 = (w0 * g.sw - g.pad_l) * g.cin;
  const size_t img = (size_t)n0 * g.H * g.rowlen;
  const int dq = PROD_THREADS / g.wcols, dm = PROD_THREADS - dq * g.wcols;
  int wr = ptid / g.wcols, wc = ptid - wr * g.wcols;
  int c = wc % 3;   // uint8 images: channel of the value (a window row is whole 3-channel pixels)
#pragma unroll
  for (int j = 0; j < STEM_FILL; ++j) {
    const int ih = ih0 + wr, col = col0 + wc;
    const bool in = ptid + PROD_THREADS * j < g.nwin && ih >= 0 && ih < g.H && col >= 0 && col < g.rowlen;
    const size_t off = img + (size_t)(ih * g.rowlen + col);
    if constexpr (IN == STEM_F32) raw[j] = in ? __float_as_uint(__ldg(g.x + off)) : 0u;
    else raw[j] = in ? (uint32_t)__ldg(g.u8 + off + (IN == STEM_U8_CAFFE ? 2 - 2 * c : 0)) : 0x100u;
    wr += dq;
    wc += dm;
    if (wc >= g.wcols) { wc -= g.wcols; ++wr; }
    c = c == 0 ? 2 : c - 1;   // (c + 128) % 3
  }
}

// ... converted to the conv input's values and stored at window[e].  float(byte) is exact via the 2^23 magic number; then
// the one rounded add (caffe) or keras_tf_preprocess (tf).
template <int IN>
__device__ __forceinline__ void stem_fill_store(const StemGeo& g, uint32_t win, int ptid, const uint32_t (&raw)[STEM_FILL]) {
  int c = (ptid % g.wcols) % 3;
#pragma unroll
  for (int j = 0; j < STEM_FILL; ++j) {
    const int e = ptid + PROD_THREADS * j;
    if (e < g.nwin) {
      const float b = __fsub_rn(__uint_as_float(0x4B000000u | raw[j]), 8388608.f);
      float v;
      if constexpr (IN == STEM_F32) v = __uint_as_float(raw[j]);
      else if constexpr (IN == STEM_U8_CAFFE) v = raw[j] > 255u ? 0.f : __fadd_rn(b, c == 0 ? g.s0 : (c == 1 ? g.s1 : g.s2));
      else v = raw[j] > 255u ? 0.f : keras_tf_preprocess(b);
      asm volatile("st.shared.f32 [%0], %1;" ::"r"(win + 4u * (uint32_t)e), "f"(v) : "memory");
    }
    c = c == 0 ? 2 : c - 1;
  }
}

// patch row r of k-block kb (128 rows x 64 k, bf16 hi / lo planes) from the window; row_base = th * sh * wcols + tw * sw * cin
template <int NPLANES>
__device__ __forceinline__ void stem_build(const StemGeo& g, uint32_t win, uint32_t a_dst, int r, int row_base, int kb) {
  int k = kb * BK;
  int a = k / g.run, jj = k - a * g.run;
  uint32_t src = win + 4u * (uint32_t)(row_base + a * g.wcols + jj);
  const uint32_t wrap = 4u * (uint32_t)(g.wcols - g.run);   // end of a kernel row's run -> start of the next one
#pragma unroll 1
  for (int ch = 0; ch < 8; ++ch) {
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      v[e] = 0.f;
      if (k < g.K) asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v[e]) : "r"(src));
      ++k;
      src += 4u;
      if (++jj == g.run) { jj = 0; src += wrap; }
    }
    const uint32_t off = (uint32_t)r * 128u + ((uint32_t)(ch ^ (r & 7)) << 4);
    uint32_t h[4], l[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (NPLANES == 2) split_bf16x2(v[2 * q], v[2 * q + 1], h[q], l[q]);
      else h[q] = pack_bf16x2(v[2 * q], v[2 * q + 1]);
    }
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a_dst + off), "r"(h[0]), "r"(h[1]), "r"(h[2]), "r"(h[3])
                 : "memory");
    if (NPLANES == 2)
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a_dst + Smem<NPLANES, 64>::A_PLANE + off), "r"(l[0]),
                   "r"(l[1]), "r"(l[2]), "r"(l[3])
                   : "memory");
  }
}

template <int NPLANES, int IN>
__device__ __forceinline__ void stem_body(const MegaOp* ops, int stages, int pdl) {
  using L = Smem<NPLANES, 64>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t ring = smem_u32(smem);
  const uint32_t stg = ring + stages * L::STAGE;
  const uint32_t win0 = stg + STG_BYTES;
  const uint32_t bar_base = win0 + 2 * STEM_WIN_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (stages + s); };

  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), CONS_THREADS / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (pdl) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  }

  const MegaOp& op = ops[0];
  const KParams& p = op.p;
  const int total = op.m_tiles * op.n_tiles;
  const int k_blocks = p.k_blocks;
  uint32_t it = 0;   // k-blocks through the ring so far (same sequence in both roles)

  if (tid >= CONS_THREADS) {
    // =================================================================== producer: window fill + patch rows
    const int ptid = tid - CONS_THREADS;
    const StemGeo g = stem_geo(op);
    // rows past tile_h x tile_w (a map narrower than the tile) build pixel (0, 0): the epilogue stores no such row
    int th = ptid / p.tile_w, tw = ptid - th * p.tile_w;
    if (th >= p.tile_h) th = tw = 0;
    const int row_base = th * g.sh * g.wcols + tw * g.sw * g.cin;
    uint32_t raw[STEM_FILL];
    int n0, h0, w0;
    if ((int)blockIdx.x < total) {
      stem_tile_origin(p, (int)blockIdx.x % op.m_tiles, n0, h0, w0);
      stem_fill_load<IN>(g, ptid, n0, h0, w0, raw);
      stem_fill_store<IN>(g, win0, ptid, raw);
    }
    int wb = 0;
    for (int t = blockIdx.x; t < total; t += gridDim.x, wb ^= 1) {
      const int t_next = t + (int)gridDim.x;
      if (t_next < total) {   // the next tile's window: in flight while this tile is built
        stem_tile_origin(p, t_next % op.m_tiles, n0, h0, w0);
        stem_fill_load<IN>(g, ptid, n0, h0, w0, raw);
      }
      prod_bar_sync();   // window wb is complete
      const uint32_t win = win0 + (uint32_t)wb * STEM_WIN_BYTES;
      const int c_base = (t / op.m_tiles) * 64;
      for (int kb = 0; kb < k_blocks; ++kb, ++it) {
        const int stage = (int)(it % (uint32_t)stages);
        mbar_wait(empty_bar(stage), ((it / (uint32_t)stages) & 1u) ^ 1u, 1);
        const uint32_t a_dst = ring + stage * L::STAGE;
        const uint32_t b_dst = a_dst + NPLANES * L::A_PLANE;
        if (ptid == 0) {
          mbar_expect_tx(full_bar(stage), NPLANES * (uint32_t)L::B_PLANE);
          tma_load_3d(b_dst, &op.tmw[0], full_bar(stage), kb * BK, c_base, 0);
          if (NPLANES == 2) tma_load_3d(b_dst + L::B_PLANE, &op.tmw[1], full_bar(stage), kb * BK, c_base, 0);
        }
        stem_build<NPLANES>(g, win, a_dst, ptid, row_base, kb);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> wgmma reads
        prod_bar_sync();   // also: every producer is done reading window wb ^ 1 (built by the previous tile)
        if (ptid == 0) mbar_arrive(full_bar(stage));
      }
      if (t_next < total) stem_fill_store<IN>(g, win0 + (uint32_t)(wb ^ 1) * STEM_WIN_BYTES, ptid, raw);
    }
    return;
  }

  // ===================================================================== consumers
  const int wg = tid >> 7;
  const int lane = tid & 31;
  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    int prev_stage = -1;
    for (int kb = 0; kb < k_blocks; ++kb, ++it) {
      const int stage = (int)(it % (uint32_t)stages);
      mbar_wait(full_bar(stage), (it / (uint32_t)stages) & 1u, 2);
      const uint32_t a_addr = ring + stage * L::STAGE + wg * (64 * 128);
      const uint32_t b_addr = ring + stage * L::STAGE + NPLANES * L::A_PLANE;
      wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t a_hi = make_sw128_desc(a_addr + k * 32);
        const uint64_t b_hi = make_sw128_desc(b_addr + k * 32);
        wgmma_bf16<64>(acc, a_hi, b_hi);
        if (NPLANES == 2) {
          wgmma_bf16<64>(acc, make_sw128_desc(a_addr + L::A_PLANE + k * 32), b_hi);
          wgmma_bf16<64>(acc, a_hi, make_sw128_desc(b_addr + L::B_PLANE + k * 32));
        }
      }
      wg_commit();
      wg_wait<1>();   // the previous k-block's wgmmas are done: its stage may be refilled
      acc_fence(acc);
      if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar(prev_stage));
      prev_stage = stage;
    }
    wg_wait<0>();
    acc_fence(acc);
    if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar(prev_stage));
    int n0, h0, w0;
    stem_tile_origin(p, t % op.m_tiles, n0, h0, w0);
    epi_tile<NPLANES, 64, false, true>(p, epi_args(op), stg, acc, 0xffffu, (t / op.m_tiles) * 64, n0, h0, w0);
  }
}

template <int NPLANES>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_stem_kernel(const MegaOp* __restrict__ ops, int stages, int pdl) {
  stem_body<NPLANES, STEM_F32>(ops, stages, pdl);
}

// the fused stem reading a uint8 RGB image: Keras caffe preprocessing applied as the window is filled
template <int NPLANES>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_stem_u8_kernel(const MegaOp* __restrict__ ops, int stages, int pdl) {
  stem_body<NPLANES, STEM_U8_CAFFE>(ops, stages, pdl);
}

// ... preprocessing it in Keras tf mode instead
template <int NPLANES>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_stem_u8tf_kernel(const MegaOp* __restrict__ ops, int stages, int pdl) {
  stem_body<NPLANES, STEM_U8_TF>(ops, stages, pdl);
}

// weights: fp32 HWIO [tap][cin][cout]  ->  bf16 [plane][tap][cout][cin]
__global__ void __launch_bounds__(256) weight_transform_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out,
                                                               int taps, int cin, int cout, int nplanes) {
  size_t total = (size_t)taps * cin * cout;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;   // index in the OUTPUT layout (coalesced writes)
  if (i >= total) return;
  int ci = (int)(i % cin);
  size_t t2 = i / cin;
  int co = (int)(t2 % cout);
  int tap = (int)(t2 / cout);
  float v = w[((size_t)tap * cin + ci) * cout + co];
  __nv_bfloat16 hi = __float2bfloat16_rn(v);
  out[i] = hi;
  if (nplanes == 2) out[total + i] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// ---------------------------------------------------------------------------------------------- host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

int encode_map(CUtensorMap* map, void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
               const uint32_t* box, const uint32_t* estr) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return DEFER_ERR_CUDA;
  }
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, base, (const cuuint64_t*)dims,
                   (const cuuint64_t*)strides_bytes, (const cuuint32_t*)box, (const cuuint32_t*)estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d): rank %d dims [%llu,%llu,%llu,%llu] box [%u,%u,%u,%u]", (int)r,
              rank, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)(rank > 2 ? dims[2] : 0),
              (unsigned long long)(rank > 3 ? dims[3] : 0), box[0], box[1], rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
    return DEFER_ERR_CUDA;
  }
  return DEFER_OK;
}

typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                     CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                     CUtensorMapFloatOOBfill);

PFN_encodeIm2col get_encode_im2col() {
  static PFN_encodeIm2col fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeIm2col)p;
  }
  return fn;
}

// The im2col bounding box of a conv over an h x w input, in (W, H) order.  The pixel walk of a tile visits the input
// corners (ow * sw - pad_l, oh * sh - pad_t) of its output pixels in (n, oh, ow) order: in a row it steps by the stride up
// to the corner of the last output column, then goes on at the lower corner of the next row (and of the next image after
// the last row).  So the box runs from (-pad_l, -pad_t) to the corner of the last output pixel; TMA takes its lower
// corner as an offset from input pixel (0, 0) and its upper corner as an offset from pixel (w - 1, h - 1).
void im2col_corners(int h, int w, int ho, int wo, int sh, int sw, int pad_t, int pad_l, int lower[2], int upper[2]) {
  lower[0] = -pad_l;
  lower[1] = -pad_t;
  upper[0] = (wo - 1) * sw - pad_l - (w - 1);
  upper[1] = (ho - 1) * sh - pad_t - (h - 1);
}

// a rank-4 im2col tensor map holds each corner in [-128, 127] (the tap offsets of kernels up to 7 x 7 are far inside
// what the load instruction takes)
bool im2col_corners_encodable(const int lower[2], const int upper[2]) {
  for (int i = 0; i < 2; ++i)
    if (lower[i] < -128 || lower[i] > 127 || upper[i] < -128 || upper[i] > 127) return false;
  return true;
}

// A operand of a non-flat conv: the NHWC plane at `base` as (C, W, H, N), walked 128 pixels x 64 channels per load
int encode_im2col_map(CUtensorMap* map, void* base, const UmmaConvPlan& P) {
  PFN_encodeIm2col enc = get_encode_im2col();
  if (!enc) {
    set_error("cuTensorMapEncodeIm2col entry point not available");
    return DEFER_ERR_CUDA;
  }
  const uint64_t dims[4] = {(uint64_t)P.cin, (uint64_t)P.w, (uint64_t)P.h, (uint64_t)P.n};
  const uint64_t strides[3] = {(uint64_t)P.cin * 2, (uint64_t)P.w * P.cin * 2, (uint64_t)P.h * P.w * P.cin * 2};
  const uint32_t es[4] = {1, (uint32_t)P.sw, (uint32_t)P.sh, 1};
  int lower[2], upper[2];
  im2col_corners(P.h, P.w, P.ho, P.wo, P.sh, P.sw, P.pad_t, P.pad_l, lower, upper);
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, base, (const cuuint64_t*)dims, (const cuuint64_t*)strides, lower,
                   upper, (cuuint32_t)BK, (cuuint32_t)BM, (const cuuint32_t*)es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeIm2col failed (CUresult %d): dims [%llu,%llu,%llu,%llu] corners (%d,%d)..(%d,%d) stride %dx%d",
              (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
              (unsigned long long)dims[3], lower[0], lower[1], upper[0], upper[1], P.sh, P.sw);
    return DEFER_ERR_CUDA;
  }
  return DEFER_OK;
}

template <auto kernel>
int set_smem_attr(bool cluster16 = false) {
  static bool attr_set[64] = {false};   // one flag array per kernel instantiation
  int dev = 0;
  DEFER_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && !attr_set[dev]) {
    DEFER_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_CAP));
    if (cluster16) DEFER_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    prefer_max_smem(kernel);
    attr_set[dev] = true;
  }
  return DEFER_OK;
}

int sm_count() {
  static int sms[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev >= 64) return 1;
  if (!sms[dev]) cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
  return sms[dev] > 0 ? sms[dev] : 1;
}

void fill_op(const UmmaConvPlan& P, const UmmaConvLaneArgs& a, MegaOp* out) {
  MegaOp& op = *out;
  memset(&op, 0, sizeof op);
  op.tmx[0] = a.tmap_x[0];
  op.tmx[1] = a.tmap_x[1];
  op.tmw[0] = P.tmap_w[0];
  op.tmw[1] = P.tmap_w[1];
  KParams& kp = op.p;
  kp.n = P.n; kp.ho = P.ho; kp.wo = P.wo; kp.cout = P.cout;
  kp.im2col = P.im2col;
  kp.m_total = P.n * P.ho * P.wo;
  kp.kh = P.kh; kp.kw = P.kw; kp.sh = P.sh; kp.sw = P.sw; kp.pad_t = P.pad_t; kp.pad_l = P.pad_l;
  kp.cblocks = P.cin / 64;
  kp.k_blocks = P.k_blocks;
  kp.splits = P.splits;
  kp.cluster = P.cluster;
  kp.flags = P.flags;
  kp.scale = P.scale; kp.shift = P.shift;
  kp.res = (P.flags & DEFER_FLAG_RESIDUAL) ? a.res : nullptr;
  kp.y = a.y;
  kp.partial = a.partial;
  kp.counters = a.counters;
  kp.plane_out = (size_t)P.n * P.ho * P.wo * P.cout;
  op.m_tiles = P.m_tiles;
  op.n_tiles = P.cout / P.bn;
  op.scale2 = P.scale2;
  op.shift2 = P.shift2;
  op.y2 = a.y2;
  op.relu2 = P.relu2;
  op.store_first = P.aff ? P.store_first : 1;
}

template <int NPLANES, int BN, bool AFF = false>
int launch_op_t(const UmmaConvPlan& P, const UmmaConvLaneArgs& a, cudaStream_t st) {
  using L = Smem<NPLANES, BN>;
  constexpr auto kernel = AFF ? &conv_umma_aff_kernel<NPLANES, BN> : &conv_umma_kernel<NPLANES, BN>;
  DEFER_TRY((set_smem_attr<kernel>()));
  MegaOp op;
  fill_op(P, a, &op);
  // >= 2: a consumer releases a stage only once the NEXT k-block's wgmmas are issued (wgmma.wait_group 1)
  int stages = P.stages < 2 ? 2 : (P.stages > L::max_stages() ? L::max_stages() : P.stages);
  const size_t smem = (size_t)L::total(stages, P.cluster != 0);
  dim3 grid(op.m_tiles, op.n_tiles, P.splits);
  static const int pdl = env_int("DEFER_PDL", 0);
  if (pdl || P.cluster) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.gridDim = grid;
    cfg.blockDim = dim3(NUM_THREADS, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (pdl) {
      attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attr[na].val.programmaticStreamSerializationAllowed = 1;
      ++na;
    }
    if (P.cluster) {   // the `splits` CTAs of one output tile (grid.z) are one thread-block cluster
      attr[na].id = cudaLaunchAttributeClusterDimension;
      attr[na].val.clusterDim.x = 1;
      attr[na].val.clusterDim.y = 1;
      attr[na].val.clusterDim.z = (unsigned)P.splits;
      ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    DEFER_CUDA(cudaLaunchKernelEx(&cfg, kernel, op, stages, pdl));
    return DEFER_OK;
  }
  kernel<<<grid, NUM_THREADS, smem, st>>>(op, stages, 0);
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

// persistent grid over the tiles of one op in device memory: every CTA walks ceil(n_tiles / grid) tiles, so the launch
// lasts `rounds` tile-times whatever the grid is; take the SMALLEST grid that still finishes in the minimum number of
// rounds and leave the other SMs to the lanes running next to this one
template <auto kernel>
int launch_grid(const void* dev_op, int n_tiles, int stages, size_t smem, cudaStream_t st) {
  DEFER_TRY((set_smem_attr<kernel>()));
  const int sms = sm_count();
  int grid = sms < n_tiles ? sms : n_tiles;
  const int rounds = (n_tiles + grid - 1) / grid;
  grid = (n_tiles + rounds - 1) / rounds;
  static const int pdl = env_int("DEFER_PDL", 0);
  if (pdl) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.gridDim = dim3(grid, 1, 1);
    cfg.blockDim = dim3(NUM_THREADS, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    DEFER_CUDA(cudaLaunchKernelEx(&cfg, kernel, reinterpret_cast<const MegaOp*>(dev_op), stages, 1));
    return DEFER_OK;
  }
  kernel<<<grid, NUM_THREADS, smem, st>>>(reinterpret_cast<const MegaOp*>(dev_op), stages, 0);
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

template <int NPLANES, int BN, bool AFF = false>
int launch_persist_t(const void* dev_op, int n_tiles, int stages, cudaStream_t st) {
  using L = Smem<NPLANES, BN>;
  constexpr auto kernel = AFF ? &conv_stream_aff_kernel<NPLANES, BN> : &conv_stream_kernel<NPLANES, BN>;
  if (stages > L::max_stages()) stages = L::max_stages();
  if (stages < 2) stages = 2;
  return launch_grid<kernel>(dev_op, n_tiles, stages, (size_t)L::total(stages, false), st);
}

template <int NPLANES, int IN>
int launch_stem_t(const void* dev_op, int n_tiles, int stages, cudaStream_t st) {
  using L = StemSmem<NPLANES>;
  constexpr auto kernel = IN == STEM_U8_TF      ? &conv_stem_u8tf_kernel<NPLANES>
                          : IN == STEM_U8_CAFFE ? &conv_stem_u8_kernel<NPLANES>
                                                : &conv_stem_kernel<NPLANES>;
  if (stages > L::max_stages()) stages = L::max_stages();
  if (stages < 2) stages = 2;
  return launch_grid<kernel>(dev_op, n_tiles, stages, (size_t)L::total(stages), st);
}

template <int NPLANES>
int launch_mega_t(const void* dev_ops, int n_ops, int stages, cudaStream_t st) {
  using L = Smem<NPLANES, MEGA_BN>;
  DEFER_TRY(set_smem_attr<conv_mega_kernel<NPLANES>>(true));
  if (stages < 2) stages = 2;   // see launch_op_t
  if (stages > L::max_stages()) stages = L::max_stages();
  const int cluster = umma_mega_cluster_size();
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = dim3(cluster, 1, 1);
  cfg.blockDim = dim3(NUM_THREADS, 1, 1);
  cfg.dynamicSmemBytes = L::total(stages, false);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  DEFER_CUDA(cudaLaunchKernelEx(&cfg, conv_mega_kernel<NPLANES>, reinterpret_cast<const MegaOp*>(dev_ops), n_ops, stages));
  return DEFER_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------- public
bool umma_conv_supported(int fmt, int n, int h, int w, int cin, int ho, int wo, int cout, int kh, int kw, int sh, int sw,
                         int pad_t, int pad_l) {
  if (fmt != FMT_BF16X2 && fmt != FMT_BF16) return false;
  if (cin % 64 != 0 || cout % 64 != 0) return false;
  if (sh < 1 || sw < 1 || sh > 2 || sw > 2) return false;
  if (kh > 7 || kw > 7) return false;
  if (n < 1 || ho < 1 || wo < 1 || h < 1 || w < 1) return false;
  if ((size_t)n * ho * wo * cout >= (1ull << 40)) return false;
  int lower[2], upper[2];
  im2col_corners(h, w, ho, wo, sh, sw, pad_t, pad_l, lower, upper);
  return im2col_corners_encodable(lower, upper);
}

int umma_conv_prepare(UmmaConvPlan* plan, int fmt, int n, int h, int w, int cin, int ho, int wo, int cout, int kh, int kw,
                      int sh, int sw, int pad_t, int pad_l, uint32_t flags, const float* w_hwio_dev, const float* scale_dev,
                      const float* shift_dev, bool mega, int stream_bn) {
  UmmaConvPlan& P = *plan;
  P = UmmaConvPlan();
  P.fmt = fmt;
  P.nplanes = fmt == FMT_BF16X2 ? 2 : 1;
  P.n = n; P.h = h; P.w = w; P.cin = cin; P.ho = ho; P.wo = wo; P.cout = cout;
  P.kh = kh; P.kw = kw; P.sh = sh; P.sw = sw; P.pad_t = pad_t; P.pad_l = pad_l;
  P.flags = flags;
  P.scale = scale_dev;
  P.shift = shift_dev;
  const int taps = kh * kw;
  P.k_blocks = taps * (cin / 64);

  // ---- M tiling: 128 consecutive output pixels per tile.  A 1x1/stride-1 conv whose output grid IS the input grid reads
  // them as 128 consecutive rows of the [M, C] view; every other conv through TMA im2col (a fused asymmetric ZeroPadding2D
  // gives ho != h even with pad_t == pad_l == 0: the bounding box and its out-of-bounds zero fill are the padding).
  P.im2col = (kh == 1 && kw == 1 && sh == 1 && sw == 1 && pad_t == 0 && pad_l == 0 && ho == h && wo == w) ? 0 : 1;
  P.m_tiles = (int)(((long long)n * ho * wo + BM - 1) / BM);
  if (P.im2col) {
    int lower[2], upper[2];
    im2col_corners(h, w, ho, wo, sh, sw, pad_t, pad_l, lower, upper);
    if (!im2col_corners_encodable(lower, upper)) {
      set_error("umma conv: im2col box corners (%d,%d)..(%d,%d) outside [-128, 127]", lower[0], lower[1], upper[0], upper[1]);
      return DEFER_ERR_INVALID;
    }
  }
  const int m_tiles = P.m_tiles;

  // ---- N tile, split-K and ring depth.  The A tile is re-read once per N tile and the weights once per M tile, so
  // wide N tiles cut L2 -> SM traffic; split-K adds partial-tile traffic and is kept for launches of very few CTAs.
  P.bn = (cout % 128 == 0 && (long long)m_tiles * (cout / 128) >= env_int("DEFER_UMMA_BN128_MIN_CTAS", 1)) ? 128 : 64;
  int force_bn = env_int("DEFER_UMMA_BN", 0);
  if (force_bn == 64 || (force_bn == 128 && cout % 128 == 0)) P.bn = force_bn;
  int ctas = m_tiles * (cout / P.bn);
  P.splits = 1;
  int target = env_int("DEFER_UMMA_TARGET_CTAS", 4);
  if (env_int("DEFER_UMMA_SPLITK", 1) && ctas < target && P.k_blocks >= 8) {
    int s = (target + ctas - 1) / ctas;
    int max_s = P.k_blocks / 4;          // keep >= 4 k-blocks (256 K elements) per split
    if (s > max_s) s = max_s;
    if (s > 16) s = 16;
    if (s < 1) s = 1;
    int per = (P.k_blocks + s - 1) / s;  // make every split non-empty
    P.splits = (P.k_blocks + per - 1) / per;
  }
  int force_split = env_int("DEFER_UMMA_FORCE_SPLITS", 0);
  if (force_split > 0 && force_split <= P.k_blocks) {
    int per = (P.k_blocks + force_split - 1) / force_split;
    P.splits = (P.k_blocks + per - 1) / per;
  }
  // ---- cluster split-K (opt-in, DEFER_UMMA_CLUSTER=1): S CTAs per output tile split the K loop and the epilogue;
  // the partial tiles meet in distributed shared memory.  S = largest of {8, 4, 2} that leaves >= DEFER_UMMA_CSPLIT_KB
  // k-blocks per CTA.
  P.cluster = 0;
  if (env_int("DEFER_UMMA_CLUSTER", 0) && force_split <= 0 && !mega) {
    const int min_kb = env_int("DEFER_UMMA_CSPLIT_KB", 4);
    int max_s = env_int("DEFER_UMMA_CSPLIT_MAX", 8);
    if (max_s > 8) max_s = 8;
    const int max_ctas = env_int("DEFER_UMMA_CSPLIT_MAX_CTAS", 256);
    int s = 1;
    for (int c = 2; c <= max_s; c *= 2)
      if (P.k_blocks / c >= min_kb && (long long)ctas * c <= max_ctas) s = c;
    int force_c = env_int("DEFER_UMMA_FORCE_CSPLIT", 0);
    if ((force_c == 2 || force_c == 4 || force_c == 8) && P.k_blocks >= force_c) s = force_c;
    P.splits = s;
    P.cluster = s > 1 ? 1 : 0;
  }
  if (mega) {   // megakernel tiles: one N-tile width, the whole K loop inside the tile
    P.bn = MEGA_BN;
    P.splits = 1;
    P.cluster = 0;
  }
  if (stream_bn > 0) {   // streaming persistent kernel: whole K loop inside the tile, N tile chosen by the caller
    P.bn = (stream_bn == 128 && cout % 128 == 0) ? 128 : 64;
    P.splits = 1;
    P.cluster = 0;
    P.stream = 1;
  }
  {
    int kb_per = (P.k_blocks + P.splits - 1) / P.splits;
    int st = kb_per <= 2 ? 2 : (kb_per <= 6 ? 3 : 4);
    int force_st = env_int("DEFER_UMMA_STAGES", 0);
    if (force_st > 0) st = force_st;
    P.stages = st;
  }

  // ---- weights: fp32 HWIO -> bf16 [plane][tap][cout][cin]
  size_t welems = (size_t)taps * cin * cout;
  DEFER_CUDA(cudaMalloc(&P.w_dev, welems * 2 * P.nplanes));
  {
    unsigned grid = (unsigned)((welems + 255) / 256);
    prefer_max_smem(weight_transform_kernel);
    weight_transform_kernel<<<grid, 256>>>(w_hwio_dev, (__nv_bfloat16*)P.w_dev, taps, cin, cout, P.nplanes);
    DEFER_CUDA(cudaGetLastError());
  }
  for (int pl = 0; pl < P.nplanes; ++pl) {
    uint64_t dims[3] = {(uint64_t)cin, (uint64_t)cout, (uint64_t)taps};
    uint64_t strides[2] = {(uint64_t)cin * 2, (uint64_t)cin * cout * 2};
    uint32_t box[3] = {64, (uint32_t)P.bn, 1};
    uint32_t es[3] = {1, 1, 1};
    DEFER_TRY(encode_map(&P.tmap_w[pl], (uint8_t*)P.w_dev + pl * welems * 2, 3, dims, strides, box, es));
  }
  if (P.nplanes == 1) P.tmap_w[1] = P.tmap_w[0];
  P.ready = true;
  return DEFER_OK;
}

int umma_conv_bind(const UmmaConvPlan& P, UmmaConvLaneArgs* a, const void* x, const void* res, void* y) {
  if (!P.ready) {
    set_error("umma_conv_bind: plan not prepared");
    return DEFER_ERR_STATE;
  }
  size_t xelems = (size_t)P.n * P.h * P.w * P.cin;
  for (int pl = 0; pl < P.nplanes; ++pl) {
    uint8_t* base = (uint8_t*)x + pl * xelems * 2;
    if (P.im2col) {
      DEFER_TRY(encode_im2col_map(&a->tmap_x[pl], base, P));
    } else {
      uint64_t m = (uint64_t)P.n * P.h * P.w;
      uint64_t dims[4] = {(uint64_t)P.cin, m, 1, 1};
      uint64_t strides[3] = {(uint64_t)P.cin * 2, m * P.cin * 2, m * P.cin * 2};
      uint32_t box[4] = {64, BM, 1, 1};
      uint32_t es[4] = {1, 1, 1, 1};
      DEFER_TRY(encode_map(&a->tmap_x[pl], base, 4, dims, strides, box, es));
    }
  }
  if (P.nplanes == 1) a->tmap_x[1] = a->tmap_x[0];
  a->res = res;
  a->y = y;
  a->partial = nullptr;
  a->counters = nullptr;
  if (P.splits > 1 && !P.cluster) {
    size_t tiles = (size_t)P.m_tiles * (P.cout / P.bn);
    DEFER_CUDA(cudaMalloc((void**)&a->partial, tiles * P.splits * BM * P.bn * sizeof(float)));
    DEFER_CUDA(cudaMalloc((void**)&a->counters, tiles * sizeof(unsigned int)));
    DEFER_CUDA(cudaMemset(a->counters, 0, tiles * sizeof(unsigned int)));
  }
  return DEFER_OK;
}

void umma_conv_unbind(UmmaConvLaneArgs* a) {
  if (a->partial) cudaFree(a->partial);
  if (a->counters) cudaFree(a->counters);
  a->partial = nullptr;
  a->counters = nullptr;
}

int launch_conv_umma(const UmmaConvPlan& P, const UmmaConvLaneArgs& a, cudaStream_t st) {
  if (P.aff) {
    if (P.nplanes == 2) return P.bn == 128 ? launch_op_t<2, 128, true>(P, a, st) : launch_op_t<2, 64, true>(P, a, st);
    return P.bn == 128 ? launch_op_t<1, 128, true>(P, a, st) : launch_op_t<1, 64, true>(P, a, st);
  }
  if (P.nplanes == 2) return P.bn == 128 ? launch_op_t<2, 128>(P, a, st) : launch_op_t<2, 64>(P, a, st);
  return P.bn == 128 ? launch_op_t<1, 128>(P, a, st) : launch_op_t<1, 64>(P, a, st);
}

// ---- persistent / megakernel host side
size_t umma_mega_op_bytes() { return sizeof(MegaOp); }

int umma_mega_fill(void* host_dst, const UmmaConvPlan& P, const UmmaConvLaneArgs& a) {
  if (!P.ready || (P.bn != MEGA_BN && !P.stream) || P.splits != 1) {
    set_error("umma_mega_fill: plan is not a persistent-kernel plan (bn %d, splits %d)", P.bn, P.splits);
    return DEFER_ERR_STATE;
  }
  MegaOp op;
  fill_op(P, a, &op);
  memcpy(host_dst, &op, sizeof op);
  return DEFER_OK;
}

// 8 CTAs is the portable cluster size; up to 16 are allowed on H100 where a GPC has the SMs free
int umma_mega_cluster_size() {
  static int cached = 0;
  if (cached) return cached;
  int want = env_int("DEFER_MEGA_CLUSTER", 8);
  if (want < 1) want = 1;
  if (want > 16) want = 16;
  cached = want;
  return cached;
}

// ONE op on a persistent grid (many tiles: batched microbatches / large feature maps), 64-wide N tiles
int launch_conv_persistent(int nplanes, const void* dev_op, int n_tiles, bool aff, cudaStream_t st) {
  const int stages = env_int("DEFER_PERSIST_STAGES", MAX_STAGES);
  if (aff)
    return nplanes == 2 ? launch_persist_t<2, 64, true>(dev_op, n_tiles, stages, st)
                        : launch_persist_t<1, 64, true>(dev_op, n_tiles, stages, st);
  return nplanes == 2 ? launch_persist_t<2, 64>(dev_op, n_tiles, stages, st) : launch_persist_t<1, 64>(dev_op, n_tiles, stages, st);
}

// ONE op on the streaming persistent grid: the epilogue stages through its own shared-memory tile, outside the operand
// ring, so the producer keeps the next tile's operands in flight during this tile's epilogue
int launch_conv_stream(int nplanes, int bn, const void* dev_op, int n_tiles, int k_blocks, bool aff, cudaStream_t st) {
  (void)k_blocks;
  const int stages = env_int("DEFER_STREAM_STAGES", MAX_STAGES);
  if (aff) {
    if (bn == 128) return nplanes == 2 ? launch_persist_t<2, 128, true>(dev_op, n_tiles, stages, st)
                                       : launch_persist_t<1, 128, true>(dev_op, n_tiles, stages, st);
    if (bn == 64) return nplanes == 2 ? launch_persist_t<2, 64, true>(dev_op, n_tiles, stages, st)
                                      : launch_persist_t<1, 64, true>(dev_op, n_tiles, stages, st);
  }
  if (bn == 128) return nplanes == 2 ? launch_persist_t<2, 128>(dev_op, n_tiles, stages, st) : launch_persist_t<1, 128>(dev_op, n_tiles, stages, st);
  if (bn == 64) return nplanes == 2 ? launch_persist_t<2, 64>(dev_op, n_tiles, stages, st) : launch_persist_t<1, 64>(dev_op, n_tiles, stages, st);
  set_error("conv_stream: unsupported N tile %d", bn);
  return DEFER_ERR_INVALID;
}

// ---- fused stem: host side
// M tile of the fused stem: 8 rows x 16 columns of output pixels of one image (fewer columns and more rows on a map
// narrower than 16), and the image window it reads
static void stem_tile(int ho, int wo, int kh, int kw, int sh, int sw, int cin, int* tile_h, int* tile_w, int* win_rows,
                      int* win_cols) {
  *tile_w = wo < STEM_TILE_W ? wo : STEM_TILE_W;
  *tile_h = BM / *tile_w < ho ? BM / *tile_w : ho;
  *win_rows = (*tile_h - 1) * sh + kh;
  *win_cols = ((*tile_w - 1) * sw + kw) * cin;
}

bool umma_stem_fusable(int fmt, int cin, int ho, int wo, int cout, int kh, int kw, int sh, int sw, uint32_t flags) {
  if (fmt != FMT_BF16X2 && fmt != FMT_BF16) return false;
  if (cout != 64 || (flags & DEFER_FLAG_RESIDUAL) || kh * kw * cin > 256) return false;
  int tile_h, tile_w, win_rows, win_cols;
  stem_tile(ho, wo, kh, kw, sh, sw, cin, &tile_h, &tile_w, &win_rows, &win_cols);
  return (long long)win_rows * win_cols <= STEM_WIN_VALS;
}

int umma_mega_set_stem(void* host_op, const float* x, int h, int w, int cin, int kh, int kw, int sh, int sw, int pad_t,
                       int pad_l) {
  MegaOp* op = reinterpret_cast<MegaOp*>(host_op);
  KParams& p = op->p;
  op->stem_x = x;
  op->stem_h = h; op->stem_w = w; op->stem_cin = cin;
  op->stem_kh = kh; op->stem_kw = kw; op->stem_sh = sh; op->stem_sw = sw;
  op->stem_pad_t = pad_t; op->stem_pad_l = pad_l;
  op->stem_K = kh * kw * cin;
  // the real output map replaces the plan's flat view of the patch matrix: tile_h x tile_w pixels of one image
  stem_tile(p.ho, p.wo, kh, kw, sh, sw, cin, &p.tile_h, &p.tile_w, &op->stem_win_rows, &op->stem_win_cols);
  p.tiles_h = (p.ho + p.tile_h - 1) / p.tile_h;
  p.tiles_w = (p.wo + p.tile_w - 1) / p.tile_w;
  op->m_tiles = p.n * p.tiles_h * p.tiles_w;
  return op->m_tiles * op->n_tiles;
}

void umma_mega_set_stem_u8(void* host_op, const uint8_t* x, const float shift[3]) {
  MegaOp* op = reinterpret_cast<MegaOp*>(host_op);
  op->stem_x = nullptr;
  op->stem_u8 = x;
  for (int c = 0; c < 3; ++c) op->stem_shift[c] = shift[c];
}

int launch_conv_stem(int nplanes, const void* dev_op, int n_tiles, bool u8, bool tf, cudaStream_t st) {
  const int stages = env_int("DEFER_STREAM_STAGES", MAX_STAGES);
  if (u8 && tf)
    return nplanes == 2 ? launch_stem_t<2, STEM_U8_TF>(dev_op, n_tiles, stages, st)
                        : launch_stem_t<1, STEM_U8_TF>(dev_op, n_tiles, stages, st);
  if (u8)
    return nplanes == 2 ? launch_stem_t<2, STEM_U8_CAFFE>(dev_op, n_tiles, stages, st)
                        : launch_stem_t<1, STEM_U8_CAFFE>(dev_op, n_tiles, stages, st);
  return nplanes == 2 ? launch_stem_t<2, STEM_F32>(dev_op, n_tiles, stages, st) : launch_stem_t<1, STEM_F32>(dev_op, n_tiles, stages, st);
}

int launch_conv_mega(int nplanes, const void* dev_ops, int n_ops, cudaStream_t st) {
  int stages = env_int("DEFER_MEGA_STAGES", 4);
  return nplanes == 2 ? launch_mega_t<2>(dev_ops, n_ops, stages, st) : launch_mega_t<1>(dev_ops, n_ops, stages, st);
}

void umma_conv_release(UmmaConvPlan& P) {
  if (P.w_dev) cudaFree(P.w_dev);
  P.w_dev = nullptr;
  P.ready = false;
}

}  // namespace defer
